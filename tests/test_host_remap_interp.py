"""INTER_CUBIC and INTER_LANCZOS4 on the CPU.  tests/host/remap_interp.cu runs the per-thread body of k_gather_taps
(gather_taps_frames, with the weight tables build_interp_tabs makes) over the device's grid, from the library's own
headers, and every image must equal live cv2.remap / cv2.warpPerspective byte for byte:

- every one of the 1024 fraction classes, 2,000 samples each, for both kernels and 1, 3 and 4 channels;
- sources narrower or shorter than the kernel, windows across every edge, batches across GATHER_NB;
- int16-extreme and out-of-frame maps (the BEV fuzz corpus's map recipes);
- the random calibrations of tests/calib_cases.py through their maps (mode 0) and their camera model (mode 1);
- cv2.warpPerspective with the corpus's homographies (mode 2).

nvcc compiles the harness; only host code runs."""
import os
import shutil
import struct
import subprocess

import cv2
import numpy as np
import pytest

from cameracalibration_b200.build import GENCODE
from tests import bev_cases as B
from tests import calib_cases as CC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KS = {cv2.INTER_CUBIC: 4, cv2.INTER_LANCZOS4: 8}
INTERS = (cv2.INTER_CUBIC, cv2.INTER_LANCZOS4)


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    nvcc = next((c for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc") if c and os.path.exists(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("host_remap_interp") / "remap_interp"
    build = subprocess.run([nvcc, "-O2", "-std=c++17", "--fmad=false", "-Xcompiler", "-ffp-contract=off", *GENCODE, "-o", str(out),
                            os.path.join(ROOT, "tests", "host", "remap_interp.cu")], capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stdout + build.stderr
    return str(out)


def _stack(frames, row_pad=0, img_pad=0):
    """n frames uint8[n][h][w][ch] in one buffer with padded rows and images; the padding holds noise."""
    n, h, w, ch = frames.shape
    srow = w * ch + row_pad
    simg = h * srow + img_pad
    size = (n - 1) * simg + (h - 1) * srow + w * ch
    buf = np.random.default_rng(n * 7 + h * 3 + w).integers(0, 256, size, dtype=np.uint8)
    for f in range(n):
        np.lib.stride_tricks.as_strided(buf[f * simg:], (h, w, ch), (srow, ch, 1))[...] = frames[f]
    return buf, srow, simg


def _record(mode, inter, frames, dw, dh, extra, row_pad=0, img_pad=0):
    n, sh, sw, ch = frames.shape
    buf, srow, simg = _stack(frames, row_pad, img_pad)
    return (struct.pack("<8i", mode, ch, KS[inter], sw, sh, dw, dh, n) + struct.pack("<2q", srow, simg) + extra + buf.tobytes(),
            dict(mode=mode, n=n, dw=dw, dh=dh, ch=ch))


def _maps_record(inter, frames, m1, m2, **pad):
    dh, dw = m2.shape
    extra = np.ascontiguousarray(m1, np.int16).tobytes() + np.ascontiguousarray(m2, np.uint16).tobytes()
    return _record(0, inter, frames, dw, dh, extra, **pad)


def _run(exe, tmp_path, recs):
    """Runs the records; returns per record the n output images and, for mode 1, the model's maps."""
    (tmp_path / "in.bin").write_bytes(b"".join(r for r, _ in recs))
    r = subprocess.run([exe, "run", str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True,
                       timeout=1800)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr[-2000:])
    raw, p, res = np.fromfile(tmp_path / "out.bin", np.uint8), 0, []
    for _, c in recs:
        k = c["n"] * c["dh"] * c["dw"] * c["ch"]
        imgs = raw[p:p + k].reshape(c["n"], c["dh"], c["dw"], c["ch"])
        p += k
        maps = None
        if c["mode"] == 1:
            npx = c["dh"] * c["dw"]
            m1 = raw[p:p + 4 * npx].view(np.int16).reshape(c["dh"], c["dw"], 2)
            m2 = raw[p + 4 * npx:p + 6 * npx].view(np.uint16).reshape(c["dh"], c["dw"])
            p += 6 * npx
            maps = (m1, m2)
        res.append((imgs, maps))
    assert p == raw.size
    return res


def _remap(frame, m1, m2, inter):
    f = frame[..., 0] if frame.shape[2] == 1 else frame
    return cv2.remap(f, m1, m2, inter).reshape(m2.shape + (frame.shape[2],))


def _check(got, frames, m1, m2, inter, what):
    assert got.shape[0] == frames.shape[0] >= 1
    for f in range(frames.shape[0]):
        want = _remap(frames[f], m1, m2, inter)
        assert (got[f] == want).all(), (what, f, int((got[f] != want).sum()))


@pytest.mark.parametrize("inter", INTERS, ids=["cubic", "lanczos4"])
def test_every_fraction_class(exe, tmp_path, inter):
    """2,000 samples of each of the 1024 classes per channel count, windows inside and across the edges."""
    rng = np.random.default_rng(10 + inter)
    recs, want = [], []
    for ch in (1, 3, 4):
        sw, sh = int(rng.integers(40, 90)), int(rng.integers(30, 70))
        frames = rng.integers(0, 256, (1, sh, sw, ch), dtype=np.uint8)
        dh, dw = 1000, 2048                               # 2,048,000 pixels: every class exactly 2,000 times
        m2 = rng.permutation(np.repeat(np.arange(1024, dtype=np.uint16), 2000)).reshape(dh, dw)
        m1 = np.stack([rng.integers(-9, sw + 9, (dh, dw)), rng.integers(-9, sh + 9, (dh, dw))], -1).astype(np.int16)
        assert (np.bincount(m2.ravel(), minlength=1024) >= 2000).all()
        recs.append(_maps_record(inter, frames, m1, m2, row_pad=int(rng.integers(0, 5))))
        want.append((frames, m1, m2))
    for (got, _), (frames, m1, m2) in zip(_run(exe, tmp_path, recs), want):
        _check(got, frames, m1, m2, inter, ("classes", frames.shape))


@pytest.mark.parametrize("inter", INTERS, ids=["cubic", "lanczos4"])
def test_small_sources_and_batches(exe, tmp_path, inter):
    """W, H in 1..8 (smaller than the kernel), every window position around the frame, batches of 1, 3, 8, 9 and 17
    with padded rows and images."""
    rng = np.random.default_rng(20 + inter)
    recs, want = [], []
    for i, (sw, sh) in enumerate([(w, h) for w in range(1, 9) for h in (1, 2, 5, 8)]):
        ch = (1, 3, 4)[i % 3]
        n = (1, 3, 8, 9, 17)[i % 5]
        frames = rng.integers(0, 256, (n, sh, sw, ch), dtype=np.uint8)
        xs, ys = np.meshgrid(np.arange(-9, sw + 9), np.arange(-9, sh + 9))
        m1 = np.stack([xs, ys], -1).astype(np.int16)
        m2 = rng.integers(0, 1024, xs.shape).astype(np.uint16)
        recs.append(_maps_record(inter, frames, m1, m2, row_pad=i % 4, img_pad=(i * 5) % 7))
        want.append((frames, m1, m2))
    for (got, _), (frames, m1, m2) in zip(_run(exe, tmp_path, recs), want):
        _check(got, frames, m1, m2, inter, ("small", frames.shape))


@pytest.mark.parametrize("inter", INTERS, ids=["cubic", "lanczos4"])
def test_extreme_and_local_maps(exe, tmp_path, inter):
    """The BEV fuzz corpus's map recipes: int16-extreme taps (+-40000 clipped to int16) with a band of ordinary ones,
    random taps within 6 px of the frame, and taps exactly on the edges; map2 over all 16 bits (cv2 reads its low 10)."""
    rng = np.random.default_rng(30 + inter)
    recs, want = [], []
    for i, kind in enumerate(("extreme", "local", "extreme", "local")):
        FW, FH = (33, 64, 97, 116)[i], (21, 40, 65, 52)[i]
        ch = (1, 3, 4, 3)[i]
        for m1, m2 in B._maps(rng, kind, 2, FW, FH, 77, 45):
            m2 = (m2 | (rng.integers(0, 64, m2.shape) << 10)).astype(np.uint16) if i % 2 else m2
            frames = rng.integers(0, 256, (2, FH, FW, ch), dtype=np.uint8)
            recs.append(_maps_record(inter, frames, m1, m2, row_pad=i))
            want.append((frames, m1, m2))
    for (got, _), (frames, m1, m2) in zip(_run(exe, tmp_path, recs), want):
        _check(got, frames, m1, m2, inter, "extreme/local")


def _calib_cases():
    # the scaled and strong cameras (frames up to 1920 x 1080; the 4K mild ones add time, not new arithmetic)
    return [c for c in CC.corpus() if c.kind != "mild"][::2]


@pytest.mark.parametrize("inter", INTERS, ids=["cubic", "lanczos4"])
def test_calibrations_maps_and_model(exe, tmp_path, inter):
    """Mode 0 through cv2's own maps; mode 1 through the camera model, against cv2.remap over the maps the model gives
    (k_undistort_map's arithmetic), and against cv2.remap over cv2's maps at every pixel where the two map entries agree
    (fisheye: all of them; pinhole: all but fraction entries of off-frame taps, DESIGN.md section 7)."""
    recs, want = [], []
    for i, c in enumerate(_calib_cases()):
        ch = (1, 3, 4)[i % 3]
        frames = CC.frames(c.name, ch, 1)
        m1, m2 = CC.cv2_maps(c.name)
        recs.append(_maps_record(inter, frames, m1, m2))
        want.append((c, frames, 0))
        extra = np.r_[c.K.ravel(), c.d5, c.P.ravel(), float(c.model)].astype("<f8").tobytes()
        recs.append(_record(1, inter, frames, c.UW, c.UH, extra))
        want.append((c, frames, 1))
    agree = 0
    for (got, maps), (c, frames, mode) in zip(_run(exe, tmp_path, recs), want):
        w1, w2 = CC.cv2_maps(c.name)
        if mode == 0:
            _check(got, frames, w1, w2, inter, (c.name, 0))
            continue
        _check(got, frames, maps[0], maps[1], inter, (c.name, 1))
        same = (maps[0] == w1).all(-1) & (maps[1] == w2)
        assert not c.fisheye or same.all(), c.name
        theirs = _remap(frames[0], w1, w2, inter)
        assert (got[0][same] == theirs[same]).all(), c.name
        agree += int(same.sum())
    assert agree > 0


@pytest.mark.parametrize("inter", INTERS, ids=["cubic", "lanczos4"])
def test_warp_perspective(exe, tmp_path, inter):
    """Mode 2: cv2.warpPerspective(src, H, (BW, BH), flags) with the corpus's homographies, horizons inside the canvas
    and exact W = 0 lines included."""
    recs, want = [], []
    for i, c in enumerate(CC.corpus()[12::3]):
        ch = (1, 3, 4)[i % 3]
        sw, sh = min(c.UW, 1000), min(c.UH, 800)
        frames = CC.frames(c.name, ch, 1, (sw, sh))
        recs.append(_record(2, inter, frames, c.BW, c.BH, np.asarray(c.H, "<f8").tobytes()))
        want.append((c, frames))
    for (got, _), (c, frames) in zip(_run(exe, tmp_path, recs), want):
        f = frames[0][..., 0] if frames.shape[3] == 1 else frames[0]
        w = cv2.warpPerspective(f, c.H, (c.BW, c.BH), flags=inter).reshape(c.BH, c.BW, frames.shape[3])
        assert (got[0] == w).all(), (c.name, int((got[0] != w).sum()))


def test_cv2_reads_area_as_linear():
    """The premise of the library's INTER_AREA: cv2.remap and cv2.warpPerspective give INTER_LINEAR's bytes."""
    rng = np.random.default_rng(5)
    img = rng.integers(0, 256, (60, 80, 3), dtype=np.uint8)
    m1 = np.stack([rng.integers(-3, 83, (40, 50)), rng.integers(-3, 63, (40, 50))], -1).astype(np.int16)
    m2 = rng.integers(0, 1024, (40, 50)).astype(np.uint16)
    assert (cv2.remap(img, m1, m2, cv2.INTER_AREA) == cv2.remap(img, m1, m2, cv2.INTER_LINEAR)).all()
    H = CC.corpus()[13].H
    assert (cv2.warpPerspective(img, H, (70, 50), flags=cv2.INTER_AREA) ==
            cv2.warpPerspective(img, H, (70, 50), flags=cv2.INTER_LINEAR)).all()
