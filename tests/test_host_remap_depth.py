"""16U, 16S and 32F images on the CPU.  tests/host/remap_depth.cu runs the per-thread bodies of k_gather and
k_gather_taps at those depths (gather_frames / gather_taps_frames with T = uint16_t, int16_t, float) over the device's
grid, from the library's own headers, and every image must equal live cv2.remap / cv2.warpPerspective / cv2.warpAffine
bit for bit (float32: the same bit pattern, or NaN where cv2 gives NaN; NEAREST keeps even a NaN's payload):

- every depth x channel count (1, 3, 4) x interpolation (NEAREST, LINEAR, CUBIC, LANCZOS4) x MODE 0-5, except the
  warps the library refuses because cv2 4.13 leaves remap's arithmetic there (cv2_warp_differs);
- every one of the 1024 fraction classes, for every depth, channel count and interpolation;
- sources narrower or shorter than the kernel, windows across every edge, batches across GATHER_NB with padded rows and
  images;
- int16-extreme and out-of-frame maps (the BEV fuzz corpus's map recipes);
- the random calibrations of tests/calib_cases.py (maps and camera model) and the rectified stereo pairs of
  tests/float_map_cases.py (cv2's CV_16SC2, CV_32FC1 and CV_32FC2 maps);
- cv2.warpPerspective with the corpus's homographies and cv2.warpAffine with and without WARP_INVERSE_MAP;
- value extremes: 0, 65535, -32768, 32767, +-inf, NaN (with zero weights too), -0.0, denormals and FLT_MAX.

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
from tests import float_map_cases as FM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INTERS = (cv2.INTER_NEAREST, cv2.INTER_LINEAR, cv2.INTER_CUBIC, cv2.INTER_LANCZOS4)
DEPTHS = {2: np.uint16, 3: np.int16, 5: np.float32}
DEPTH_IDS = ["16u", "16s", "32f"]


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    nvcc = next((c for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc") if c and os.path.exists(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("host_remap_depth") / "remap_depth"
    build = subprocess.run([nvcc, "-O2", "-std=c++17", "--fmad=false", "-Xcompiler", "-ffp-contract=off", *GENCODE, "-o", str(out),
                            os.path.join(ROOT, "tests", "host", "remap_depth.cu")], capture_output=True, text=True, timeout=900)
    assert build.returncode == 0, build.stdout + build.stderr
    return str(out)


def values(rng, depth, shape, special=0.0):
    """Random elements of a depth over its whole range; a fraction `special` of them replaced by the depth's extremes."""
    dt = DEPTHS[depth]
    if depth == 5:
        v = (rng.standard_normal(shape) * 10.0 ** rng.uniform(-3, 4, shape)).astype(np.float32)
        ext = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1e-45, -1e-40, 1.17549435e-38, 3.4028235e38, -3.4028235e38,
                        65535.0, -32768.0], np.float32)
    else:
        info = np.iinfo(dt)
        v = rng.integers(info.min, int(info.max) + 1, shape).astype(dt)
        ext = np.array([info.min, info.max, 0, info.max - 1], dt)
    if special:
        m = rng.random(shape) < special
        v[m] = rng.choice(ext, int(m.sum()))
    return v


def _stack(frames, row_pad=0, img_pad=0):
    """n frames [n][h][w][ch] in one byte buffer with rows and images padded by whole elements of noise."""
    n, h, w, ch = frames.shape
    es = frames.itemsize
    srow = (w * ch + row_pad) * es
    simg = h * srow + img_pad * es
    size = (n - 1) * simg + (h - 1) * srow + w * ch * es
    buf = np.random.default_rng(n * 7 + h * 3 + w).integers(0, 256, size, dtype=np.uint8)
    typed = buf.view(frames.dtype)
    for f in range(n):
        np.lib.stride_tricks.as_strided(typed[f * simg // es:], (h, w, ch), (srow, ch * es, es))[...] = frames[f]
    return buf, srow, simg


def _record(mode, inter, frames, dw, dh, extra, arg=0, row_pad=0, img_pad=0):
    n, sh, sw, ch = frames.shape
    depth = {np.dtype(v): k for k, v in DEPTHS.items()}[frames.dtype]
    buf, srow, simg = _stack(frames, row_pad, img_pad)
    return (struct.pack("<10i", mode, ch, inter, depth, sw, sh, dw, dh, n, arg) + struct.pack("<2q", srow, simg) + extra +
            buf.tobytes(), dict(mode=mode, n=n, dw=dw, dh=dh, ch=ch, dtype=frames.dtype))


def _maps_record(inter, frames, m1, m2, **pad):
    dh, dw = m1.shape[:2]
    extra = np.ascontiguousarray(m1, np.int16).tobytes() + (b"" if m2 is None else np.ascontiguousarray(m2, np.uint16).tobytes())
    return _record(0, inter, frames, dw, dh, extra, int(m2 is not None), **pad)


def _fmaps_record(inter, frames, x, y, **pad):
    """mode 4: CV_32FC1 planes (x, y), or CV_32FC2 pairs in x when y is None"""
    dh, dw = x.shape[:2]
    extra = np.ascontiguousarray(x, np.float32).tobytes() + (b"" if y is None else np.ascontiguousarray(y, np.float32).tobytes())
    return _record(4, inter, frames, dw, dh, extra, cv2.CV_32FC2 if y is None else cv2.CV_32FC1, **pad)


def _model_record(mode, inter, frames, K, d5, P, model, dw, dh):
    extra = np.r_[np.ravel(K), d5, np.ravel(P), float(model)].astype("<f8").tobytes()
    return _record(mode, inter, frames, dw, dh, extra)


def _run(exe, tmp_path, recs):
    """Runs the records; returns per record the n output images and, for modes 1 and 5, the model's maps."""
    (tmp_path / "in.bin").write_bytes(b"".join(r for r, _ in recs))
    r = subprocess.run([exe, "run", str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True,
                       timeout=1800)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr[-2000:])
    raw, p, res = np.fromfile(tmp_path / "out.bin", np.uint8), 0, []
    for _, c in recs:
        npx = c["dh"] * c["dw"]
        k = c["n"] * npx * c["ch"] * c["dtype"].itemsize
        imgs = raw[p:p + k].view(c["dtype"]).reshape(c["n"], c["dh"], c["dw"], c["ch"])
        p += k
        maps = None
        if c["mode"] == 1:
            maps = (raw[p:p + 4 * npx].view(np.int16).reshape(c["dh"], c["dw"], 2),
                    raw[p + 4 * npx:p + 6 * npx].view(np.uint16).reshape(c["dh"], c["dw"]))
            p += 6 * npx
        elif c["mode"] == 5:
            maps = (raw[p:p + 4 * npx].view(np.float32).reshape(c["dh"], c["dw"]),
                    raw[p + 4 * npx:p + 8 * npx].view(np.float32).reshape(c["dh"], c["dw"]))
            p += 8 * npx
        res.append((imgs, maps))
    assert p == raw.size
    return res


def same(got, want, inter):
    """Bit for bit; a float32 NaN matches any NaN except under NEAREST, which moves the bits themselves."""
    if got.shape != want.shape:
        return False
    if got.dtype != np.float32 or inter == cv2.INTER_NEAREST:
        return got.tobytes() == want.tobytes()
    g, w = got.view(np.uint32), want.view(np.uint32)
    return bool(((g == w) | (np.isnan(got) & np.isnan(want))).all())


def ndiff(got, want):
    if got.dtype == np.float32:
        return int((~((got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want)))).sum())
    return int((got != want).sum())


def _cv(call, frame):
    """cv2 on one frame [h][w][ch] (ch 1 passed as [h][w]); the result as [h][w][ch]."""
    ch = frame.shape[2]
    out = call(frame[..., 0] if ch == 1 else frame)
    return out.reshape(out.shape[:2] + (ch,))


def _check(got, frames, inter, call, what):
    assert got.shape[0] == frames.shape[0] >= 1
    for f in range(frames.shape[0]):
        want = _cv(call, frames[f])
        assert same(got[f], want, inter), (what, f, ndiff(got[f], want))


def _remap_call(m1, m2, inter):
    return lambda f: cv2.remap(f, m1, m2, inter)


def cv2_warp_differs(mode, depth, inter, ch):
    """The warps bevk refuses (BEVK_ERR_UNSUPPORTED): cv2 4.13 computes them with warp-specific bodies whose pixels differ
    from cv2.remap's through the same positions -- warpPerspective (MODE 2) LINEAR at 16UC3 / 16UC4 and NEAREST at 32FC1 /
    32FC4, warpAffine (MODE 3) NEAREST at 16UC4 and at 16S with any channel count.  test_cv2_warps_leave_remap pins it."""
    nearest, linear = inter == cv2.INTER_NEAREST, inter in (cv2.INTER_LINEAR, cv2.INTER_AREA)
    if mode == 2:
        return (depth == 2 and linear and ch != 1) or (depth == 5 and nearest and ch != 3)
    return mode == 3 and nearest and (depth == 3 or (depth == 2 and ch == 4))


def _mild_camera(W, H, fisheye):
    K = np.array([[0.6 * W, 0, W / 2 + 0.3], [0, 0.61 * W, H / 2 - 0.2], [0, 0, 1]])
    d5 = np.array([0.03, -0.01, 0.002, -0.001, 0.0]) if fisheye else np.array([-0.2, 0.05, 0.001, -0.002, 0.01])
    P = K.copy()
    P[0, 0] *= 0.8
    P[1, 1] *= 0.8
    return K, d5, P, 0 if fisheye else 1


@pytest.mark.parametrize("depth", DEPTHS, ids=DEPTH_IDS)
def test_every_combination(exe, tmp_path, depth):
    """Every channel count x interpolation x MODE 0-5 at this depth, windows inside and across the edges."""
    rng = np.random.default_rng(100 + depth)
    recs, want = [], []
    sw, sh, dw, dh = 37, 29, 45, 33
    for mode in range(6):
        for ch in (1, 3, 4):
            for inter in INTERS:
                if cv2_warp_differs(mode, depth, inter, ch):
                    continue
                frames = values(rng, depth, (2, sh, sw, ch), 0.05)
                if mode == 0:
                    m1 = np.stack([rng.integers(-5, sw + 5, (dh, dw)), rng.integers(-5, sh + 5, (dh, dw))], -1).astype(np.int16)
                    m2 = None if inter == cv2.INTER_NEAREST and ch == 3 else rng.integers(0, 1024, (dh, dw)).astype(np.uint16)
                    recs.append(_maps_record(inter, frames, m1, m2, row_pad=ch, img_pad=3))
                    want.append((frames, inter, _remap_call(m1, m2, inter)))
                elif mode in (1, 5):
                    K, d5, P, model = _mild_camera(sw, sh, fisheye=(ch != 3))
                    recs.append(_model_record(mode, inter, frames, K, d5, P, model, dw, dh))
                    want.append((frames, inter, None))
                elif mode == 2:
                    H = np.array([[0.9, 0.05, 1.3], [-0.04, 1.1, -2.2], [1e-3, -2e-3, 1.0]])
                    recs.append(_record(2, inter, frames, dw, dh, H.astype("<f8").tobytes()))
                    want.append((frames, inter, lambda f, H=H, i=inter: cv2.warpPerspective(f, H, (dw, dh), flags=i)))
                elif mode == 3:
                    inv = ch == 4
                    M = cv2.getRotationMatrix2D((sw / 2, sh / 2), 17.0 + ch, 1.1)
                    flags = inter | (cv2.WARP_INVERSE_MAP if inv else 0)
                    recs.append(_record(3, inter, frames, dw, dh, M.astype("<f8").tobytes(), int(inv)))
                    want.append((frames, inter, lambda f, M=M, fl=flags: cv2.warpAffine(f, M, (dw, dh), flags=fl)))
                else:
                    x = rng.uniform(-5, sw + 5, (dh, dw)).astype(np.float32)
                    y = rng.uniform(-5, sh + 5, (dh, dw)).astype(np.float32)
                    if ch == 3:   # CV_32FC2
                        xy = np.stack([x, y], -1)
                        recs.append(_fmaps_record(inter, frames, xy, None))
                        want.append((frames, inter, _remap_call(xy, None, inter)))
                    else:
                        recs.append(_fmaps_record(inter, frames, x, y))
                        want.append((frames, inter, _remap_call(x, y, inter)))
    for (got, maps), (frames, inter, call), (_, c) in zip(_run(exe, tmp_path, recs), want, recs):
        if call is None:   # the camera model: cv2.remap over the maps the model gives
            call = _remap_call(maps[0], maps[1], inter)
        _check(got, frames, inter, call, (c["mode"], c["ch"], inter))


@pytest.mark.parametrize("depth", DEPTHS, ids=DEPTH_IDS)
def test_every_fraction_class(exe, tmp_path, depth):
    """40 samples of each of the 1024 classes per channel count and interpolation, windows inside and across the edges."""
    rng = np.random.default_rng(200 + depth)
    recs, want = [], []
    for inter in INTERS:
        for ch in (1, 3, 4):
            sw, sh = int(rng.integers(20, 60)), int(rng.integers(15, 40))
            frames = values(rng, depth, (1, sh, sw, ch), 0.02)
            dh, dw = 40, 1024
            m2 = rng.permutation(np.repeat(np.arange(1024, dtype=np.uint16), 40)).reshape(dh, dw)
            m1 = np.stack([rng.integers(-9, sw + 9, (dh, dw)), rng.integers(-9, sh + 9, (dh, dw))], -1).astype(np.int16)
            recs.append(_maps_record(inter, frames, m1, m2, row_pad=int(rng.integers(0, 5))))
            want.append((frames, inter, _remap_call(m1, m2, inter)))
    for (got, _), (frames, inter, call) in zip(_run(exe, tmp_path, recs), want):
        _check(got, frames, inter, call, ("classes", inter, frames.shape))


@pytest.mark.parametrize("depth", DEPTHS, ids=DEPTH_IDS)
def test_small_sources_and_batches(exe, tmp_path, depth):
    """W, H in 1..8 (smaller than the kernels), every window position around the frame, batches of 1, 3, 8, 9 and 17
    with padded rows and images, through CV_16SC2 and float maps."""
    rng = np.random.default_rng(300 + depth)
    recs, want = [], []
    for i, (sw, sh) in enumerate([(w, h) for w in (1, 2, 3, 5, 8) for h in (1, 2, 5, 8)]):
        ch = (1, 3, 4)[i % 3]
        n = (1, 3, 8, 9, 17)[i % 5]
        inter = INTERS[i % 4]
        frames = values(rng, depth, (n, sh, sw, ch), 0.05)
        xs, ys = np.meshgrid(np.arange(-9, sw + 9), np.arange(-9, sh + 9))
        m1 = np.stack([xs, ys], -1).astype(np.int16)
        m2 = rng.integers(0, 1024, xs.shape).astype(np.uint16)
        recs.append(_maps_record(inter, frames, m1, m2, row_pad=i % 4, img_pad=(i * 5) % 7))
        want.append((frames, inter, _remap_call(m1, m2, inter)))
        x = (xs + rng.uniform(-1, 1, xs.shape)).astype(np.float32)
        y = (ys + rng.uniform(-1, 1, ys.shape)).astype(np.float32)
        recs.append(_fmaps_record(INTERS[(i + 1) % 4], frames, x, y, row_pad=(i + 1) % 4, img_pad=i % 5))
        want.append((frames, INTERS[(i + 1) % 4], _remap_call(x, y, INTERS[(i + 1) % 4])))
    for (got, _), (frames, inter, call) in zip(_run(exe, tmp_path, recs), want):
        _check(got, frames, inter, call, ("small", inter, frames.shape))


@pytest.mark.parametrize("depth", DEPTHS, ids=DEPTH_IDS)
def test_extreme_and_local_maps(exe, tmp_path, depth):
    """The BEV fuzz corpus's map recipes: int16-extreme taps with a band of ordinary ones, random taps within 6 px of the
    frame, and taps exactly on the edges; map2 over all 16 bits (cv2 reads its low 10)."""
    rng = np.random.default_rng(400 + depth)
    recs, want = [], []
    for i, kind in enumerate(("extreme", "local", "extreme", "local")):
        FW, FH = (33, 64, 97, 116)[i], (21, 40, 65, 52)[i]
        ch = (1, 3, 4, 3)[i]
        for j, (m1, m2) in enumerate(B._maps(rng, kind, 2, FW, FH, 77, 45)):
            m2 = (m2 | (rng.integers(0, 64, m2.shape) << 10)).astype(np.uint16) if i % 2 else m2
            inter = INTERS[(2 * i + j) % 4]
            frames = values(rng, depth, (2, FH, FW, ch), 0.05)
            recs.append(_maps_record(inter, frames, m1, m2, row_pad=i))
            want.append((frames, inter, _remap_call(m1, m2, inter)))
    for (got, _), (frames, inter, call) in zip(_run(exe, tmp_path, recs), want):
        _check(got, frames, inter, call, ("extreme/local", inter))


@pytest.mark.parametrize("depth", DEPTHS, ids=DEPTH_IDS)
def test_calibrations_and_stereo_pairs(exe, tmp_path, depth):
    """The random calibrations through cv2's maps (MODE 0) and their camera model (MODE 1, and MODE 5 through float
    maps), against cv2.remap over the maps the model gives; the rectified stereo pairs through cv2's CV_16SC2, CV_32FC1
    and CV_32FC2 maps (MODE 0 and 4)."""
    rng = np.random.default_rng(500 + depth)
    recs, want = [], []
    cases = [c for c in CC.corpus() if c.kind != "mild" and c.FW * c.FH <= 1280 * 1024][::3]
    for i, c in enumerate(cases):
        ch, inter = (1, 3, 4)[i % 3], INTERS[i % 4]
        frames = values(rng, depth, (1, c.FH, c.FW, ch), 0.01)
        m1, m2 = CC.cv2_maps(c.name)
        recs.append(_maps_record(inter, frames, m1, m2))
        want.append((frames, inter, _remap_call(m1, m2, inter)))
        mode = (1, 5)[i % 2]
        recs.append(_model_record(mode, INTERS[(i + 1) % 4], frames, c.K, c.d5, c.P, c.model, c.UW, c.UH))
        want.append((frames, INTERS[(i + 1) % 4], None))
    for j, c in enumerate(x for x in FM.corpus() if x.name.startswith("stereo")):
        ch = (3, 1, 4, 3)[j]
        frames = values(rng, depth, (1, c.SH, c.SW, ch), 0.01)
        for k, m1type in enumerate((cv2.CV_16SC2, cv2.CV_32FC1, cv2.CV_32FC2)):
            inter = INTERS[(j + k) % 4]
            m1, m2 = FM.cv2_maps(c.name, m1type)
            if m1type == cv2.CV_16SC2:
                recs.append(_maps_record(inter, frames, m1, m2))
            else:
                recs.append(_fmaps_record(inter, frames, m1, m2))
            want.append((frames, inter, _remap_call(m1, m2, inter)))
    for (got, maps), (frames, inter, call), (_, c) in zip(_run(exe, tmp_path, recs), want, recs):
        if call is None:
            call = _remap_call(maps[0], maps[1], inter)
        _check(got, frames, inter, call, ("calib", c["mode"], inter))


@pytest.mark.parametrize("depth", DEPTHS, ids=DEPTH_IDS)
def test_warps(exe, tmp_path, depth):
    """MODE 2: cv2.warpPerspective with the corpus's homographies (horizons inside the canvas, exact W = 0 lines);
    MODE 3: cv2.warpAffine with random rotations, scales and shears, with and without WARP_INVERSE_MAP."""
    rng = np.random.default_rng(600 + depth)
    recs, want = [], []
    for i, c in enumerate(CC.corpus()[12::4]):
        ch, inter = (1, 3, 4)[i % 3], INTERS[i % 4]
        if cv2_warp_differs(2, depth, inter, ch):
            inter = cv2.INTER_CUBIC
        sw, sh = min(c.UW, 600), min(c.UH, 400)
        frames = values(rng, depth, (1, sh, sw, ch), 0.01)
        bw, bh = min(c.BW, 500), min(c.BH, 500)
        recs.append(_record(2, inter, frames, bw, bh, np.asarray(c.H, "<f8").tobytes()))
        want.append((frames, inter, lambda f, H=c.H, i=inter, s=(bw, bh): cv2.warpPerspective(f, H, s, flags=i)))
    for i in range(16):
        ch, inter, inv = (1, 3, 4)[i % 3], INTERS[i % 4], bool(i & 4)
        if cv2_warp_differs(3, depth, inter, ch):
            inter = cv2.INTER_LANCZOS4
        sw, sh, dw, dh = int(rng.integers(5, 90)), int(rng.integers(5, 70)), int(rng.integers(5, 90)), int(rng.integers(5, 70))
        frames = values(rng, depth, (1 + i % 3, sh, sw, ch), 0.02)
        M = np.array([[rng.uniform(-1.5, 1.5), rng.uniform(-1, 1), rng.uniform(-20, 40)],
                      [rng.uniform(-1, 1), rng.uniform(-1.5, 1.5), rng.uniform(-20, 40)]])
        recs.append(_record(3, inter, frames, dw, dh, M.astype("<f8").tobytes(), int(inv), row_pad=i % 3, img_pad=i % 2))
        fl = inter | (cv2.WARP_INVERSE_MAP if inv else 0)
        want.append((frames, inter, lambda f, M=M, fl=fl, s=(dw, dh): cv2.warpAffine(f, M, s, flags=fl)))
    for (got, _), (frames, inter, call), (_, c) in zip(_run(exe, tmp_path, recs), want, recs):
        _check(got, frames, inter, call, ("warp", c["mode"], inter))


@pytest.mark.parametrize("depth", DEPTHS, ids=DEPTH_IDS)
def test_value_extremes(exe, tmp_path, depth):
    """Sources dense with the depth's extremes (CUBIC and LANCZOS4 overshoot them and must saturate); float sources of
    +-inf, NaN, -0.0, denormals and FLT_MAX, among them NaN and inf taps whose weight is 0 (fraction 0, inside the frame
    and across its edges), windows of -0.0 only and of denormals only."""
    rng = np.random.default_rng(700 + depth)
    recs, want = [], []
    sw, sh, dw, dh = 23, 17, 64, 48
    fills = [values(rng, depth, (1, sh, sw, 4), 0.6)]
    if depth == 5:
        fills += [np.full((1, sh, sw, 4), -0.0, np.float32), np.full((1, sh, sw, 4), 1e-41, np.float32),
                  np.where(rng.random((1, sh, sw, 4)) < 0.5, np.float32(-0.0), np.float32(3e-39)).astype(np.float32)]
    else:
        info = np.iinfo(DEPTHS[depth])
        cb = (np.indices((sh, sw)).sum(0) % 2).astype(bool)[None, :, :, None]
        fills += [np.where(cb, info.max, info.min).astype(DEPTHS[depth]).repeat(4, -1)]
    for fi, base in enumerate(fills):
        for ch in (1, 3, 4):
            frames = np.ascontiguousarray(base[..., :ch])
            for inter in INTERS:
                m1 = np.stack([rng.integers(-9, sw + 9, (dh, dw)), rng.integers(-9, sh + 9, (dh, dw))], -1).astype(np.int16)
                m2 = rng.integers(0, 1024, (dh, dw)).astype(np.uint16)
                m2[rng.random((dh, dw)) < 0.3] = 0                     # zero weights beside the anchor tap
                m2[rng.random((dh, dw)) < 0.1] &= 31                   # fy = 0 only
                recs.append(_maps_record(inter, frames, m1, m2, row_pad=fi))
                want.append((frames, inter, _remap_call(m1, m2, inter)))
    for (got, _), (frames, inter, call) in zip(_run(exe, tmp_path, recs), want):
        _check(got, frames, inter, call, ("extremes", inter, frames.shape))


def test_cv2_warps_leave_remap():
    """The premise of the refusals, case by case, over 8 random homographies and affine matrices (both directions).  The
    source holds the values 0..255 at every depth, so that a warp that follows cv2.remap's arithmetic gives, at NEAREST,
    the bits of cv2's 8-bit warp (whose positions the gathers match at every depth) and, at LINEAR, the 16U result
    rint(32F result) (both are the same float sum, 16U rounded half to even; the 32F warps follow remap).  Every refused
    case (cv2_warp_differs) differs from that reference for some matrix; every other channel count, depth 16U / 16S / 32F
    at NEAREST, and 16U at LINEAR, equals it for all of them."""
    rng = np.random.default_rng(9)
    cases = []
    for _ in range(8):
        sw, sh, dw, dh = (int(v) for v in rng.integers(8, 80, 4))
        H = np.eye(3) + rng.normal(0, [[0.2, 0.2, 5], [0.2, 0.2, 5], [1e-3, 1e-3, 0]])
        M = np.array([[rng.uniform(-1.5, 1.5), rng.uniform(-1, 1), rng.uniform(-20, 40)],
                      [rng.uniform(-1, 1), rng.uniform(-1.5, 1.5), rng.uniform(-20, 40)]])
        cases.append((rng.integers(0, 256, (sh, sw, 4)), (dw, dh), H, M))
    warps = [(2, 0, lambda f, H, M, s, i: cv2.warpPerspective(f, H, s, flags=i)),
             (3, 0, lambda f, H, M, s, i: cv2.warpAffine(f, M, s, flags=i)),
             (3, cv2.WARP_INVERSE_MAP, lambda f, H, M, s, i: cv2.warpAffine(f, M, s, flags=i | cv2.WARP_INVERSE_MAP))]
    for mode, inv, warp in warps:
        for ch in (1, 3, 4):
            for inter, depths in ((cv2.INTER_NEAREST, (2, 3, 5)), (cv2.INTER_LINEAR, (2,))):
                for depth in depths:
                    differ = False
                    for img, s, H, M in cases:
                        src = img[..., :ch] if ch > 1 else img[..., 0]
                        got = warp(src.astype(DEPTHS[depth]), H, M, s, inter).astype(np.float64)
                        if inter == cv2.INTER_NEAREST:
                            ref = warp(src.astype(np.uint8), H, M, s, inter).astype(np.float64)
                        else:
                            ref = np.rint(warp(src.astype(np.float32), H, M, s, inter).astype(np.float64))
                        differ |= bool((got != ref).any())
                    assert differ == cv2_warp_differs(mode, depth, inter, ch), (mode, inv, depth, ch, inter)


def test_cv2_float_arithmetic_premises():
    """The premises the float gathers rest on, read off cv2: the -0.0 sign rule of each kernel inside the frame, a NaN
    tap with zero weight poisoning LINEAR, and CV_8S, CV_16F and CV_64F: the first two refused by cv2.remap."""
    img = np.full((12, 12), -0.0, np.float32)
    m1 = np.full((1, 1, 2), 4, np.int16)
    m2 = np.zeros((1, 1), np.uint16)
    sign = lambda i: bool(np.signbit(cv2.remap(img, m1, m2, i)[0, 0]))
    assert sign(cv2.INTER_LINEAR) and sign(cv2.INTER_CUBIC) and not sign(cv2.INTER_LANCZOS4)
    nan = np.zeros((4, 4), np.float32)
    nan[1, 2] = np.nan
    assert np.isnan(cv2.remap(nan, np.full((1, 1, 2), 1, np.int16), np.zeros((1, 1), np.uint16), cv2.INTER_LINEAR)[0, 0])
    for dt in (np.int8, np.float16):
        with pytest.raises(cv2.error):
            cv2.remap(np.zeros((4, 4), dt), np.zeros((2, 2, 2), np.int16), np.zeros((2, 2), np.uint16), cv2.INTER_LINEAR)
