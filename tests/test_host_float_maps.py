"""cv2's float maps on the CPU: tests/host/float_maps.cu runs the kernels' own code (undistort_map_f32_px<LENS> after
the library's camera set-up, convert_map_px, and MODE 4 of gather_frames, gather_taps_frames and gather4_frames; host
forms, no FMA contraction) over tests/float_map_cases.py, compared with live cv2.initUndistortRectifyMap,
cv2.convertMaps and cv2.remap bit for bit."""
import os
import shutil
import subprocess

import cv2
import numpy as np
import pytest

from cameracalibration_b200.build import GENCODE
from tests import float_map_cases as FC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INTERPS = (cv2.INTER_NEAREST, cv2.INTER_LINEAR, cv2.INTER_CUBIC, cv2.INTER_AREA, cv2.INTER_LANCZOS4)


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    nvcc = next((c for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc") if c and os.path.exists(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("float_maps") / "float_maps"
    build = subprocess.run([nvcc, "-O2", "-std=c++17", "--fmad=false", "-Xcompiler", "-ffp-contract=off", *GENCODE, "-o", str(out),
                            os.path.join(ROOT, "tests", "host", "float_maps.cu")], capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stdout + build.stderr
    return str(out)


def _run(exe, args, stdin=""):
    r = subprocess.run([exe] + [str(a) for a in args], input=stdin, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)


def host_maps(exe, tmp_path, c, m1type):
    out = tmp_path / "maps.bin"
    values = list(np.ravel(c.K)) + list(np.ravel(c.D)) + ([] if c.R is None else list(np.ravel(c.R))) + list(np.ravel(c.P))
    _run(exe, ["maps", c.model, c.W, c.H, c.D.size, int(c.R is not None), m1type, out], " ".join(float(v).hex() for v in values))
    raw = np.fromfile(out, np.float32)
    if m1type == cv2.CV_32FC2:
        return raw.reshape(c.H, c.W, 2), None
    n = c.W * c.H
    return raw[:n].reshape(c.H, c.W), raw[n:].reshape(c.H, c.W)


def test_float_map_corpus_reaches_every_class():
    k = FC.classes()
    assert k["pinhole_n"] == {4, 5, 8, 12, 14}
    assert k["pinhole_n_with_R"] == {4, 5, 8, 12, 14} and k["pinhole_n_without_R"] == {4, 5, 8, 12, 14}
    assert k["stereo"] == 2 and k["stereo_vertical"] == 2
    assert k["fisheye_R"] >= 2 and k["fisheye_no_R"] >= 1 and k["fisheye_inf"] >= 1
    assert k["w_mod8"] >= {0, 1, 7} and k["one_row"] >= 2
    for cls in ("tie32", "tie1", "nan", "inf", "-inf", "3e9", "near_1024", "near_32768", "near_32767"):
        assert k[cls] > 0, cls


def test_float_maps_vs_cv2(exe, tmp_path):
    """CV_32FC1 (both models) and CV_32FC2 (pinhole) maps of every camera == cv2's, bit for bit; a pinhole entry may
    differ only far outside the frame (float_map_cases.far_outside_only), with the same remapped image."""
    n_diff = 0
    for c in FC.corpus():
        for t in (cv2.CV_32FC1,) if c.fisheye else (cv2.CV_32FC1, cv2.CV_32FC2):
            got, want = host_maps(exe, tmp_path, c, t), FC.cv2_maps(c.name, t)
            if FC.same(got[0], want[0]) and FC.same(got[1], want[1]):
                continue
            assert FC.far_outside_only(c, got, want), c.name
            n_diff += int(sum((g != w).sum() for g, w in zip(FC.planes(got), FC.planes(want))))
            f = FC.frames(c, 3)[0]
            for i in (cv2.INTER_LINEAR, cv2.INTER_NEAREST):
                assert (cv2.remap(f, *got, i) == cv2.remap(f, *want, i)).all(), c.name
    assert n_diff < 100


def _convert(exe, tmp_path, m1, m2, intype, outtype, nn):
    h, w = m1.shape[:2]
    src, out = tmp_path / "cin.bin", tmp_path / "cout.bin"
    with open(src, "wb") as f:
        f.write(np.ascontiguousarray(m1).tobytes())
        if m2 is not None:
            f.write(np.ascontiguousarray(m2).tobytes())
    _run(exe, ["convert", intype, int(m2 is not None), outtype, int(nn), w, h, src, out])
    raw = np.fromfile(out, np.uint8)
    n = w * h
    if outtype == cv2.CV_16SC2:
        o1 = raw[:4 * n].view(np.int16).reshape(h, w, 2)
        return o1, (None if nn else raw[4 * n:].view(np.uint16).reshape(h, w))
    if outtype == cv2.CV_32FC2:
        return raw.view(np.float32).reshape(h, w, 2), None
    f = raw.view(np.float32)
    return f[:n].reshape(h, w), f[n:].reshape(h, w)


def _cv2_convert(m1, m2, t, nn):
    a, b = cv2.convertMaps(m1, m2, t, nninterpolation=nn)
    return a, (b if b is not None and b.size else None)


def _map_sets():
    for name, x, y, _, _ in FC.synthetic():
        yield name, x, y
    for c in FC.corpus():
        if c.W * c.H <= 400_000:
            yield c.name, *FC.cv2_maps(c.name, cv2.CV_32FC1)


def test_convert_maps_vs_cv2(exe, tmp_path):
    """convert_map_px == cv2.convertMaps for every conversion: 32FC1 <-> 32FC2, 32F -> 16SC2 (+16UC1) with and without
    nninterpolation, and 16SC2 (with map2 or none) -> 32FC1 / 32FC2."""
    for name, x, y in _map_sets():
        xy = np.dstack([x, y])
        for src, s1, s2 in ((cv2.CV_32FC1, x, y), (cv2.CV_32FC2, xy, None)):
            for t, nn in ((cv2.CV_16SC2, False), (cv2.CV_16SC2, True), (cv2.CV_32FC1 + cv2.CV_32FC2 - src, False)):
                got, want = _convert(exe, tmp_path, s1, s2, src, t, nn), _cv2_convert(s1, s2, t, nn)
                assert FC.same(got[0], want[0]) and FC.same(got[1], want[1]), (name, src, t, nn)
        i1, i2 = cv2.convertMaps(x, y, cv2.CV_16SC2)
        for m2 in (i2, None):
            # no map2 is a zero fraction; cv2 4.13 crashes converting a CV_16SC2 map1 alone to float, so the reference
            # gets the zeros explicitly
            ref2 = np.zeros(i1.shape[:2], np.uint16) if m2 is None else m2
            for t in (cv2.CV_32FC1, cv2.CV_32FC2):
                got, want = _convert(exe, tmp_path, i1, m2, cv2.CV_16SC2, t, False), _cv2_convert(i1, ref2, t, False)
                assert FC.same(got[0], want[0]) and FC.same(got[1], want[1]), (name, t, m2 is None)


def _remap(exe, tmp_path, src, m1, m2, interp, words=False):
    sh, sw = src.shape[:2]
    ch = 1 if src.ndim == 2 else src.shape[2]
    dh, dw = m1.shape[:2]
    fin, out = tmp_path / "rin.bin", tmp_path / "rout.bin"
    with open(fin, "wb") as f:
        f.write(np.ascontiguousarray(m1, np.float32).tobytes())
        if m2 is not None:
            f.write(np.ascontiguousarray(m2, np.float32).tobytes())
        f.write(np.ascontiguousarray(src).tobytes())
    t = cv2.CV_32FC1 if m2 is not None else cv2.CV_32FC2
    _run(exe, ["remap", ch, interp, t, sw, sh, dw, dh, int(words), fin, out])
    return np.fromfile(out, np.uint8).reshape((dh, dw) if ch == 1 else (dh, dw, ch))


def test_float_remap_vs_cv2(exe, tmp_path):
    """MODE 4 of the gathers == cv2.remap with float maps, for 1, 3 and 4 channels and every interpolation, through
    CV_32FC1 and CV_32FC2 maps; k_gather4's body too where it applies."""
    rng = np.random.default_rng(3)
    sets = list(FC.synthetic()) + [(c.name, *FC.cv2_maps(c.name, cv2.CV_32FC1), c.SW, c.SH)
                                   for c in FC.corpus() if c.name in ("pinhole8_R", "fisheye_behind", "pinhole5_row")]
    for name, x, y, sw, sh in sets:
        xy = np.dstack([x, y])
        for ch in (1, 3, 4):
            src = rng.integers(0, 256, (sh, sw, ch), dtype=np.uint8)
            src = src[..., 0] if ch == 1 else src
            for interp in INTERPS:
                want = cv2.remap(src, x, y, interp)
                assert (_remap(exe, tmp_path, src, x, y, interp) == want).all(), (name, ch, interp)
                assert (_remap(exe, tmp_path, src, xy, None, interp) == want).all(), (name, ch, interp, "32FC2")
            if ch == 3 and x.shape[1] % 4 == 0:
                want = cv2.remap(src, x, y, cv2.INTER_LINEAR)
                assert (_remap(exe, tmp_path, src, x, y, cv2.INTER_LINEAR, True) == want).all(), (name, "words")
                assert (_remap(exe, tmp_path, src, xy, None, cv2.INTER_LINEAR, True) == want).all(), (name, "words 32FC2")


def test_float_remap_is_convert_then_integer_remap():
    """The rule the gathers follow, pinned on cv2 itself: cv2.remap with float maps gives the bytes of
    cv2.convertMaps(..., CV_16SC2, nninterpolation = NEAREST) and the integer remap, and NEAREST is not the integer
    maps' rule (which rounds the fixed-point fraction instead)."""
    name, x, y, sw, sh = FC.synthetic()[0]
    src = np.random.default_rng(9).integers(0, 256, (sh, sw, 3), dtype=np.uint8)
    for interp in INTERPS:
        nn = interp == cv2.INTER_NEAREST
        m1, m2 = cv2.convertMaps(x, y, cv2.CV_16SC2, nninterpolation=nn)
        assert (cv2.remap(src, x, y, interp) == cv2.remap(src, m1, m2 if not nn else None, interp)).all(), interp
    m1, m2 = cv2.convertMaps(x, y, cv2.CV_16SC2)
    assert (cv2.remap(src, x, y, cv2.INTER_NEAREST) != cv2.remap(src, m1, m2, cv2.INTER_NEAREST)).any()
