"""The camera-model and homography arithmetic of the kernels on the CPU, over the seeded random calibrations of
tests/calib_cases.py: tests/host/kernel_math.cu runs the very coordinate code the kernels run (undistort_point,
quantise_uv, warp_point, warp_maps_pixel; host forms, no FMA contraction) and the result is compared with cv2 byte for
byte.  A difference here is a formula or evaluation-order difference; one that only tests/test_gpu_calib_fuzz.py shows
comes from the device math library."""
import os
import shutil
import subprocess

import cv2
import numpy as np
import pytest

from cameracalibration_b200.build import GENCODE
from oracle import restate as R
from tests import calib_cases as CC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    nvcc = next((c for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc") if c and os.path.exists(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("calib_math") / "kernel_math"
    build = subprocess.run([nvcc, "-O2", "-std=c++17", "--fmad=false", "-Xcompiler", "-ffp-contract=off", *GENCODE, "-o", str(out),
                            os.path.join(ROOT, "tests", "host", "kernel_math.cu")], capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stdout + build.stderr
    return str(out)


def _run(exe, args, values):
    r = subprocess.run([exe] + [str(a) for a in args], input=" ".join(float(v).hex() for v in values), capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)


def _planes(path, w, h):
    raw = np.fromfile(path, np.uint8)
    return raw[:w * h * 4].view(np.int16).reshape(h, w, 2), raw[w * h * 4:].view(np.uint16).reshape(h, w)


def test_calib_corpus_reaches_every_class():
    """The corpus holds every class of input that moves the coordinate arithmetic, so that thinning it fails here."""
    cases = CC.corpus()
    fish = [c for c in cases if c.fisheye]
    pin = [c for c in cases if not c.fisheye]
    # mild distortion at real sizes: 3840x2160, and 2560x2048 at SIZE_SCALE 2; SIZE_SCALE 1.5; offsets of the principal point
    assert any((c.UW, c.UH) == (3840, 2160) for c in fish)
    assert any((c.UW, c.UH, c.SS) == (2560, 2048, 2.0) for c in cases)
    assert {c.SS for c in cases} >= {1.0, 1.5, 2.0} and {c.model for c in cases if c.SS != 1} == {0, 1}
    assert any(c.P[0, 2] != c.UW / 2 for c in cases)
    # pinhole vector body: widths with W % 8 in {0, 1, 7}; int16 saturation of map1 (saturating pack) and, on fisheye
    # maps and the scalar tail, entries that wrap; cvRound's INT_MIN for |u*32| >= 2^31
    assert {c.UW % 8 for c in pin if c.kind == "strong"} >= {0, 1, 7}
    big = {}
    for c in cases:
        if c.kind == "strong":
            u, v = CC.uv32(c)
            big[c.name] = np.nanmax(np.abs(np.where(np.isfinite(u), u, 0)))
            big[c.name + "v"] = np.nanmax(np.abs(np.where(np.isfinite(v), v, 0)))
    assert any(b >= 2.0 ** 31 for b in big.values())
    assert any(32768 * 32 <= b < 2.0 ** 31 for b in big.values())
    m1s = [(c, CC.cv2_maps(c.name)[0]) for c in cases if c.kind == "strong"]
    assert any(((m1 == 32767) | (m1 == -32768)).any() for c, m1 in m1s if not c.fisheye)
    # fisheye rays behind the camera (_w <= 0 gives infinities) are not reachable with R = I; wraps show as sign flips
    assert any((np.abs(np.diff(m1[..., 0].astype(np.int32), axis=1)) > 30000).any() for c, m1 in m1s if c.fisheye)
    # canvases: widths that are not multiples of 64 (and one that is), W % 4 != 0; strong perspective with the horizon
    # inside the canvas, W == 0 exactly at some pixels; pre-images that leave the undistorted frame
    assert any(c.BW % 64 == 0 for c in cases) and any(c.BW % 64 and c.BW < 64 for c in cases)
    assert any(c.UW % 4 for c in cases) and any(c.BW % 4 for c in cases)
    assert {c.horizon for c in fish} == {"none", "inside", "zero"} and {c.horizon for c in pin} == {"none", "inside", "zero"}
    leave = 0
    for c in cases:
        Hi = np.linalg.inv(c.H)
        yy, xx = np.mgrid[0:c.BH, 0:c.BW]
        W = Hi[2, 0] * xx + Hi[2, 1] * yy + Hi[2, 2]
        assert (c.horizon != "none") == bool((W <= 0).any()), c.name
        assert c.horizon != "zero" or (W == 0).any(), c.name
        with np.errstate(all="ignore"):
            X = (Hi[0, 0] * xx + Hi[0, 1] * yy + Hi[0, 2]) / W
            Y = (Hi[1, 0] * xx + Hi[1, 1] * yy + Hi[1, 2]) / W
        leave += bool((((X < 0) | (X >= c.UW) | (Y < 0) | (Y >= c.UH)) & (W > 0)).any())
    assert leave >= len(cases) // 3


def test_undistort_map_code_vs_cv2_random_calibrations(exe, tmp_path):
    """k_undistort_map / the fused gathers' camera model (kernel_math maps) == cv2.fisheye.initUndistortRectifyMap /
    cv2.initUndistortRectifyMap, every entry of every case (about 73 M).  The one tolerated difference, for the pinhole
    model whose cv2 build contracts into FMAs in its AVX2 dispatch (DESIGN.md section 7): map2 fractions of an axis whose
    map1 (equal to cv2's) lies outside any frame, with identical remapped images -- a handful of entries in all."""
    n = n_tolerated = 0
    for c in CC.corpus():
        out = tmp_path / "maps.bin"
        _run(exe, ["maps", c.model, c.UW, c.UH, out], list(c.K.ravel()) + list(c.d5) + list(c.P.ravel()))
        got, want = _planes(out, c.UW, c.UH), CC.cv2_maps(c.name)
        n += c.UW * c.UH
        same = (got[0] == want[0]).all() and (got[1] == want[1]).all()
        if not same:
            assert CC.pinhole_outside_only(c, got, want), CC.first_diffs(c, got, want)
            assert CC.remaps_agree(c, got, want), c.name
            n_tolerated += int((got[1] != want[1]).sum())
    assert n > 70_000_000 and n_tolerated < 10


def test_bev_lut_code_vs_cv2_random_calibrations(exe, tmp_path):
    """Camera.get_bev_maps the way bevk_bev_set_camera builds it (k_warp_maps<1>: the fisheye model at the four taps,
    FP32 plane interpolation) == cv2.warpPerspective of cv2's map planes, every fisheye case; and k_warp_maps<0> on
    cv2's planes of every case that fits in 1.5 M entries."""
    for c in CC.corpus():
        want = CC.cv2_bev_maps(c.name)
        if c.fisheye:
            out = tmp_path / "bev.bin"
            _run(exe, ["bevmaps", c.UW, c.UH, c.BW, c.BH, out], list(c.K.ravel()) + list(c.D) + list(c.P.ravel()) + list(c.H.ravel()))
            got = _planes(out, c.BW, c.BH)
            assert (got[0] == want[0]).all() and (got[1] == want[1]).all(), (c.name, CC.first_diffs(c, got, want))
        if c.UW * c.UH <= 1_500_000:
            m1, m2 = CC.cv2_maps(c.name)
            (tmp_path / "planes.bin").write_bytes(m1.tobytes() + m2.tobytes())
            _run(exe, ["warpmaps", c.UW, c.UH, c.BW, c.BH, tmp_path / "planes.bin", tmp_path / "warped.bin"], list(c.H.ravel()))
            got = _planes(tmp_path / "warped.bin", c.BW, c.BH)
            assert (got[0] == want[0]).all() and (got[1] == want[1]).all(), c.name


def test_warp_point_code_vs_cv2_random_homographies(exe, tmp_path):
    """warp_point (cv2.warpPerspective's fixed-point pre-image, 64-pixel blocks, W == 0 guard) for every case's
    homography, units 32 and 1, against the restated coordinates and against cv2.warpPerspective of an index image."""
    for c in CC.corpus():
        out = tmp_path / "warp.bin"
        for unit in (32, 1):
            _run(exe, ["warp", c.BW, c.BH, unit, out], list(c.H.ravel()))
            xy = np.fromfile(out, np.int32).reshape(c.BH, c.BW, 2)
            X, Y = R.warp_coords(c.H, c.BW, c.BH, unit)
            assert (xy[..., 0] == X).all() and (xy[..., 1] == Y).all(), (c.name, unit)
        sw, sh = min(c.UW, 2048), min(c.UH, 2048)
        idx = (np.arange(sw * sh, dtype=np.int64) % 251).astype(np.uint8).reshape(sh, sw)
        want = cv2.warpPerspective(idx, c.H, (c.BW, c.BH), flags=cv2.INTER_NEAREST)
        sx, sy = xy[..., 0], xy[..., 1]
        inside = (sx >= 0) & (sx < sw) & (sy >= 0) & (sy < sh)
        assert (np.where(inside, idx[np.clip(sy, 0, sh - 1), np.clip(sx, 0, sw - 1)], 0) == want).all(), c.name
