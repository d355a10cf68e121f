"""cv2's point functions on the CPU: tests/host/points.cu runs the kernels' own per-point code (point_op of k_points,
after points_camera; host forms, no FMA contraction) over tests/points_cases.py and compares it with live cv2 bit for
bit, at float32 and float64 (the host has glibc's tan / atan, so the fisheye is exact at both)."""
import os
import shutil
import subprocess

import cv2
import numpy as np
import pytest

from cameracalibration_b200.build import GENCODE
from tests import points_cases as PC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OP = {"undistort": 0, "project": 1, "distort": 2, "perspective": 3}


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    nvcc = next((c for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc") if c and os.path.exists(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("points") / "points"
    build = subprocess.run([nvcc, "-O2", "-std=c++17", "--fmad=false", "-Xcompiler", "-ffp-contract=off", *GENCODE, "-o", str(out),
                            os.path.join(ROOT, "tests", "host", "points.cu")], capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stdout + build.stderr
    return str(out)


def host_points(exe, tmp_path, c, pts):
    """The kernel's per-point code on case c's points: [N][1][2], or the exit code when points_camera refuses."""
    pts = np.ascontiguousarray(pts)
    n = pts.shape[0] * pts.shape[1]
    D = [] if c.D is None else list(np.ravel(c.D))
    if c.op == "project":
        R = list(c.rvec)
    else:
        R = [] if c.R is None else list(np.ravel(c.R))
    K = PC.K if c.op != "perspective" else c.M
    vals = list(np.ravel(K)) + D + R + ([] if c.P is None else list(np.ravel(c.P))) + list(c.tvec) + [c.alpha, c.criteria[2]]
    src, dst = tmp_path / "in.bin", tmp_path / "out.bin"
    pts.tofile(src)
    args = [exe, "run", OP[c.op], int(c.model == "pinhole"), 6 if pts.dtype == np.float64 else 5, n, len(D), len(R),
            int(c.P is not None), c.criteria[0], c.criteria[1], src, dst]
    r = subprocess.run([str(a) for a in args], input=" ".join(float(v).hex() for v in vals), capture_output=True, text=True,
                       timeout=600)
    if r.returncode:
        return r.returncode
    return np.fromfile(dst, pts.dtype).reshape(-1, 1, 2)


def test_points_corpus_reaches_every_class():
    k = PC.classes()
    assert k["pinhole_n"] == {0, 4, 5, 8, 12, 14} and k["tilt"] >= 1
    assert k["fisheye_R"] >= 1 and k["fisheye_rvec"] >= 1 and k["fisheye_P"] >= 1 and k["fisheye_plain"] >= 1
    assert k["crit"] == {1, 3}
    assert k["ops"] == set(PC.OPS)
    for cls in ("z0", "z_neg", "w_small", "nan", "inf", "theta_clamped", "theta_flipped", "not_converged", "icdist_neg",
                "principal"):
        assert k[cls] > 0, cls
    assert 0 in PC.SIZES and 1 in PC.SIZES and max(PC.SIZES) >= 1 << 20
    assert set(PC.LAYOUTS) == {"N12", "1N2", "N2"} and {np.dtype(d) for d in PC.DTYPES} == {np.dtype(np.float32), np.dtype(np.float64)}


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_points_vs_cv2(exe, tmp_path, dtype):
    """Every case of the corpus == cv2 bit for bit (NaN as NaN), special points included."""
    for c in PC.corpus():
        pts = PC.points(c, 4000, dtype, seed=len(c.name))
        got, want = host_points(exe, tmp_path, c, pts), PC.cv2_points(c, pts)
        assert PC.same(got, want.reshape(-1, 1, 2)), (c.name, np.dtype(dtype).name)


def test_points_reach_the_special_branches(exe, tmp_path):
    """The corpus's points reach icdist < 0 (the restart), the fisheye's theta clamp, its -1e6 rule and its
    |theta_d| <= eps shortcut, and perspectiveTransform's zero output."""
    c = next(c for c in PC.corpus() if c.name == "und_pin5_barrel")
    pts = PC.points(c, 4000, np.float64)
    got = host_points(exe, tmp_path, c, pts).reshape(-1, 2)
    raw = (pts.reshape(-1, 2) - [PC.K[0, 2], PC.K[1, 2]]) * [1 / PC.K[0, 0], 1 / PC.K[1, 1]]
    assert (got == raw).all(1).sum() > 100   # restarted points come back as the raw normalised point
    f = next(c for c in PC.corpus() if c.name == "und_fish_noconv")
    fp = PC.points(f, 4000, np.float64)
    out = host_points(exe, tmp_path, f, fp).reshape(-1, 2)
    assert (out == -1e6).all(1).any()
    s = next(c for c in PC.corpus() if c.name == "und_fish_strong")
    assert (host_points(exe, tmp_path, s, PC.points(s, 10, np.float64)).reshape(-1, 2)[11] == 0).all()   # |theta_d| < eps
    p = next(c for c in PC.corpus() if c.name == "persp")
    pp = PC.points(p, 10, np.float32)
    assert (host_points(exe, tmp_path, p, pp).reshape(-1, 2)[10:18] == 0).all(1).any()


def test_rodrigues_vs_cv2(exe):
    rng = np.random.default_rng(5)
    for rv in [np.zeros(3), np.array([1e-17, 0, 0]), np.array([np.pi, 0, 0])] + list(rng.normal(0, 1.5, (50, 3))):
        r = subprocess.run([exe, "rodrigues"], input=" ".join(float(v).hex() for v in rv), capture_output=True, text=True)
        R = np.array([float.fromhex(x) for x in r.stdout.split()]).reshape(3, 3)
        assert PC.same(R, cv2.Rodrigues(np.asarray(rv, np.float64))[0]), rv


def test_refused_cameras(exe, tmp_path):
    """D lengths cv2 refuses, a criteria without COUNT (cv2 would iterate without bound), more than 1000 iterations and
    the pinhole EPS criterion (its reprojection-error stop is not restated) are refused."""
    pts = PC.points(PC.Case("x", "undistort"), 4, np.float32)
    for c in (PC.Case("d3", "undistort", D=np.zeros(3)), PC.Case("d6", "project", D=np.zeros(6)),
              PC.Case("f5", "undistort", "fisheye", np.zeros(5)), PC.Case("eps", "undistort", "fisheye", PC.D_FISH,
                                                                            criteria=(2, 10, 1e-8)),
              PC.Case("many", "undistort", D=np.zeros(5), criteria=(1, 1001, 0.)),
              PC.Case("pin_eps", "undistort", D=np.zeros(5), criteria=(3, 5, 0.01))):
        assert host_points(exe, tmp_path, c, pts if c.op != "project" else PC.points(c, 4, np.float32)) == 3, c.name
