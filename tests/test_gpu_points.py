"""cv2's point functions on the GPU: the corpus of tests/points_cases.py through every ops wrapper on NumPy and CUDA
points, compared with live cv2 bit for bit (float32 fisheye included, with no tolerance), plus every accepted layout,
n = 0, 1 and 1 M, in-place calls, one CUDA-graph capture replayed on new points, and the refusals."""
import ctypes as C

import cv2
import numpy as np
import pytest

from cameracalibration_b200 import _lib as L
from cameracalibration_b200 import ops
from tests import points_cases as PC

pytestmark = pytest.mark.gpu


def _ops_call(c, pts, inplace=False):
    if c.op == "undistort" and c.model == "pinhole":
        return ops.undistort_points_iter(pts, PC.K, c.D, c.R, c.P, c.criteria, inplace=inplace)
    if c.op == "undistort":
        return ops.fisheye_undistort_points(pts, PC.K, c.D, R=c.R, P=c.P, criteria=c.criteria, inplace=inplace)
    if c.op == "project" and c.model == "pinhole":
        pts_, jac = ops.project_points(pts, c.rvec, c.tvec, PC.K, c.D)
        assert jac is None
        return pts_
    if c.op == "project":
        return ops.fisheye_project_points(pts, c.rvec, c.tvec, PC.K, c.D, alpha=c.alpha)[0]
    if c.op == "distort":
        return ops.fisheye_distort_points(pts, PC.K, c.D, alpha=c.alpha, inplace=inplace)
    return ops.perspective_transform(pts, c.M, inplace=inplace)


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _host(t):
    import torch
    torch.cuda.synchronize()
    return t.cpu().numpy()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_points_corpus_vs_cv2(dtype):
    for c in PC.corpus():
        pts = PC.points(c, 20000, dtype, seed=len(c.name))
        if not PC.supported(c, dtype):
            with pytest.raises(L.BevkError):
                _ops_call(c, pts)
            continue
        want = PC.cv2_points(c, pts)
        assert PC.same(_ops_call(c, pts), want), (c.name, "numpy")
        assert PC.same(_host(_ops_call(c, _cuda(pts))), want), (c.name, "cuda")


def test_points_million_float32():
    """1 M points of every op (float32, device-resident) == cv2."""
    for name in ("und_pin14_tilt_RP", "und_fish_RP", "proj_pin8", "proj_fish_alpha", "dist_fish", "persp"):
        c = next(c for c in PC.corpus() if c.name == name)
        pts = PC.points(c, 1 << 20, np.float32, seed=7)
        assert PC.same(_host(_ops_call(c, _cuda(pts))), PC.cv2_points(c, pts)), name


def test_layouts_and_sizes():
    c = next(c for c in PC.corpus() if c.name == "und_pin5_RP")
    f = next(c for c in PC.corpus() if c.name == "und_fish_P")
    p = PC.points(c, 100, np.float32)
    flat = p.reshape(-1, 2)
    for src in (p, p.reshape(1, -1, 2), flat, flat[:1], p[:1]):
        want = cv2.undistortPoints(src, PC.K, c.D, R=c.R, P=c.P)
        got = ops.undistort_points(src, PC.K, c.D, R=c.R, P=c.P)
        assert PC.same(got, want), src.shape
        assert PC.same(_host(ops.undistort_points(_cuda(src), PC.K, c.D, R=c.R, P=c.P)), want), src.shape
    for src in (p, p.reshape(1, -1, 2)):
        want = cv2.fisheye.undistortPoints(src, PC.K, f.D, P=f.P)
        assert PC.same(ops.fisheye_undistort_points(src, PC.K, f.D, P=f.P), want), src.shape
        assert PC.same(ops.perspective_transform(src, PC.H), cv2.perspectiveTransform(src, PC.H)), src.shape
    with pytest.raises(L.BevkError):
        ops.fisheye_undistort_points(flat, PC.K, f.D)           # cv2's fisheye takes [N][1][2] / [1][N][2] only
    obj = PC.points(next(c for c in PC.corpus() if c.op == "project"), 50, np.float64)
    for src in (obj, obj.reshape(1, -1, 3), obj.reshape(-1, 3)):
        want = cv2.projectPoints(src, np.array([0.1, 0.2, 0.3]), np.zeros(3), PC.K, None)[0]
        assert PC.same(ops.project_points(src, np.array([0.1, 0.2, 0.3]), np.zeros(3), PC.K, None)[0], want)
    empty = ops.undistort_points(np.zeros((0, 1, 2), np.float32), PC.K, c.D)
    assert empty.shape == (0, 1, 2) and empty.dtype == np.float32
    assert _host(ops.perspective_transform(_cuda(np.zeros((0, 1, 2), np.float32)), PC.H)).shape == (0, 1, 2)


def _layout(p, layout):
    return {"N12": p, "1N2": p.reshape(1, -1, p.shape[-1]), "N2": p.reshape(-1, p.shape[-1])}[layout]


def test_every_op_layout_size_and_dtype():
    """One case of every op at each of PC.SIZES (0, 1, 1 M), PC.LAYOUTS cv2 accepts for it and PC.DTYPES."""
    for name in ("und_pin5_RP", "und_fish_P", "proj_pin5", "proj_fish", "dist_fish", "persp"):
        c = next(c for c in PC.corpus() if c.name == name)
        for dtype in PC.DTYPES:
            for n in PC.SIZES:
                base = PC.points(c, n, dtype, seed=n)[:n]
                for layout in PC.LAYOUTS:
                    if layout == "N2" and (c.model == "fisheye" or c.op in ("distort", "perspective")):
                        continue   # cv2 takes [N][2] in its pinhole functions only
                    pts = _layout(base, layout)
                    if not PC.supported(c, dtype):
                        with pytest.raises(L.BevkError):
                            _ops_call(c, pts)
                        continue
                    got, dev = _ops_call(c, pts), _host(_ops_call(c, _cuda(pts)))
                    if n == 0:   # cv2 returns None or raises on no points; the library returns an empty array
                        assert got.size == 0 and dev.size == 0 and got.dtype == np.dtype(dtype)
                        continue
                    want = PC.cv2_points(c, pts)
                    assert PC.same(got, want) and PC.same(dev, want), (name, np.dtype(dtype).name, n, layout)


def test_in_place():
    for name in ("und_pin8_RP", "und_fish_RP", "dist_fish", "persp"):
        c = next(c for c in PC.corpus() if c.name == name)
        pts = PC.points(c, 5000, np.float32, seed=3)
        want = PC.cv2_points(c, pts)
        h = pts.copy()
        assert _ops_call(c, h, inplace=True) is h and PC.same(h.reshape(-1, 1, 2), want.reshape(-1, 1, 2)), name
        d = _cuda(pts)
        _ops_call(c, d, inplace=True)
        assert PC.same(_host(d).reshape(-1, 1, 2), want.reshape(-1, 1, 2)), name


def test_graph_capture_replays_on_new_points():
    """One capture of a device call on the ctx stream, replayed after the points were overwritten."""
    import torch
    ctx = L.Context(0)
    a = PC.points(PC.Case("p", "perspective", M=PC.H), 4096, np.float32, seed=1)
    b = PC.points(PC.Case("p", "perspective", M=PC.H), 4096, np.float32, seed=2)
    src, dst = _cuda(a), torch.empty(a.shape, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    with ctx.graph_capture() as g:
        L.check(ctx.lib.bevk_perspective_transform(ctx.h, C.c_void_p(src.data_ptr()), C.c_void_p(dst.data_ptr()), a.shape[0],
                                                   5, L.dptr(PC.H), 1))   # 5: BEVK_CV_32F
    g.launch()
    ctx.sync()
    assert PC.same(dst.cpu().numpy(), cv2.perspectiveTransform(a, PC.H))
    src.copy_(torch.from_numpy(b))
    torch.cuda.synchronize()
    g.launch()
    ctx.sync()
    assert PC.same(dst.cpu().numpy(), cv2.perspectiveTransform(b, PC.H))
    g.destroy()


def test_refusals():
    p32 = np.zeros((4, 1, 2), np.float32)
    p64 = p32.astype(np.float64)
    for call in (lambda: ops.undistort_points(p32, PC.K, np.zeros(3)),                          # D length cv2 refuses
                 lambda: ops.fisheye_undistort_points(p32, PC.K, np.zeros(5)),
                 lambda: ops.fisheye_undistort_points(p64, PC.K, PC.D_FISH),                   # float64 fisheye
                 lambda: ops.fisheye_distort_points(p64, PC.K, PC.D_FISH),
                 lambda: ops.fisheye_project_points(np.zeros((4, 1, 3)), np.zeros(3), np.zeros(3), PC.K, PC.D_FISH),
                 lambda: ops.undistort_points_iter(p32, PC.K, np.zeros(5), None, None, (1, 1001, 0.)),  # > 1000
                 lambda: ops.undistort_points_iter(p32, PC.K, np.zeros(5), None, None, (3, 5, 0.01)),   # pinhole EPS
                 lambda: ops.fisheye_undistort_points(p32, PC.K, PC.D_FISH, criteria=(2, 10, 1e-8)),  # no COUNT
                 lambda: ops.undistort_points(p32.astype(np.float16), PC.K, None),
                 lambda: ops.perspective_transform(np.zeros((4, 1, 3), np.float32), PC.H)):
        with pytest.raises(L.BevkError):
            call()
    # in place needs a writeable C-contiguous destination of the points' dtype
    big = np.zeros((8, 1, 2), np.float32)
    ro = p32.copy()
    ro.flags.writeable = False
    for bad in (big[::2], big[::-1], ro):
        before = big.copy()
        with pytest.raises(L.BevkError):
            ops.perspective_transform(bad, PC.H, inplace=True)
        assert (big == before).all()
    ctx = L.default_context()
    a = np.zeros(8, np.float32)
    # overlapping but not identical input and output
    assert ctx.lib.bevk_perspective_transform(ctx.h, L.vptr(a), C.c_void_p(a.ctypes.data + 4), 3, 5, L.dptr(PC.H), 0) == -1
    assert ctx.lib.bevk_perspective_transform(ctx.h, L.vptr(a), L.vptr(a), -1, 5, L.dptr(PC.H), 0) != 0
