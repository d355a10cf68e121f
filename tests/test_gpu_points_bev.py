"""Points between camera frames and the BEV canvas on the GPU: BevEngine.camera_to_canvas / canvas_to_camera,
BevGenerator.points_to_bev / points_from_bev and InCalibrator.undistort_points against the cv2 chains they are defined
as, written out here, for the four reference cameras of tests/golden/fixtures.npz (and a pinhole with their D5) over
the whole canvas grid and the whole raw-frame grid, NumPy and CUDA points, bit for bit."""
import cv2
import numpy as np
import pytest

from cameracalibration_b200 import ops
from cameracalibration_b200.IntrinsicCalibration.intrinsicCalib import InCalibrator
from cameracalibration_b200.SurroundBirdEyeView.surroundBEV import BevGenerator
from oracle import cv2_path as C
from tests import points_cases as PC
from tests.helpers import NAMES

pytestmark = pytest.mark.gpu


def _grid(w, h, dtype=np.float32):
    ys, xs = np.mgrid[0:h, 0:w]
    return np.stack([xs, ys], -1).reshape(-1, 1, 2).astype(dtype)


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _host(t):
    import torch
    torch.cuda.synchronize()
    return t.cpu().numpy()


def _to_canvas(model, K, D, P, H, pts):
    und = cv2.fisheye.undistortPoints(pts, K, D, P=P) if model == "fisheye" else cv2.undistortPoints(pts, K, D, P=P)
    return cv2.perspectiveTransform(und, H)


def _from_canvas(model, K, D, P, H, pts):
    xy = cv2.undistortPoints(cv2.perspectiveTransform(pts, cv2.invert(H)[1]), P, None)
    if model == "fisheye":
        return cv2.fisheye.distortPoints(xy, K, D)
    xyz = np.concatenate([xy, np.ones_like(xy[..., :1])], -1)
    return cv2.projectPoints(xyz, np.zeros(3), np.zeros(3), K, D)[0]


def _check(eng, cam, model, K, D, P, H, g, dtype):
    raw, canvas = _grid(g.FW, g.FH, dtype), _grid(g.BW, g.BH, dtype)
    for pts, got_fn, want_fn in ((raw, eng.camera_to_canvas, _to_canvas), (canvas, eng.canvas_to_camera, _from_canvas)):
        want = want_fn(model, K, D, P, H, pts)
        assert PC.same(got_fn(cam, pts), want), (cam, got_fn.__name__, "numpy")
        assert PC.same(_host(got_fn(cam, _cuda(pts))), want), (cam, got_fn.__name__, "cuda")


def test_bev_engine_point_mappings_vs_cv2_chains(fx):
    g = fx.geometry()
    calib = fx.scaled_calib(g)
    eng = ops.BevEngine(5, (g.FW, g.FH), (g.BW, g.BH))
    und = (int(g.FW * g.SS), int(g.FH * g.SS))
    for i, n in enumerate(NAMES):
        K, D, H = calib[n]
        P = C.dst_camera_matrix(K, g.FW, g.FH, g.FS, g.SS)
        eng.set_camera(i, K, D, P, und, H)
        _check(eng, i, "fisheye", K, np.asarray(D, np.float64).reshape(-1)[:4], P, H, g, np.float32)
    K, _, H = calib["front"]
    P = C.dst_camera_matrix(K, g.FW, g.FH, g.FS, g.SS)
    eng.set_camera(4, K, fx.D5, P, und, H, model="pinhole")
    for dtype in (np.float32, np.float64):
        _check(eng, 4, "pinhole", K, np.asarray(fx.D5, np.float64).reshape(-1), P, H, g, dtype)


def test_bev_generator_and_incalibrator_points(fx):
    gen = BevGenerator(calib=fx.calib)
    g = gen._g
    pts = np.ascontiguousarray(_grid(g.FW, g.FH)[::7])   # cv2.fisheye.undistortPoints misreads strided views
    canvas = np.ascontiguousarray(_grid(g.BW, g.BH)[::5])
    for name, cam in zip(NAMES, gen.cameras):
        D = np.asarray(cam.dist_coeff, np.float64).reshape(-1)[:4]
        assert PC.same(gen.points_to_bev(name, pts),
                       _to_canvas("fisheye", cam.camera_mat, D, cam.camera_mat_dst, cam.homography, pts)), name
        assert PC.same(gen.points_from_bev(name, canvas),
                       _from_canvas("fisheye", cam.camera_mat, D, cam.camera_mat_dst, cam.homography, canvas)), name
    for kind, D in (("fisheye", fx.calib["front"][1]), ("normal", fx.D5)):
        inc = InCalibrator(kind)
        K = fx.calib["front"][0]
        inc.set_calibration(K, D)
        P = inc.camera._get_camera_mat_dst(K)
        d = np.asarray(D, np.float64)
        want = cv2.fisheye.undistortPoints(pts, K, d, P=P) if kind == "fisheye" else cv2.undistortPoints(pts, K, d, P=P)
        assert PC.same(inc.undistort_points(pts), want), kind
        assert PC.same(_host(inc.undistort_points(_cuda(pts))), want), kind
