"""GPU test of cv2's rational, thin-prism and tilted pinhole models and of rectification rotations: the maps of
bevk_undistort_rectify_map, Undistorter slots (map-resident and fused) on host frames, device batches, a captured graph
and the JPEG / PNG encoders, and BEV cameras of the pinhole model (bevk_bev_set_camera_model), every output byte equal
to cv2 with cv2's own maps (tests/lens_cases.py)."""
import ctypes

import cv2
import numpy as np
import pytest

from oracle import cv2_path as C
from oracle import restate as RS
from tests import calib_cases as CC
from tests import lens_cases as LC

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


def _small(name, w=None, h=None):
    """The case's camera at a small undistorted size (K and P scaled with it), and cv2's maps there."""
    c = LC.case_by_name(name)
    w, h = w or c.UW, h or c.UH
    S = np.diag([w / c.UW, h / c.UH, 1.0])
    K, P = S @ c.K, S @ c.P
    R = np.eye(3) if c.R is None else c.R
    if c.fisheye:
        maps = cv2.fisheye.initUndistortRectifyMap(K, c.D.reshape(4, 1), R, P, (w, h), cv2.CV_16SC2)
    else:
        maps = cv2.initUndistortRectifyMap(K, c.D, R, P, (w, h), cv2.CV_16SC2)
    return c, K, P, maps


def _want(maps, frame, interp=cv2.INTER_LINEAR):
    out = cv2.remap(np.ascontiguousarray(frame), maps[0], maps[1], interp)
    return out.reshape(out.shape[0], out.shape[1], -1)


def test_rectify_maps_vs_cv2():
    """bevk_undistort_rectify_map == cv2.initUndistortRectifyMap / cv2.fisheye.initUndistortRectifyMap with R, every
    case: no tolerance for the fisheye (whose rotated rays are walked row by row), pinhole_outside_only for the pinhole."""
    from cameracalibration_b200 import ops
    for c in LC.corpus():
        fn = ops.fisheye_init_undistort_rectify_map if c.fisheye else ops.init_undistort_rectify_map
        got = fn(c.K, c.D, c.P, (c.UW, c.UH), R=np.eye(3) if c.R is None else c.R)
        want = LC.cv2_maps(c.name)
        if not ((got[0] == want[0]).all() and (got[1] == want[1]).all()):
            assert not c.fisheye and LC.outside_only(c, got, want), LC.first_diffs(c, got, want)


INTERPS = (cv2.INTER_NEAREST, cv2.INTER_LINEAR, cv2.INTER_CUBIC, cv2.INTER_LANCZOS4)


@pytest.mark.parametrize("name", ["real14_8", "strong12_1", "strong8_9", "stereo5_1", "rotated3"])
@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("size", [(200, 120), (201, 121), (207, 119)])
def test_undistorter_slots(torch, name, fused, size):
    """Undistorter map-resident and fused slots (a rotated fisheye: map-resident only), 1/3/4 channels, NEAREST /
    LINEAR / CUBIC / LANCZOS4, on host frames and device batches of 1, 3 and 9, widths with W % 8 in {0, 1, 7} (the
    pinhole vector body's saturating pack ends at W - W % 8), against cv2.remap through cv2's maps.  The slot's maps()
    equal cv2's, or differ only as calib_cases.pinhole_outside_only allows: then the images are compared with cv2.remap
    through the slot's maps, since CUBIC and LANCZOS4 windows of an entry at map1 = -2 still reach into the frame."""
    from cameracalibration_b200 import ops
    from cameracalibration_b200 import _lib as L
    w, h = size
    c, K, P, maps = _small(name, w, h)
    model = "fisheye" if c.fisheye else "pinhole"
    if fused and c.fisheye:
        with pytest.raises(L.BevkError, match="map-resident"):
            ops.Undistorter(K, c.D, P, size, model=model, fused=True, R=c.R)
        return
    u = ops.Undistorter(K, c.D, P, size, model=model, fused=fused, R=c.R)
    m = u.maps()
    exact = (m[0] == maps[0]).all() and (m[1] == maps[1]).all()
    assert exact or (not c.fisheye and LC.outside_only(c, m, maps)), LC.first_diffs(c, m, maps)
    if not exact:
        maps = m
    rng = np.random.default_rng(5 + fused)
    for ch in (1, 3, 4):
        host = rng.integers(0, 256, (9, 160, 240, ch), dtype=np.uint8)
        for interp in INTERPS:
            one = u(host[0] if ch > 1 else host[0, :, :, 0], interpolation=interp)
            assert (one.reshape(h, w, -1) == _want(maps, host[0], interp)).all(), (ch, interp)
            for n in (1, 3, 9):
                got = u.cuda(torch.from_numpy(host[:n]).cuda(), interpolation=interp).cpu().numpy()
                for i in range(n):
                    assert (got[i].reshape(h, w, -1) == _want(maps, host[i], interp)).all(), (ch, interp, n, i)
    u.close()


def test_graph_replay_fused_rational(torch):
    """A fused 14-coefficient slot captured in a CUDA graph and replayed over rewritten frames."""
    from cameracalibration_b200 import ops
    c, K, P, maps = _small("real14_2", 128, 96)
    u = ops.Undistorter(K, c.D, P, (128, 96), model="pinhole", fused=True)
    rng = np.random.default_rng(3)
    n = 4
    frames = torch.from_numpy(rng.integers(0, 256, (n, 100, 140, 3), dtype=np.uint8)).cuda()
    out = torch.empty((n, 96, 128, 3), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    lib, ctx = u.ctx.lib, u.ctx
    call = lambda: lib.bevk_undistort_stack(ctx.h, u.slot, ctypes.c_void_p(frames.data_ptr()), 100 * 140 * 3, 140, 100, 140 * 3,
                                            3, n, ctypes.c_void_p(out.data_ptr()), 96 * 128 * 3, 128, 96, 128 * 3, 1)
    assert call() == 0
    ctx.sync()
    with ctx.graph_capture() as g:
        assert call() == 0
    for rep in range(2):
        host = rng.integers(0, 256, (n, 100, 140, 3), dtype=np.uint8)
        frames.copy_(torch.from_numpy(host))
        out.fill_(0)
        torch.cuda.synchronize()
        g.launch()
        ctx.sync()
        got = out.cpu().numpy()
        for i in range(n):
            assert (got[i] == _want(maps, host[i])).all(), (rep, i)
    g.destroy()
    u.close()


def test_jpeg_png_streams(torch):
    """.jpeg / .png / .cuda_to_jpeg of a tilted-model slot == cv2.imencode of cv2.remap."""
    from cameracalibration_b200 import ops
    c, K, P, maps = _small("real14_5", 160, 96)
    u = ops.Undistorter(K, c.D, P, (160, 96), model="pinhole", R=c.R)
    rng = np.random.default_rng(9)
    host = rng.integers(0, 256, (3, 90, 150, 3), dtype=np.uint8)
    want = [_want(maps, f) for f in host]
    assert u.jpeg(host[0], quality=90) == cv2.imencode(".jpg", want[0], [cv2.IMWRITE_JPEG_QUALITY, 90])[1].tobytes()
    assert u.png(host[1]) == cv2.imencode(".png", want[1])[1].tobytes()
    streams = u.cuda_to_jpeg(torch.from_numpy(host).cuda(), quality=75)
    for s, w in zip(streams, want):
        assert s == cv2.imencode(".jpg", w, [cv2.IMWRITE_JPEG_QUALITY, 75])[1].tobytes()
    u.close()


def test_old_entry_points_take_8_coefficients():
    """bevk_undistort_map, bevk_undistorter_set and InCalibrator("normal") with 8 coefficients == the new entry point."""
    from cameracalibration_b200 import ops
    from cameracalibration_b200.IntrinsicCalibration.intrinsicCalib import InCalibrator
    c, K, P, maps = _small("real8_0", 200, 160)
    new = ops.init_undistort_rectify_map(K, c.D, P, (200, 160), R=np.eye(3))
    old = ops.init_undistort_rectify_map(K, c.D, P, (200, 160))
    assert (new[0] == old[0]).all() and (new[1] == old[1]).all()
    assert ((new[0] == maps[0]).all() and (new[1] == maps[1]).all()) or LC.outside_only(c, new, maps)
    for fused in (False, True):
        u = ops.Undistorter(K, c.D, P, (200, 160), model="pinhole", fused=fused)
        m = u.maps()
        assert (m[0] == new[0]).all() and (m[1] == new[1]).all(), fused
        u.close()
    ic = InCalibrator("normal")
    d = ic.set_calibration(c.K, c.D)
    m = d._und.maps()
    want = ops.init_undistort_rectify_map(c.K, c.D, ic.camera._get_camera_mat_dst(c.K), (m[0].shape[1], m[0].shape[0]),
                                          R=np.eye(3))
    assert (m[0] == want[0]).all() and (m[1] == want[1]).all()


def test_rectify_refusals():
    """D lengths cv2 refuses, on every new entry point; the fused rotated fisheye names the map-resident slot."""
    from cameracalibration_b200 import ops
    from cameracalibration_b200 import _lib as L
    c, K, P, _ = _small("real8_0", 64, 48)
    for n in (3, 6, 15):
        with pytest.raises(L.BevkError, match="coefficients"):
            ops.init_undistort_rectify_map(K, np.full(n, 0.01), P, (64, 48), R=np.eye(3))
        with pytest.raises(L.BevkError, match="coefficients"):
            ops.Undistorter(K, np.full(n, 0.01), P, (64, 48), model="pinhole", R=np.eye(3))
    with pytest.raises(L.BevkError, match="coefficients"):
        ops.fisheye_init_undistort_rectify_map(K, np.full(5, 0.01), P, (64, 48), R=np.eye(3))
    eng = ops.BevEngine(1, (64, 48), (40, 30))
    with pytest.raises(L.BevkError, match="coefficients"):
        eng.set_camera(0, K, np.full(6, 0.01), P, (64, 48), np.eye(3), model="pinhole")
    r, Kr, Pr, _ = _small("rotated1", 128, 96)
    with pytest.raises(L.BevkError, match="map-resident"):
        ops.Undistorter(Kr, r.D, Pr, (128, 96), fused=True, R=r.R)


def _pinhole_calib(fx, g, n):
    """fx's four cameras scaled to geometry g, as pinhole cameras with n coefficients (seeded per camera)."""
    calib = fx.scaled_calib(g)
    out = {}
    for i, name in enumerate(("front", "back", "left", "right")):
        K, D4, H = calib[name]
        rng = np.random.default_rng(100 * n + i)
        out[name] = (K, LC._pinhole_D(rng, n, False), H)
    return calib, out


@pytest.mark.parametrize("n", [5, 8, 14])
def test_bev_pinhole_cameras(fx, n):
    """bevk_bev_set_camera_model with pinhole cameras: each LUT == cv2.warpPerspective of the camera's map planes, and
    the four-camera canvases (blend, BALANCE, car) == the cv2 oracle with cv2's own maps; BevGenerator with 4-tuple
    calibs.  The map planes are the library's, which equal cv2's up to calib_cases.pinhole_outside_only: map2 fractions
    of entries whose taps lie outside every frame, which cv2's FMA-contracted pinhole build rounds its own way.  Warped
    into the LUT they stay outside every frame, so the canvases are cv2's byte for byte."""
    from cameracalibration_b200 import ops
    from cameracalibration_b200.SurroundBirdEyeView import surroundBEV as SB
    g = fx.geometry()   # the module defaults, which BevGenerator reads
    fish, calib = _pinhole_calib(fx, g, n)
    ref = C.RefBev(fish, g, blend=True, masks=[RS.blend_mask(nm, g.BW, g.BH, g.CW, g.CH) for nm in SB.NAMES])
    eng = ops.BevEngine(4, (g.FW, g.FH), (g.BW, g.BH))
    size = (int(g.FW * g.SS), int(g.FH * g.SS))
    for i, (name, cam) in enumerate(zip(SB.NAMES, ref.cameras)):
        K, D, H = calib[name]
        P = C.dst_camera_matrix(K, g.FW, g.FH, g.FS, g.SS)
        cam.undistort_maps = cv2.initUndistortRectifyMap(K, D, np.eye(3), P, size, cv2.CV_16SC2)
        cam.bev_maps = (cam.warp_homography(cam.undistort_maps[0]), cam.warp_homography(cam.undistort_maps[1]))
        mine = ops.init_undistort_rectify_map(K, D, P, size, R=np.eye(3))
        assert CC.pinhole_outside_only(LC.case_by_name("real8_0"), mine, cam.undistort_maps), name
        eng.set_camera(i, K, D, P, size, H, model="pinhole")
        got = eng.get_maps(i)
        assert (got[0] == cam.warp_homography(mine[0])).all() and (got[1] == cam.warp_homography(mine[1])).all(), name
        eng.set_mask(i, ref.masks[i])
    eng.finalize()
    frames = fx.frames(g.FW, g.FH)
    car = fx.car(g.BW, g.BH)
    for balance in (False, True):
        ref.balance = balance
        got = eng.run([frames], car, balance)[0]
        assert (got == ref(*frames, car)).all(), balance
    # BevGenerator with {name: (K, D, H, "pinhole")}
    gen = SB.BevGenerator(blend=True, balance=True, calib={k: (*v, "pinhole") for k, v in calib.items()})
    assert all(cam.model == "pinhole" for cam in gen.cameras)
    assert (gen(*frames, car) == ref(*frames, car)).all()
