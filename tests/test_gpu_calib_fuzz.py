"""The kernels' camera-model and homography arithmetic on the device, over the seeded random calibrations of
tests/calib_cases.py, byte for byte against cv2: k_undistort_map (ops, Undistorter.maps of map and fused slots), the
fused gathers (k_gather4<1> / k_gather<1>), k_warp_maps<1> (BevEngine.set_camera), k_warp_maps<0>
(ops.warp_perspective_maps) and the homography gathers (ops.warp_perspective).  The host build of the same code runs
in tests/test_host_calib_fuzz.py; a difference only here would come from the device math library (atan, sqrt,
division)."""
import cv2
import numpy as np
import pytest

from oracle import cv2_path as C
from oracle import restate as R
from tests import calib_cases as CC
from tests.helpers import NAMES

pytestmark = pytest.mark.gpu


def _check_maps(c, got, want):
    same = (got[0] == want[0]).all() and (got[1] == want[1]).all()
    assert same or (CC.pinhole_outside_only(c, got, want) and CC.remaps_agree(c, got, want)), CC.first_diffs(c, got, want)


def test_undistort_maps_vs_cv2_random_calibrations():
    from cameracalibration_b200 import ops
    n = 0
    for c in CC.corpus():
        want = CC.cv2_maps(c.name)
        f = ops.fisheye_init_undistort_rectify_map if c.fisheye else ops.init_undistort_rectify_map
        _check_maps(c, f(c.K, c.D if c.fisheye else c.d5, c.P, (c.UW, c.UH)), want)
        model = "fisheye" if c.fisheye else "pinhole"
        for fused in (False, True):
            u = ops.Undistorter(c.K, c.D if c.fisheye else c.d5, c.P, (c.UW, c.UH), model=model, fused=fused)
            _check_maps(c, u.maps(), want)
            u.close()
        n += 3 * c.UW * c.UH
    print(f"map entries compared: {n}")


def test_undistorted_images_vs_cv2_remap_random_calibrations():
    """Undistorter.__call__ (one frame) and .cuda (9 frames) for map and fused slots, both models, 1 / 3 / 4 channels,
    LINEAR and NEAREST, against cv2.remap through cv2's maps; both gathers (word path for 3-channel LINEAR at W % 4 == 0).
    The 2560x2048 cases (mild5 holds the entries the running row sums decide) take one frame per call."""
    import torch
    from cameracalibration_b200 import ops
    n = 0
    for c in CC.corpus():
        large = c.UW * c.UH > 1_400_000
        if large and (c.UW, c.UH) != (2560, 2048):
            continue
        want_maps = CC.cv2_maps(c.name)
        d = c.D if c.fisheye else c.d5
        for fused in (False, True):
            u = ops.Undistorter(c.K, d, c.P, (c.UW, c.UH), model="fisheye" if c.fisheye else "pinhole", fused=fused)
            for ch in ((1, 3) if large else (1, 3, 4)):
                fr = CC.frames(c.name, ch, 1 if large else 9)
                for inter in (cv2.INTER_LINEAR, cv2.INTER_NEAREST):
                    want = [cv2.remap(f, *want_maps, inter) for f in fr]
                    want = [w if w.ndim == 3 else w[..., None] for w in want]
                    got1 = u(fr[0], interpolation=inter)
                    assert (got1.reshape(want[0].shape) == want[0]).all(), (c.name, fused, ch, inter)
                    word = ch == 3 and inter == cv2.INTER_LINEAR and c.UW % 4 == 0
                    assert u.last_path() == ("word" if word else "byte"), (c.name, ch, inter)
                    n += c.UW * c.UH
                    if large:
                        continue
                    got9 = u.cuda(torch.from_numpy(fr).cuda(), interpolation=inter)
                    torch.cuda.synchronize()
                    assert u.last_path() == ("word" if word else "byte"), (c.name, ch, inter)
                    assert (got9.cpu().numpy() == np.stack(want)).all(), (c.name, fused, ch, inter)
                    n += 9 * c.UW * c.UH
            u.close()
    print(f"undistorted pixels compared: {n}")


def test_undistorted_jpeg_vs_cv2_random_calibrations():
    """Undistorter.cuda_to_jpeg == cv2.imencode of cv2.remap through cv2's maps, byte for byte, on a few cases."""
    import torch
    from cameracalibration_b200 import ops
    for name in ("scaled4", "strong_fisheye1", "strong_pinhole3", "scaled5"):
        c = CC.case_by_name(name)
        u = ops.Undistorter(c.K, c.D if c.fisheye else c.d5, c.P, (c.UW, c.UH), model="fisheye" if c.fisheye else "pinhole",
                            fused=True)
        fr = CC.frames(name, 3, 2)
        got = u.cuda_to_jpeg(torch.from_numpy(fr).cuda(), quality=90)
        for f, g in zip(fr, got):
            ok, want = cv2.imencode(".jpg", cv2.remap(f, *CC.cv2_maps(name), cv2.INTER_LINEAR), [cv2.IMWRITE_JPEG_QUALITY, 90])
            assert ok and g == want.tobytes(), name
        u.close()


def test_bev_luts_and_warps_vs_cv2_random_calibrations():
    """BevEngine.set_camera -> get_maps == cv2.warpPerspective of cv2's planes (fisheye cases); ops.warp_perspective_maps
    on cv2's planes; ops.warp_perspective of images, 1 / 3 / 4 channels, both interpolations."""
    from cameracalibration_b200 import _lib as L
    from cameracalibration_b200 import ops
    ctx = L.default_context()
    n = 0
    paths = set()
    for c in CC.corpus():
        want = CC.cv2_bev_maps(c.name)
        if c.fisheye:
            e = ops.BevEngine(1, (c.FW, c.FH), (c.BW, c.BH))
            e.set_camera(0, c.K, c.D, c.P, (c.UW, c.UH), c.H)
            got = e.get_maps(0)
            assert (got[0] == want[0]).all() and (got[1] == want[1]).all(), (c.name, CC.first_diffs(c, got, want))
        got = ops.warp_perspective_maps(*CC.cv2_maps(c.name), c.H, (c.BW, c.BH))
        assert (got[0] == want[0]).all() and (got[1] == want[1]).all(), c.name
        n += 2 * c.BW * c.BH
        for ch in (1, 3, 4):
            src = CC.frames(c.name, ch, 1, (min(c.UW, 1024), min(c.UH, 768)))[0]
            src = src[..., 0] if ch == 1 else src
            for inter in (cv2.INTER_LINEAR, cv2.INTER_NEAREST):
                got = ops.warp_perspective(src, c.H, (c.BW, c.BH), flags=inter)
                word = ch == 3 and inter == cv2.INTER_LINEAR and c.BW % 4 == 0 and src.shape[1] % 4 == 0   # 4-byte rows
                assert ctx.lib.bevk_undistort_last_path(ctx.h) == (4 if word else 1), (c.name, ch, inter)
                paths.add(word)
                assert (got == cv2.warpPerspective(src, c.H, (c.BW, c.BH), flags=inter)).all(), (c.name, ch, inter)
    assert paths == {True, False}
    print(f"BEV map entries compared: {n}")


def _rig(seed, g):
    """Four random fisheye cameras of geometry g (|D| <= 0.1, strong-perspective homographies, one with the horizon
    inside the canvas): a calib dict as BevGenerator and C.RefBev take it."""
    rng = np.random.default_rng(seed)
    calib = {}
    for k, name in enumerate(NAMES):
        K = np.array([[rng.uniform(0.3, 0.7) * g.FW, 0, g.FW / 2 + rng.uniform(-20, 20)],
                      [0, rng.uniform(0.3, 0.7) * g.FW, g.FH / 2 + rng.uniform(-20, 20)], [0, 0, 1.0]])
        D = rng.uniform(-0.1, 0.1, (4, 1))
        H = CC._homography(rng, int(g.FW * g.SS), int(g.FH * g.SS), g.BW, g.BH, "inside" if k == 1 else "none")
        calib[name] = (K, D, H)
    return calib


@pytest.mark.parametrize("seed", [0, 1])
def test_bev_engine_from_random_cameras_vs_ref_bev(seed):
    """BevEngine built with set_camera from four random fisheye cameras, rendered through run and run_cuda with
    BALANCE off and on and with the car, == C.RefBev (the reference's cv2 call sequence) canvas for canvas."""
    import torch
    from cameracalibration_b200 import ops
    g = C.Geometry(FW=(640, 332)[seed], FH=(512, 250)[seed], BW=(333, 480)[seed], BH=(257, 400)[seed], CW=83, CH=102,
                   FS=(0.8, 1.0)[seed], SS=(2.0, 1.5)[seed])
    calib = _rig(10 + seed, g)
    masks = [R.blend_mask(n, g.BW, g.BH, g.CW, g.CH) for n in NAMES]
    e = ops.BevEngine(4, (g.FW, g.FH), (g.BW, g.BH))
    for i, n in enumerate(NAMES):
        K, D, H = calib[n]
        e.set_camera(i, K, D, C.dst_camera_matrix(K, g.FW, g.FH, g.FS, g.SS), (int(g.FW * g.SS), int(g.FH * g.SS)), H)
        e.set_mask(i, masks[i])
    e.finalize()
    rng = np.random.default_rng(20 + seed)
    sets = [[rng.integers(0, 256, (g.FH, g.FW, 3), dtype=np.uint8) for _ in NAMES] for _ in range(3)]
    car = rng.integers(0, 256, (g.BH, g.BW, 3), dtype=np.uint8)
    car[rng.integers(0, 2, (g.BH, g.BW)) == 0] = 0
    d = torch.from_numpy(np.stack([np.stack(s) for s in sets])).cuda()
    for balance in (False, True):
        ref = C.RefBev(calib, g, True, balance, masks=masks)
        for with_car in (False, True):
            cr = car if with_car else None
            want = np.stack([ref(*s, cr) for s in sets])
            assert (e.run(sets, cr, balance) == want).all(), ("run", balance, with_car)
            got = e.run_cuda(d, torch.from_numpy(car).cuda() if with_car else None, balance)
            torch.cuda.synchronize()
            assert (got.cpu().numpy() == want).all(), ("run_cuda", balance, with_car)


def test_bev_generator_with_a_random_calibration(fx):
    """BevGenerator(calib=...) with a random four-camera calibration at the default geometry == C.RefBev."""
    from cameracalibration_b200.SurroundBirdEyeView import surroundBEV as S
    g = fx.geometry()
    calib = _rig(30, g)
    bev = S.BevGenerator(blend=True, balance=True, calib=calib)
    masks = [R.blend_mask(n, g.BW, g.BH, g.CW, g.CH) for n in NAMES]
    ref = C.RefBev(calib, g, True, True, masks=masks)
    rng = np.random.default_rng(31)
    frames = [rng.integers(0, 256, (g.FH, g.FW, 3), dtype=np.uint8) for _ in NAMES]
    car = fx.car()
    assert (bev(*frames, car) == ref(*frames, car)).all()
