"""GPU test of the edge cases of tests/lens_edge_cases.py: every kernel instance that evaluates the camera model, against
cv2 with cv2's own maps.  The map builds (k_undistort_map<LENS>, k_walk_rays for both models) of every case, the 4K
walked fisheye included, also equal the host build of the same code (tests/host/lens_models.cu) bit for bit; Undistorter
slots (map-resident and fused) reach k_gather4, k_gather and k_gather_taps; BEV cameras reach k_warp_maps<1, LENS> and
a four-camera render through run_stack; fused fisheye slots whose rays depend on the row are refused."""
import cv2
import numpy as np
import pytest

from oracle import cv2_path as C
from oracle import restate as RS
from tests import calib_cases as CC
from tests import lens_cases as LC
from tests import lens_edge_cases as E
from tests.test_host_lens_models import _maps, exe  # noqa: F401  (exe: the host build, a module fixture)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


def test_edge_maps_vs_cv2_and_host(exe, tmp_path):
    """ops.init_undistort_rectify_map / ops.fisheye_init_undistort_rectify_map with R of every edge case == cv2's maps
    (no tolerance for the fisheye, pinhole_outside_only for the pinhole) and == the host build, bit for bit."""
    from cameracalibration_b200 import ops
    n = 0
    for c in E.corpus():
        fn = ops.fisheye_init_undistort_rectify_map if c.fisheye else ops.init_undistort_rectify_map
        got = fn(c.K, c.D, c.P, (c.UW, c.UH), R=np.eye(3) if c.R is None else c.R)
        want = E.cv2_maps(c.name)
        if not ((got[0] == want[0]).all() and (got[1] == want[1]).all()):
            assert not c.fisheye and LC.outside_only(c, got, want), LC.first_diffs(c, got, want)
        host, _ = _maps(exe, tmp_path, c.model, c.K, c.D, c.R, c.P, c.UW, c.UH)
        assert (got[0] == host[0]).all() and (got[1] == host[1]).all(), (c.name, LC.first_diffs(c, got, host))
        n += c.UW * c.UH
    assert n > 9_000_000


def _small(c, size):
    """c's camera at undistorted size `size` (K and P scaled with it), and cv2's maps there."""
    w, h = size
    S = np.diag([w / c.UW, h / c.UH, 1.0])
    K, P = S @ c.K, S @ c.P
    R = np.eye(3) if c.R is None else c.R
    if c.fisheye:
        return K, P, cv2.fisheye.initUndistortRectifyMap(K, c.D.reshape(4, 1), R, P, (w, h), cv2.CV_16SC2)
    return K, P, cv2.initUndistortRectifyMap(K, c.D, R, P, (w, h), cv2.CV_16SC2)


def _want(maps, frame, interp):
    out = cv2.remap(np.ascontiguousarray(frame), maps[0], maps[1], interp)
    return out.reshape(out.shape[0], out.shape[1], -1)


INTERPS = (cv2.INTER_NEAREST, cv2.INTER_LINEAR, cv2.INTER_CUBIC, cv2.INTER_LANCZOS4)
SLOT_CASES = ("pole8", "pole14", "prism12", "tilt0", "rotpin8_1", "rotfish4_4", "neardyadic320", "dyadic_pin", "dyadic_fish",
              "wmod7", "only_ty", "flip_pin", "eye_fish")


def _path(ch, interp, w, odd):
    if interp in (cv2.INTER_CUBIC, cv2.INTER_LANCZOS4):
        return "taps"
    return "word" if ch == 3 and interp == cv2.INTER_LINEAR and w % 4 == 0 and not odd else "byte"


@pytest.mark.parametrize("name", SLOT_CASES)
@pytest.mark.parametrize("fused", [False, True])
def test_edge_undistorter_slots(torch, name, fused):
    """Map-resident and fused Undistorter slots of the edge cameras (a fused fisheye slot whose rays depend on the row is
    refused with the map-resident message; a fused pinhole slot keeps its block starts), 1/3/4 channels, NEAREST / LINEAR / CUBIC / LANCZOS4, host frames and device batches
    of 1, 9 and 17 (across GATHER_NB) at an aligned and an odd base, W % 4 == 0 and not: k_gather4, k_gather and
    k_gather_taps, each asserted by last_path(), against cv2.remap through cv2's maps (or the slot's, where they differ
    as pinhole_outside_only allows).  The dyadic cameras keep their size, so that _w == 0 stays exact."""
    from cameracalibration_b200 import ops
    from cameracalibration_b200 import _lib as L
    c = E.case_by_name(name)
    model = "fisheye" if c.fisheye else "pinhole"
    sizes = [(c.UW, c.UH)] if name.startswith("dyadic") else [(120, 72), (121, 73)]
    rng = np.random.default_rng(11 + fused)
    for size in sizes:
        w, h = size
        K, P, maps = _small(c, size) if size != (c.UW, c.UH) else (c.K, c.P, E.cv2_maps(c.name))
        if fused and c.fisheye and LC.walks(c):
            with pytest.raises(L.BevkError, match="map-resident"):
                ops.Undistorter(K, c.D, P, size, model=model, fused=True, R=c.R)
            return
        u = ops.Undistorter(K, c.D, P, size, model=model, fused=fused, R=c.R)
        m = u.maps()
        exact = (m[0] == maps[0]).all() and (m[1] == maps[1]).all()
        assert exact or (not c.fisheye and LC.outside_only(c, m, maps)), LC.first_diffs(c, m, maps)
        ref = maps if exact else m
        for ch in (1, 3, 4):
            host = rng.integers(0, 256, (17, 90, 160, ch), dtype=np.uint8)   # rows of 4-byte multiples: the word path
            d = torch.from_numpy(host).cuda()
            flat = torch.zeros(host.size + 1, dtype=torch.uint8, device="cuda")
            flat[1:] = d.reshape(-1)
            odd_view = flat[1:].view(host.shape)
            for interp in INTERPS:
                want = [_want(ref, f, interp) for f in host]
                one = u(host[0] if ch > 1 else host[0, :, :, 0], interpolation=interp)
                assert (one.reshape(h, w, -1) == want[0]).all(), (size, ch, interp)
                for n in (1, 9, 17):
                    for odd, src in ((False, d), (True, odd_view)):
                        got = u.cuda(src[:n], interpolation=interp)
                        assert u.last_path() == _path(ch, interp, w, odd), (size, ch, interp, n, odd)
                        got = got.cpu().numpy()
                        for i in range(n):
                            assert (got[i].reshape(h, w, -1) == want[i]).all(), (size, ch, interp, n, odd, i)
        u.close()


def test_edge_fused_slots_of_walking_rays():
    """A fused fisheye slot whose R makes the rays depend on the row is refused with the map-resident message and launches
    no kernel.  A fused pinhole slot of such a camera (rotated, stereo-rectified, dyadic, near-dyadic, narrow) keeps its
    block starts and evaluates per pixel exactly what the map-resident slot's map holds, bit for bit."""
    from cameracalibration_b200 import ops
    from cameracalibration_b200 import _lib as L
    ctx = L.Context(0)
    for name in ("rotfish4_3", "dyadic_fish", "fishodd97", "thinfish33x1"):
        c = E.case_by_name(name)
        assert LC.walks(c), name
        ctx.sync()
        before = ctx.launches
        with pytest.raises(L.BevkError, match="map-resident"):
            ops.Undistorter(c.K, c.D, c.P, (c.UW, c.UH), model="fisheye", fused=True, R=c.R, ctx=ctx)
        assert ctx.launches == before, name
    rng = np.random.default_rng(3)
    for name in ("rotpin5_0", "rotpin14_2", "stereov0", "dyadic_pin", "neardyadic327", "narrow3", "wmod5", "thinpin41x1"):
        c = E.case_by_name(name)
        assert LC.walks(c), name
        res = ops.Undistorter(c.K, c.D, c.P, (c.UW, c.UH), model="pinhole", fused=False, R=c.R, ctx=ctx)
        fus = ops.Undistorter(c.K, c.D, c.P, (c.UW, c.UH), model="pinhole", fused=True, R=c.R, ctx=ctx)
        m, f = res.maps(), fus.maps()
        assert (m[0] == f[0]).all() and (m[1] == f[1]).all(), name
        frame = rng.integers(0, 256, (c.UH + 7, c.UW + 9, 3), dtype=np.uint8)
        for interp in INTERPS:
            assert (fus(frame, interpolation=interp) == res(frame, interpolation=interp)).all(), (name, interp)
        res.close()
        fus.close()


BEV_CAMERAS = ("pole8", "pole12", "tilt0", "prism14")


def test_edge_bev_pinhole_cameras(torch, fx):
    """bevk_bev_set_camera_model with pinhole edge cameras (8 / 12 / 14 coefficients: poles, tilt of 1 rad, saturating
    thin prism) under homographies whose horizon crosses the canvas (calib_cases._homography "inside", and _H_ZERO with
    W == 0 exactly): each LUT (k_warp_maps<1, 1>) == cv2.warpPerspective of cv2's map planes, and one four-camera render
    through run_stack == RefBev with cv2's maps, BALANCE off and on."""
    from cameracalibration_b200 import ops
    from cameracalibration_b200.SurroundBirdEyeView import surroundBEV as SB
    g = fx.geometry()
    rng = np.random.default_rng(77)
    cams = [E.case_by_name(n) for n in BEV_CAMERAS]
    Hs = [CC._H_ZERO.copy() if i == 1 else CC._homography(rng, c.UW, c.UH, g.BW, g.BH, "inside") for i, c in enumerate(cams)]
    fish = fx.scaled_calib(g)
    ref = C.RefBev(fish, g, blend=True, masks=[RS.blend_mask(nm, g.BW, g.BH, g.CW, g.CH) for nm in SB.NAMES])
    eng = ops.BevEngine(4, (g.FW, g.FH), (g.BW, g.BH))
    for i, (c, H, cam) in enumerate(zip(cams, Hs, ref.cameras)):
        m = E.cv2_maps(c.name)
        cam.undistort_maps = m
        cam.bev_maps = (cv2.warpPerspective(m[0], H, (g.BW, g.BH)), cv2.warpPerspective(m[1], H, (g.BW, g.BH)))
        eng.set_camera(i, c.K, c.D, c.P, (c.UW, c.UH), H, model="pinhole")
        got = eng.get_maps(i)
        assert (got[0] == cam.bev_maps[0]).all() and (got[1] == cam.bev_maps[1]).all(), c.name
        eng.set_mask(i, ref.masks[i])
    eng.finalize()
    frames = fx.frames(g.FW, g.FH)
    car = fx.car(g.BW, g.BH)
    d = torch.from_numpy(np.stack(frames)).cuda()
    dcar = torch.from_numpy(np.ascontiguousarray(car)).cuda()
    out = torch.empty((1, g.BH, g.BW, 3), dtype=torch.uint8, device="cuda")
    for balance in (False, True):
        ref.balance = balance
        want = ref(*frames, car)
        eng.run_stack(d.data_ptr(), g.FW * g.FH * 3, 1, out.data_ptr(), dcar.data_ptr(), balance)
        eng.ctx.sync()
        assert (out.cpu().numpy()[0] == want).all(), balance
