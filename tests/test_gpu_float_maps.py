"""GPU test of cv2's float maps (CV_32FC1 / CV_32FC2), every byte against cv2: the map builds, ops.remap with float
maps on host images and device batches (padded rows and images, CUDA or NumPy maps), a captured graph, map-resident and
fused Undistorter slots, their JPEG and PNG streams, ops.convert_maps, and the refusals.  int16 maps keep their bytes.
Cameras and synthetic maps: tests/float_map_cases.py."""
import ctypes

import cv2
import numpy as np
import pytest

from tests import float_map_cases as FC

pytestmark = pytest.mark.gpu
INTERPS = (cv2.INTER_NEAREST, cv2.INTER_LINEAR, cv2.INTER_CUBIC, cv2.INTER_AREA, cv2.INTER_LANCZOS4)
ERR_ARG = -1   # BEVK_ERR_ARG


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


def _as3(a):
    return a.reshape(a.shape[0], a.shape[1], -1)


def _build(ops, c, m1type):
    fn = ops.fisheye_init_undistort_rectify_map if c.fisheye else ops.init_undistort_rectify_map
    return fn(c.K, c.D, c.P, (c.W, c.H), R=c.R, m1type=m1type)


def test_float_maps_vs_cv2():
    """ops.init_undistort_rectify_map / fisheye_init_undistort_rectify_map with m1type CV_32FC1 (both models) and
    CV_32FC2 (pinhole) == cv2's maps bit for bit (NaN and inf included); a pinhole entry may differ only as
    float_map_cases.far_outside_only allows."""
    from cameracalibration_b200 import ops
    for c in FC.corpus():
        for t in (cv2.CV_32FC1,) if c.fisheye else (cv2.CV_32FC1, cv2.CV_32FC2):
            got, want = _build(ops, c, t), FC.cv2_maps(c.name, t)
            if not (FC.same(got[0], want[0]) and FC.same(got[1], want[1])):
                assert FC.far_outside_only(c, got, want), (c.name, t)
        if c.fisheye and c.name == "fisheye_behind":
            assert np.isinf(got[0]).any()


def _map_sets():
    for name, x, y, sw, sh in FC.synthetic():
        yield name, x, y, sw, sh
    for n in ("pinhole8_R", "fisheye_behind", "stereo_vertical_left"):
        c = FC.case_by_name(n)
        yield n, *FC.cv2_maps(n, cv2.CV_32FC1), c.SW, c.SH


def _padded(torch, host, pad_row=12, pad_img=256):
    """host [N][H][W][C] as a CUDA view with padded rows and images."""
    n, h, w, ch = host.shape
    row = w * ch + pad_row
    img = h * row + pad_img
    pool = torch.zeros(n * img, dtype=torch.uint8, device="cuda")
    view = pool.as_strided((n, h, w, ch), (img, row, ch, 1))
    view.copy_(torch.from_numpy(host))
    return view


def test_remap_float_host_and_device(torch):
    """ops.remap with float maps: NumPy images (CV_32FC1 and CV_32FC2 maps) and CUDA batches of 1, 3 and 9 with padded
    rows and images (CUDA and NumPy maps), 1, 3 and 4 channels, every interpolation, == cv2.remap per frame; 3-channel
    INTER_LINEAR of widths % 4 == 0 takes the word path."""
    from cameracalibration_b200 import ops
    rng = np.random.default_rng(11)
    for name, x, y, sw, sh in _map_sets():
        xy = np.dstack([x, y])
        dx, dy, dxy = (torch.from_numpy(a).cuda() for a in (x, y, xy))
        for ch in (1, 3, 4):
            host = rng.integers(0, 256, (9, sh, sw, ch), dtype=np.uint8)
            for interp in INTERPS:
                want = [_as3(cv2.remap(host[i] if ch > 1 else host[i, :, :, 0], x, y, interp)) for i in range(9)]
                one = host[0] if ch > 1 else host[0, :, :, 0]
                assert (_as3(ops.remap(one, x, y, interp)) == want[0]).all(), (name, ch, interp)
                assert (_as3(ops.remap(one, xy, None, interp)) == want[0]).all(), (name, ch, interp, "32FC2")
                for n, maps in ((1, (dx, dy)), (3, (dxy, None)), (9, (x, y))):
                    got = ops.remap(_padded(torch, host[:n]), *maps, interp).cpu().numpy()
                    for i in range(n):
                        assert (got[i] == want[i]).all(), (name, ch, interp, n, i)
                if ch == 3 and interp == cv2.INTER_LINEAR:
                    assert ops.last_path() == ("word" if x.shape[1] % 4 == 0 else "byte"), name


def test_remap_float_graph(torch):
    """bevk_remap_f32_stack captured in a CUDA graph and replayed over rewritten frames and maps."""
    from cameracalibration_b200 import _lib as L
    ctx = L.default_context()
    name, x, y, sw, sh = FC.synthetic()[0]
    h, w = x.shape
    n = 5
    frames = torch.zeros((n, sh, sw, 3), dtype=torch.uint8, device="cuda")
    out = torch.empty((n, h, w, 3), dtype=torch.uint8, device="cuda")
    mx, my = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    torch.cuda.synchronize()
    call = lambda: ctx.lib.bevk_remap_f32_stack(ctx.h, ctypes.c_void_p(frames.data_ptr()), sh * sw * 3, sw, sh, sw * 3, 3, n,
                                                ctypes.c_void_p(mx.data_ptr()), ctypes.c_void_p(my.data_ptr()),
                                                ctypes.c_void_p(out.data_ptr()), h * w * 3, w, h, w * 3, cv2.INTER_CUBIC)
    assert call() == 0
    ctx.sync()
    with ctx.graph_capture() as g:
        assert call() == 0
    rng = np.random.default_rng(4)
    for rep in range(2):
        host = rng.integers(0, 256, (n, sh, sw, 3), dtype=np.uint8)
        nx = (x + rep).astype(np.float32)
        frames.copy_(torch.from_numpy(host))
        mx.copy_(torch.from_numpy(nx))
        out.fill_(0)
        torch.cuda.synchronize()
        g.launch()
        ctx.sync()
        got = out.cpu().numpy()
        for i in range(n):
            assert (got[i] == cv2.remap(host[i], nx, y, cv2.INTER_CUBIC)).all(), (rep, i)
    g.destroy()


def _slot_cases():
    return [("stereo_left", cv2.CV_32FC1, False), ("stereo_right", cv2.CV_32FC1, True),
            ("stereo_vertical_left", cv2.CV_32FC2, False), ("pinhole14_R", cv2.CV_32FC2, True),
            ("pinhole5_row", cv2.CV_32FC1, True), ("pinhole12", cv2.CV_32FC1, True),
            ("fisheye", cv2.CV_32FC1, True), ("fisheye_behind", cv2.CV_32FC1, False)]


@pytest.mark.parametrize("name,m1type,fused", _slot_cases())
def test_undistorter_float_slots(torch, name, m1type, fused):
    """Map-resident and fused float slots: maps() == cv2's float maps (far_outside_only for the pinhole), __call__ on
    host images and cuda() on device batches == cv2.remap through cv2's float maps, 1/3/4 channels, every interpolation.
    The stereo cases are the cv2.stereoRectify snippet at 1280x720."""
    from cameracalibration_b200 import ops
    c = FC.case_by_name(name)
    model = "fisheye" if c.fisheye else "pinhole"
    u = ops.Undistorter(c.K, c.D, c.P, (c.W, c.H), model=model, fused=fused, R=c.R, m1type=m1type)
    want_maps = FC.cv2_maps(name, m1type)
    m = u.maps()
    assert (FC.same(m[0], want_maps[0]) and FC.same(m[1], want_maps[1])) or FC.far_outside_only(c, m, want_maps), name
    rng = np.random.default_rng(21)
    for ch in (1, 3, 4):
        host = rng.integers(0, 256, (3, c.SH, c.SW, ch), dtype=np.uint8)
        for interp in INTERPS if c.W * c.H < 400_000 else (cv2.INTER_NEAREST, cv2.INTER_LINEAR, cv2.INTER_LANCZOS4):
            want = [_as3(cv2.remap(f if ch > 1 else f[..., 0], *want_maps, interp)) for f in host]
            assert (_as3(u(host[0] if ch > 1 else host[0, :, :, 0], interpolation=interp)) == want[0]).all(), (ch, interp)
            got = u.cuda(_padded(torch, host), interpolation=interp).cpu().numpy()
            for i in range(3):
                assert (got[i] == want[i]).all(), (ch, interp, i)
    u.close()


def test_stereo_snippet_bytes():
    """The cv2 stereo-rectification snippet, initUndistortRectifyMap(K, D, R1, P1, size, CV_32FC1) then remap, gives
    the same bytes through Undistorter(K, D, P1, size, "pinhole", R=R1, m1type=CV_32FC1), both cameras, both slot kinds."""
    from cameracalibration_b200 import ops
    for name in ("stereo_left", "stereo_right"):
        c = FC.case_by_name(name)
        mx, my = cv2.initUndistortRectifyMap(c.K, c.D, c.R, c.P, (c.W, c.H), cv2.CV_32FC1)
        img = FC.frames(c, 3)[0]
        want = cv2.remap(img, mx, my, cv2.INTER_LINEAR)
        for fused in (False, True):
            u = ops.Undistorter(c.K, c.D, c.P, (c.W, c.H), "pinhole", fused=fused, R=c.R, m1type=cv2.CV_32FC1)
            assert (u(img) == want).all(), (name, fused)
            u.close()


def test_float_slot_streams(torch):
    """.jpeg / .png / .cuda_to_jpeg of float slots == cv2.imencode of cv2.remap through cv2's float maps."""
    from cameracalibration_b200 import ops
    for name, fused in (("stereo_vertical_right", False), ("pinhole8_R", True)):
        c = FC.case_by_name(name)
        mx, my = FC.cv2_maps(name, cv2.CV_32FC1)
        u = ops.Undistorter(c.K, c.D, c.P, (c.W, c.H), "pinhole", fused=fused, R=c.R, m1type=cv2.CV_32FC1)
        host = FC.frames(c, 3, 3)
        want = [cv2.remap(f, mx, my, cv2.INTER_LINEAR) for f in host]
        assert u.jpeg(host[0], quality=90) == cv2.imencode(".jpg", want[0], [cv2.IMWRITE_JPEG_QUALITY, 90])[1].tobytes()
        assert u.png(host[1]) == cv2.imencode(".png", want[1])[1].tobytes()
        for s, w in zip(u.cuda_to_jpeg(torch.from_numpy(host).cuda(), quality=80), want):
            assert s == cv2.imencode(".jpg", w, [cv2.IMWRITE_JPEG_QUALITY, 80])[1].tobytes()
        u.close()


def test_convert_maps_vs_cv2(torch):
    """ops.convert_maps == cv2.convertMaps bit for bit, NumPy and CUDA maps: 32FC1 <-> 32FC2, 32F -> 16SC2 with and
    without nninterpolation, 16SC2 (with map2 or none) -> 32FC1 / 32FC2."""
    from cameracalibration_b200 import ops

    def both(m1, m2, t, nn):
        host = ops.convert_maps(m1, m2, t, nn)
        dev = ops.convert_maps(torch.from_numpy(m1).cuda(), None if m2 is None else torch.from_numpy(m2).cuda(), t, nn)
        torch.cuda.synchronize()
        dev = tuple(None if d is None else d.cpu().numpy() for d in dev)
        return host, dev

    for name, x, y, _, _ in list(FC.synthetic()) + [("fisheye_behind", *FC.cv2_maps("fisheye_behind", cv2.CV_32FC1), 0, 0)]:
        xy = np.dstack([x, y])
        for s1, s2, src in ((x, y, cv2.CV_32FC1), (xy, None, cv2.CV_32FC2)):
            for t, nn in ((cv2.CV_16SC2, False), (cv2.CV_16SC2, True), (cv2.CV_32FC1 + cv2.CV_32FC2 - src, False)):
                a, b = cv2.convertMaps(s1, s2, t, nninterpolation=nn)
                want = (a, b if b is not None and b.size else None)
                for got in both(s1, s2, t, nn):
                    assert FC.same(got[0], want[0]) and FC.same(got[1], want[1]), (name, src, t, nn)
        i1, i2 = cv2.convertMaps(x, y, cv2.CV_16SC2)
        for m2 in (i2, None):
            ref2 = np.zeros(i1.shape[:2], np.uint16) if m2 is None else m2
            for t in (cv2.CV_32FC1, cv2.CV_32FC2):
                a, b = cv2.convertMaps(i1, ref2, t)
                want = (a, b if b is not None and b.size else None)
                for got in both(i1, m2, t, False):
                    assert FC.same(got[0], want[0]) and FC.same(got[1], want[1]), (name, t, m2 is None)


def test_float_refusals(torch):
    """Refusals: status, message and an untouched destination."""
    from cameracalibration_b200 import ops
    from cameracalibration_b200 import _lib as L
    ctx = L.default_context()
    lib = ctx.lib
    f = FC.case_by_name("fisheye")
    with pytest.raises(L.BevkError, match="CV_32FC2"):
        ops.fisheye_init_undistort_rectify_map(f.K, f.D, f.P, (64, 48), m1type=cv2.CV_32FC2)
    with pytest.raises(L.BevkError, match="CV_32FC2"):
        ops.Undistorter(f.K, f.D, f.P, (64, 48), m1type=cv2.CV_32FC2)
    with pytest.raises(L.BevkError, match="m1type"):
        ops.init_undistort_rectify_map(f.K, np.zeros(5), f.P, (64, 48), m1type=cv2.CV_16UC1)
    r = FC.case_by_name("fisheye_behind")
    with pytest.raises(L.BevkError, match="map-resident"):   # refused as the CV_16SC2 fused slot is
        ops.Undistorter(r.K, r.D, r.P, (r.W, r.H), fused=True, R=r.R, m1type=cv2.CV_32FC1)
    # the wrong map read-back for the slot's type
    u = ops.Undistorter(f.K, f.D, f.P, (64, 48), m1type=cv2.CV_32FC1)
    m1 = np.full((48, 64, 2), 7, np.int16)
    m2 = np.full((48, 64), 7, np.uint16)
    assert lib.bevk_undistorter_maps(ctx.h, u.slot, L.vptr(m1), L.vptr(m2)) == ERR_ARG
    assert b"bevk_undistorter_maps_f32" in lib.bevk_last_error()
    assert (m1 == 7).all() and (m2 == 7).all()
    u.close()
    # convert to the same type
    x = np.zeros((4, 4), np.float32)
    with pytest.raises(L.BevkError, match="nothing to convert"):
        ops.convert_maps(x, x, cv2.CV_32FC1)
    # a device destination that overlaps the maps, and one that overlaps the source
    h, w = 16, 32
    pool = torch.full((4 * h * w * 3 + 4 * h * w * 2,), 9, dtype=torch.uint8, device="cuda")
    src = torch.zeros((h, w, 3), dtype=torch.uint8, device="cuda")
    maps = pool[:8 * h * w].view(torch.float32).view(h, w, 2)
    maps.zero_()
    dst_ptr = pool.data_ptr() + 4 * h * w
    before = pool.clone()
    rc = lib.bevk_remap_f32_stack(ctx.h, ctypes.c_void_p(src.data_ptr()), 0, w, h, w * 3, 3, 1, ctypes.c_void_p(maps.data_ptr()),
                                  None, ctypes.c_void_p(dst_ptr), 0, w, h, w * 3, cv2.INTER_LINEAR)
    assert rc == ERR_ARG and b"overlaps the maps" in lib.bevk_last_error()
    rc = lib.bevk_remap_f32_stack(ctx.h, ctypes.c_void_p(pool.data_ptr()), 0, w, h, w * 3, 3, 1, ctypes.c_void_p(maps.data_ptr()),
                                  None, ctypes.c_void_p(pool.data_ptr() + 64), 0, w, h, w * 3, cv2.INTER_LINEAR)
    assert rc == ERR_ARG and b"overlaps" in lib.bevk_last_error()
    torch.cuda.synchronize()
    assert torch.equal(pool, before)
    # a float map1 with a map2 of another shape, and a 2-D map1 without map2
    img = np.zeros((8, 8, 3), np.uint8)
    with pytest.raises(L.BevkError, match="float"):
        ops.remap(img, np.zeros((4, 4), np.float32), np.zeros((4, 5), np.float32))
    with pytest.raises(L.BevkError, match="CV_32FC2"):
        ops.remap(img, np.zeros((4, 4), np.float32), None)


def test_int16_maps_keep_their_bytes():
    """int16 maps take the CV_16SC2 path exactly as before: cv2.remap's bytes, every interpolation, and the same gather."""
    from cameracalibration_b200 import ops
    name, x, y, sw, sh = FC.synthetic()[0]
    m1, m2 = cv2.convertMaps(x, y, cv2.CV_16SC2)
    img = np.random.default_rng(2).integers(0, 256, (sh, sw, 3), dtype=np.uint8)
    for interp in INTERPS:
        assert (ops.remap(img, m1, m2, interp) == cv2.remap(img, m1, m2, interp)).all(), interp
    assert (ops.remap(img, m1, None, cv2.INTER_NEAREST) == cv2.remap(img, m1, None, cv2.INTER_NEAREST)).all()
    ops.remap(img, m1, m2, cv2.INTER_LINEAR)
    assert ops.last_path() == "word"
