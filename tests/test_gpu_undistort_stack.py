"""GPU test of device-resident, batched undistortion (bevk_undistort_stack / _jpeg, Undistorter.cuda / cuda_to_jpeg and
the drop-in classes on CUDA tensors).  Every output byte must equal cv2.remap of its own frame through the reference's
maps (C.undistort_maps for fisheye, C.pinhole_maps for pinhole), every JPEG stream cv2.imencode of that image, and
padding and sentinels around the outputs must come back untouched."""
import ctypes

import cv2
import numpy as np
import pytest

from oracle import cv2_path as C

pytestmark = pytest.mark.gpu
FILL = 0xA5


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


def _und(fx, model="fisheye", fused=False, src=(1280, 1024), dst=(1280, 1024), fs=1.0):
    """An Undistorter for the front camera scaled to `src`, and the reference's maps for it."""
    from cameracalibration_b200 import ops
    K, D, _ = fx.calib["front"]
    K = np.diag([src[0] / 1280, src[1] / 1024, 1.0]) @ K
    P = C.dst_camera_matrix(K, dst[0], dst[1], fs, 1)
    if model == "fisheye":
        m = C.undistort_maps(K, D, P, *dst)
        u = ops.Undistorter(K, D, P, dst, model="fisheye", fused=fused)
    else:
        m = C.pinhole_maps(K, fx.D5, P, *dst)
        u = ops.Undistorter(K, fx.D5, P, dst, model="pinhole", fused=fused)
    return u, m


def _want(maps, frame, interp=cv2.INTER_LINEAR):
    out = cv2.remap(np.ascontiguousarray(frame), maps[0], maps[1], interp)
    return out.reshape(out.shape[0], out.shape[1], -1)


def _frames(rng, n, h, w, c):
    return rng.integers(0, 256, (n, h, w, c), dtype=np.uint8)


@pytest.mark.parametrize("model", ["fisheye", "pinhole"])
@pytest.mark.parametrize("fused", [False, True])
def test_models_slots_channels_interpolation(fx, torch, model, fused):
    """Map and fused slots, fisheye and pinhole (pinhole: OpenCV's saturating 8-column vector body), 1/3/4 channels,
    LINEAR and NEAREST, dw % 4 == 0 and != 0."""
    from cameracalibration_b200 import ops
    rng = np.random.default_rng(7 + fused + 2 * (model == "pinhole"))
    for dst in ((96, 40), (83, 37)):
        u, maps = _und(fx, model, fused, (72, 50), dst, 0.6)
        for c in (1, 3, 4):
            host = _frames(rng, 5, 50, 72, c)
            frames = torch.from_numpy(host).cuda()
            for interp in (ops.INTER_LINEAR, ops.INTER_NEAREST):
                out = u.cuda(frames, interpolation=interp).cpu().numpy()
                assert out.shape == (5, dst[1], dst[0], c)
                for i in range(5):
                    assert (out[i] == _want(maps, host[i], interp)).all(), (dst, c, interp, i)
                words = c == 3 and interp == ops.INTER_LINEAR and dst[0] % 4 == 0
                assert u.last_path() == ("word" if words else "byte"), (dst, c, interp)
        grey = torch.from_numpy(host[0, :, :, 0].copy()).cuda()          # [H][W] -> [H][W]
        got = u.cuda(grey).cpu().numpy()
        assert got.shape == (dst[1], dst[0]) and (got == _want(maps, host[0, :, :, 0])[..., 0]).all()
        u.close()


def test_reference_size_scale_2(fx, torch):
    """The reference's frames, 1280x1024 -> 2560x2048 (SIZE_SCALE 2), map and fused slots, one batch of the four cameras."""
    from cameracalibration_b200 import ops
    K, D, _ = fx.calib["front"]
    P = C.dst_camera_matrix(K, 1280, 1024, 1, 2)
    maps = C.undistort_maps(K, D, P, 2560, 2048)
    host = np.stack([fx.img(n) for n in ("front", "back", "left", "right")])
    frames = torch.from_numpy(host).cuda()
    for fused in (False, True):
        u = ops.Undistorter(K, D, P, (2560, 2048), fused=fused)
        out = u.cuda(frames).cpu().numpy()
        assert u.last_path() == "word"
        for i in range(4):
            assert (out[i] == _want(maps, host[i])).all(), (fused, i)
        one = u.cuda(frames[2]).cpu().numpy()                              # [H][W][3]
        assert (one == out[2]).all()
        u.close()


@pytest.mark.parametrize("fused", [False, True])
def test_batch_sizes_cross_the_frame_groups(fx, torch, fused):
    rng = np.random.default_rng(11 + fused)
    u, maps = _und(fx, "fisheye", fused, (64, 48), (64, 48), 0.7)
    host = _frames(rng, 33, 48, 64, 3)
    frames = torch.from_numpy(host).cuda()
    for n in (1, 3, 4, 5, 9, 33):
        out = u.cuda(frames[:n]).cpu().numpy()
        for i in range(n):
            assert (out[i] == _want(maps, host[i])).all(), (n, i)
    u.close()


def _layout_case(torch, u, maps, rng, *, n, c, srow_pad, simg_pad, soff, drow_pad, dimg_pad, interp=1):
    """Frames at soff + f * simg in one flat device buffer, outputs into a flat buffer pre-filled with FILL that has a
    sentinel image after the last output.  Returns the path bevk_undistort_last_path reports."""
    sw, sh, dw, dh = 40, 30, u.w, u.h
    srow, drow = sw * c + srow_pad, dw * c + drow_pad
    simg, dimg = sh * srow + simg_pad, dh * drow + dimg_pad
    sbuf = rng.integers(0, 256, soff + n * simg + 64, dtype=np.uint8)
    dbuf = np.full((n + 1) * dimg + 64, FILL, np.uint8)
    ds, dd = torch.from_numpy(sbuf).cuda(), torch.from_numpy(dbuf).cuda()
    torch.cuda.synchronize()
    lib = u.ctx.lib
    rc = lib.bevk_undistort_stack(u.ctx.h, u.slot, ctypes.c_void_p(ds.data_ptr() + soff), simg, sw, sh, srow, c, n,
                                  ctypes.c_void_p(dd.data_ptr()), dimg, dw, dh, drow, interp)
    assert rc == 0, lib.bevk_last_error().decode()
    u.ctx.sync()
    out = dd.cpu().numpy()
    touched = np.zeros(out.size, bool)
    for f in range(n):
        frame = np.lib.stride_tricks.as_strided(sbuf[soff + f * simg:], (sh, sw, c), (srow, c, 1))
        got = np.lib.stride_tricks.as_strided(out[f * dimg:], (dh, dw, c), (drow, c, 1))
        assert (got == _want(maps, frame, interp)).all(), (n, c, srow_pad, simg_pad, soff, drow_pad, dimg_pad, f)
        np.lib.stride_tricks.as_strided(touched[f * dimg:], got.shape, got.strides)[...] = True
    assert (out[~touched] == FILL).all(), "padding or the sentinel image was written"
    al = (ds.data_ptr() + soff) | dd.data_ptr() | srow | drow | ((simg | dimg) if n > 1 else 0)
    words = c == 3 and interp == 1 and dw % 4 == 0 and al % 4 == 0
    assert lib.bevk_undistort_last_path(u.ctx.h) == (4 if words else 1), (n, c, srow_pad, simg_pad, soff, drow_pad, dimg_pad)
    return words


@pytest.mark.parametrize("fused", [False, True])
def test_padded_and_unaligned_layouts(fx, torch, fused):
    rng = np.random.default_rng(21 + fused)
    paths = set()
    for dw in (48, 45):
        u, maps = _und(fx, "fisheye", fused, (40, 30), (dw, 27), 0.6)
        for n in (1, 3, 5):
            for srow_pad in (0, 4, 7):                   # row pitch a multiple of 4 (0, 4) and not (7)
                paths.add(_layout_case(torch, u, maps, rng, n=n, c=3, srow_pad=srow_pad, simg_pad=0, soff=0, drow_pad=0, dimg_pad=0))
            for simg_pad in (4, 6):
                paths.add(_layout_case(torch, u, maps, rng, n=n, c=3, srow_pad=0, simg_pad=simg_pad, soff=0, drow_pad=0, dimg_pad=0))
            for soff in (1, 2, 3):
                paths.add(_layout_case(torch, u, maps, rng, n=n, c=3, srow_pad=0, simg_pad=0, soff=soff, drow_pad=0, dimg_pad=0))
            for drow_pad, dimg_pad in ((4, 0), (8, 12), (5, 3), (0, 2)):
                paths.add(_layout_case(torch, u, maps, rng, n=n, c=3, srow_pad=0, simg_pad=0, soff=0, drow_pad=drow_pad, dimg_pad=dimg_pad))
            for c in (1, 4):
                _layout_case(torch, u, maps, rng, n=n, c=c, srow_pad=3, simg_pad=5, soff=1, drow_pad=2, dimg_pad=6)
        u.close()
    assert paths == {True, False}


def test_torch_stream_ordering(fx, torch):
    """The frames are written by a torch kernel on a non-default stream just before the call; the call runs there."""
    rng = np.random.default_rng(31)
    u, maps = _und(fx, "fisheye", False, (640, 512), (640, 512), 1.0)
    host = _frames(rng, 6, 512, 640, 3)
    big = torch.from_numpy(host).cuda()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        frames = torch.zeros_like(big)
        frames.copy_(big)
        frames.add_(1)                                       # in place on s; the gather must see it
        out = u.cuda(frames)
    s.synchronize()
    got = out.cpu().numpy()
    for i in range(6):
        assert (got[i] == _want(maps, host[i] + np.uint8(1))).all(), i
    u.close()


def test_graph_capture_and_replay_after_rewrite(fx, torch):
    rng = np.random.default_rng(41)
    u, maps = _und(fx, "fisheye", True, (96, 64), (96, 64), 0.8)
    n = 5
    frames = torch.from_numpy(_frames(rng, n, 64, 96, 3)).cuda()
    out = torch.empty((n, 64, 96, 3), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    lib, ctx = u.ctx.lib, u.ctx
    call = lambda: lib.bevk_undistort_stack(ctx.h, u.slot, ctypes.c_void_p(frames.data_ptr()), 64 * 96 * 3, 96, 64, 96 * 3, 3, n,
                                            ctypes.c_void_p(out.data_ptr()), 64 * 96 * 3, 96, 64, 96 * 3, 1)
    assert call() == 0
    ctx.sync()
    with ctx.graph_capture() as g:
        assert call() == 0
    for rep in range(3):
        host = _frames(rng, n, 64, 96, 3)
        frames.copy_(torch.from_numpy(host))                  # rewritten in place, same pointers
        out.fill_(0)
        torch.cuda.synchronize()
        g.launch()
        ctx.sync()
        got = out.cpu().numpy()
        for i in range(n):
            assert (got[i] == _want(maps, host[i])).all(), (rep, i)
    g.destroy()
    u.close()


def test_dropin_classes_take_cuda_tensors(fx, torch):
    """InCalibrator.undistort and Camera.undistort on CUDA tensors: results stay on the device and equal the NumPy path."""
    from cameracalibration_b200.IntrinsicCalibration import InCalibrator
    from cameracalibration_b200.SurroundBirdEyeView import surroundBEV as S
    K, D, _ = fx.calib["front"]
    a = InCalibrator.get_args()
    a.FRAME_WIDTH, a.FRAME_HEIGHT, a.FOCAL_SCALE, a.SIZE_SCALE = 1280, 1024, 0.5, 1
    cal = InCalibrator("fisheye")
    cal.set_calibration(K, D)
    raw = fx.img("raw0")
    t = torch.from_numpy(raw).cuda()
    got = cal.undistort(t)
    assert isinstance(got, torch.Tensor) and got.is_cuda
    assert (got.cpu().numpy() == cal.undistort(raw)).all()
    batch = cal.undistort(torch.stack([t, t.flip(0).contiguous()]))
    assert (batch[1].cpu().numpy() == cal.undistort(np.ascontiguousarray(raw[::-1]))).all()
    cam = S.Camera("front", fx.calib["front"])
    got = cam.undistort(torch.from_numpy(fx.img("front")).cuda())
    assert got.is_cuda and (got.cpu().numpy() == cam.undistort(fx.img("front"))).all()
    maps = C.undistort_maps(K, D, cam.camera_mat_dst, *cam._g.und_size)
    assert (got.cpu().numpy() == _want(maps, fx.img("front"))).all()


def test_jpeg_decode_then_undistort(fx, torch):
    """ops.jpeg_decode -> Undistorter.cuda: the chain include/bevk.h describes, against cv2.remap of the decoded frames."""
    from cameracalibration_b200 import ops
    jpegs = [cv2.imencode(".jpg", fx.img(n), [cv2.IMWRITE_JPEG_QUALITY, 90])[1].tobytes() for n in ("front", "back", "left")]
    K, D, _ = fx.calib["front"]
    P = C.dst_camera_matrix(K, 1280, 1024, 1, 1)
    u = ops.Undistorter(K, D, P, (1280, 1024))
    decoded = ops.jpeg_decode(jpegs, 1280, 1024, ctx=u.ctx)
    out = u.cuda(decoded).cpu().numpy()
    host = decoded.cpu().numpy()
    maps = C.undistort_maps(K, D, P, 1280, 1024)
    for i in range(3):
        assert (out[i] == _want(maps, host[i])).all(), i
    u.close()


@pytest.mark.parametrize("chunk", [None, "3"])
def test_cuda_to_jpeg_streams(fx, torch, monkeypatch, chunk):
    """Streams equal cv2.imencode(cv2.remap(...)) at q 1/50/95/100 for batches that cross a chunk boundary."""
    if chunk:
        monkeypatch.setenv("BEVK_JPEG_CHUNK", chunk)
    rng = np.random.default_rng(51)
    for fused in (False, True):
        u, maps = _und(fx, "fisheye", fused, (320, 256), (324, 250), 0.8)
        host = np.stack([cv2.resize(fx.img(n), (320, 256)) for n in ("front", "back", "left", "right")] * 3)[:10]
        host[5:] = _frames(rng, 5, 256, 320, 3)
        frames = torch.from_numpy(host).cuda()
        for q in (1, 50, 95, 100):
            streams = u.cuda_to_jpeg(frames, q)
            assert len(streams) == 10
            for i in range(10):
                want = cv2.imencode(".jpg", _want(maps, host[i]), [cv2.IMWRITE_JPEG_QUALITY, q])[1].tobytes()
                assert streams[i] == want, (fused, q, i)
        assert u.cuda_to_jpeg(frames[3]) == u.cuda_to_jpeg(frames[3:4])
        u.close()


def test_jpeg_capacity_rule(fx, torch):
    from cameracalibration_b200 import ops
    u, maps = _und(fx, "fisheye", False, (200, 160), (200, 160), 0.8)
    frames = torch.from_numpy(_frames(np.random.default_rng(61), 11, 160, 200, 3)).cuda()
    torch.cuda.synchronize()
    streams = u.cuda_to_jpeg(frames, 90)
    total = sum(len(s) for s in streams)
    lib = u.ctx.lib
    cap = total - 1
    out = np.full(total + 4096, 0x5A, np.uint8)
    sizes = (ctypes.c_uint64 * 11)()
    rc = lib.bevk_undistort_stack_jpeg(u.ctx.h, u.slot, ctypes.c_void_p(frames.data_ptr()), 160 * 200 * 3, 200, 160, 200 * 3, 11,
                                       ops.INTER_LINEAR, 90, out.ctypes.data_as(ctypes.c_void_p), cap, sizes)
    assert rc != 0 and "capacity" in lib.bevk_last_error().decode()
    assert list(sizes) == [len(s) for s in streams]
    lead = b"".join(streams[:-1])                               # every stream but the last fits
    assert out[:len(lead)].tobytes() == lead
    assert (out[len(lead):] == 0x5A).all(), "bytes written at or past capacity"
    rc = lib.bevk_undistort_stack_jpeg(u.ctx.h, u.slot, ctypes.c_void_p(frames.data_ptr()), 160 * 200 * 3, 200, 160, 200 * 3, 11,
                                       ops.INTER_LINEAR, 90, out.ctypes.data_as(ctypes.c_void_p), total, sizes)
    assert rc == 0 and out[:total].tobytes() == b"".join(streams)
    u.close()


def test_errors(fx, torch):
    from cameracalibration_b200 import _lib as L
    u, _ = _und(fx, "fisheye", False, (64, 48), (64, 48), 0.8)
    lib, h, s = u.ctx.lib, u.ctx.h, u.slot
    src = torch.zeros((4, 48, 64, 3), dtype=torch.uint8, device="cuda")
    dst = torch.zeros((4, 48, 64, 3), dtype=torch.uint8, device="cuda")
    sp, dp = ctypes.c_void_p(src.data_ptr()), ctypes.c_void_p(dst.data_ptr())
    img, row = 48 * 64 * 3, 64 * 3

    def call(src=sp, simg=img, srow=row, ch=3, n=4, dst=dp, dimg=img, dw=64, dh=48, drow=row, interp=1):
        rc = lib.bevk_undistort_stack(h, s, src, simg, 64, 48, srow, ch, n, dst, dimg, dw, dh, drow, interp)
        return rc, lib.bevk_last_error().decode()

    assert call()[0] == 0
    for kw, msg in [(dict(dw=63), "map"), (dict(dh=49), "map"), (dict(ch=2), "channels"), (dict(n=0), "n must"),
                    (dict(dst=ctypes.c_void_p(src.data_ptr() + img)), "overlaps"), (dict(dst=sp), "overlaps"),
                    (dict(srow=row - 1), "stride"), (dict(drow=row - 3), "stride"), (dict(simg=img - 1), "image stride"),
                    (dict(dimg=img - row), "image stride"), (dict(interp=2), "interp")]:
        rc, err = call(**kw)
        assert rc != 0 and msg in err, (kw, err)
    assert call(n=1, simg=0, dimg=0)[0] == 0                     # image strides are not read for one frame
    with pytest.raises(L.BevkError, match="CUDA array"):
        u.cuda(np.zeros((48, 64, 3), np.uint8))
    with pytest.raises(L.BevkError, match="shape"):
        u.cuda(src, out=torch.zeros((4, 48, 63, 3), dtype=torch.uint8, device="cuda"))
    with pytest.raises(L.BevkError):
        u.cuda(torch.zeros((48, 64, 2), dtype=torch.uint8, device="cuda"))
    with pytest.raises(L.BevkError, match="3"):
        u.cuda_to_jpeg(torch.zeros((2, 48, 64, 1), dtype=torch.uint8, device="cuda"))
    lib.bevk_graph_begin(h)
    try:
        out, sizes = np.zeros(1 << 16, np.uint8), (ctypes.c_uint64 * 4)()
        rc = lib.bevk_undistort_stack_jpeg(h, s, sp, img, 64, 48, row, 4, 1, 95, out.ctypes.data_as(ctypes.c_void_p), out.size, sizes)
        assert rc != 0 and "graph" in lib.bevk_last_error().decode()
    finally:
        gid = ctypes.c_int(-1)
        if lib.bevk_graph_end(h, ctypes.byref(gid)) == 0:
            lib.bevk_graph_destroy(h, gid)
    u.close()
    with pytest.raises(L.BevkError, match="closed"):
        u.cuda(src)
    with pytest.raises(L.BevkError, match="closed"):
        u(src)
