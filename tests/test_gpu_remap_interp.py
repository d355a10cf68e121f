"""INTER_CUBIC and INTER_LANCZOS4 on the GPU (k_gather_taps): every entry point against live cv2, byte for byte.

ops.remap and ops.warp_perspective; Undistorter called on NumPy frames and through .cuda, map and fused slots, fisheye
and pinhole, 1/3/4 channels; batches across GATHER_NB with padded rows and images and odd base pointers; .jpeg, .png and
.cuda_to_jpeg against cv2.imencode of cv2.remap; a captured CUDA graph; the refusals.  For pinhole slots the oracle is
cv2.remap over Undistorter.maps() (cv2's own pinhole maps differ in fraction entries of off-frame taps, DESIGN.md
section 7); cv2's own maps are the oracle too wherever the two map pairs agree."""
import ctypes

import cv2
import numpy as np
import pytest

from oracle import cv2_path as C
from tests import bev_cases as B
from tests import calib_cases as CC

pytestmark = pytest.mark.gpu
INTERS = (cv2.INTER_CUBIC, cv2.INTER_LANCZOS4)
FILL = 0xA5


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


def _remap(frame, m1, m2, inter):
    out = cv2.remap(np.ascontiguousarray(frame), m1, m2, inter)
    return out.reshape(out.shape[0], out.shape[1], -1)


def _und(fx, model, fused, src, dst, fs):
    """An Undistorter for the front camera scaled to `src`, its own maps and cv2's maps."""
    from cameracalibration_b200 import ops
    K, D, _ = fx.calib["front"]
    K = np.diag([src[0] / 1280, src[1] / 1024, 1.0]) @ K
    P = C.dst_camera_matrix(K, dst[0], dst[1], fs, 1)
    if model == "fisheye":
        theirs = C.undistort_maps(K, D, P, *dst)
        u = ops.Undistorter(K, D, P, dst, model="fisheye", fused=fused)
    else:
        theirs = C.pinhole_maps(K, fx.D5, P, *dst)
        u = ops.Undistorter(K, fx.D5, P, dst, model="pinhole", fused=fused)
    return u, u.maps(), theirs


def _check_und(got, frame, ours, theirs, inter, model, what):
    """got == cv2.remap over the library's maps, and over cv2's maps wherever the entries agree (fisheye: everywhere)."""
    want = _remap(frame, *ours, inter)
    got = got.reshape(want.shape)
    assert (got == want).all(), (what, int((got != want).sum()))
    same = (ours[0] == theirs[0]).all(-1) & (ours[1] == theirs[1])
    assert model != "fisheye" or same.all(), what
    assert (got[same] == _remap(frame, *theirs, inter)[same]).all(), what
    return 1


@pytest.mark.parametrize("inter", INTERS, ids=["cubic", "lanczos4"])
def test_ops_remap(inter):
    from cameracalibration_b200 import ops
    rng = np.random.default_rng(50 + inter)
    compared = 0
    for i, kind in enumerate(("local", "extreme", "local", "extreme")):
        FW, FH = ((5, 3), (64, 40), (97, 65), (7, 8))[i]
        for ch in (1, 3, 4):
            for m1, m2 in B._maps(rng, kind, 1, FW, FH, 77, 45):
                src = rng.integers(0, 256, (FH, FW, ch), dtype=np.uint8)
                img = src[..., 0] if ch == 1 else src
                got = ops.remap(img, m1, m2, inter)
                want = cv2.remap(img, m1, m2, inter)
                assert (got == want).all(), (kind, FW, FH, ch, int((got != want).sum()))
                ctx = ops.L.default_context()
                assert ctx.lib.bevk_undistort_last_path(ctx.h) == 2
                compared += 1
    # INTER_AREA is INTER_LINEAR, as cv2.remap reads it
    src = rng.integers(0, 256, (40, 64, 3), dtype=np.uint8)
    m1, m2 = B._maps(rng, "local", 1, 64, 40, 77, 45)[0]
    got = ops.remap(src, m1, m2, ops.INTER_AREA)
    assert (got == cv2.remap(src, m1, m2, cv2.INTER_AREA)).all() and (got == ops.remap(src, m1, m2, ops.INTER_LINEAR)).all()
    assert compared == 12


@pytest.mark.parametrize("inter", INTERS, ids=["cubic", "lanczos4"])
def test_ops_warp_perspective(inter):
    from cameracalibration_b200 import ops
    compared = 0
    for i, c in enumerate(CC.corpus()[12::4]):
        ch = (1, 3, 4)[i % 3]
        sw, sh = min(c.UW, 1000), min(c.UH, 800)
        f = CC.frames(c.name, ch, 1, (sw, sh))[0]
        img = f[..., 0] if ch == 1 else f
        got = ops.warp_perspective(img, c.H, (c.BW, c.BH), inter)
        want = cv2.warpPerspective(img, c.H, (c.BW, c.BH), flags=inter)
        assert (got == want).all(), (c.name, ch, int((got != want).sum()))
        compared += 1
    c = CC.corpus()[13]
    img = CC.frames(c.name, 3, 1, (400, 300))[0]
    got = ops.warp_perspective(img, c.H, (c.BW, c.BH), ops.INTER_AREA)
    assert (got == cv2.warpPerspective(img, c.H, (c.BW, c.BH), flags=cv2.INTER_AREA)).all()
    assert compared > 0


@pytest.mark.parametrize("model", ["fisheye", "pinhole"])
@pytest.mark.parametrize("fused", [False, True])
def test_undistorter_numpy_and_cuda(fx, torch, model, fused):
    """Map and fused slots, both models, 1/3/4 channels, both kernels; NumPy frames and a CUDA batch of 5."""
    rng = np.random.default_rng(60 + fused + 2 * (model == "pinhole"))
    compared = 0
    for dst in ((96, 40), (83, 37)):
        u, ours, theirs = _und(fx, model, fused, (72, 50), dst, 0.6)
        for ch in (1, 3, 4):
            host = rng.integers(0, 256, (5, 50, 72, ch), dtype=np.uint8)
            frames = torch.from_numpy(host).cuda()
            for inter in INTERS:
                one = host[0][..., 0] if ch == 1 else host[0]
                compared += _check_und(u(one, inter), one, ours, theirs, inter, model, (dst, ch, inter, "numpy"))
                assert u.last_path() == "taps"
                out = u.cuda(frames, interpolation=inter).cpu().numpy()
                assert u.last_path() == "taps"
                for i in range(5):
                    compared += _check_und(out[i], host[i], ours, theirs, inter, model, (dst, ch, inter, i))
        u.close()
    assert compared == 2 * 3 * 2 * 6


@pytest.mark.parametrize("fused", [False, True])
def test_reference_size(fx, torch, fused):
    """The reference's four frames, 1280x1024 -> 2560x2048 (SIZE_SCALE 2), as one batch."""
    from cameracalibration_b200 import ops
    K, D, _ = fx.calib["front"]
    P = C.dst_camera_matrix(K, 1280, 1024, 1, 2)
    maps = C.undistort_maps(K, D, P, 2560, 2048)
    host = np.stack([fx.img(n) for n in ("front", "back", "left", "right")])
    frames = torch.from_numpy(host).cuda()
    u = ops.Undistorter(K, D, P, (2560, 2048), fused=fused)
    for inter in INTERS:
        out = u.cuda(frames, interpolation=inter).cpu().numpy()
        for i in range(4):
            assert (out[i] == _remap(host[i], *maps, inter)).all(), (fused, inter, i)
    u.close()


def _layout_case(torch, u, ours, rng, inter, *, n, c, srow_pad, simg_pad, soff, drow_pad, dimg_pad):
    """bevk_undistort_stack_interp over frames at soff + f * simg of one device buffer, into a FILL-ed buffer with a sentinel
    image after the last output."""
    sw, sh, dw, dh = 40, 30, u.w, u.h
    srow, drow = sw * c + srow_pad, dw * c + drow_pad
    simg, dimg = sh * srow + simg_pad, dh * drow + dimg_pad
    sbuf = rng.integers(0, 256, soff + n * simg + 64, dtype=np.uint8)
    dbuf = np.full((n + 1) * dimg + 64, FILL, np.uint8)
    ds, dd = torch.from_numpy(sbuf).cuda(), torch.from_numpy(dbuf).cuda()
    torch.cuda.synchronize()
    lib = u.ctx.lib
    rc = lib.bevk_undistort_stack_interp(u.ctx.h, u.slot, ctypes.c_void_p(ds.data_ptr() + soff), simg, sw, sh, srow, c, n,
                                         ctypes.c_void_p(dd.data_ptr()), dimg, dw, dh, drow, inter)
    assert rc == 0, lib.bevk_last_error().decode()
    u.ctx.sync()
    assert lib.bevk_undistort_last_path(u.ctx.h) == 2
    out = dd.cpu().numpy()
    touched = np.zeros(out.size, bool)
    for f in range(n):
        frame = np.lib.stride_tricks.as_strided(sbuf[soff + f * simg:], (sh, sw, c), (srow, c, 1))
        got = np.lib.stride_tricks.as_strided(out[f * dimg:], (dh, dw, c), (drow, c, 1))
        assert (got == _remap(frame, *ours, inter)).all(), (n, c, srow_pad, simg_pad, soff, drow_pad, dimg_pad, f)
        np.lib.stride_tricks.as_strided(touched[f * dimg:], got.shape, got.strides)[...] = True
    assert (out[~touched] == FILL).all(), "padding or the sentinel image was written"
    return n


@pytest.mark.parametrize("inter", INTERS, ids=["cubic", "lanczos4"])
@pytest.mark.parametrize("fused", [False, True])
def test_batches_padding_odd_bases(fx, torch, inter, fused):
    rng = np.random.default_rng(70 + inter + fused)
    u, ours, _ = _und(fx, "pinhole" if fused else "fisheye", fused, (40, 30), (45, 27), 0.6)
    compared = 0
    for i, n in enumerate((1, 3, 8, 9, 17)):
        for c in (1, 3, 4):
            compared += _layout_case(torch, u, ours, rng, inter, n=n, c=c, srow_pad=(0, 4, 7)[i % 3], simg_pad=(0, 5, 12)[(i + c) % 3],
                                     soff=(0, 1, 3)[(i + c) % 3], drow_pad=(0, 3)[i % 2], dimg_pad=(0, 9)[(i + 1) % 2])
    assert compared == 3 * (1 + 3 + 8 + 9 + 17)
    u.close()


@pytest.mark.parametrize("fused", [False, True])
def test_jpeg_png_and_cuda_to_jpeg(fx, torch, fused):
    rng = np.random.default_rng(80 + fused)
    u, ours, _ = _und(fx, "fisheye", fused, (120, 90), (128, 96), 0.7)
    host = rng.integers(0, 256, (3, 90, 120, 3), dtype=np.uint8)
    frames = torch.from_numpy(host).cuda()
    jparams = [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, cv2.IMWRITE_JPEG_OPTIMIZE, 1]
    pparams = [cv2.IMWRITE_PNG_COMPRESSION, 9]
    compared = 0
    for inter in INTERS:
        ref = [_remap(h, *ours, inter) for h in host]
        got = u.jpeg(host[0], 90, inter, jparams)
        assert got == cv2.imencode(".jpg", ref[0], [cv2.IMWRITE_JPEG_QUALITY, 90] + jparams)[1].tobytes(), inter
        got = u.png(host[1], pparams, inter)
        assert got == cv2.imencode(".png", ref[1], pparams)[1].tobytes(), inter
        streams = u.cuda_to_jpeg(frames, 85, inter, jparams)
        assert len(streams) == 3
        for i in range(3):
            assert streams[i] == cv2.imencode(".jpg", ref[i], [cv2.IMWRITE_JPEG_QUALITY, 85] + jparams)[1].tobytes(), (inter, i)
            compared += 1
    assert compared == 6
    u.close()


def test_graph_capture_cubic(fx, torch):
    """One Undistorter.cuda(..., interpolation=INTER_CUBIC) captured into a CUDA graph and replayed over rewritten
    frames: the tables were uploaded with the ctx, so the call only enqueues its kernel."""
    from cameracalibration_b200 import ops
    rng = np.random.default_rng(90)
    u, ours, _ = _und(fx, "fisheye", True, (96, 64), (96, 64), 0.8)
    n = 9
    frames = torch.from_numpy(rng.integers(0, 256, (n, 64, 96, 3), dtype=np.uint8)).cuda()
    out = torch.empty((n, 64, 96, 3), dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with u.ctx.on_stream(s.cuda_stream):
        u.cuda(frames, out=out, interpolation=ops.INTER_CUBIC, stream=s.cuda_stream)
        u.ctx.sync()
        with u.ctx.graph_capture() as g:
            u.cuda(frames, out=out, interpolation=ops.INTER_CUBIC, stream=s.cuda_stream)
        for rep in range(2):
            host = rng.integers(0, 256, (n, 64, 96, 3), dtype=np.uint8)
            frames.copy_(torch.from_numpy(host))
            out.fill_(0)
            torch.cuda.synchronize()
            g.launch()
            u.ctx.sync()
            got = out.cpu().numpy()
            for i in range(n):
                assert (got[i] == _remap(host[i], *ours, cv2.INTER_CUBIC)).all(), (rep, i)
        g.destroy()
    u.close()


def test_refusals(fx, torch):
    from cameracalibration_b200 import _lib as L
    from cameracalibration_b200 import ops
    src = np.zeros((20, 30, 3), np.uint8)
    m1 = np.zeros((10, 12, 2), np.int16)
    for inter in INTERS:
        with pytest.raises(L.BevkError, match="needs map2"):
            ops.remap(src, m1, None, inter)
    for bad in (5, 7, -1, 16):
        with pytest.raises(L.BevkError, match="not supported"):
            ops.remap(src, m1, np.zeros((10, 12), np.uint16), bad)
    ctx = L.default_context()
    out = np.empty((10, 12, 3), np.uint8)
    m2 = np.zeros((10, 12), np.uint16)
    for bad in (5, 7, -1):   # the C entry points refuse unknown flags on their own
        assert ctx.lib.bevk_remap(ctx.h, L.vptr(src), 30, 20, 90, 3, L.vptr(m1), L.vptr(m2), 12, 10, L.vptr(out), 36, bad) == -4
        H = np.eye(3)
        assert ctx.lib.bevk_warp_perspective(ctx.h, L.vptr(src), 30, 20, 90, 3, L.dptr(H), L.vptr(out), 12, 10, 36, bad) == -4
    assert ctx.lib.bevk_remap(ctx.h, L.vptr(src), 30, 20, 90, 3, L.vptr(m1), None, 12, 10, L.vptr(out), 36, ops.INTER_CUBIC) == -1
    u, _, _ = _und(fx, "fisheye", False, (30, 20), (12, 10), 0.6)
    frames = torch.zeros((2, 20, 30, 3), dtype=torch.uint8, device="cuda")
    for bad in (5, 7):
        with pytest.raises(L.BevkError):
            u.cuda(frames, interpolation=bad)
        assert ctx.lib.bevk_undistort_stack_interp(u.ctx.h, u.slot, ctypes.c_void_p(frames.data_ptr()), 1800, 30, 20, 90, 3, 2,
                                                   ctypes.c_void_p(frames.data_ptr()), 1800, 12, 10, 36, bad) == -4
    # bevk_undistort_stack keeps its contract: NEAREST and LINEAR only
    out = torch.zeros((2, 10, 12, 3), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    for inter in (ops.INTER_CUBIC, ops.INTER_AREA, ops.INTER_LANCZOS4):
        args = (u.ctx.h, u.slot, ctypes.c_void_p(frames.data_ptr()), 1800, 30, 20, 90, 3, 2, ctypes.c_void_p(out.data_ptr()), 360, 12,
                10, 36, inter)
        assert ctx.lib.bevk_undistort_stack(*args) == -4 and "bevk_undistort_stack_interp" in L.load().bevk_last_error().decode()
        assert ctx.lib.bevk_undistort_stack_interp(*args) == 0, L.load().bevk_last_error().decode()
    u.ctx.sync()
    u.close()
    # the BEV engine keeps NEAREST and LINEAR only
    e = ops.BevEngine(1, (64, 48), (32, 32))
    for inter in INTERS:
        with pytest.raises(L.BevkError):
            e.set_interpolation(inter)
