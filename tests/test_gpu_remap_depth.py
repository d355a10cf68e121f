"""16U, 16S and 32F images through the device gathers, against cv2 bit for bit (float32: the bit pattern, NaN where
cv2 gives NaN): ops.remap (CV_16SC2 maps with and without map2, float maps), Undistorter slots (map-resident and fused,
CV_16SC2 and float maps, both lens models), ops.warp_perspective and ops.warp_affine (WARP_INVERSE_MAP too), each on
NumPy images and, where the call has one, on CUDA batches with padded rows and images at odd element-aligned offsets; a
captured and replayed graph; the refusals; and the uint8 calls' paths unchanged."""
import ctypes

import cv2
import numpy as np
import pytest

from tests import float_map_cases as FC
from tests.test_host_remap_depth import DEPTHS, DEPTH_IDS, INTERS, cv2_warp_differs, same, values

pytestmark = pytest.mark.gpu
ERR_ARG, ERR_UNSUPPORTED = -1, -4


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


def _as3(a):
    return a.reshape(a.shape[0], a.shape[1], -1)


def _padded(torch, host, off=3, pad_row=5, pad_img=7):
    """host [N][H][W][C] as a CUDA view at an odd element offset, rows and images padded by whole elements."""
    n, h, w, ch = host.shape
    row = w * ch + pad_row
    img = h * row + pad_img
    t = torch.from_numpy(np.ascontiguousarray(host))
    pool = torch.zeros(off + n * img, dtype=t.dtype, device="cuda")
    view = pool.as_strided((n, h, w, ch), (img, row, ch, 1), off)
    view.copy_(t)
    return view


def _cv(call, f):
    return _as3(call(f if f.shape[2] > 1 else f[..., 0]))


def _check_both(torch, rng, depth, sw, sh, host_call, device_call, want_call, inter, what, n=3, skip=lambda ch: False):
    """One NumPy image through host_call and an n-frame CUDA batch through device_call (None: no device form), at every
    channel count but those skip() names."""
    for ch in (1, 3, 4):
        if skip(ch):
            continue
        frames = values(rng, depth, (n, sh, sw, ch), 0.03)
        want = [_cv(want_call, f) for f in frames]
        got = _as3(host_call(frames[0] if ch > 1 else frames[0, :, :, 0]))
        assert got.dtype == frames.dtype and same(got, want[0], inter), (what, ch, inter, "host")
        if device_call is not None:
            out = device_call(_padded(torch, frames))
            assert out.dtype == getattr(torch, np.dtype(DEPTHS[depth]).name)
            got = out.cpu().numpy()
            for i in range(n):
                assert same(got[i], want[i], inter), (what, ch, inter, "device", i)


@pytest.mark.parametrize("depth", DEPTHS, ids=DEPTH_IDS)
def test_remap(torch, depth):
    """ops.remap: CV_16SC2 maps (map2 omitted for NEAREST too) on NumPy images; CV_32FC1 / CV_32FC2 maps on NumPy images
    and CUDA batches (CUDA and NumPy maps)."""
    from cameracalibration_b200 import ops
    rng = np.random.default_rng(1 + depth)
    sw, sh, dw, dh = 61, 47, 72, 53
    x = rng.uniform(-6, sw + 6, (dh, dw)).astype(np.float32)
    y = rng.uniform(-6, sh + 6, (dh, dw)).astype(np.float32)
    m1, m2 = cv2.convertMaps(x, y, cv2.CV_16SC2)
    xy = np.dstack([x, y])
    dx, dy = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    for inter in INTERS:
        _check_both(torch, rng, depth, sw, sh, lambda f: ops.remap(f, m1, m2, inter), None,
                    lambda f: cv2.remap(f, m1, m2, inter), inter, "16SC2")
        _check_both(torch, rng, depth, sw, sh, lambda f: ops.remap(f, x, y, inter), lambda d: ops.remap(d, dx, dy, inter),
                    lambda f: cv2.remap(f, x, y, inter), inter, "32FC1")
        _check_both(torch, rng, depth, sw, sh, lambda f: ops.remap(f, xy, None, inter), lambda d: ops.remap(d, xy, None, inter),
                    lambda f: cv2.remap(f, xy, None, inter), inter, "32FC2")
    n1, _ = cv2.convertMaps(x, y, cv2.CV_16SC2, nninterpolation=True)
    _check_both(torch, rng, depth, sw, sh, lambda f: ops.remap(f, n1, None, cv2.INTER_NEAREST), None,
                lambda f: cv2.remap(f, n1, None, cv2.INTER_NEAREST), cv2.INTER_NEAREST, "16SC2 without map2")


@pytest.mark.parametrize("depth", DEPTHS, ids=DEPTH_IDS)
def test_warps(torch, depth):
    """ops.warp_perspective (NumPy) and ops.warp_affine (NumPy and CUDA, with and without WARP_INVERSE_MAP) at every
    interpolation and channel count the library takes at this depth; the cases cv2 computes with other bodies than
    cv2.remap's (cv2_warp_differs) are refused with BEVK_ERR_UNSUPPORTED on both forms."""
    from cameracalibration_b200 import ops
    from cameracalibration_b200 import _lib as L
    rng = np.random.default_rng(10 + depth)
    sw, sh, dw, dh = 57, 43, 64, 49
    H = np.array([[0.9, 0.05, 1.3], [-0.04, 1.1, -2.2], [1e-3, -2e-3, 1.0]])
    M = cv2.getRotationMatrix2D((sw / 2, sh / 2), 23.0, 1.07)
    for inter in INTERS:
        for ch in (1, 3, 4):   # the refused cases, one channel count at a time
            img = values(rng, depth, (sh, sw, ch))
            if cv2_warp_differs(2, depth, inter, ch):
                with pytest.raises(L.BevkError, match="another body"):
                    ops.warp_perspective(img, H, (dw, dh), inter)
            if cv2_warp_differs(3, depth, inter, ch):
                for fl in (inter, inter | cv2.WARP_INVERSE_MAP):
                    with pytest.raises(L.BevkError, match="another body"):
                        ops.warp_affine(img, M, (dw, dh), fl)
                    with pytest.raises(L.BevkError, match="another body"):
                        ops.warp_affine(_padded(torch, img[None]), M, (dw, dh), fl)
        _check_both(torch, rng, depth, sw, sh, lambda f: ops.warp_perspective(f, H, (dw, dh), inter), None,
                    lambda f: cv2.warpPerspective(f, H, (dw, dh), flags=inter), inter, "perspective",
                    skip=lambda ch: cv2_warp_differs(2, depth, inter, ch))
        for fl in (inter, inter | cv2.WARP_INVERSE_MAP):
            _check_both(torch, rng, depth, sw, sh, lambda f: ops.warp_affine(f, M, (dw, dh), fl),
                        lambda d: ops.warp_affine(d, M, (dw, dh), fl),
                        lambda f: cv2.warpAffine(f, M, (dw, dh), flags=fl), inter, ("affine", fl),
                        skip=lambda ch: cv2_warp_differs(3, depth, inter, ch))


def _slot_cases():
    return [("stereo_vertical_left", cv2.CV_16SC2, False), ("pinhole14_R", cv2.CV_16SC2, True),
            ("stereo_vertical_right", cv2.CV_32FC1, False), ("pinhole12", cv2.CV_32FC2, True),
            ("fisheye_R", cv2.CV_32FC1, False), ("fisheye", cv2.CV_32FC1, True), ("fisheye", cv2.CV_16SC2, True)]


@pytest.mark.parametrize("depth", DEPTHS, ids=DEPTH_IDS)
@pytest.mark.parametrize("name,m1type,fused", _slot_cases())
def test_undistorter_slots(torch, depth, name, m1type, fused):
    """Map-resident and fused slots of both models, CV_16SC2 and float maps: __call__ on NumPy images and cuda() on CUDA
    batches == cv2.remap through the slot's own maps (which the existing tests hold to cv2's)."""
    from cameracalibration_b200 import ops
    c = FC.case_by_name(name)
    u = ops.Undistorter(c.K, c.D, c.P, (c.W, c.H), model="fisheye" if c.fisheye else "pinhole", fused=fused, R=c.R,
                        m1type=m1type)
    maps = u.maps()
    rng = np.random.default_rng(20 + depth)
    for inter in INTERS:
        _check_both(torch, rng, depth, c.SW, c.SH, lambda f: u(f, interpolation=inter),
                    lambda d: u.cuda(d, interpolation=inter), lambda f: cv2.remap(f, *maps, inter), inter, (name, m1type),
                    n=2)
    u.close()


def test_graph_capture(torch):
    """bevk_undistort_stack_interp_typed (CV_32FC3, LANCZOS4) captured in a CUDA graph and replayed over rewritten frames."""
    from cameracalibration_b200 import ops
    from cameracalibration_b200 import _lib as L
    ctx = L.default_context()
    c = FC.case_by_name("pinhole12")
    u = ops.Undistorter(c.K, c.D, c.P, (c.W, c.H), model="pinhole", m1type=cv2.CV_32FC1, ctx=ctx)
    maps = u.maps()
    n, es = 3, 4
    frames = torch.zeros((n, c.SH, c.SW, 3), dtype=torch.float32, device="cuda")
    out = torch.empty((n, c.H, c.W, 3), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    call = lambda: ctx.lib.bevk_undistort_stack_interp_typed(
        ctx.h, u.slot, ctypes.c_void_p(frames.data_ptr()), c.SH * c.SW * 3 * es, c.SW, c.SH, c.SW * 3 * es, 5 + (2 << 3), n,
        ctypes.c_void_p(out.data_ptr()), c.H * c.W * 3 * es, c.W, c.H, c.W * 3 * es, cv2.INTER_LANCZOS4)
    assert call() == 0
    ctx.sync()
    with ctx.graph_capture() as g:
        assert call() == 0
    rng = np.random.default_rng(4)
    for rep in range(2):
        host = values(rng, 5, (n, c.SH, c.SW, 3), 0.01)
        frames.copy_(torch.from_numpy(host))
        out.fill_(0)
        torch.cuda.synchronize()
        g.launch()
        ctx.sync()
        got = out.cpu().numpy()
        for i in range(n):
            assert same(got[i], cv2.remap(host[i], *maps, cv2.INTER_LANCZOS4), cv2.INTER_LANCZOS4), (rep, i)
    g.destroy()
    u.close()


def test_refusals_write_nothing(torch):
    """CV_8S, CV_16F and CV_64F: BEVK_ERR_UNSUPPORTED; base pointers, row strides and image strides that are not
    multiples of the element: BEVK_ERR_ARG; the destination is left untouched."""
    from cameracalibration_b200 import _lib as L
    ctx = L.default_context()
    vp = ctypes.c_void_p
    m1 = np.zeros((8, 8, 2), np.int16)
    m2 = np.zeros((8, 8), np.uint16)
    src = np.ones(64 * 64, np.float64)
    dst = np.full(64 * 64, 7, np.float64)
    for t in (1, 7, 6, 6 + (2 << 3)):   # CV_8S, CV_16F, CV_64F, CV_64FC3
        assert ctx.lib.bevk_remap_typed(ctx.h, L.vptr(src), 8, 8, 64, t, L.vptr(m1), L.vptr(m2), 8, 8, L.vptr(dst), 64,
                                        cv2.INTER_LINEAR) == ERR_UNSUPPORTED, t
    base = src.ctypes.data
    for sp, ss, dp, ds in ((base + 1, 32, dst.ctypes.data, 32), (base, 33, dst.ctypes.data, 32),
                           (base, 32, dst.ctypes.data + 1, 32), (base, 32, dst.ctypes.data, 35)):
        assert ctx.lib.bevk_remap_typed(ctx.h, vp(sp), 8, 8, ss, 2, L.vptr(m1), L.vptr(m2), 8, 8, vp(dp), ds,
                                        cv2.INTER_LINEAR) == ERR_ARG
        assert ctx.lib.bevk_warp_affine_typed(ctx.h, vp(sp), 8, 8, ss, 5, L.dptr(np.eye(2, 3)), vp(dp), 8, 8, ds,
                                              cv2.INTER_LINEAR) == ERR_ARG
    assert (dst == 7).all()
    d_src = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    d_dst = torch.full((4096,), 9, dtype=torch.uint8, device="cuda")
    M = np.eye(2, 3)
    for off, rs, img in ((1, 32, 512), (0, 34, 512), (0, 32, 510)):   # CV_32FC1 8x8 frames, n = 2
        assert ctx.lib.bevk_warp_affine_stack_typed(ctx.h, vp(d_src.data_ptr() + off), img, 8, 8, rs, 5, 2, L.dptr(M),
                                                    vp(d_dst.data_ptr() + 2048), 512, 8, 8, 32, cv2.INTER_LINEAR) == ERR_ARG
    torch.cuda.synchronize()
    assert (d_dst == 9).all()


def test_uint8_paths_unchanged(torch):
    """The uint8 calls still take their paths (word, byte, taps) and give cv2's bytes; a uint16 call of the same shape
    takes the byte path."""
    from cameracalibration_b200 import ops
    rng = np.random.default_rng(3)
    img = rng.integers(0, 256, (40, 64, 3), dtype=np.uint8)
    x = rng.uniform(-2, 66, (32, 64)).astype(np.float32)
    y = rng.uniform(-2, 42, (32, 64)).astype(np.float32)
    for inter, path in ((cv2.INTER_LINEAR, "word"), (cv2.INTER_NEAREST, "byte"), (cv2.INTER_CUBIC, "taps")):
        assert (ops.remap(torch.from_numpy(img).cuda(), x, y, inter).cpu().numpy() == cv2.remap(img, x, y, inter)).all()
        assert ops.last_path() == path
    got = ops.remap(torch.from_numpy(img.astype(np.uint16)).cuda(), x, y, cv2.INTER_LINEAR).cpu().numpy()
    assert ops.last_path() == "byte" and (got == cv2.remap(img.astype(np.uint16), x, y, cv2.INTER_LINEAR)).all()
