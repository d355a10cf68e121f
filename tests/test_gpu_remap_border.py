"""cv2's border modes through the device gathers, against cv2 bit for bit (float32: the bit pattern, NaN where cv2 gives
NaN): ops.remap (CV_16SC2 and float maps, NumPy and CUDA sources), Undistorter slots (map-resident and fused, __call__
and cuda()), ops.warp_perspective and ops.warp_affine_border, at every depth and channel count, each under every border mode
with border values beyond the depth's range, at .5 and NaN; BORDER_TRANSPARENT over a filled ``out`` on the host and in
place on the device; padded CUDA batches; the word path under BORDER_REPLICATE; the C _border entry points; one
captured graph; the refusals."""
import ctypes

import cv2
import numpy as np
import pytest

from tests import float_map_cases as FC
from tests.test_host_remap_border import DEPTHS, DEPTH_IDS, INTERS, MODES, cv2_border_differs, values
from tests.test_host_remap_depth import cv2_warp_differs, same

pytestmark = pytest.mark.gpu
ERR_ARG, ERR_UNSUPPORTED = -1, -4
BVALS = [(0, 0, 0, 0), (300, -2, 7.5, 8.5), (np.nan, 65535.5, -1, 2.5), (17.25,), 9]


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


def _as3(a):
    return a.reshape(a.shape[0], a.shape[1], -1)


def _padded(torch, host, pad_row=4, pad_img=8):
    """host [N][H][W][C] as a CUDA view with rows and images padded by whole elements (4-byte aligned for uint8)."""
    n, h, w, ch = host.shape
    row = w * ch + pad_row
    img = h * row + pad_img
    t = torch.from_numpy(np.ascontiguousarray(host))
    pool = torch.zeros(n * img, dtype=t.dtype, device="cuda")
    view = pool.as_strided((n, h, w, ch), (img, row, ch, 1), 0)
    view.copy_(t)
    return view


def _squeeze(f):
    return f if f.shape[2] > 1 else f[..., 0]


def _check(torch, rng, depth, sw, sh, dw, dh, host_call, device_call, cv_call, inter, border, bval, what, n=2):
    """Every channel count: one NumPy image through host_call(src, out, mode, value) and (device_call not None) an
    n-frame padded CUDA batch through device_call(frames, out, mode, value), against cv_call(src, dst, mode, value).
    Under BORDER_TRANSPARENT ``out`` starts filled with noise, and cv2 gets the same noise as its dst."""
    for ch in (1, 3, 4):
        frames = values(rng, depth, (n, sh, sw, ch), 0.03)
        fill = values(rng, depth, (n, dh, dw, ch))
        want = [_as3(cv_call(_squeeze(frames[i]), _squeeze(fill[i]).copy(), border, bval)) for i in range(n)]
        out = _squeeze(fill[0]).copy() if border == cv2.BORDER_TRANSPARENT else None
        got = _as3(host_call(_squeeze(frames[0]), out, border, bval))
        assert same(got, want[0], inter), (what, ch, inter, border, bval, "host")
        if device_call is not None:
            dout = None
            if border == cv2.BORDER_TRANSPARENT:
                dout = _padded(torch, fill, 8, 16)
            res = device_call(_padded(torch, frames), dout, border, bval)
            got = res.cpu().numpy()
            for i in range(n):
                assert same(got[i], want[i], inter), (what, ch, inter, border, bval, "device", i)


@pytest.mark.parametrize("depth", DEPTHS, ids=DEPTH_IDS)
def test_remap(torch, depth):
    """ops.remap with CV_16SC2 maps (host) and float maps (host and CUDA batches), every mode and interpolation."""
    from cameracalibration_b200 import ops
    rng = np.random.default_rng(40 + depth)
    sw, sh, dw, dh = 23, 17, 36, 28
    m1 = np.stack([rng.integers(-12, sw + 12, (dh, dw)), rng.integers(-12, sh + 12, (dh, dw))], -1).astype(np.int16)
    m2 = rng.integers(0, 1024, (dh, dw)).astype(np.uint16)
    fx = rng.uniform(-12, sw + 12, (dh, dw)).astype(np.float32)
    fy = rng.uniform(-12, sh + 12, (dh, dw)).astype(np.float32)
    for k, border in enumerate(MODES):
        for j, inter in enumerate(INTERS):
            if cv2_border_differs(0, depth, inter, border):
                continue
            bval = BVALS[(k + j) % len(BVALS)]
            _check(torch, rng, depth, sw, sh, dw, dh,
                   lambda s, o, b, v: ops.remap(s, m1, m2, inter, out=o, borderMode=b, borderValue=v), None,
                   lambda s, d, b, v: cv2.remap(s, m1, m2, inter, dst=d, borderMode=b, borderValue=v), inter, border, bval,
                   "remap16")
            _check(torch, rng, depth, sw, sh, dw, dh,
                   lambda s, o, b, v: ops.remap(s, fx, fy, inter, out=o, borderMode=b, borderValue=v),
                   lambda s, o, b, v: ops.remap(s, fx, fy, inter, out=o, borderMode=b, borderValue=v),
                   lambda s, d, b, v: cv2.remap(s, fx, fy, inter, dst=d, borderMode=b, borderValue=v), inter, border, bval,
                   "remapf32")


@pytest.mark.parametrize("depth", DEPTHS, ids=DEPTH_IDS)
def test_warps(torch, depth):
    """ops.warp_perspective (host) and ops.warp_affine_border (host and CUDA batches, WARP_INVERSE_MAP too), zoomed out so that
    most pixels fall outside the source."""
    from cameracalibration_b200 import ops
    rng = np.random.default_rng(50 + depth)
    sw, sh, dw, dh = 21, 15, 40, 32
    H = np.array([[2.1, 0.2, 3.0], [-0.1, 2.3, 1.5], [2e-3, 1e-3, 1.0]])
    M = cv2.getRotationMatrix2D((sw / 2, sh / 2), 23.0, 1.7)
    for k, border in enumerate(MODES):
        for j, inter in enumerate(INTERS):
            bval = BVALS[(k + 2 * j) % len(BVALS)]
            differs = lambda mode: any(cv2_warp_differs(mode, depth, inter, c) for c in (1, 3, 4)) or \
                cv2_border_differs(mode, depth, inter, border)
            if not differs(2):
                _check(torch, rng, depth, sw, sh, dw, dh,
                       lambda s, o, b, v: ops.warp_perspective(s, H, (dw, dh), inter, out=o, borderMode=b, borderValue=v),
                       None,
                       lambda s, d, b, v: cv2.warpPerspective(s, H, (dw, dh), dst=d, flags=inter, borderMode=b,
                                                              borderValue=v), inter, border, bval, "persp")
            if differs(3):
                continue
            fl = inter | (cv2.WARP_INVERSE_MAP if k % 2 else 0)
            _check(torch, rng, depth, sw, sh, dw, dh,
                   lambda s, o, b, v: ops.warp_affine_border(s, M, (dw, dh), fl, out=o, borderMode=b, borderValue=v),
                   lambda s, o, b, v: ops.warp_affine_border(s, M, (dw, dh), fl, out=o, borderMode=b, borderValue=v),
                   lambda s, d, b, v: cv2.warpAffine(s, M, (dw, dh), dst=d, flags=fl, borderMode=b, borderValue=v),
                   inter, border, bval, "affine")


@pytest.mark.parametrize("fused", [0, 1])
@pytest.mark.parametrize("m1type", [cv2.CV_16SC2, cv2.CV_32FC1])
def test_undistorter_slots(torch, m1type, fused):
    """Map-resident and fused slots, CV_16SC2 and float maps: __call__ and cuda() == cv2.remap through the slot's maps,
    every depth, mode and interpolation."""
    from cameracalibration_b200 import ops
    c = FC.case_by_name("pinhole12")
    u = ops.Undistorter(c.K, c.D, c.P, (c.W, c.H), model="pinhole", fused=fused, R=c.R, m1type=m1type)
    maps = u.maps()
    rng = np.random.default_rng(60 + fused)
    for depth in DEPTHS:
        for k, border in enumerate(MODES):
            inter = INTERS[(k + depth) % 4]
            if cv2_border_differs(0, depth, inter, border):
                inter = cv2.INTER_CUBIC
            _check(torch, rng, depth, c.SW, c.SH, c.W, c.H,
                   lambda s, o, b, v: u(s, inter, out=o, borderMode=b, borderValue=v),
                   lambda s, o, b, v: u.cuda(s, out=o, interpolation=inter, borderMode=b, borderValue=v),
                   lambda s, d, b, v: cv2.remap(s, *maps, inter, dst=d, borderMode=b, borderValue=v), inter, border,
                   BVALS[k % len(BVALS)], ("slot", m1type, fused, depth))
    u.close()


def test_transparent_keeps_out_and_word_path(torch):
    """BORDER_TRANSPARENT leaves the bytes of ``out`` it does not write, on the host and in place on the device, and takes
    the byte path; 3-channel uint8 LINEAR under BORDER_REPLICATE stays on the word path."""
    from cameracalibration_b200 import ops
    rng = np.random.default_rng(7)
    src = rng.integers(0, 256, (30, 40, 3), dtype=np.uint8)
    M = np.array([[0.5, 0.1, 30.0], [-0.1, 0.5, 20.0]])
    fill = rng.integers(0, 256, (48, 64, 3), dtype=np.uint8)
    want = cv2.warpAffine(src, M, (64, 48), dst=fill.copy(), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_TRANSPARENT)
    assert (want == fill).all(-1).sum() > 100   # the premise: most of the canvas is untouched
    out = fill.copy()
    got = ops.warp_affine_border(src, M, (64, 48), cv2.INTER_LINEAR, borderMode=cv2.BORDER_TRANSPARENT, out=out)
    assert got is out and np.array_equal(out, want)
    d_src = torch.from_numpy(src[None]).cuda()
    d_out = torch.from_numpy(fill[None]).cuda()
    ops.warp_affine_border(d_src, M, (64, 48), cv2.INTER_LINEAR, borderMode=cv2.BORDER_TRANSPARENT, out=d_out)
    torch.cuda.synchronize()
    assert ops.last_path() == "byte"
    assert np.array_equal(d_out.cpu().numpy()[0], want)
    rep = ops.warp_affine_border(d_src, M, (64, 48), cv2.INTER_LINEAR, borderMode=cv2.BORDER_REPLICATE, borderValue=(1, 2, 3))
    torch.cuda.synchronize()
    assert ops.last_path() == "word"
    assert np.array_equal(rep.cpu().numpy()[0], cv2.warpAffine(src, M, (64, 48), flags=cv2.INTER_LINEAR,
                                                                borderMode=cv2.BORDER_REPLICATE, borderValue=(1, 2, 3)))


def test_c_entry_points(torch):
    """The host _border entry points bevk_remap_border, bevk_remap_f32_border, bevk_undistort_border,
    bevk_warp_perspective_border and bevk_warp_affine_border at CV_16UC3 under BORDER_WRAP with value (7, 8, 9, 10);
    NULL for border_value means zeros."""
    from cameracalibration_b200 import ops
    from cameracalibration_b200 import _lib as L
    ctx = L.default_context()
    lib = ctx.lib
    rng = np.random.default_rng(8)
    sw, sh, dw, dh = 19, 13, 24, 20
    src = rng.integers(0, 65536, (sh, sw, 3)).astype(np.uint16)
    t = 2 + (2 << 3)
    bv = (ctypes.c_double * 4)(7, 8, 9, 10)
    m1 = np.stack([rng.integers(-30, sw + 30, (dh, dw)), rng.integers(-30, sh + 30, (dh, dw))], -1).astype(np.int16)
    m2 = rng.integers(0, 1024, (dh, dw)).astype(np.uint16)
    fx, fy = (m1[..., 0] + 0.3).astype(np.float32), (m1[..., 1] - 0.6).astype(np.float32)
    H = np.array([[1.3, 0.1, -4.0], [0.05, 1.2, 3.0], [1e-3, 0, 1.0]])
    M = np.array([[0.8, 0.3, -5.0], [-0.2, 0.9, 7.0]])
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    DP = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    kw = dict(borderMode=cv2.BORDER_WRAP, borderValue=(7, 8, 9, 10))
    calls = [
        (lambda o: lib.bevk_remap_border(ctx.h, P(src), sw, sh, sw * 6, t, P(m1), P(m2), dw, dh, P(o), dw * 6, 2, 3, bv),
         cv2.remap(src, m1, m2, cv2.INTER_CUBIC, **kw)),
        (lambda o: lib.bevk_remap_f32_border(ctx.h, P(src), sw, sh, sw * 6, t, P(fx), P(fy), dw, dh, P(o), dw * 6, 1, 3, bv),
         cv2.remap(src, fx, fy, cv2.INTER_LINEAR, **kw)),
        (lambda o: lib.bevk_warp_perspective_border(ctx.h, P(src), sw, sh, sw * 6, t, DP(H), P(o), dw, dh, dw * 6, 4, 3, bv),
         cv2.warpPerspective(src, H, (dw, dh), flags=cv2.INTER_LANCZOS4, **kw)),
        (lambda o: lib.bevk_warp_affine_border(ctx.h, P(src), sw, sh, sw * 6, t, DP(M), P(o), dw, dh, dw * 6, 0, 3, bv),
         cv2.warpAffine(src, M, (dw, dh), flags=cv2.INTER_NEAREST, **kw)),
        (lambda o: lib.bevk_remap_border(ctx.h, P(src), sw, sh, sw * 6, t, P(m1), P(m2), dw, dh, P(o), dw * 6, 1, 0, None),
         cv2.remap(src, m1, m2, cv2.INTER_LINEAR)),
    ]
    for i, (call, want) in enumerate(calls):
        o = np.zeros((dh, dw, 3), np.uint16)
        assert call(o) == 0, (i, lib.bevk_last_error())
        assert np.array_equal(o, want), i
    c = FC.case_by_name("pinhole12")
    u = ops.Undistorter(c.K, c.D, c.P, (c.W, c.H), model="pinhole", R=c.R)
    s2 = rng.integers(0, 65536, (c.SH, c.SW, 3)).astype(np.uint16)
    o = np.zeros((c.H, c.W, 3), np.uint16)
    assert lib.bevk_undistort_border(ctx.h, u.slot, P(s2), c.SW, c.SH, c.SW * 6, t, P(o), c.W, c.H, c.W * 6, 1, 3, bv) == 0
    assert np.array_equal(o, cv2.remap(s2, *u.maps(), cv2.INTER_LINEAR, **kw))
    u.close()


def test_graph_capture(torch):
    """bevk_warp_affine_stack_border (CV_8UC4, CUBIC, BORDER_REFLECT_101 with a value) captured in a graph and replayed
    over rewritten frames."""
    from cameracalibration_b200 import _lib as L
    ctx = L.default_context()
    n, sw, sh, dw, dh = 3, 33, 21, 40, 30
    M = np.array([[1.4, 0.2, -6.0], [-0.1, 1.3, -4.0]])
    frames = torch.zeros((n, sh, sw, 4), dtype=torch.uint8, device="cuda")
    out = torch.empty((n, dh, dw, 4), dtype=torch.uint8, device="cuda")
    bv = (ctypes.c_double * 4)(5, 250, 77, 1)
    torch.cuda.synchronize()
    call = lambda: ctx.lib.bevk_warp_affine_stack_border(
        ctx.h, ctypes.c_void_p(frames.data_ptr()), sh * sw * 4, sw, sh, sw * 4, 3 << 3, n, M.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
        ctypes.c_void_p(out.data_ptr()), dh * dw * 4, dw, dh, dw * 4, cv2.INTER_CUBIC, cv2.BORDER_REFLECT_101, bv)
    assert call() == 0
    ctx.sync()
    with ctx.graph_capture() as g:
        assert call() == 0
    rng = np.random.default_rng(9)
    for rep in range(2):
        host = rng.integers(0, 256, (n, sh, sw, 4), dtype=np.uint8)
        frames.copy_(torch.from_numpy(host))
        out.fill_(0)
        torch.cuda.synchronize()
        g.launch()
        ctx.sync()
        got = out.cpu().numpy()
        for i in range(n):
            want = cv2.warpAffine(host[i], M, (dw, dh), flags=cv2.INTER_CUBIC, borderMode=cv2.BORDER_REFLECT_101,
                                  borderValue=(5, 250, 77, 1))
            assert np.array_equal(got[i], want), (rep, i)
    g.destroy()


def test_refusals(torch):
    """Mode 7 and REFLECT | BORDER_ISOLATED: BevkError from Python, BEVK_ERR_ARG from C; BORDER_TRANSPARENT without out;
    the cases cv2 computes another way (cv2_border_differs): BEVK_ERR_UNSUPPORTED.  Nothing is written."""
    from cameracalibration_b200 import ops
    from cameracalibration_b200 import _lib as L
    ctx = L.default_context()
    src = np.zeros((8, 8), np.uint8)
    m1 = np.zeros((4, 4, 2), np.int16)
    m2 = np.zeros((4, 4), np.uint16)
    for mode in (7, cv2.BORDER_REFLECT | cv2.BORDER_ISOLATED):
        with pytest.raises(L.BevkError):
            ops.remap(src, m1, m2, cv2.INTER_LINEAR, borderMode=mode)
    with pytest.raises(L.BevkError):
        ops.remap(src, m1, m2, cv2.INTER_LINEAR, borderMode=cv2.BORDER_TRANSPARENT)
    with pytest.raises(L.BevkError):
        ops.remap(src, m1, m2, cv2.INTER_LINEAR, borderValue=(1, 2, 3, 4, 5))
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    o = np.full((4, 4), 0xAB, np.uint8)
    assert ctx.lib.bevk_remap_border(ctx.h, P(src), 8, 8, 8, 0, P(m1), P(m2), 4, 4, P(o), 4, 1, 7, None) == ERR_ARG
    assert ctx.lib.bevk_remap_border(ctx.h, P(src), 8, 8, 8, 0, P(m1), P(m2), 4, 4, P(o), 4, 1, 18, None) == ERR_ARG
    assert ctx.lib.bevk_remap_border(ctx.h, P(src), 8, 8, 8, 0, P(m1), P(m2), 4, 4, P(o), 4, 1, -1, None) == ERR_ARG
    f = np.zeros((8, 8), np.float32)
    fo = np.full((4, 4), 3.0, np.float32)
    assert ctx.lib.bevk_remap_border(ctx.h, P(f), 8, 8, 32, 5, P(m1), P(m2), 4, 4, P(fo), 16, 1, 5, None) == ERR_UNSUPPORTED
    s16 = np.zeros((8, 8), np.int16)
    o16 = np.full((4, 4), 5, np.int16)
    H = np.eye(3)
    for inter in (cv2.INTER_NEAREST, cv2.INTER_LINEAR):
        for mode in (cv2.BORDER_REPLICATE, cv2.BORDER_TRANSPARENT):
            assert ctx.lib.bevk_warp_perspective_border(ctx.h, P(s16), 8, 8, 16, 3, H.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), P(o16), 4, 4, 8, inter, mode,
                                                        None) == ERR_UNSUPPORTED
    assert (o == 0xAB).all() and (fo == 3.0).all() and (o16 == 5).all()
    with pytest.raises(L.BevkError):
        ops.warp_perspective(s16, H, (4, 4), cv2.INTER_LINEAR, borderMode=cv2.BORDER_REPLICATE)
