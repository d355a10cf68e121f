"""Grey and BGRA images through the device JPEG and PNG encoders (bevk_jpeg_encode_channels, bevk_png_encode_channels,
ops.imencode) against live cv2.imencode, byte for byte, on one context reused across sizes, channel counts and formats."""
import ctypes as C

import cv2
import numpy as np
import pytest

from cameracalibration_b200 import _lib as L
from cameracalibration_b200 import ops
from tests import encode_channels_cases as E

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
ERR_ARG, ERR_UNSUPPORTED = -1, -4   # BEVK_ERR_ARG, BEVK_ERR_UNSUPPORTED


@pytest.fixture(scope="module")
def ctx():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    c = L.Context(0)
    yield c
    c.close()


def raw_call(ctx, ext, dev, params, capacity=None):
    """The C entry on a uint8 CUDA tensor [N][H][W][C] (any strides with dense pixels): (status, streams, sizes)."""
    n, h, w, c = dev.shape
    quality, arr, k = ops._imencode_jpeg_params(params) if ext != ".png" else (None, *ops._jpeg_params(params))
    bound = ops.imencode_bound(ext, w, h, c, params)
    cap = n * bound if capacity is None else capacity
    out = np.zeros(max(cap, 1), np.uint8)
    sizes = (C.c_uint64 * n)()
    torch.cuda.synchronize()
    args = (C.c_void_p(dev.data_ptr()), dev.stride(0), dev.stride(1), c, n, w, h)
    if ext == ".png":
        r = ctx.lib.bevk_png_encode_channels(ctx.h, arr, k, *args, L.vptr(out), cap, sizes)
    else:
        r = ctx.lib.bevk_jpeg_encode_channels(ctx.h, arr, k, *args, int(quality), L.vptr(out), cap, sizes)
    return r, ops._split(out, list(sizes)) if r == 0 else None, list(sizes), bound


def test_corpus_matches_cv2(ctx):
    cases = E.cases()
    bad = []
    for name, ext, imgs, params in cases:
        want = E.cv2_streams(ext, imgs, params)
        got = ops.imencode(ext, imgs, params, ctx=ctx)
        dev = torch.from_numpy(imgs).cuda()
        r, raw, sizes, bound = raw_call(ctx, ext, dev, params)
        assert r == 0, (name, L.load().bevk_last_error().decode())
        assert all(len(s) <= bound for s in want), name
        if got != want or raw != want:
            bad.append(name)
    assert not bad, (len(bad), bad[:20])


@pytest.mark.parametrize("c", [1, 4])
@pytest.mark.parametrize("ext,params", [(".jpg", []), (".jpg", [E.P, 1, E.R, 2]), (".png", []), (".png", [E.PC, 9])])
def test_padded_pitches(ctx, c, ext, params):
    rng = np.random.default_rng(5 + c)
    imgs = np.stack([E.image(rng, 23, 37, c, k) for k in ("smooth", "noise")])
    n, h, w, _ = imgs.shape
    row, img = w * c + 13, h * (w * c + 13) + 29
    base = torch.full((n * img + 64,), 0xA5, dtype=torch.uint8, device="cuda")
    view = base.as_strided((n, h, w, c), (img, row, c, 1))
    view.copy_(torch.from_numpy(imgs).cuda())
    want = E.cv2_streams(ext, imgs, params)
    assert ops.imencode(ext, view, params, ctx=ctx) == want
    assert raw_call(ctx, ext, view, params)[1] == want


def test_rank2_and_single_channel_forms(ctx):
    rng = np.random.default_rng(9)
    g = E.image(rng, 31, 45, 1)[..., 0]
    for ext in (".jpg", ".png", ".jpeg", ".jpe", ".JPG"):
        want = cv2.imencode(ext, g)[1].tobytes()
        assert ops.imencode(ext, g, ctx=ctx) == [want]
        assert ops.imencode(ext, g[..., None], ctx=ctx) == [want]
        assert ops.imencode(ext, torch.from_numpy(g).cuda(), ctx=ctx) == [want]


def test_bgra_jpeg_equals_bgr(ctx):
    rng = np.random.default_rng(12)
    imgs = np.stack([E.image(rng, 40, 51, 4, k) for k in ("smooth", "noise")])
    for params in ([], [E.P, 1], [E.O, 1, E.SF, 0x211111], [E.R, 3, E.Q, 70]):
        assert ops.imencode(".jpg", imgs, params, ctx=ctx) == ops.imencode(".jpg", imgs[..., :3].copy(), params, ctx=ctx)


def test_three_channels_match_existing_wrappers(ctx):
    rng = np.random.default_rng(13)
    imgs = np.stack([E.image(rng, 33, 47, 3, k) for k in ("smooth", "noise")])
    for params in ([], [E.P, 1, E.R, 2], [E.O, 1], [E.LQ, 40, E.CQ, 90]):
        assert ops.imencode(".jpg", imgs, params, ctx=ctx) == ops.jpeg_encode_params(imgs, params, 95, ctx=ctx)
    assert ops.imencode(".jpg", imgs, [E.Q, 60], ctx=ctx) == ops.jpeg_encode_params(imgs, [], 60, ctx=ctx)
    for params in ([], [E.PC, 9], [E.PS, 2]):
        assert ops.imencode(".png", imgs, params, ctx=ctx) == ops.png_encode(imgs, ctx=ctx, params=params)


def test_undistorted_grey_and_bgra_frames(ctx):
    """Undistorter.cuda then ops.imencode equals cv2.remap then cv2.imencode."""
    from oracle import cv2_path as CP
    from tests.helpers import Fixtures
    fx = Fixtures()
    K, D, _ = fx.calib["front"]
    K = np.diag([320 / 1280, 256 / 1024, 1.0]) @ K
    P = CP.dst_camera_matrix(K, 320, 256, 1.0, 1)
    m1, m2 = CP.undistort_maps(K, D, P, 320, 256)
    rng = np.random.default_rng(21)
    u = ops.Undistorter(K, D, P, (320, 256), ctx=ctx)
    try:
        for c in (1, 4):
            frames = np.stack([E.image(rng, 256, 320, c, k) for k in ("smooth", "noise")])
            und = u.cuda(torch.from_numpy(frames).cuda())
            for ext, params in ((".jpg", []), (".jpg", [E.P, 1]), (".png", []), (".png", [E.PC, 6])):
                want = []
                for f in frames:
                    r = cv2.remap(f[..., 0] if c == 1 else f, m1, m2, cv2.INTER_LINEAR)
                    want.append(cv2.imencode(ext, r, params)[1].tobytes())
                assert ops.imencode(ext, und, params, ctx=ctx) == want, (c, ext, params)
    finally:
        u.close()


def test_errors(ctx):
    img2 = np.zeros((2, 8, 8, 2), np.uint8)
    with pytest.raises(L.BevkError):
        ops.imencode(".jpg", img2, ctx=ctx)
    with pytest.raises(L.BevkError):
        ops.imencode(".bmp", np.zeros((8, 8), np.uint8), ctx=ctx)
    with pytest.raises(L.BevkError):
        ops.imencode(".tiff", np.zeros((8, 8, 3), np.uint8), ctx=ctx)
    dev = torch.zeros((1, 8, 8, 2), dtype=torch.uint8, device="cuda")
    out = np.zeros(4096, np.uint8)
    sizes = (C.c_uint64 * 1)()
    arr, k = ops._jpeg_params([])
    for c in (0, 2, 5):
        assert ctx.lib.bevk_jpeg_encode_channels(ctx.h, arr, k, C.c_void_p(dev.data_ptr()), 128, 16, c, 1, 8, 8, 95,
                                                 L.vptr(out), 4096, sizes) == ERR_UNSUPPORTED
        assert ctx.lib.bevk_png_encode_channels(ctx.h, arr, k, C.c_void_p(dev.data_ptr()), 128, 16, c, 1, 8, 8,
                                                L.vptr(out), 4096, sizes) == ERR_UNSUPPORTED
        n = C.c_uint64()
        assert L.load().bevk_jpeg_encode_channels_bound(8, 8, c, arr, k, C.byref(n)) == ERR_UNSUPPORTED
        assert L.load().bevk_png_encode_channels_bound(8, 8, c, C.byref(n)) == ERR_UNSUPPORTED
    # refused PNG lists, grey and BGRA alike
    for c in (1, 4):
        img = np.zeros((8, 8, c), np.uint8)
        for params in ([E.PC, 0], [E.PC, 2], [E.PS, 0], [cv2.IMWRITE_PNG_BILEVEL, 1], [cv2.IMWRITE_PNG_ZLIBBUFFER_SIZE, 8192]):
            with pytest.raises(L.BevkError):
                ops.imencode(".png", img, params, ctx=ctx)
    # capacity: sizes filled, nothing written, BEVK_ERR_ARG
    rng = np.random.default_rng(3)
    for ext, c in ((".jpg", 1), (".png", 4), (".jpg", 4), (".png", 1)):
        imgs = torch.from_numpy(np.stack([E.image(rng, 20, 30, c, "noise") for _ in range(2)])).cuda()
        want = E.cv2_streams(ext, imgs.cpu().numpy(), [])
        cap = len(want[0]) + len(want[1]) - 1
        r, _, sizes, _ = raw_call(ctx, ext, imgs, [], capacity=cap)
        assert r == ERR_ARG and sizes == [len(s) for s in want]
        r, raw, sizes, _ = raw_call(ctx, ext, imgs, [], capacity=cap + 1)
        assert r == 0 and raw == want
    # the timing covers the call
    ops.imencode(".jpg", np.zeros((16, 16), np.uint8), ctx=ctx)
    ms = C.c_float()
    assert ctx.lib.bevk_last_kernel_ms(ctx.h, C.byref(ms)) == 0 and ms.value > 0
