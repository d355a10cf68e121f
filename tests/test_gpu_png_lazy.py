"""GPU test of the device PNG encoder's hash-chain path (bevk_png_encode_params, ops.png_encode at levels 4..9 under
the DEFAULT, FILTERED and FIXED strategies): the seeded corpus of tests/png_lazy_cases.py, one context reused across
sizes and lists, mixed batches with padded rows and images, batches spanning several groups, the capacity rule, calls
interleaved with bevk_png_set_params / bevk_png_encode, 1000 x 1000 canvases and 1920 x 1080 undistorted frames at
levels 6 and 9, and Tools/undistort.py -dstformat png -- every stream byte-identical to cv2.imencode(".png", img,
params)."""
import ctypes

import cv2
import numpy as np
import pytest

from tests import png_cases as P
from tests import png_lazy_cases as PL
from tests.helpers import h16

pytestmark = pytest.mark.gpu
C, S = cv2.IMWRITE_PNG_COMPRESSION, cv2.IMWRITE_PNG_STRATEGY


@pytest.fixture(scope="module")
def torch():
    import torch as t
    return t


@pytest.fixture(scope="module")
def ops():
    from cameracalibration_b200 import ops as o
    return o


@pytest.fixture(scope="module")
def L():
    from cameracalibration_b200 import _lib
    return _lib


def cv2_png(img, params):
    return cv2.imencode(".png", img, list(params))[1].tobytes()


def padded(torch, imgs, row_pad, img_pad, offset):
    n, h, w, _ = imgs.shape
    row = 3 * w + row_pad
    istride = h * row + img_pad
    buf = torch.full((offset + n * istride + 64,), 0xA5, dtype=torch.uint8, device="cuda")
    view = torch.as_strided(buf, (n, h, w, 3), (istride, row, 3, 1), offset)
    view.copy_(torch.from_numpy(imgs).cuda())
    return buf, view


def encode_params(ctx, L, params, d, n, w, h, istride, rstride, capacity, out=None):
    out = np.full(capacity + 16, 0x5A, np.uint8) if out is None else out
    sizes = (ctypes.c_uint64 * n)()
    arr = (ctypes.c_int * max(1, len(params)))(*params)
    r = ctx.lib.bevk_png_encode_params(ctx.h, arr, len(params), ctypes.c_void_p(d), istride, rstride, n, w, h, L.vptr(out),
                                       capacity, sizes)
    return r, out, list(sizes)


def test_png_lazy_corpus(ops, torch):
    n = 0
    for name, img, params in PL.cases():
        want = cv2_png(img, params)
        assert ops.png_encode(img, params=params) == [want], name
        n += 1
    assert n > 80


@pytest.mark.parametrize("row_pad,img_pad,offset", [(1, 0, 1), (13, 7, 3)])
def test_png_lazy_padded_mixed_batches(ops, torch, row_pad, img_pad, offset):
    rng = np.random.default_rng(row_pad)
    makers = [P._smooth, P._noise, P._flat, P._blocks, P._stripes, P._runs3]
    imgs = np.stack([makers[i % len(makers)](rng, 90, 150) for i in range(7)])
    _, view = padded(torch, imgs, row_pad, img_pad, offset)
    for params in ([C, 9], [C, 4, S, PL.FILTERED], [C, 6, S, PL.FIXED], [C, 7, cv2.IMWRITE_PNG_FILTER, 8]):
        assert ops.png_encode(view, params=params) == [cv2_png(i, params) for i in imgs], params


def test_png_lazy_batch_spans_groups(ops, torch):
    """1000 x 1000 canvases: more filtered bytes than one group of the hash-chain pipeline holds."""
    rng = np.random.default_rng(6)
    imgs = np.stack([P._blocks(rng, 1000, 1000) if i % 2 else P._smooth(rng, 1000, 1000) for i in range(13)])
    d = torch.from_numpy(imgs).cuda()
    for params in ([C, 6], [C, 9]):
        assert ops.png_encode(d, params=params) == [cv2_png(i, params) for i in imgs], params


@pytest.mark.parametrize("side", [1, 9])
def test_png_lazy_many_tiny_images(ops, torch, side):
    """2^17 + 1 images of 1 x 1 or 9 x 9 in one call: the hash-chain path runs them in groups of at most 2^16 images,
    so its (image, hash) sort keys stay within 32 bits."""
    from concurrent.futures import ThreadPoolExecutor
    rng = np.random.default_rng(side)
    n = (1 << 17) + 1
    imgs = rng.integers(0, 256, (n, side, side, 3), dtype=np.uint8)
    imgs[::3] = imgs[0]
    got = ops.png_encode(torch.from_numpy(imgs).cuda(), params=[C, 9])
    with ThreadPoolExecutor() as ex:
        want = list(ex.map(lambda i: cv2_png(i, [C, 9]), imgs, chunksize=4096))
    assert len(got) == n
    bad = [k for k in range(n) if got[k] != want[k]]
    assert not bad, bad[:10]


def test_png_lazy_context_reuse_capacity_and_interleaving(ops, torch, L):
    ctx = L.Context(0)
    rng = np.random.default_rng(10)
    for (w, h), params in [((64, 50), [C, 9]), ((300, 7), [C, 5, S, PL.FILTERED]), ((64, 50), []),
                           ((1, 1), [C, 4]), ((500, 400), [C, 8, S, PL.FIXED]), ((64, 50), [C, 6]),
                           ((500, 400), [S, cv2.IMWRITE_PNG_STRATEGY_HUFFMAN_ONLY])]:
        imgs = rng.integers(0, 256, (2, h, w, 3), dtype=np.uint8)
        imgs[1] = P._smooth(rng, h, w)
        assert ops.png_encode(imgs, ctx=ctx, params=params) == [cv2_png(i, params) for i in imgs], (w, h, params)
    imgs = np.stack([P._stripes(rng, 60, 90), P._blocks(rng, 60, 90)])
    d = torch.from_numpy(imgs).cuda()
    want = [cv2_png(i, [C, 9]) for i in imgs]
    total = sum(map(len, want))
    # capacity one byte short: fails, writes nothing, sizes filled; then exact
    r, out, sizes = encode_params(ctx, L, [C, 9], d.data_ptr(), 2, 90, 60, 60 * 90 * 3, 90 * 3, total - 1)
    assert r == -1 and sizes == [len(x) for x in want] and (out == 0x5A).all()
    r, out, sizes = encode_params(ctx, L, [C, 9], d.data_ptr(), 2, 90, 60, 60 * 90 * 3, 90 * 3, total)
    assert r == 0 and out[:total].tobytes() == b"".join(want) and (out[total:] == 0x5A).all()
    ms = ctypes.c_float()
    assert ctx.lib.bevk_last_kernel_ms(ctx.h, ctypes.byref(ms)) == 0 and ms.value > 0
    # the ctx's bevk_png_set_params list is neither read nor changed by the params entry
    ops.png_set_params(ctx, P.PARAMS["huff"])
    huff = [cv2_png(i, P.PARAMS["huff"]) for i in imgs]
    for params in ([C, 9], [C, 5, S, PL.FILTERED]):
        r, out, _ = encode_params(ctx, L, params, d.data_ptr(), 2, 90, 60, 60 * 90 * 3, 90 * 3, 1 << 20)
        assert r == 0 and out[:sum(len(cv2_png(i, params)) for i in imgs)].tobytes() == b"".join(cv2_png(i, params) for i in imgs)
        out = np.zeros(1 << 20, np.uint8)
        sizes = (ctypes.c_uint64 * 2)()
        assert ctx.lib.bevk_png_encode(ctx.h, ctypes.c_void_p(d.data_ptr()), 60 * 90 * 3, 90 * 3, 2, 90, 60, L.vptr(out),
                                       out.size, sizes) == 0
        assert out[:sum(map(len, huff))].tobytes() == b"".join(huff)
    # refusals: levels 0..3 under hash-chain strategies, BILEVEL, ZLIBBUFFER_SIZE; odd lists are argument errors
    for bad, code in (([C, 3], -4), ([C, 0], -4), ([S, 0], -4), ([S, 1, C, 2], -4), ([C, 9, cv2.IMWRITE_PNG_BILEVEL, 1], -4),
                      ([C, 9, cv2.IMWRITE_PNG_ZLIBBUFFER_SIZE, 4096], -4), ([C], -1), ([99, 1], -1)):
        r, _, _ = encode_params(ctx, L, bad, d.data_ptr(), 2, 90, 60, 60 * 90 * 3, 90 * 3, 1 << 20)
        assert r == code, bad
    with pytest.raises(L.BevkError):
        ops.png_encode(imgs, ctx=ctx, params=[C, 3])
    ub = ctypes.c_uint64()
    assert ctx.lib.bevk_png_encode_bound(90, 60, None, 0, ctypes.byref(ub)) == 0 and ub.value >= max(map(len, want))


def test_png_lazy_canvases_and_undistorted_frames(ops, torch, fx):
    """1000 x 1000 BEV-like canvases and 1920 x 1080 undistorted fixture frames at levels 6 and 9."""
    rng = np.random.default_rng(11)
    canvases = np.stack([P._blocks(rng, 1000, 1000), P._smooth(rng, 1000, 1000)])
    K, D, _ = fx.calib["front"]
    Pm = np.array(K, np.float64)
    Pm[0, 2], Pm[1, 2] = 960.0, 540.0
    und = ops.Undistorter(K, D, Pm, (1920, 1080))
    frame = und(fx.img("front"))
    assert frame.shape == (1080, 1920, 3)
    for params in ([C, 6], [C, 9]):
        assert ops.png_encode(torch.from_numpy(canvases).cuda(), params=params) == [cv2_png(i, params) for i in canvases]
        assert und.png(fx.img("front"), params) == cv2_png(frame, params)
    und.close()


@pytest.mark.parametrize("quality", [9, 6])
def test_png_lazy_tools_undistort_cli(fx, tmp_path, quality):
    """Tools/undistort.py -dstformat png at -quality 4..9 encodes on the device: the file is the one cv2.imwrite writes
    for the reference's undistorted image."""
    from cameracalibration_b200.Tools import undistort as T
    (tmp_path / "in").mkdir()
    (tmp_path / "out").mkdir()
    K, D, _ = fx.calib["front"]
    np.save(tmp_path / "K.npy", K)
    np.save(tmp_path / "D.npy", D)
    cv2.imwrite(str(tmp_path / "in" / "front.png"), fx.img("front"))
    T.main(["-path_read", str(tmp_path / "in") + "/", "-path_save", str(tmp_path / "out") + "/", "-path_k",
            str(tmp_path / "K.npy"), "-path_d", str(tmp_path / "D.npy"), "-srcformat", "png", "-dstformat", "png",
            "-quality", str(quality)])
    data = (tmp_path / "out" / "front.png").read_bytes()
    img = cv2.imread(str(tmp_path / "out" / "front.png"))
    assert h16(img) == fx.gold["tools_undistort_front"]
    assert data == cv2_png(img, [C, quality])
