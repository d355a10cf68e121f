"""GPU test of the device PNG encoder (bevk_png_encode, ops.png_encode): the seeded corpus of tests/png_cases.py through
ops.png_encode from NumPy and from torch CUDA tensors, padded rows and images at an odd base address, batches of 1, 3
and 32 mixed images, one context reused across sizes and params, the capacity rule and a refused list that leaves the
previous params in force -- every stream byte-identical to cv2.imencode(".png", img, params)."""
import ctypes

import cv2
import numpy as np
import pytest

from tests import png_cases as P

pytestmark = pytest.mark.gpu


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
    """CUDA view of imgs [n][h][w][3] with row_pad bytes after each row, img_pad after each image, starting offset
    bytes into its allocation."""
    n, h, w, _ = imgs.shape
    row = 3 * w + row_pad
    istride = h * row + img_pad
    buf = torch.full((offset + n * istride + 64,), 0xA5, dtype=torch.uint8, device="cuda")
    view = torch.as_strided(buf, (n, h, w, 3), (istride, row, 3, 1), offset)
    view.copy_(torch.from_numpy(imgs).cuda())
    return buf, view


def test_png_corpus_numpy_and_cuda(ops, torch):
    n = 0
    for name, img, params in P.cases():
        want = cv2_png(img, params)
        assert ops.png_encode(img, params=params) == [want], name
        assert ops.png_encode(torch.from_numpy(img).cuda(), params=params) == [want], name
        n += 2
    assert n > 150


@pytest.mark.parametrize("row_pad,img_pad,offset", [(1, 0, 1), (13, 7, 3), (64, 256, 0)])
def test_png_padded_layouts(ops, torch, row_pad, img_pad, offset):
    rng = np.random.default_rng(row_pad)
    imgs = np.stack([P._stripes(rng, 45, 77), P._noise(rng, 45, 77), P._flat(rng, 45, 77)])
    _, view = padded(torch, imgs, row_pad, img_pad, offset)
    for params in ([], P.PARAMS["huff"], P.PARAMS["rle_l5"]):
        assert ops.png_encode(view, params=params) == [cv2_png(i, params) for i in imgs]


@pytest.mark.parametrize("n", [1, 3, 32])
def test_png_batches_of_mixed_content(ops, torch, n):
    rng = np.random.default_rng(n)
    makers = [P._smooth, P._noise, P._flat, P._blocks, P._stripes, P._runs3]
    imgs = np.stack([makers[i % len(makers)](rng, 120, 200) for i in range(n)])
    for params in ([], P.PARAMS["huff"], P.PARAMS["filter_all"]):
        assert ops.png_encode(torch.from_numpy(imgs).cuda(), params=params) == [cv2_png(i, params) for i in imgs]


def test_png_large_batch_spans_groups(ops, torch):
    """1000 x 1000 canvases: more filtered bytes than one group of the pipeline holds, so the batch runs in groups."""
    rng = np.random.default_rng(5)
    imgs = np.stack([P._blocks(rng, 1000, 1000) if i % 2 else P._smooth(rng, 1000, 1000) for i in range(48)])
    assert ops.png_encode(torch.from_numpy(imgs).cuda()) == [cv2_png(i, []) for i in imgs]


def test_png_context_reuse_and_capacity(ops, torch, L):
    ctx = L.Context(0)
    rng = np.random.default_rng(9)
    for (w, h), params in [((64, 50), []), ((300, 7), P.PARAMS["huff"]), ((64, 50), P.PARAMS["filter_paeth"]),
                           ((1, 1), []), ((500, 400), P.PARAMS["rle_l5"]), ((64, 50), [])]:
        imgs = rng.integers(0, 256, (2, h, w, 3), dtype=np.uint8)
        imgs[1] = P._smooth(rng, h, w)
        assert ops.png_encode(imgs, ctx=ctx, params=params) == [cv2_png(i, params) for i in imgs]
    # capacity one byte short: fails, writes nothing, sizes filled
    imgs = np.stack([P._stripes(rng, 60, 90), P._noise(rng, 60, 90)])
    want = [cv2_png(i, []) for i in imgs]
    d = torch.from_numpy(imgs).cuda()
    total = sum(map(len, want))
    ops.png_set_params(ctx, None)
    out = np.full(total + 16, 0x5A, np.uint8)
    sizes = (ctypes.c_uint64 * 2)()
    r = ctx.lib.bevk_png_encode(ctx.h, ctypes.c_void_p(d.data_ptr()), 60 * 90 * 3, 90 * 3, 2, 90, 60, L.vptr(out),
                                total - 1, sizes)
    assert r == -1 and list(sizes) == [len(x) for x in want] and (out == 0x5A).all()
    r = ctx.lib.bevk_png_encode(ctx.h, ctypes.c_void_p(d.data_ptr()), 60 * 90 * 3, 90 * 3, 2, 90, 60, L.vptr(out),
                                total, sizes)
    assert r == 0 and out[:total].tobytes() == b"".join(want) and (out[total:] == 0x5A).all()
    # a refused list leaves the previous params in force
    ops.png_set_params(ctx, P.PARAMS["huff"])
    for bad, code in (([cv2.IMWRITE_PNG_COMPRESSION, 5], -4), ([cv2.IMWRITE_PNG_STRATEGY, 3, 99, 1], -1), ([17], -1)):
        arr = (ctypes.c_int * len(bad))(*bad)
        assert ctx.lib.bevk_png_set_params(ctx.h, arr, len(bad)) == code
    r = ctx.lib.bevk_png_encode(ctx.h, ctypes.c_void_p(d.data_ptr()), 60 * 90 * 3, 90 * 3, 2, 90, 60, L.vptr(out),
                                out.size, sizes)
    assert r == 0
    huff = [cv2_png(i, P.PARAMS["huff"]) for i in imgs]
    assert out[:sum(map(len, huff))].tobytes() == b"".join(huff)
    ms = ctypes.c_float()
    assert ctx.lib.bevk_last_kernel_ms(ctx.h, ctypes.byref(ms)) == 0 and ms.value > 0
    with pytest.raises(L.BevkError):
        ops.png_encode(imgs, ctx=ctx, params=[cv2.IMWRITE_PNG_COMPRESSION, 3])
