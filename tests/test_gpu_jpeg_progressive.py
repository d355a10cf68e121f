"""GPU test of progressive JPEG on the device (bevk_jpeg_encode_params with IMWRITE_JPEG_PROGRESSIVE): the seeded corpus of
tests/jpeg_progressive_cases.py through bevk_jpeg_encode_params (padded row pitches and image strides, one context reused
across sizes) and ops.jpeg_encode_params (NumPy and torch input), every stream byte-identical to
cv2.imencode(".jpg", img, [IMWRITE_JPEG_QUALITY, q] + params) and within bevk_jpeg_encode_params_bound.  Also: the
capacity error, baseline lists through the new call equal to bevk_jpeg_encode, the ctx's list left alone, and the refused
keys."""
import ctypes
from contextlib import contextmanager

import cv2
import numpy as np
import pytest

from tests import jpeg_progressive_cases as J

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


@contextmanager
def _context(L):
    ctx = L.Context(L.default_context().device)
    try:
        yield ctx
    finally:
        ctx.close()


def _cv2(img, q, params=()):
    return cv2.imencode(".jpg", np.ascontiguousarray(img), [cv2.IMWRITE_JPEG_QUALITY, q] + list(params))[1].tobytes()


def _ints(params):
    return (ctypes.c_int * max(len(params), 1))(*params), len(params)


def _padded(torch, imgs, pad_row, pad_img):
    """A CUDA copy of imgs [N][H][W][3] with pad_row bytes after each row and pad_img after each image."""
    n, H, W, _ = imgs.shape
    pitch, istride = W * 3 + pad_row, H * (W * 3 + pad_row) + pad_img
    rows = torch.full((n, H, pitch), 0x5A, dtype=torch.uint8, device="cuda")
    rows[:, :, :W * 3] = torch.from_numpy(np.ascontiguousarray(imgs).reshape(n, H, W * 3)).cuda()
    buf = torch.full((n, istride), 0x5A, dtype=torch.uint8, device="cuda")
    buf[:, :H * pitch] = rows.reshape(n, H * pitch)
    return buf.reshape(-1), pitch, istride


def _encode(L, ctx, ptr, istride, pitch, n, W, H, q, params, cap):
    arr, k = _ints(params)
    buf = np.full(cap + 4096, 0xA5, np.uint8)
    sizes = (ctypes.c_uint64 * n)()
    rc = ctx.lib.bevk_jpeg_encode_params(ctx.h, arr, k, ctypes.c_void_p(ptr), istride, pitch, n, W, H, q, L.vptr(buf), cap, sizes)
    return rc, buf, list(sizes)


def _bound(L, W, H, params):
    arr, k = _ints(params)
    b = ctypes.c_uint64()
    assert L.load().bevk_jpeg_encode_params_bound(W, H, arr, k, ctypes.byref(b)) == 0
    return b.value


def test_corpus_direct_padded(torch, L):
    """Every corpus case through bevk_jpeg_encode_params with padded rows and images, on one context."""
    with _context(L) as ctx:
        for k, c in enumerate(J.cases()):
            imgs = np.stack(c.images)
            n, H, W, _ = imgs.shape
            big = W * H > 1 << 20
            buf_d, pitch, istride = (torch.from_numpy(imgs).cuda(), W * 3, H * W * 3) if big else \
                _padded(torch, imgs, 5 + k % 11, 64 + 3 * (k % 5))
            want = [_cv2(im, c.quality, c.params) for im in imgs]
            total, bound = sum(map(len, want)), _bound(L, W, H, c.params)
            assert all(len(s) <= bound for s in want), c.name
            rc, buf, sizes = _encode(L, ctx, buf_d.data_ptr(), istride, pitch, n, W, H, c.quality, c.params, total)
            assert rc == 0, (c.name, ctx.lib.bevk_last_error().decode())
            assert sizes == [len(s) for s in want], c.name
            got = bytes(buf[:total])
            assert got == b"".join(want), (c.name, [bytes(buf[sum(sizes[:i]):sum(sizes[:i + 1])]) == w for i, w in enumerate(want)])
            assert (buf[total:] == 0xA5).all(), c.name


def test_corpus_ops_numpy_and_torch(torch, ops):
    for c in J.cases(small=True):
        imgs = np.stack(c.images)
        want = [_cv2(im, c.quality, c.params) for im in imgs]
        assert ops.jpeg_encode_params(imgs, c.params, quality=c.quality) == want, c.name
        assert ops.jpeg_encode_params(torch.from_numpy(imgs).cuda(), c.params, quality=c.quality) == want, c.name
        assert ops.jpeg_encode_params(imgs[0], c.params, quality=c.quality) == want[:1], c.name


def test_capacity_error(torch, L):
    imgs = np.stack([J.smooth(np.random.default_rng(k), 56, 40) for k in range(3)])
    d = torch.from_numpy(imgs).cuda()
    want = [_cv2(im, 90, J.P) for im in imgs]
    total = sum(map(len, want))
    with _context(L) as ctx:
        rc, buf, sizes = _encode(L, ctx, d.data_ptr(), 40 * 56 * 3, 56 * 3, 3, 56, 40, 90, J.P, total - 1)
        assert rc == -1 and "capacity" in ctx.lib.bevk_last_error().decode()
        assert sizes == [len(s) for s in want] and (buf == 0xA5).all()
        rc, buf, sizes = _encode(L, ctx, d.data_ptr(), 40 * 56 * 3, 56 * 3, 3, 56, 40, 90, J.P, total)
        assert rc == 0 and bytes(buf[:total]) == b"".join(want)
        ms = ctypes.c_float()
        assert ctx.lib.bevk_last_kernel_ms(ctx.h, ctypes.byref(ms)) == 0 and ms.value > 0


def test_baseline_lists_equal_jpeg_encode(torch, L):
    """Lists without PROGRESSIVE (or with it off) write bevk_jpeg_encode's streams under the same bevk_jpeg_set_params
    list, and the ctx's list is neither read nor changed."""
    rng = np.random.default_rng(11)
    imgs = rng.integers(0, 256, (3, 37, 45, 3), dtype=np.uint8)
    d = torch.from_numpy(imgs).cuda()
    ctx_list = [J.SAMPLING, 0x111111, J.RST, 1]
    with _context(L) as ctx:
        arr, k = _ints(ctx_list)
        assert ctx.lib.bevk_jpeg_set_params(ctx.h, arr, k) == 0
        for params in ([], [J.OPTIMIZE, 1], [J.SAMPLING, 0x211111, J.RST, 3], [J.PROGRESSIVE, 0, J.OPTIMIZE, 1],
                       [J.LUMA, 90, J.CHROMA, 60]):
            want = [_cv2(im, 85, params) for im in imgs]
            total = sum(map(len, want))
            rc, buf, sizes = _encode(L, ctx, d.data_ptr(), 37 * 45 * 3, 45 * 3, 3, 45, 37, 85, params, total)
            assert rc == 0 and bytes(buf[:total]) == b"".join(want), params
            # bevk_jpeg_encode under the same list as the ctx's list gives the same streams
            a2, k2 = _ints(params)
            assert ctx.lib.bevk_jpeg_set_params(ctx.h, a2, k2) == 0
            buf2 = np.zeros(total, np.uint8)
            s2 = (ctypes.c_uint64 * 3)()
            assert ctx.lib.bevk_jpeg_encode(ctx.h, ctypes.c_void_p(d.data_ptr()), 37 * 45 * 3, 45 * 3, 3, 45, 37, 85, L.vptr(buf2),
                                            total, s2) == 0
            assert bytes(buf2) == bytes(buf[:total]), params
            assert ctx.lib.bevk_jpeg_set_params(ctx.h, arr, k) == 0
        # the ctx's list is still in force for bevk_jpeg_encode after progressive calls
        _encode(L, ctx, d.data_ptr(), 37 * 45 * 3, 45 * 3, 3, 45, 37, 85, J.P, 1 << 20)
        want = [_cv2(im, 85, ctx_list) for im in imgs]
        total = sum(map(len, want))
        buf2 = np.zeros(total, np.uint8)
        s2 = (ctypes.c_uint64 * 3)()
        assert ctx.lib.bevk_jpeg_encode(ctx.h, ctypes.c_void_p(d.data_ptr()), 37 * 45 * 3, 45 * 3, 3, 45, 37, 85, L.vptr(buf2),
                                        total, s2) == 0
        assert bytes(buf2) == b"".join(want)


def test_refused_keys(torch, L, ops):
    d = torch.zeros((16, 16, 3), dtype=torch.uint8, device="cuda")
    with _context(L) as ctx:
        for bad in ([1, 90], [J.PROGRESSIVE], [8, 1], [0, 0], [J.PROGRESSIVE, 1, 1, 50]):
            rc, _, _ = _encode(L, ctx, d.data_ptr(), 0, 48, 1, 16, 16, 90, bad, 1 << 16)
            assert rc == -1, bad
            arr, k = _ints(bad)
            b = ctypes.c_uint64()
            assert ctx.lib.bevk_jpeg_encode_params_bound(16, 16, arr, k, ctypes.byref(b)) == -1, bad
            with pytest.raises(L.BevkError):
                ops.jpeg_encode_params(np.zeros((16, 16, 3), np.uint8), bad)
