"""GPU test of the device JPEG encoder under cv2.imwrite's JPEG parameters (bevk_jpeg_set_params, params= of the Python
wrappers): the seeded corpus of tests/jpeg_params_cases.py through ops.jpeg_encode (NumPy and CUDA input, padded and
byte-offset layouts) and bevk_jpeg_encode, Undistorter.jpeg / cuda_to_jpeg with the chunked pipeline, and BevGenerator /
BevEngine BEV-to-JPEG with and without BALANCE (k_gain, then the encoder) and the car, under sampling factors, luma / chroma qualities,
optimised tables and restart intervals -- every stream byte-identical to
cv2.imencode(".jpg", img, [IMWRITE_JPEG_QUALITY, q] + params).  Also: the capacity error, params not leaking between
wrapper calls on one context, and the refusals."""
import ctypes
import os
from contextlib import contextmanager

import cv2
import numpy as np
import pytest

from oracle import cv2_path as C
from oracle import restate as R
from tests import bev_cases as B
from tests import calib_cases as CC
from tests import jpeg_params_cases as J
from tests.helpers import NAMES

pytestmark = pytest.mark.gpu

P444, P422, P440, P411 = [J.SAMPLING, 0x111111], [J.SAMPLING, 0x211111], [J.SAMPLING, 0x121111], [J.SAMPLING, 0x411111]
PARAM_SETS = [P444, P422, P440, P411, [J.LUMA, 90, J.CHROMA, 70], [J.LUMA, 80] + P422, [J.OPTIMIZE, 1], [J.RST, 3],
              P444 + [J.OPTIMIZE, 1, J.RST, 1], P411 + [J.RST, 2, J.OPTIMIZE, 1]]


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
def _env(env):
    old = {k: os.environ.get(k) for k in env}
    for k, v in env.items():
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = v
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


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


def _layout(torch, imgs, kind):
    """(CUDA view of the images in layout kind, device pointer, image stride, row stride, buffer kept alive)."""
    n, H, W, _ = imgs.shape
    dense = torch.from_numpy(imgs).cuda()
    if kind == "dense":
        return dense, dense.data_ptr(), H * W * 3, W * 3, dense
    pitch, istride, off = (3 * W + 13, (H + 1) * (3 * W + 13) + 5, 0) if kind == "padded" else (3 * W, 3 * W * H, 3)
    base = torch.full((off + n * istride + 64,), 0x5A, dtype=torch.uint8, device="cuda")
    view = torch.as_strided(base, (n, H, W, 3), (istride, pitch, 3, 1), off)
    view.copy_(dense)
    return view, base.data_ptr() + off, istride, pitch, base


def _direct(L, ctx, ptr, istride, pitch, n, W, H, q, params, want, what):
    """bevk_jpeg_set_params, then bevk_jpeg_encode into a buffer of exactly the streams' total followed by sentinels."""
    arr, k = _ints(params)
    assert ctx.lib.bevk_jpeg_set_params(ctx.h, arr, k) == 0, what
    total = sum(len(s) for s in want)
    buf = np.full(total + 4096, 0xA5, np.uint8)
    sizes = (ctypes.c_uint64 * n)()
    rc = ctx.lib.bevk_jpeg_encode(ctx.h, ctypes.c_void_p(ptr), istride, pitch, n, W, H, q, L.vptr(buf), total, sizes)
    assert rc == 0, (what, ctx.lib.bevk_last_error().decode())
    assert list(sizes) == [len(s) for s in want], what
    assert buf[:total].tobytes() == b"".join(want), what
    assert (buf[total:] == 0xA5).all(), what
    bound = ctypes.c_uint64()
    assert ctx.lib.bevk_jpeg_encode_bound_params(W, H, arr, k, ctypes.byref(bound)) == 0
    assert max(len(s) for s in want) <= bound.value, what


def test_corpus_byte_equal_to_cv2(torch, ops, L):
    """Every corpus case through ops.jpeg_encode (NumPy; CUDA dense, padded rows and images, byte offset 3) and
    bevk_jpeg_encode, all on one context."""
    n_img = 0
    with _context(L) as ctx:
        for i, c in enumerate(J.cases()):
            imgs = np.stack(c.images)
            n, H, W, _ = imgs.shape
            want = [_cv2(im, c.quality, c.params) for im in c.images]
            assert ops.jpeg_encode(imgs, c.quality, ctx=ctx, params=c.params) == want, (c.name, "numpy")
            kind = ("dense", "padded", "offset")[i % 3]
            view, ptr, istride, pitch, _keep = _layout(torch, imgs, kind)
            assert ops.jpeg_encode(view, c.quality, ctx=ctx, params=c.params) == want, (c.name, kind)
            _direct(L, ctx, ptr, istride, pitch, n, W, H, c.quality, c.params, want, c.name)
            n_img += n
    print(f"{n_img} images compared")


def test_params_do_not_leak_between_calls(torch, ops, L):
    """Wrappers set the context's params on every call (the empty list for params=None), and
    bevk_jpeg_set_params(ctx, NULL, 0) restores cv2's defaults for the direct calls."""
    rng = np.random.default_rng(77)
    imgs = rng.integers(0, 256, (3, 40, 56, 3), dtype=np.uint8)
    default = [_cv2(im, 90) for im in imgs]
    with _context(L) as ctx:
        for p in PARAM_SETS:
            assert ops.jpeg_encode(imgs, 90, ctx=ctx, params=p) == [_cv2(im, 90, p) for im in imgs], p
            assert ops.jpeg_encode(imgs, 90, ctx=ctx) == default, p
        d = torch.from_numpy(imgs).cuda()
        arr, k = _ints(P444)
        assert ctx.lib.bevk_jpeg_set_params(ctx.h, arr, k) == 0
        assert ctx.lib.bevk_jpeg_set_params(ctx.h, None, 0) == 0
        _direct(L, ctx, d.data_ptr(), 40 * 56 * 3, 56 * 3, 3, 56, 40, 90, [], default, "reset")


def test_refusals_and_capacity(torch, ops, L):
    """QUALITY in the list, odd n, unknown keys: BEVK_ERR_ARG; PROGRESSIVE: BEVK_ERR_UNSUPPORTED; a refused list leaves
    the params as they were.  The capacity error behaves as without params: sizes filled, nothing written."""
    rng = np.random.default_rng(78)
    imgs = rng.integers(0, 256, (2, 40, 56, 3), dtype=np.uint8)
    d = torch.from_numpy(imgs).cuda()
    keep = P444 + [J.OPTIMIZE, 1, J.RST, 2]
    want = [_cv2(im, 90, keep) for im in imgs]
    with _context(L) as ctx:
        arr, k = _ints(keep)
        assert ctx.lib.bevk_jpeg_set_params(ctx.h, arr, k) == 0
        for bad, rc in (([1, 90], -1), ([J.SAMPLING], -1), ([8, 1], -1), ([0, 0], -1), ([J.PROGRESSIVE, 1], -4),
                        ([J.PROGRESSIVE, 3, J.OPTIMIZE, 1], -4), ([J.RST, 1, 1, 50], -1)):
            a, n = _ints(bad)
            assert ctx.lib.bevk_jpeg_set_params(ctx.h, a, n) == rc, bad
            b = ctypes.c_uint64()
            assert ctx.lib.bevk_jpeg_encode_bound_params(56, 40, a, n, ctypes.byref(b)) == rc, bad
            with pytest.raises(L.BevkError):
                ops.jpeg_encode(imgs, 90, ctx=ctx, params=bad)
        total = sum(len(s) for s in want)
        buf = np.full(total + 64, 0xA5, np.uint8)
        sizes = (ctypes.c_uint64 * 2)()
        rc = ctx.lib.bevk_jpeg_encode(ctx.h, ctypes.c_void_p(d.data_ptr()), 40 * 56 * 3, 56 * 3, 2, 56, 40, 90, L.vptr(buf),
                                      total - 1, sizes)
        assert rc == -1 and "capacity" in ctx.lib.bevk_last_error().decode()
        assert list(sizes) == [len(s) for s in want] and (buf == 0xA5).all()
        _direct(L, ctx, d.data_ptr(), 40 * 56 * 3, 56 * 3, 2, 56, 40, 90, keep, want, "after refusals")
    assert ops.jpeg_encode_bound(56, 40) == ops.jpeg_encode_bound(56, 40, [])
    assert ops.jpeg_encode_bound(56, 40, P444) > ops.jpeg_encode_bound(56, 40)
    assert ops.jpeg_encode_bound(56, 40, P444 + [J.OPTIMIZE, 1, J.RST, 1]) > ops.jpeg_encode_bound(56, 40, P444)


def test_undistorter_jpeg_and_stack_chunks(torch, ops, L):
    """Undistorter.jpeg and cuda_to_jpeg under every parameter set, with BEVK_JPEG_CHUNK 1, 3 and 0, against
    cv2.imencode(cv2.remap(...), params); and bevk_undistort_stack_jpeg directly after bevk_jpeg_set_params."""
    c = min((c for c in CC.corpus() if c.fisheye), key=lambda c: c.UW * c.UH)
    u = ops.Undistorter(c.K, c.D, c.P, (c.UW, c.UH), model="fisheye")
    fr = CC.frames(c.name, 3, 7)
    und = [cv2.remap(f, *CC.cv2_maps(c.name), cv2.INTER_LINEAR) for f in fr]
    d = torch.from_numpy(fr).cuda()
    for k, p in enumerate(PARAM_SETS):
        q = (95, 100, 75, 50)[k % 4]
        want = [_cv2(x, q, p) for x in und]
        assert u.jpeg(fr[0], quality=q, params=p) == want[0], p
        for chunk in ("1", "3", "0"):
            with _env({"BEVK_JPEG_CHUNK": chunk}):
                got = u.cuda_to_jpeg(d, quality=q, params=p)
            assert got == want, (p, chunk)
        assert u.jpeg(fr[1], quality=q) == _cv2(und[1], q), p                  # params=None: the defaults again
    u.close()


@pytest.mark.parametrize("balance", [False, True])
def test_bevgenerator_jpeg_with_params(fx, balance):
    """BevGenerator.jpeg / jpeg_batch / jpeg_cuda with and without the car under the parameter sets: each stream equals
    cv2.imencode of the reference's cv2-path canvas with the same params."""
    import torch
    from cameracalibration_b200.SurroundBirdEyeView import surroundBEV as S
    g = fx.geometry()
    bev = S.BevGenerator(blend=True, balance=balance, calib=fx.calib)
    masks = [R.blend_mask(n, g.BW, g.BH, g.CW, g.CH) for n in NAMES]
    ref = C.RefBev(fx.calib, g, True, balance, masks=masks)
    F, car = fx.frames(), fx.car()
    canv = {c: ref(*F, None if c is None else car) for c in (None, "car")}
    rev = ref(*F[::-1], car)
    d = torch.from_numpy(np.stack([np.stack(F)])).cuda()
    for p in PARAM_SETS:
        assert bev.jpeg(*F, None, params=p) == _cv2(canv[None], 95, p), p
        assert bev.jpeg(*F, car, params=p) == _cv2(canv["car"], 95, p), p
        assert bev.jpeg_batch([F, F[::-1]], car, quality=90, params=p) == [_cv2(canv["car"], 90, p), _cv2(rev, 90, p)], p
        assert bev.jpeg_cuda(d, torch.from_numpy(car).cuda(), params=p) == [_cv2(canv["car"], 95, p)], p
    assert bev.jpeg(*F, car) == _cv2(canv["car"], 95)


def test_balance_tiny_canvases_with_params(torch, ops):
    """BALANCE on 24x16 canvases (one CTA's 128 blocks span many images), batch 129, car on, through cuda_to_jpeg
    (BEVK_JPEG_CHUNK 0 and default) and run_to_jpeg, under 4:4:4, 4:1:1, luma / chroma qualities, and optimised tables
    with and without one MCU per restart interval: k_gain over the tiny canvases, then the encoder in the general MCU
    layouts, per-image tables over batches of 129 images that each get their own."""
    rng = np.random.default_rng(600)
    FW, FH, BW, BH = 64, 40, 24, 16
    maps = B._maps(rng, "extreme", 4, FW, FH, BW, BH)
    masks = B._masks(rng, 4, BW, BH, 1)
    sets = B._frames(rng, 4, FW, FH, True, 129)
    car = rng.integers(0, 256, (BH, BW, 3), dtype=np.uint8)
    car[rng.integers(0, 2, (BH, BW)) == 0] = 0
    case = B.Case("gain_params", "extreme", FW, FH, BW, BH, False, maps, masks, sets, car)
    e = ops.BevEngine(4, (FW, FH), (BW, BH))
    for k, ((m1, m2), mk) in enumerate(zip(maps, masks)):
        e.set_maps(k, m1, m2)
        e.set_mask(k, mk)
    e.finalize()
    frames = torch.from_numpy(np.stack([np.stack(s) for s in sets])).cuda()
    car_d = torch.from_numpy(car).cuda()
    canv = [B.oracle(case, s, True, True) for s in range(129)]
    n_cmp = 0
    for p in (P444, P411, [J.LUMA, 95, J.CHROMA, 60], [J.OPTIMIZE, 1, J.RST, 1], P411 + [J.OPTIMIZE, 1]):
        want = [None if w is None else _cv2(w, 90, p) for w in canv]
        runs = [({"BEVK_JPEG_CHUNK": "0"}, lambda: e.cuda_to_jpeg(frames, 90, car_d, True, params=p)),
                ({"BEVK_JPEG_CHUNK": None}, lambda: e.cuda_to_jpeg(frames, 90, car_d, True, params=p)),
                ({}, lambda: e.run_to_jpeg(sets, 90, car, True, params=p))]
        for env, run in runs:
            with _env(env):
                got = run()
            for s, w in enumerate(want):
                if w is not None:
                    assert got[s] == w, (p, env, s)
                    n_cmp += 1
    e.ctx.close()
    assert n_cmp > 1000, n_cmp


def test_optimised_large_frames_and_batch_tables(torch, ops, L):
    """Optimised tables at 2560x2048 4:4:4 (one image's counts cover millions of symbols, several CTAs' shared
    counts per image) and a batch of 40 mixed images whose tables all differ, with restart intervals of one MCU row."""
    rng = np.random.default_rng(99)
    big = np.stack([rng.integers(0, 256, (2048, 2560, 3), dtype=np.uint8),
                    np.ascontiguousarray(np.broadcast_to(J.image(rng, 2560, 1, "gradient"), (2048, 2560, 3)))])
    p = P444 + [J.OPTIMIZE, 1, J.RST, 320]
    with _context(L) as ctx:
        got = ops.jpeg_encode(torch.from_numpy(big).cuda(), 95, ctx=ctx, params=p)
        assert got == [_cv2(b, 95, p) for b in big]
        imgs = np.stack([J.image(rng, 72, 40, ("noise", "flat", "checker", "gradient")[i % 4]) for i in range(40)])
        p = [J.OPTIMIZE, 1, J.RST, 5]
        want = [_cv2(im, 85, p) for im in imgs]
        assert len({w[:700] for w in want}) > 4
        assert ops.jpeg_encode(imgs, 85, ctx=ctx, params=p) == want
