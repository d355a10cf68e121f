"""GPU test of what the encoders of one context share: the two output slots and their page-locked sizes (every JPEG,
progressive JPEG and PNG call), and the JPEG work buffers with their header and table cache.  Calls of every encoder at
different sizes are interleaved on one context, one chunked call fails on capacity partway through, and every stream
must still equal cv2's byte for byte.  Every encoding entry refuses inside a graph capture, and OPTIMIZE / PROGRESSIVE
at -1 are read as cv2 reads them (off) by the calls that use the context's list."""
import ctypes
import os
from contextlib import contextmanager

import cv2
import numpy as np
import pytest

from tests import bev_cases as B

pytestmark = pytest.mark.gpu

OPTIMIZE, PROGRESSIVE, RST, SAMPLING = cv2.IMWRITE_JPEG_OPTIMIZE, cv2.IMWRITE_JPEG_PROGRESSIVE, cv2.IMWRITE_JPEG_RST_INTERVAL, \
    cv2.IMWRITE_JPEG_SAMPLING_FACTOR


@pytest.fixture(scope="module")
def ops():
    from cameracalibration_b200 import ops as o
    return o


@pytest.fixture(scope="module")
def L():
    from cameracalibration_b200 import _lib
    return _lib


@pytest.fixture(scope="module")
def torch():
    import torch as t
    return t


def _jpg(img, q, params=()):
    return cv2.imencode(".jpg", np.ascontiguousarray(img), [cv2.IMWRITE_JPEG_QUALITY, q] + list(params))[1].tobytes()


def _png(img, params=()):
    return cv2.imencode(".png", np.ascontiguousarray(img), list(params))[1].tobytes()


@contextmanager
def _chunk(n):
    old = os.environ.get("BEVK_JPEG_CHUNK")
    os.environ["BEVK_JPEG_CHUNK"] = str(n)
    try:
        yield
    finally:
        if old is None:
            os.environ.pop("BEVK_JPEG_CHUNK")
        else:
            os.environ["BEVK_JPEG_CHUNK"] = old


def _engine(ops, case):
    e = ops.BevEngine(case.NC, (case.FW, case.FH), (case.BW, case.BH))
    for k, ((m1, m2), mk) in enumerate(zip(case.maps, case.masks)):
        e.set_maps(k, m1, m2)
        e.set_mask(k, mk)
    if case.nearest:
        e.set_interpolation(ops.INTER_NEAREST)
    e.finalize()
    return e


def _undistorter(ops, ctx):
    K = np.array([[70.0, 0, 44], [0, 70.0, 30], [0, 0, 1]])
    return ops.Undistorter(K, np.array([-0.2, 0.05, 0.001, -0.002, 0.0]), K, (88, 60), model="pinhole", ctx=ctx)


def test_interleaved_encoders_and_a_capacity_failure(ops, L, torch):
    """One context: the chunked BEV-to-JPEG call, bevk_jpeg_encode under a context list, progressive
    bevk_jpeg_encode_params, bevk_png_encode_params at level 9 and bevk_png_encode, at four image sizes, in one order,
    then the chunked call failing on capacity after its first chunk, then the others in the reverse order."""
    case = B.case_by_name("smooth4")
    e = _engine(ops, case)
    ctx, lib, nb = e.ctx, e.ctx.lib, 5
    d = torch.from_numpy(np.stack([np.stack(s) for s in case.sets[:nb]])).cuda()
    bev_want = [_jpg(B.oracle(case, s), 90) for s in range(nb)]
    fb = case.FW * case.FH * 3
    table = (ctypes.c_void_p * (nb * case.NC))(*[d.data_ptr() + i * fb for i in range(nb * case.NC)])
    rng = np.random.default_rng(41)
    a = rng.integers(0, 256, (3, 72, 88, 3), dtype=np.uint8)
    b = rng.integers(0, 256, (2, 40, 56, 3), dtype=np.uint8)
    c = np.repeat(np.repeat(rng.integers(0, 256, (4, 9, 12, 3), dtype=np.uint8), 4, 1), 4, 2)   # compressible
    base_params, prog_params, png_params = [SAMPLING, 0x111111, RST, 3], [PROGRESSIVE, 1], [cv2.IMWRITE_PNG_COMPRESSION, 9]
    da = torch.from_numpy(a).cuda()
    torch.cuda.synchronize()   # the raw calls below run on the context's stream

    def bev(cap=None):
        out = np.full(sum(map(len, bev_want)) + 64, 0x5A, np.uint8)
        sizes = (ctypes.c_uint64 * nb)()
        cap = sum(map(len, bev_want)) if cap is None else cap
        ops.jpeg_set_params(ctx)   # the context's list: cv2's defaults again after check_baseline set its own
        with _chunk(2):
            rc = lib.bevk_bev_frames_to_jpeg(ctx.h, table, nb, None, 0, 90, L.vptr(out), cap, sizes)
        return rc, out, list(sizes)

    def check_bev():
        rc, out, sizes = bev()
        assert rc == 0, lib.bevk_last_error().decode()
        assert sizes == [len(s) for s in bev_want] and out[:sum(sizes)].tobytes() == b"".join(bev_want)

    def check_baseline():
        assert ops.jpeg_encode(a, 85, ctx=ctx, params=base_params) == [_jpg(x, 85, base_params) for x in a]

    def check_progressive():
        assert ops.jpeg_encode_params(b, prog_params, 80, ctx=ctx) == [_jpg(x, 80, prog_params) for x in b]

    def check_png_level9():
        assert ops.png_encode(c, ctx=ctx, params=png_params) == [_png(x, png_params) for x in c]

    def check_png_default():
        ops.png_set_params(ctx)
        cap = 3 * ops.png_encode_bound(88, 72)
        out, sizes = np.empty(cap, np.uint8), (ctypes.c_uint64 * 3)()
        L.check(lib.bevk_png_encode(ctx.h, ctypes.c_void_p(da.data_ptr()), 72 * 88 * 3, 88 * 3, 3, 88, 72, L.vptr(out), cap, sizes))
        assert ops._split(out, sizes) == [_png(x) for x in a]

    steps = [check_bev, check_baseline, check_progressive, check_png_level9, check_png_default]
    for step in steps:
        step()
    # capacity for the first two streams and one byte: the first chunk's streams are written, nothing after them
    lead = len(bev_want[0]) + len(bev_want[1])
    rc, out, sizes = bev(lead + 1)
    assert rc == -1 and "capacity" in lib.bevk_last_error().decode()
    assert sizes == [len(s) for s in bev_want]
    assert out[:lead].tobytes() == b"".join(bev_want[:2]) and (out[lead:] == 0x5A).all()
    for step in reversed(steps):
        step()


def test_baseline_progressive_baseline_at_one_size(ops):
    """The header / frame prefix and tables are cached per (size, options): a progressive call between two baseline
    calls at the same size and quality switches them both ways."""
    from cameracalibration_b200 import _lib as L
    ctx = L.Context(L.default_context().device)
    img = np.random.default_rng(42).integers(0, 256, (2, 48, 64, 3), dtype=np.uint8)
    base = [_jpg(x, 90) for x in img]
    prog = [_jpg(x, 90, [PROGRESSIVE, 1]) for x in img]
    assert ops.jpeg_encode(img, 90, ctx=ctx) == base
    assert ops.jpeg_encode_params(img, [PROGRESSIVE, 1], 90, ctx=ctx) == prog
    assert ops.jpeg_encode(img, 90, ctx=ctx) == base
    assert ops.jpeg_encode_params(img, [], 90, ctx=ctx) == base
    assert ops.jpeg_encode_params(img, [PROGRESSIVE, 1], 90, ctx=ctx) == prog


def test_every_encoding_entry_refuses_inside_a_capture(ops, L, torch):
    case = B.case_by_name("smooth4")
    e = _engine(ops, case)
    ctx, lib = e.ctx, e.ctx.lib
    u = _undistorter(ops, ctx)
    d = torch.from_numpy(np.stack([np.stack(s) for s in case.sets[:2]])).cuda()
    fb = case.FW * case.FH * 3
    table = (ctypes.c_void_p * (2 * case.NC))(*[d.data_ptr() + i * fb for i in range(2 * case.NC)])
    keep = [np.ascontiguousarray(f) for fs in case.sets[:2] for f in fs]
    host_tab = (ctypes.c_void_p * (2 * case.NC))(*[k.ctypes.data for k in keep])
    src = np.random.default_rng(43).integers(0, 256, (60, 88, 3), dtype=np.uint8)
    dsrc = torch.from_numpy(src).cuda()
    dp = ctypes.c_void_p(dsrc.data_ptr())
    torch.cuda.synchronize()   # the raw calls below run on the context's stream
    cap = 1 << 22
    out, sizes = np.empty(cap, np.uint8), (ctypes.c_uint64 * 2)()
    pj, pp = (ctypes.c_int * 2)(PROGRESSIVE, 1), (ctypes.c_int * 2)(cv2.IMWRITE_PNG_COMPRESSION, 9)
    o = (L.vptr(out), cap, sizes)
    calls = {
        "bevk_jpeg_encode": lambda: lib.bevk_jpeg_encode(ctx.h, dp, 0, 88 * 3, 1, 88, 60, 95, *o),
        "bevk_jpeg_encode_params": lambda: lib.bevk_jpeg_encode_params(ctx.h, pj, 2, dp, 0, 88 * 3, 1, 88, 60, 95, *o),
        "bevk_png_encode": lambda: lib.bevk_png_encode(ctx.h, dp, 0, 88 * 3, 1, 88, 60, *o),
        "bevk_png_encode_params": lambda: lib.bevk_png_encode_params(ctx.h, pp, 2, dp, 0, 88 * 3, 1, 88, 60, *o),
        "bevk_undistort_jpeg": lambda: lib.bevk_undistort_jpeg(ctx.h, u.slot, L.vptr(src), 88, 60, 88 * 3, ops.INTER_LINEAR, 95, *o),
        "bevk_undistort_stack_jpeg": lambda: lib.bevk_undistort_stack_jpeg(ctx.h, u.slot, dp, 0, 88, 60, 88 * 3, 1,
                                                                           ops.INTER_LINEAR, 95, *o),
        "bevk_bev_run_to_jpeg": lambda: lib.bevk_bev_run_to_jpeg(ctx.h, host_tab, case.FW * 3, 2, None, 0, 95, *o),
        "bevk_bev_frames_to_jpeg": lambda: lib.bevk_bev_frames_to_jpeg(ctx.h, table, 2, None, 0, 95, *o),
    }
    for name, call in calls.items():   # eagerly first: each call works here
        assert call() == 0, (name, lib.bevk_last_error().decode())
    L.check(lib.bevk_graph_begin(ctx.h))
    try:
        for name, call in calls.items():
            assert call() == -1, name
            assert "graph" in lib.bevk_last_error().decode(), name
    finally:
        gid = ctypes.c_int(-1)
        if lib.bevk_graph_end(ctx.h, ctypes.byref(gid)) == 0:
            lib.bevk_graph_destroy(ctx.h, gid)
    assert ops.jpeg_encode(dsrc, 95, ctx=ctx) == [_jpg(src, 95)]
    assert e.cuda_to_jpeg(d[:1], 95) == [_jpg(B.oracle(case, 0), 95)]
    u.close()


@pytest.mark.parametrize("params", [[OPTIMIZE, -1], [PROGRESSIVE, -1], [OPTIMIZE, 2], [PROGRESSIVE, 0, OPTIMIZE, -3]])
def test_context_list_flags_read_as_cv2(ops, torch, params):
    """The calls that use the context's list read OPTIMIZE and PROGRESSIVE as cv2 does: off at or below 0."""
    case = B.case_by_name("smooth4")
    e = _engine(ops, case)
    img = np.random.default_rng(44).integers(0, 256, (2, 40, 56, 3), dtype=np.uint8)
    assert ops.jpeg_encode(img, 90, ctx=e.ctx, params=params) == [_jpg(x, 90, params) for x in img]
    u = _undistorter(ops, e.ctx)
    src = np.random.default_rng(45).integers(0, 256, (60, 88, 3), dtype=np.uint8)
    assert u.jpeg(src, 90, params=params) == _jpg(u(src), 90, params)
    u.close()
    d = torch.from_numpy(np.stack([np.stack(s) for s in case.sets[:2]])).cuda()
    assert e.cuda_to_jpeg(d, 90, params=params) == [_jpg(B.oracle(case, s), 90, params) for s in range(2)]
