"""GPU test of the BEV-to-JPEG entry points (bevk_bev_run_to_jpeg / bevk_bev_frames_to_jpeg, BevEngine.run_to_jpeg /
cuda_to_jpeg, BevGenerator.jpeg / jpeg_batch / jpeg_cuda): every stream must equal cv2.imencode of the oracle canvas
byte for byte -- the reference's cv2 path on its own data, and the fuzz corpus of tests/bev_cases.py -- through the host
chunk pipeline (chunk tails, pageable / page-locked / zero-copy frames, padded rows), device stacks and pointer tables,
both fused kernels, BALANCE with colour balance and the car applied before the encoder, the capacity rule, quality clamping
and the refusal inside a graph capture."""
import ctypes
import os
from contextlib import contextmanager

import cv2
import numpy as np
import pytest

from oracle import cv2_path as C
from oracle import restate as R
from tests import bev_cases as B
from tests.helpers import NAMES

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from cameracalibration_b200 import ops as o
    return o


@pytest.fixture(scope="module")
def torch():
    import torch as t
    return t


def _jpg(img, q):
    return cv2.imencode(".jpg", np.ascontiguousarray(img), [cv2.IMWRITE_JPEG_QUALITY, q])[1].tobytes()


@contextmanager
def _env(env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _engine(ops, case, env=None):
    e = ops.BevEngine(case.NC, (case.FW, case.FH), (case.BW, case.BH))
    for k, ((m1, m2), mk) in enumerate(zip(case.maps, case.masks)):
        e.set_maps(k, m1, m2)
        e.set_mask(k, mk)
    if case.nearest:
        e.set_interpolation(ops.INTER_NEAREST)
    with _env(env or {}):
        e.finalize()
    return e


class Want:
    """cv2.imencode of the oracle canvas per (frame-set, balance, car, quality)."""

    def __init__(self, case):
        self.case, self.memo = case, {}

    def __call__(self, s, balance, car, q):
        k = (s, balance, car, q)
        if k not in self.memo:
            canvas = B.oracle(self.case, s, balance, car)
            self.memo[k] = None if canvas is None else _jpg(canvas, q)
        return self.memo[k]

    def check(self, got, balance, car, q, what):
        compared = 0
        for s, stream in enumerate(got):
            w = self(s, balance, car, q)
            if w is None:          # BALANCE of a canvas with a zero channel mean: the reference divides by zero
                continue
            assert stream == w, (self.case.name, what, s, balance, car, q, len(stream), len(w))
            compared += 1
        assert compared > 0, (self.case.name, what, "no frame-set has a defined oracle")
        return compared


def _stack(torch, case, n):
    return torch.from_numpy(np.stack([np.stack(s) for s in case.sets[:n]])).cuda()


def _views(torch, case, n):
    """Frame-sets 0..n-1 as nested lists of device views into one buffer at a 16-byte aligned stride (a stack for any
    frame size), and the buffer."""
    fb = case.FW * case.FH * 3
    step = (fb + 15) // 16 * 16
    buf = torch.zeros(n * case.NC * step + 64, dtype=torch.uint8, device="cuda")
    frames = []
    for b, fs in enumerate(case.sets[:n]):
        row = []
        for k, f in enumerate(fs):
            v = buf[(b * case.NC + k) * step:(b * case.NC + k) * step + fb]
            v.copy_(torch.from_numpy(f.reshape(-1)).cuda())
            row.append(v.view(case.FH, case.FW, 3))
        frames.append(row)
    return frames, buf


def _pinned(sets):
    from cameracalibration_b200 import _lib as L
    out = []
    for fs in sets:
        row = []
        for f in fs:
            p = L.pinned_empty(f.shape)
            p[...] = f
            row.append(p)
        out.append(row)
    return out


@pytest.mark.parametrize("blend", [False, True])
@pytest.mark.parametrize("balance", [False, True])
def test_bevgenerator_jpeg_on_reference_data(fx, blend, balance):
    """BevGenerator.jpeg / jpeg_batch / jpeg_cuda with and without the car on the reference's data/ frames: each stream
    equals cv2.imencode of the reference's cv2 path and of BevGenerator.__call__'s canvas."""
    import torch
    from cameracalibration_b200.SurroundBirdEyeView import surroundBEV as S
    g = fx.geometry()
    bev = S.BevGenerator(blend=blend, balance=balance, calib=fx.calib)
    masks = [R.blend_mask(n, g.BW, g.BH, g.CW, g.CH) if blend else C.plain_mask(n, g) for n in NAMES]
    ref = C.RefBev(fx.calib, g, blend, balance, masks=masks)
    F, car = fx.frames(), fx.car()
    for c in (None, car):
        want = _jpg(ref(*F, c), 95)
        got = bev.jpeg(*F, c)
        assert got == want, (blend, balance, c is not None)
        assert got == _jpg(bev(*F, c), 95)
        assert cv2.imdecode(np.frombuffer(got, np.uint8), cv2.IMREAD_COLOR).shape == (g.BH, g.BW, 3)
    assert bev.jpeg_batch([F, F[::-1]], car, quality=90) == [_jpg(ref(*F, car), 90), _jpg(ref(*F[::-1], car), 90)]
    d = torch.from_numpy(np.stack([np.stack(F)])).cuda()
    assert bev.jpeg_cuda(d, torch.from_numpy(car).cuda()) == [_jpg(ref(*F, car), 95)]


def test_run_to_jpeg_chunks_and_ingest(ops):
    """Host frames through the chunk pipeline: batches 1, 3, 4, 5, 9 at BEVK_CHUNK 1 and 3 (ragged last chunks), pageable
    and page-locked frames (zero-copy span ingest on and off), frames with a padded row stride, BALANCE on and off."""
    case = B.case_by_name("smooth4")
    want = Want(case)
    e, ez = _engine(ops, case), _engine(ops, case, {"BEVK_ZEROCOPY": "0"})
    pinned = _pinned(case.sets)
    padded = []
    for fs in case.sets:
        row = []
        for f in fs:
            p = np.zeros((case.FH, case.FW + 7, 3), np.uint8)[:, :case.FW]
            p[...] = f
            row.append(p)
        padded.append(row)
    assert padded[0][0].strides[0] == (case.FW + 7) * 3
    n_cmp = 0
    for chunk in ("1", "3"):
        with _env({"BEVK_CHUNK": chunk}):
            for n in (1, 3, 4, 5, 9):
                for balance in (False, True):
                    for frames, eng, what in ((case.sets, e, "pageable"), (pinned, e, "zero-copy"), (pinned, ez, "page-locked DMA"),
                                              (padded, e, "padded rows")):
                        got = eng.run_to_jpeg(frames[:n], 75, case.car, balance)
                        assert len(got) == n
                        assert eng.last_path() == "tma", (what, n, chunk)
                        n_cmp += want.check(got, balance, True, 75, f"{what} chunk {chunk} batch {n}")
                got = e.run_to_jpeg(case.sets[:n], 100)
                n_cmp += want.check(got, False, False, 100, f"no car chunk {chunk} batch {n}")
    assert e.last_h2d_bytes() > 0
    print(f"run_to_jpeg: {n_cmp} streams compared")


def test_cuda_to_jpeg_stack_table_and_gather(ops, torch):
    """Device frames: a stack takes k_bev_tma (path 2), nested lists of frames that form no stack and BEVK_TMA=0 take
    k_bev (path 1); BALANCE renders from its balanced copies, a stack, so it takes k_bev_tma unless BEVK_TMA=0."""
    from cameracalibration_b200 import _lib as L
    case = B.case_by_name("smooth4")
    want = Want(case)
    e, eg = _engine(ops, case), _engine(ops, case, {"BEVK_TMA": "0"})
    d = _stack(torch, case, 9)
    car = torch.from_numpy(case.car).cuda()
    fb = case.FW * case.FH * 3
    step = (fb + 32 + 15) // 16 * 16
    buf = torch.zeros(9 * case.NC * step + 64, dtype=torch.uint8, device="cuda")
    nested = []
    for b, fs in enumerate(case.sets):
        row = []
        for k, f in enumerate(fs):
            i = b * case.NC + k
            o = i * step + (16 if i % 2 else 0)
            buf[o:o + fb].copy_(torch.from_numpy(f.reshape(-1)).cuda())
            row.append(buf[o:o + fb].view(case.FH, case.FW, 3))
        nested.append(row)
    for balance in (False, True):
        for n in (1, 4, 9):
            got = e.cuda_to_jpeg(d[:n], 75, car, balance)
            assert L.load().bevk_bev_last_path(e.ctx.h) == 2
            want.check(got, balance, True, 75, f"stack batch {n}")
            got = e.cuda_to_jpeg(nested[:n], 100, None, balance)
            assert e.last_path() == ("tma" if balance else "gather"), balance
            want.check(got, balance, False, 100, f"nested batch {n}")
            got = eg.cuda_to_jpeg(d[:n], 75, car, balance)
            assert L.load().bevk_bev_last_path(eg.ctx.h) == 1
            want.check(got, balance, True, 75, f"BEVK_TMA=0 batch {n}")
        for chunk in ("0", "1", "4"):              # the whole device batch at once, and chunks of canvases
            with _env({"BEVK_JPEG_CHUNK": chunk}):
                want.check(e.cuda_to_jpeg(d, 95, car, balance), balance, True, 95, f"BEVK_JPEG_CHUNK {chunk}")


def test_balance_to_jpeg_launches_the_two_step_kernels(ops, torch):
    """BALANCE to JPEG launches as many kernels as run_stack + ops.jpeg_encode (the render ending in k_gain, then the
    encoder), with identical streams."""
    case = B.case_by_name("smooth4")
    e = _engine(ops, case)
    n, fb = 5, case.FW * case.FH * 3
    d = _stack(torch, case, n)
    car = torch.from_numpy(case.car).cuda()
    out = torch.empty((n, case.BH, case.BW, 3), dtype=torch.uint8, device="cuda")

    def two_calls():
        e.run_stack(d.data_ptr(), fb, n, out.data_ptr(), car.data_ptr(), True)
        return ops.jpeg_encode(out, 95, ctx=e.ctx)

    for _ in range(2):                             # every table, buffer and tensor map exists afterwards
        two_calls()
        e.cuda_to_jpeg(d, 95, car, True)
    l0 = e.ctx.launches
    sep = two_calls()
    l1 = e.ctx.launches
    one = e.cuda_to_jpeg(d, 95, car, True)
    l2 = e.ctx.launches
    assert one == sep
    assert l1 - l0 == l2 - l1, (l1 - l0, l2 - l1)
    Want(case).check(one, True, True, 95, "BALANCE to JPEG")


@pytest.mark.parametrize("seed", range(B.N_CASES))
def test_fuzz_corpus_both_entry_points(ops, torch, seed):
    """Every corpus case through run_to_jpeg (7 host frame-sets, BEVK_CHUNK 3) and cuda_to_jpeg (9 device frame-sets as a
    16-byte aligned stack of views) at q75 and q100, with the car, BALANCE on and off on the 4-camera cases."""
    case = B.make_case(seed)
    want = Want(case)
    e = _engine(ops, case)
    frames, _keep = _views(torch, case, 9)
    car = torch.from_numpy(case.car).cuda()
    for balance in ((False, True) if case.NC == 4 else (False,)):
        for q in (75, 100):
            with _env({"BEVK_CHUNK": "3"}):
                want.check(e.run_to_jpeg(case.sets[:7], q, case.car, balance), balance, True, q, "run_to_jpeg")
            want.check(e.cuda_to_jpeg(frames, q, car, balance), balance, True, q, "cuda_to_jpeg")
            assert e.last_path() == ("tma" if case.tma_friendly else "gather"), (balance, q)


def test_capacity_quality_and_graph_capture(ops, torch):
    """Capacity: total - 1 fails with "capacity", fills sizes[], writes the whole leading streams that fit and nothing at
    or past capacity; exactly total succeeds.  Quality is clamped as cv2 does.  A call inside a capture is refused."""
    from cameracalibration_b200 import _lib as L
    case = B.case_by_name("smooth4")
    want = Want(case)
    e = _engine(ops, case)
    lib, n = e.ctx.lib, 5
    streams = [want(s, True, True, 90) for s in range(n)]
    total = sum(len(s) for s in streams)
    d = _stack(torch, case, n)
    car_d = torch.from_numpy(case.car).cuda()
    fb = case.FW * case.FH * 3
    dev_tab = (ctypes.c_void_p * (n * case.NC))(*[d.data_ptr() + i * fb for i in range(n * case.NC)])
    keep = [np.ascontiguousarray(f) for fs in case.sets[:n] for f in fs]
    host_tab = (ctypes.c_void_p * (n * case.NC))(*[k.ctypes.data for k in keep])
    car_h = np.ascontiguousarray(case.car)

    def call(which, cap, buf, sizes, q=90):
        if which == "host":
            return lib.bevk_bev_run_to_jpeg(e.ctx.h, host_tab, case.FW * 3, n, L.vptr(car_h), L.FLAG_BALANCE, q, L.vptr(buf), cap, sizes)
        return lib.bevk_bev_frames_to_jpeg(e.ctx.h, dev_tab, n, ctypes.c_void_p(car_d.data_ptr()), L.FLAG_BALANCE, q, L.vptr(buf), cap,
                                           sizes)

    for which, env in (("host", {"BEVK_CHUNK": "1"}), ("host", {"BEVK_CHUNK": "3"}), ("device", {}), ("device", {"BEVK_JPEG_CHUNK": "2"})):
        with _env(env):
            for cap, lead in ((total - 1, n - 1), (len(streams[0]) + len(streams[1]) - 1, 1), (len(streams[0]) - 1, 0)):
                buf = np.full(total + 64, 0xA5, np.uint8)
                sizes = (ctypes.c_uint64 * n)()
                assert call(which, cap, buf, sizes) == -1, (which, env, cap)
                assert "capacity" in lib.bevk_last_error().decode()
                assert list(sizes) == [len(s) for s in streams], (which, env, cap)
                written = sum(len(s) for s in streams[:lead])
                assert buf[:written].tobytes() == b"".join(streams[:lead]), (which, env, cap)
                assert (buf[written:] == 0xA5).all(), (which, env, cap)
            buf = np.full(total + 64, 0xA5, np.uint8)
            sizes = (ctypes.c_uint64 * n)()
            assert call(which, total, buf, sizes) == 0, lib.bevk_last_error().decode()
            assert buf[:total].tobytes() == b"".join(streams) and (buf[total:] == 0xA5).all()
    for q in (-5, 0, 150):
        want_q = [_jpg(B.oracle(case, s, False, True), q) for s in range(3)]
        assert e.run_to_jpeg(case.sets[:3], q, case.car) == want_q, q
        assert e.cuda_to_jpeg(d[:3], q, car_d) == want_q, q
    buf, sizes = np.empty(total, np.uint8), (ctypes.c_uint64 * n)()
    L.check(lib.bevk_graph_begin(e.ctx.h))
    try:
        for which in ("host", "device"):
            assert call(which, total, buf, sizes) == -1
            assert "graph" in lib.bevk_last_error().decode()
    finally:
        gid = ctypes.c_int(-1)
        if lib.bevk_graph_end(e.ctx.h, ctypes.byref(gid)) == 0:
            lib.bevk_graph_destroy(e.ctx.h, gid)
    assert e.cuda_to_jpeg(d[:1], 95, car_d, True) == [want(0, True, True, 95)]
