"""GPU tests of the packed YUV 4:2:2 render (YUYV, UYVY) on the 4:2:2 corpus of tests/yuv422_cases.py (yuv422_corpus: the
even-width fuzz corpus cases and a supplement with odd heights down to 1, FW % 4 == 2, FW % 32 == 16, 1-8 cameras,
int16-extreme and edge taps, bright frames): k_vsum_yuv, k_yuv_spans, the page-locked windows (k_fetch_yuv) and the
pageable DMA rectangles, then k_bev_tma or k_bev on the converted copy stack.  Every case runs in both byte orders
through run_stack (dense, and at an odd base and stride), run_cuda, run on page-locked and pageable frames with padded
rows, and run_cuda_planes (a pool view and a table of separate surfaces, rows padded to a 2048-byte pitch).  Each canvas
is compared byte for byte with the cv2 / NumPy oracle of cv2.cvtColor(COLOR_YUV2BGR_YUY2 / _UYVY) of every frame; the
run_stack canvases of 9 frame-sets also with the same engine's BGR render of the cvtColor frames.  Every render must have
run k_bev_tma exactly when the copy stack's pitch is 16-byte friendly (FW % 16 == 0).

As in test_gpu_yuv_fuzz, consecutive checked calls on one engine take frame-sets 0.. and 1.. in turn, and calls in the
other byte order, in NV12 (even heights) and in BGR with BALANCE, on the frame-sets in reverse order, overwrite the copy
stack in between, so that no check can pass on an earlier call's conversion."""
import ctypes

import cv2
import numpy as np
import pytest

from oracle import restate as R
from tests import bev_cases as B
from tests import yuv422_cases as YC
from tests import yuv422_frames as Y2
from tests import yuv_frames as Y
from tests.helpers import NAMES
from tests.test_gpu_bev_fuzz import Want, _engines, _render, ops, torch  # noqa: F401  (module fixtures)
from tests.test_gpu_yuv_fuzz import _bgr_stack, _Pools

pytestmark = pytest.mark.gpu
BATCHES = (1, 4, 9)
CASES = [c.name for c in YC.yuv422_corpus()]
V = ctypes.c_void_p


def _stack(torch, case, order, odd):
    """The packed frame-sets `order` as one device stack: dense, or at byte 1 of the buffer with a frame stride of frame
    bytes + 3 (odd) and 0xFF padding.  Returns (buffer, byte offset of the first frame, stride)."""
    fb = case.FW * case.FH * 2
    stride, base = (fb + 3, 1) if odd else (fb, 0)
    host = np.full(base + len(order) * case.NC * stride, 0xFF, np.uint8)
    for i, f in enumerate(f for s in order for f in case.yuv[s]):
        host[base + i * stride:base + i * stride + fb] = f.reshape(-1)
    return torch.from_numpy(host).cuda(), base, stride


def _host(case, alloc, pad):
    """Every frame-set as host arrays from alloc(shape), rows 2 FW + pad bytes apart (views [FH][FW][2])."""
    out = []
    for fs in case.yuv:
        row = []
        for f in fs:
            p = alloc((case.FH, 2 * case.FW + pad))[:, :2 * case.FW].reshape(case.FH, case.FW, 2)
            p[...] = f
            row.append(p)
        out.append(row)
    return out


def _pitch(FW):
    """Rows padded to a multiple of 2048 bytes, as decoder and capture surfaces often are."""
    return (2 * FW + 2048) // 2048 * 2048


def _planes_pool(torch, frame_sets):
    """Frame-sets (lists of [FH][FW][2] frames) as a strided [batch][NC][FH][FW][2] view into one pool of rows padded to
    _pitch (0xA5 padding).  Returns (pool, view)."""
    a = np.stack([np.stack(fs) for fs in frame_sets])
    nb, NC, FH, FW = a.shape[:4]
    P = _pitch(FW)
    pool = torch.full((nb * NC * FH * P,), 0xA5, dtype=torch.uint8, device="cuda")
    view = pool.as_strided((nb, NC, FH, FW, 2), (NC * FH * P, FH * P, P, 2, 1))
    view.copy_(torch.from_numpy(a).cuda())
    return pool, view


def _planes_table(torch, case, sets):
    """The frame-sets as per-frame 1-tuples of [FH][FW][2] views into separate allocations (no common frame stride)."""
    P = _pitch(case.FW)
    keep, out = [], []
    for j, s in enumerate(sets):
        row = []
        for k, f in enumerate(case.yuv[s]):
            buf = torch.full(((case.FH + 1 + (j * case.NC + k) % 3) * P,), 0x5A, dtype=torch.uint8, device="cuda")
            v = buf.as_strided((case.FH, case.FW, 2), (P, 2, 1), P * ((j * case.NC + k) % 3))
            v.copy_(torch.from_numpy(f).cuda())
            keep.append(buf)
            row.append((v,))
        out.append(row)
    return keep, out


@pytest.mark.parametrize("fmt", Y2.FORMATS)
@pytest.mark.parametrize("name", CASES)
def test_yuv422_case_every_entry_point(ops, torch, name, fmt):
    """One 4:2:2 corpus case in one byte order through every entry point that takes packed frames; BALANCE on the
    4-camera cases, car on and off, BGR and (even canvases) NV12 / I420 canvases from run_cuda_planes."""
    from cameracalibration_b200 import _lib as L
    case = YC.yuv422_case(name, fmt)
    other = "uyvy" if fmt == "yuyv" else "yuyv"
    other_case = YC.yuv422_case(name, other)
    want, want_other = Want(case), Want(other_case)
    path = "tma" if case.FW % 16 == 0 else "gather"
    balances = (False, True) if case.NC == 4 else (False,)
    outs = ("bgr", "nv12", "i420") if case.BW % 2 == 0 and case.BH % 2 == 0 else ("bgr",)
    rev = list(range(YC.N_SETS))[::-1]
    n_cmp = 0
    with _engines(ops) as make:
        e = make(case)
        pick = _Pools()
        d_rev, base_rev, stride_rev = _stack(torch, other_case, rev, False)
        db_rev, sb_rev = _bgr_stack(torch, other_case, rev)
        nv12_rev = None
        if case.FH % 2 == 0:   # the same engine's NV12 path, on frames of its own
            rng = np.random.default_rng(len(name))
            nv = [[Y.random_yuv(rng, case.FW, case.FH) for _ in range(case.NC)] for _ in range(9)]
            nv12_rev = (torch.from_numpy(np.stack([f for fs in nv for f in fs]).reshape(-1)).cuda(),
                        [[Y.to_bgr(f, "nv12") for f in fs] for fs in nv])

        def overwrite():
            """The copy stack rewritten on other frames: the other byte order, NV12, and (4 cameras) BGR with BALANCE."""
            got = _render(torch, e, d_rev, stride_rev, 9, case.car, False, pixel_format=other, base=base_rev)
            assert e.last_path() == path, other
            n = want_other.check(got, False, True, f"{other} run_stack", rev)
            if nv12_rev is not None:
                got = _render(torch, e, nv12_rev[0], case.FW * case.FH * 3 // 2, 9, None, False, pixel_format="nv12")
                ref = _render(torch, e, *_bgr_frames(torch, case, nv12_rev[1]), 9, None, False)
                assert (got == ref).all(), "nv12"
            if case.NC == 4:
                got = _render(torch, e, db_rev, sb_rev, 9, case.car, True)
                n += want_other.check(got, True, True, "bgr BALANCE run_stack", rev)
            return n

        # run_stack: a dense stack, then one at an odd base address and an odd frame stride
        for odd in (False, True):
            d, base, stride = _stack(torch, case, range(YC.N_SETS), odd)
            what = "odd stack" if odd else "dense stack"
            for balance in balances:
                for n in BATCHES:
                    for car in (None, case.car):
                        sets = pick(n)
                        got = _render(torch, e, d, stride, n, car, balance, pixel_format=fmt, base=base + sets[0] * case.NC * stride)
                        assert e.last_path() == path, (what, n, balance)
                        n_cmp += want.check(got, balance, car is not None, f"run_stack {what} batch {n}", sets)
                        if n == 9 and car is not None:   # the same engine's render of the cvtColor frames
                            db, sb = _bgr_stack(torch, case, sets)
                            ref = _render(torch, e, db, sb, n, car, balance)
                            assert (got == ref).all(), (what, balance, int((got != ref).sum()))
            n_cmp += overwrite()
        # run_cuda on one [batch][NC][FH][FW][2] array, with the car
        car_t = torch.from_numpy(case.car).cuda()
        for balance in balances:
            sets = pick(7)
            d = torch.from_numpy(np.stack([np.stack(case.yuv[s]) for s in sets])).cuda()
            out = e.run_cuda(d, car_t, balance, pixel_format=fmt)
            torch.cuda.synchronize()
            assert e.last_path() == path, ("run_cuda", balance)
            n_cmp += want.check(out.cpu().numpy(), balance, True, "run_cuda", sets)
        n_cmp += overwrite()
        # host frames: page-locked (zero-copy windows when the rows are 16-byte friendly) and pageable, rows padded
        for pad in (0, 16, 4):
            for kind, alloc in (("page-locked", L.pinned_empty), ("pageable", lambda shape: np.zeros(shape, np.uint8))):
                frames = _host(case, alloc, pad)
                for balance in balances:
                    sets = pick(5)
                    got = e.run([frames[s] for s in sets], case.car, balance, pixel_format=fmt)
                    assert e.last_path() == path, (pad, kind, balance)
                    n_cmp += want.check(got, balance, True, f"run {kind} rows 2 FW + {pad}", sets)
        n_cmp += overwrite()
        # run_cuda_planes: a pool view and a table of separate surfaces, rows at a 2048-byte pitch
        k = 0
        for entry in ("pool", "table"):
            for balance in balances:
                for ofmt in outs:
                    sets = pick(3)
                    if entry == "pool":
                        keep, y = _planes_pool(torch, [case.yuv[s] for s in sets])
                    else:
                        keep, y = _planes_table(torch, case, sets)
                    car = car_t if k % 2 else None
                    got = e.run_cuda_planes(y, pixel_format=fmt, car=car, balance=balance, out_format=ofmt)
                    torch.cuda.synchronize()
                    assert e.last_path() == path, (entry, balance, ofmt)
                    got = got.cpu().numpy()
                    for i, s in enumerate(sets):
                        w = want(s, balance, car is not None)
                        if w is not None:
                            assert (got[i] == _as_out(w, ofmt)).all(), (name, fmt, entry, balance, ofmt, s)
                            n_cmp += 1
                    del keep
                    k += 1
    assert n_cmp > 0
    print(f"{name} {fmt}: {n_cmp} canvases compared")


def _bgr_frames(torch, case, sets):
    """BGR frame-sets (lists of frames) as one device stack at a 16-byte stride: (buffer, stride)."""
    fb = case.FW * case.FH * 3
    stride = (fb + 15) // 16 * 16
    host = np.zeros((sum(len(fs) for fs in sets), stride), np.uint8)
    host[:, :fb] = np.stack([f.reshape(-1) for fs in sets for f in fs])
    return torch.from_numpy(host.reshape(-1)).cuda(), stride


def _as_out(bgr, ofmt):
    if ofmt == "bgr":
        return bgr
    i420 = cv2.cvtColor(bgr, cv2.COLOR_BGR2YUV_I420)
    return i420 if ofmt == "i420" else Y.i420_to_nv12(i420)


def _fixture_engine(ops, fx, FW, FH, BW=1000, BH=1000):
    from tests.test_gpu_tma import _engine
    g = fx.geometry(FW, FH, BW, BH)
    e, masks = _engine(ops, fx, g, True)
    return e, g


@pytest.mark.parametrize("fmt", Y2.FORMATS)
def test_bench_geometry_paths_and_copy_bytes(ops, torch, fx, fmt):
    """1920 x 1080 -> 1000^2 with the fixture's cameras (the bench geometry), camera-like frames: run from page-locked
    frames (the SMs fetch the 16-byte windows) and pageable ones (DMA rectangles), run_cuda and run_cuda_planes on a
    pitched pool all equal the BGR render of the cvtColor frames, with BALANCE and the car, BGR and NV12 canvases.
    last_h2d_bytes: pageable calls move host_copy_bytes per frame-set (the rectangle sum), page-locked ones fewer (the
    windows), BALANCE whole frames at 2 bytes per pixel; the 4:2:2 upload is at most 0.72x the BGR one."""
    from cameracalibration_b200 import _lib as L
    e, g = _fixture_engine(ops, fx, 1920, 1080)
    try:
        bgr_in = fx.frames(1920, 1080)
        n = 3
        yuv = [[Y2.from_bgr(np.roll(f, 31 * b, axis=1), fmt) for f in bgr_in] for b in range(n)]
        bgr = [[Y2.to_bgr(f, fmt) for f in fs] for fs in yuv]
        car = fx.car(1000, 1000)
        pinned = [[L.pinned_empty(f.shape) for f in fs] for fs in yuv]
        for fs, ps in zip(yuv, pinned):
            for f, p in zip(fs, ps):
                p[...] = f
        h2d, _ = e.host_copy_bytes(False, fmt)
        h2d_bal, _ = e.host_copy_bytes(True, fmt)
        h2d_bgr, _ = e.host_copy_bytes(False)
        assert h2d_bal == 4 * 1920 * 1080 * 2 and h2d <= 0.72 * h2d_bgr, (h2d, h2d_bal, h2d_bgr)
        for balance in (False, True):
            want = e.run(bgr, car, balance)
            got = e.run(yuv, car, balance, pixel_format=fmt)
            assert e.last_path() == "tma"
            assert e.last_h2d_bytes() == n * (h2d_bal if balance else h2d)
            assert (got == want).all(), (fmt, balance, "pageable")
            got = e.run(pinned, car, balance, pixel_format=fmt)
            if balance:
                assert e.last_h2d_bytes() == n * h2d_bal
            else:
                assert 0 < e.last_h2d_bytes() < n * h2d, (e.last_h2d_bytes(), h2d)
            assert (got == want).all(), (fmt, balance, "page-locked")
            car_t = torch.from_numpy(car).cuda()
            d = torch.from_numpy(np.stack([np.stack(fs) for fs in yuv])).cuda()
            for ofmt in ("bgr", "nv12"):
                ref = e.run_cuda(d, car_t, balance, pixel_format=fmt, out_format=ofmt)
                torch.cuda.synchronize()
                assert (ref.cpu().numpy() == (want if ofmt == "bgr" else np.stack([_as_out(w, ofmt) for w in want]))).all()
                keep, y = _planes_pool(torch, yuv)
                got = e.run_cuda_planes(y, pixel_format=fmt, car=car_t, balance=balance, out_format=ofmt)
                torch.cuda.synchronize()
                assert e.last_path() == "tma"
                assert (got.cpu().numpy() == ref.cpu().numpy()).all(), (fmt, balance, ofmt, "planes")
    finally:
        e.ctx.close()


@pytest.mark.parametrize("fmt", Y2.FORMATS)
def test_nearest_at_the_fixture_geometry(ops, torch, fx, fmt):
    """INTER_NEAREST with camera-like 4:2:2 frames: the render equals the BGR render of the cvtColor frames."""
    from oracle import cv2_path as C
    g = fx.geometry(1280, 1024, 1000, 1000)
    e = ops.BevEngine(4, (g.FW, g.FH), (g.BW, g.BH))
    try:
        calib = fx.scaled_calib(g)
        for i, nm in enumerate(NAMES):
            K, D, H = calib[nm]
            e.set_camera(i, K, D, C.dst_camera_matrix(K, g.FW, g.FH, g.FS, g.SS), (int(g.FW * g.SS), int(g.FH * g.SS)), H)
            e.set_mask(i, R.blend_mask(nm, g.BW, g.BH, g.CW, g.CH))
        e.set_interpolation(ops.INTER_NEAREST)
        e.finalize()
        yuv = [[Y2.from_bgr(f, fmt) for f in fx.frames(1280, 1024)]]
        bgr = [[Y2.to_bgr(f, fmt) for f in yuv[0]]]
        for balance in (False, True):
            got = e.run(yuv, fx.car(), balance, pixel_format=fmt)
            assert (got == e.run(bgr, fx.car(), balance)).all(), (fmt, balance)
    finally:
        e.ctx.close()


@pytest.mark.parametrize("balance", [False, True])
def test_graph_replay_reads_the_captured_yuv422_stack(ops, torch, fx, balance):
    """Capture a 4:2:2 run_stack on stack A, make an eager call on stack B, replay: A's canvases, which equal the BGR
    render of A's cvtColor frames."""
    from tests.test_gpu_graph_frames import _replay_after_other_stack
    e, g = _fixture_engine(ops, fx, 640, 512, 500, 500)
    try:
        n, fb = 3, 640 * 512 * 2
        car = torch.from_numpy(fx.car(500, 500)).cuda()
        for fmt in Y2.FORMATS:
            a = np.stack([np.stack([Y2.from_bgr(np.roll(f, 17 * b, axis=0), fmt) for f in fx.frames(640, 512)]) for b in range(n)])
            d_a, d_b = torch.from_numpy(a).cuda(), torch.from_numpy(np.ascontiguousarray(a[::-1]) ^ 0x21).cuda()

            def call(d, out):
                e.run_stack(d.data_ptr(), fb, n, out.data_ptr(), car.data_ptr(), balance, pixel_format=fmt)

            want_a, want_b, got = _replay_after_other_stack(torch, e, call, d_a, d_b, (n, 500, 500, 3))
            assert e.last_path() == "tma"
            bgr = [[Y2.to_bgr(f, fmt) for f in fs] for fs in a]
            assert (want_a == e.run(bgr, fx.car(500, 500), balance)).all()
            assert (got == want_a).all(), (fmt, int((got != want_a).sum()), bool((got == want_b).all()))
    finally:
        e.ctx.close()


@pytest.mark.parametrize("fmt", Y2.FORMATS)
def test_bevgenerator_yuv422_at_the_fixture_geometry(fx, fmt):
    """BevGenerator.run_batch, run_cuda and run_cuda_planes with pixel_format (blend, BALANCE, car) at 1280x1024 ->
    1000^2 with the reference's calibration: cv2.cvtColor of every frame, then the reference's call sequence (RefBev)."""
    import torch
    from cameracalibration_b200.SurroundBirdEyeView import surroundBEV as S
    from tests.test_gpu_yuv import _oracle
    g = fx.geometry()
    bev = S.BevGenerator(blend=True, balance=True, calib=fx.calib)
    masks = [R.blend_mask(n, g.BW, g.BH, g.CW, g.CH) for n in NAMES]
    car = fx.car()
    bgr_in = [fx.frames(g.FW, g.FH)] + [fx.perturbed_frames(g.FW, g.FH, 1)]
    yuv = [[Y2.from_bgr(f, fmt) for f in s] for s in bgr_in]
    want = [_oracle(fx.calib, g, masks, True, True, [Y2.to_bgr(f, fmt) for f in s], car) for s in yuv]
    got = bev.run_batch(yuv, car, pixel_format=fmt)
    d = torch.from_numpy(np.stack([np.stack(s) for s in yuv[::-1]])).cuda()
    got_d = bev.run_cuda(d, torch.from_numpy(car).cuda(), pixel_format=fmt)
    torch.cuda.synchronize()
    got_d = got_d.cpu().numpy()
    got_p = bev.run_cuda_planes([[(t,) for t in fs] for fs in d], pixel_format=fmt, car=torch.from_numpy(car).cuda())
    torch.cuda.synchronize()
    got_p = got_p.cpu().numpy()
    for b in range(2):
        assert (got[b] == want[b]).all(), (fmt, "run_batch", b, int((got[b] != want[b]).sum()))
        assert (got_d[1 - b] == want[b]).all(), (fmt, "run_cuda", b)
        assert (got_p[1 - b] == want[b]).all(), (fmt, "run_cuda_planes", b)


def test_refusals(ops, torch, fx):
    """Refused with a message, nothing enqueued and the output untouched: two input flags, an odd width, the new bits on
    every entry point that takes BGR frames only, a pitch below 2 FW, a null plane, more than 65535 frames; and the
    Python layer's shape checks."""
    from cameracalibration_b200 import _lib as L
    e, g = _fixture_engine(ops, fx, 640, 511, 500, 500)   # an odd height: 4:2:2 takes it
    lib, h = e.ctx.lib, e.ctx.h
    try:
        fb = 640 * 511 * 2
        d = torch.full((4 * fb + 64,), 7, dtype=torch.uint8, device="cuda")
        out = torch.full((500 * 500 * 3 + 64,), 0xA5, dtype=torch.uint8, device="cuda")
        o = V(out.data_ptr())
        I64 = ctypes.c_int64 * 3
        offs, pitch = I64(0, 0, 0), I64(1280, 0, 0)
        tab = (V * 12)(*[d.data_ptr() + i * fb if p == 0 else None for i in range(4) for p in range(3)])
        for flag in (L.FLAG_YUYV, L.FLAG_UYVY):
            for other in (L.FLAG_NV12, L.FLAG_I420, L.FLAG_YUYV ^ L.FLAG_UYVY ^ flag):
                both = flag | other
                assert lib.bevk_bev_run_stack(h, V(d.data_ptr()), fb, 1, None, both, o) == -1
                assert lib.bevk_bev_run_yuv_planes(h, V(d.data_ptr()), fb, offs, pitch, 1, None, both, o) == -1
                assert lib.bevk_bev_run_yuv_surfaces(h, tab, pitch, 1, None, both, o) == -1
                a, b = ctypes.c_int64(), ctypes.c_int64()
                assert lib.bevk_bev_host_copy_bytes(h, both, ctypes.byref(a), ctypes.byref(b)) == -1
                assert "exclusive" in lib.bevk_last_error().decode()
            assert lib.bevk_bev_run_stack(h, V(d.data_ptr()), fb - 1, 1, None, flag, o) == -1
            bad = I64(1279, 0, 0)
            assert lib.bevk_bev_run_yuv_planes(h, V(d.data_ptr()), fb, offs, bad, 1, None, flag, o) == -1
            assert lib.bevk_bev_run_yuv_surfaces(h, tab, bad, 1, None, flag, o) == -1
            assert lib.bevk_bev_run_yuv_planes(h, None, fb, offs, pitch, 1, None, flag, o) == -1
            t = (V * 12)(*tab); t[3 * 2] = None
            assert lib.bevk_bev_run_yuv_surfaces(h, t, pitch, 1, None, flag, o) == -1
            assert lib.bevk_bev_run_yuv_planes(h, V(d.data_ptr()), 0, offs, pitch, 16384, None, flag, o) == -1
            assert "65535" in lib.bevk_last_error().decode()
            assert lib.bevk_bev_run_stack(h, V(d.data_ptr()), fb, 16384, None, flag, o) == -1
            assert "65535" in lib.bevk_last_error().decode()
            # the entry points that read BGR frames only
            table = (V * 4)(*[d.data_ptr()] * 4)
            hp = (V * 4)(*[d.data_ptr()] * 4)
            sizes = (ctypes.c_uint64 * 4)(1, 1, 1, 1)
            streams = np.zeros(1 << 16, np.uint8)
            ssz = (ctypes.c_uint64 * 1)()
            n_own = ctypes.c_int()
            for f2 in (flag, flag | L.FLAG_BALANCE):
                rcs = {
                    "run_device": lib.bevk_bev_run_device(h, V(d.data_ptr()), 1, None, f2, o),
                    "run_frames": lib.bevk_bev_run_frames(h, table, 1, None, f2, o),
                    "run_jpeg": lib.bevk_bev_run_jpeg(h, hp, sizes, 1, None, f2, L.vptr(streams)),
                    "run_to_jpeg": lib.bevk_bev_run_to_jpeg(h, hp, 1280, 1, None, f2, 95, L.vptr(streams), streams.size, ssz),
                    "frames_to_jpeg": lib.bevk_bev_frames_to_jpeg(h, table, 1, None, f2, 95, L.vptr(streams), streams.size, ssz),
                    "run_sharded": lib.bevk_bev_run_sharded(h, V(d.data_ptr()), fb, 1, None, f2, o),
                    "run_scattered": lib.bevk_bev_run_scattered(h, V(d.data_ptr()), fb, 1, None, f2, o, ctypes.byref(n_own)),
                }
                assert all(rc == -4 for rc in rcs.values()), (flag, rcs)
                assert "BGR frames only" in lib.bevk_last_error().decode()
        e.ctx.sync()
        assert (out.cpu().numpy() == 0xA5).all(), "a refused call wrote"
        # the Python layer
        with pytest.raises(L.BevkError, match="uint8"):
            e.run([[np.zeros((511, 640, 3), np.uint8)] * 4], pixel_format="yuyv")
        with pytest.raises(L.BevkError, match="frames must be uint8"):
            e.run_cuda(torch.zeros((1, 4, 511, 1280), dtype=torch.uint8, device="cuda"), pixel_format="uyvy")
        with pytest.raises(L.BevkError, match="c and v must be None"):
            e.run_cuda_planes(torch.zeros((1, 4, 511, 640, 2), dtype=torch.uint8, device="cuda"),
                              torch.zeros((1, 4, 255, 640), dtype=torch.uint8, device="cuda"), pixel_format="yuyv")
        with pytest.raises(L.BevkError, match="dense"):
            z = torch.zeros((1, 4, 511, 640, 4), dtype=torch.uint8, device="cuda")[..., ::2]
            e.run_cuda_planes(z, pixel_format="yuyv")
        with pytest.raises(L.BevkError, match="even frame size"):
            e.run([[np.zeros((766, 640), np.uint8)] * 4], pixel_format="nv12")
    finally:
        e.ctx.close()
    # an odd width: cv2 refuses it, and so do the Python layer and the C ABI
    eo, _ = _fixture_engine(ops, fx, 641, 512, 500, 500)
    try:
        out = torch.full((500 * 500 * 3,), 0xA5, dtype=torch.uint8, device="cuda")
        d = torch.zeros(4 << 20, dtype=torch.uint8, device="cuda")
        with pytest.raises(L.BevkError, match="even frame width"):
            eo.run([[np.zeros((512, 641, 2), np.uint8)] * 4], pixel_format="yuyv")
        for flag in (L.FLAG_YUYV, L.FLAG_UYVY):
            lib = eo.ctx.lib
            assert lib.bevk_bev_run_stack(eo.ctx.h, V(d.data_ptr()), 642 * 512 * 2, 1, None, flag, V(out.data_ptr())) == -4
            assert "even width" in lib.bevk_last_error().decode()
            a, b = ctypes.c_int64(), ctypes.c_int64()
            assert lib.bevk_bev_host_copy_bytes(eo.ctx.h, flag, ctypes.byref(a), ctypes.byref(b)) == -4
            rc = lib.bevk_bev_run_yuv_planes(eo.ctx.h, V(d.data_ptr()), 642 * 512 * 2, (ctypes.c_int64 * 3)(0, 0, 0),
                                             (ctypes.c_int64 * 3)(1284, 0, 0), 1, None, flag, V(out.data_ptr()))
            assert rc == -4
            p = (V * 4)(*[np.zeros(1, np.uint8).ctypes.data] * 4)
            assert lib.bevk_bev_run(eo.ctx.h, p, 1282, 1, None, flag, L.vptr(np.zeros((500, 500, 3), np.uint8))) == -4
        eo.ctx.sync()
        assert (out.cpu().numpy() == 0xA5).all()
    finally:
        eo.ctx.close()
