"""YUV 4:2:0 canvases (out_format "nv12" / "i420", BEVK_FLAG_OUT_NV12 / _I420) on the GPU.  Every YUV canvas must equal,
byte for byte, Y.from_bgr(want, fmt) -- cv2.cvtColor(want, COLOR_BGR2YUV_I420), NV12 with its U and V planes
interleaved -- where `want` is the cv2 oracle's canvas, and the same conversion of the engine's own BGR canvas of the
same call without the output format."""
import ctypes

import numpy as np
import pytest

from tests import bev_cases as B
from tests import yuv_frames as Y
from tests.test_gpu_bev_fuzz import Want, _engines, _stack, ops, torch  # noqa: F401  (module fixtures)
from tests.test_gpu_graph_frames import _replay_after_other_stack
from tests.test_gpu_tma import _engine
from tests.test_gpu_yuv import _oracle, _sets

pytestmark = pytest.mark.gpu
IN_FORMATS = ("bgr",) + Y.FORMATS


def _yuv(canvases, fmt):
    """Y.from_bgr of every canvas of a batch."""
    return np.stack([Y.from_bgr(np.ascontiguousarray(c), fmt) for c in canvases])


def _inputs(fx, g, n, in_fmt):
    """n frame-sets in format in_fmt and the BGR frames the oracle sees (cvtColor of the YUV ones)."""
    if in_fmt == "bgr":
        bgr = [fx.frames(g.FW, g.FH)] + [fx.perturbed_frames(g.FW, g.FH, i) for i in range(1, n)]
        return bgr, bgr
    return _sets(fx, g, n, in_fmt)


def _pinned(sets):
    from cameracalibration_b200 import _lib as L
    out = []
    for s in sets:
        out.append([])
        for f in s:
            p = L.pinned_empty(f.shape)
            p[...] = f
            out[-1].append(p)
    return out


@pytest.mark.parametrize("blend", [False, True])
def test_fixture_geometry_host_frames(ops, fx, blend):
    """1280x1024 -> 1000^2 with the reference's calibration, plain and blend: BGR, NV12 and I420 frames, BALANCE on and
    off, car on and off, NV12 and I420 canvases, pageable and page-locked host frames (2 frame-sets).  host_copy_bytes
    reports 1.5 bytes per canvas pixel coming back, and the upload is that of the BGR-out call."""
    g = fx.geometry()
    e, masks = _engine(ops, fx, g, blend, calib=fx.calib)
    car = fx.car()
    n_cmp = 0
    for in_fmt in IN_FORMATS:
        frames, bgr = _inputs(fx, g, 2, in_fmt)
        pinned = _pinned(frames)
        for balance in (False, True):
            for c in (None, car):
                want = [_oracle(fx.calib, g, masks, blend, balance, s, c) for s in bgr]
                own = np.array(e.run(frames, c, balance, pixel_format=in_fmt))
                for out_fmt in Y.FORMATS:
                    for what, src in (("pageable", frames), ("page-locked", pinned)):
                        got = e.run(src, c, balance, pixel_format=in_fmt, out_format=out_fmt)
                        assert got.shape == (2, g.BH * 3 // 2, g.BW)
                        assert e.last_path() == "tma"
                        assert (got == _yuv(own, out_fmt)).all(), (in_fmt, out_fmt, what, balance, c is not None)
                        for b in range(2):
                            w = Y.from_bgr(want[b], out_fmt)
                            assert (got[b] == w).all(), (in_fmt, out_fmt, what, balance, c is not None, b, int((got[b] != w).sum()))
                            n_cmp += 1
                        if what == "pageable" and not balance:
                            assert e.last_h2d_bytes() == 2 * e.host_copy_bytes(False, in_fmt, out_fmt)[0]
                    up, down = e.host_copy_bytes(balance, in_fmt, out_fmt)
                    assert down == g.BW * g.BH * 3 // 2
                    assert (up, 2 * down) == e.host_copy_bytes(balance, in_fmt)
    assert n_cmp == 3 * 2 * 2 * 2 * 2 * 2


def test_device_entry_points(ops, fx, torch):
    """run_device (a device table), run_cuda on per-frame tensors (run_frames, a table that is no stack: k_bev) and on
    one [batch][4][FH][FW][3] tensor (run_frames on a stack), run_stack on BGR and NV12 stacks, with BALANCE on and off
    and the car; and through the raw ABI into outputs at byte offsets 1, 2 and 3, whose sentinels stay untouched."""
    from cameracalibration_b200 import _lib as L
    g = fx.geometry()
    e, masks = _engine(ops, fx, g, True, calib=fx.calib)
    dev = torch.device("cuda", e.ctx.device)
    n = 3
    frames, _ = _inputs(fx, g, n, "bgr")
    car = fx.car()
    d_car = torch.from_numpy(car).to(dev)
    d5 = torch.from_numpy(np.stack([np.stack(s) for s in frames])).to(dev)
    views = [[torch.from_numpy(f).to(dev) for f in s] for s in frames]
    table = torch.tensor([t.data_ptr() for s in views for t in s], dtype=torch.int64, device=dev)
    nv12 = torch.from_numpy(np.stack([np.stack([Y.from_bgr(f, "nv12") for f in s]) for s in frames])).to(dev)
    nv12_bgr = [[Y.to_bgr(Y.from_bgr(f, "nv12"), "nv12") for f in s] for s in frames]
    yb = g.BW * g.BH * 3 // 2
    for balance in (False, True):
        want = [_oracle(fx.calib, g, masks, True, balance, s, car) for s in frames]
        want_nv12_in = [_oracle(fx.calib, g, masks, True, balance, s, car) for s in nv12_bgr]
        for out_fmt in Y.FORMATS:
            flags = (L.FLAG_BALANCE if balance else 0) | L.OUT_FORMATS[out_fmt]
            wy = np.stack([Y.from_bgr(w, out_fmt) for w in want])
            got = {}
            out = torch.empty((n, g.BH * 3 // 2, g.BW), dtype=torch.uint8, device=dev)
            e.run_device(table.data_ptr(), n, out.data_ptr(), d_car.data_ptr(), balance, out_format=out_fmt)
            e.ctx.sync()
            got["run_device"] = out.cpu().numpy()
            got["run_cuda lists"] = e.run_cuda(views, d_car, balance, out_format=out_fmt).cpu().numpy()
            got["run_cuda tensor"] = e.run_cuda(d5, d_car, balance, out_format=out_fmt).cpu().numpy()
            assert e.last_path() == "tma"
            out = torch.empty((n, g.BH * 3 // 2, g.BW), dtype=torch.uint8, device=dev)
            e.run_stack(d5.data_ptr(), g.FW * g.FH * 3, n, out.data_ptr(), d_car.data_ptr(), balance, out_format=out_fmt)
            e.ctx.sync()
            got["run_stack"] = out.cpu().numpy()
            for off in (1, 2, 3):
                buf = torch.full((n * yb + 8,), 0xA5, dtype=torch.uint8, device=dev)
                rc = e.ctx.lib.bevk_bev_run_stack(e.ctx.h, ctypes.c_void_p(d5.data_ptr()), g.FW * g.FH * 3, n,
                                                  ctypes.c_void_p(d_car.data_ptr()), flags, ctypes.c_void_p(buf.data_ptr() + off))
                assert rc == 0, L.load().bevk_last_error()
                e.ctx.sync()
                h = buf.cpu().numpy()
                assert (h[:off] == 0xA5).all() and (h[off + n * yb:] == 0xA5).all(), off
                got[f"run_stack out + {off}"] = h[off:off + n * yb].reshape(n, g.BH * 3 // 2, g.BW)
            torch.cuda.synchronize()
            for what, x in got.items():
                assert (x == wy).all(), (what, out_fmt, balance, int((x != wy).sum()))
            # NV12 frames in, YUV canvases out
            x = e.run_cuda(nv12, d_car, balance, pixel_format="nv12", out_format=out_fmt).cpu().numpy()
            w = np.stack([Y.from_bgr(w, out_fmt) for w in want_nv12_in])
            assert (x == w).all(), ("nv12 in", out_fmt, balance)


def test_cfg4_batch_of_32_device(ops, fx, torch):
    """cfg4 (1920x1080 -> 1000^2, blend), 32 frame-sets as one device array, BGR and NV12 frames: the YUV canvases equal
    the conversion of the BGR canvases of the same frames, and the oracle at three frame-sets."""
    g = fx.geometry(1920, 1080, 1000, 1000)
    e, masks = _engine(ops, fx, g, True)
    calib = fx.scaled_calib(g)
    dev = torch.device("cuda", e.ctx.device)
    for in_fmt in ("bgr", "nv12"):
        frames, bgr = _inputs(fx, g, 32, in_fmt)
        d = torch.from_numpy(np.stack([np.stack(s) for s in frames])).to(dev)
        own = e.run_cuda(d, pixel_format=in_fmt).cpu().numpy()
        for out_fmt in Y.FORMATS:
            got = e.run_cuda(d, pixel_format=in_fmt, out_format=out_fmt)
            assert e.last_path() == "tma"
            got = got.cpu().numpy()
            assert (got == _yuv(own, out_fmt)).all(), (in_fmt, out_fmt)
            for b in (0, 13, 31):
                assert (got[b] == Y.from_bgr(_oracle(calib, g, masks, True, False, bgr[b]), out_fmt)).all(), (in_fmt, out_fmt, b)


def test_cfg3_balance_car_device_and_host(ops, fx, torch):
    """cfg3 (1920x1080 -> 1200^2, blend + BALANCE + car): a device stack and page-locked NV12 host frames."""
    g = fx.geometry(1920, 1080, 1200, 1200)
    e, masks = _engine(ops, fx, g, True)
    calib = fx.scaled_calib(g)
    car = fx.car(1200, 1200)
    dev = torch.device("cuda", e.ctx.device)
    frames, bgr = _inputs(fx, g, 2, "bgr")
    nv12, nv12_bgr = _inputs(fx, g, 2, "nv12")
    want = [_oracle(calib, g, masks, True, True, s, car) for s in bgr]
    want_nv12 = [_oracle(calib, g, masks, True, True, s, car) for s in nv12_bgr]
    d = torch.from_numpy(np.stack([np.stack(s) for s in frames])).to(dev)
    d_car = torch.from_numpy(car).to(dev)
    pinned = _pinned(nv12)
    for out_fmt in Y.FORMATS:
        out = torch.empty((2, 1800, 1200), dtype=torch.uint8, device=dev)
        e.run_stack(d.data_ptr(), 1920 * 1080 * 3, 2, out.data_ptr(), d_car.data_ptr(), True, out_format=out_fmt)
        e.ctx.sync()
        got = out.cpu().numpy()
        got_h = e.run(pinned, car, True, pixel_format="nv12", out_format=out_fmt)
        for b in range(2):
            assert (got[b] == Y.from_bgr(want[b], out_fmt)).all(), (out_fmt, "device", b)
            assert (got_h[b] == Y.from_bgr(want_nv12[b], out_fmt)).all(), (out_fmt, "host nv12", b)


@pytest.mark.parametrize("seed", range(B.N_CASES))
def test_fuzz_corpus_case(ops, torch, seed):
    """Every case of the fuzz corpus: an even canvas (BW % 4 == 0 and == 2, BW % 16 != 0) renders NV12 and I420
    canvases through run_stack (batches 1, 4 and 9, car on and off, BALANCE on the 4-camera cases) and run (pageable,
    4 frame-sets) that equal the conversion of the oracle canvases and of the same engine's BGR canvases; an odd canvas
    is refused by the Python layer and by the C ABI."""
    from cameracalibration_b200 import _lib as L
    case = B.make_case(seed)
    want = Want(case)
    balances = (False, True) if case.NC == 4 else (False,)
    with _engines(ops) as make:
        e = make(case)
        d, stride = _stack(torch, case, 9, True)
        if case.BW % 2 or case.BH % 2:
            with pytest.raises(L.BevkError, match="even"):
                e.run_stack(d.data_ptr(), stride, 1, d.data_ptr(), out_format="nv12")
            out = torch.empty(case.BW * case.BH * 3, dtype=torch.uint8, device=d.device)
            for flag in (L.FLAG_OUT_NV12, L.FLAG_OUT_I420):
                assert e.ctx.lib.bevk_bev_run_stack(e.ctx.h, ctypes.c_void_p(d.data_ptr()), stride, 1, None, flag,
                                                    ctypes.c_void_p(out.data_ptr())) == -4
            return
        d_car = torch.from_numpy(case.car).cuda()
        n_cmp = 0
        for balance in balances:
            for n in (1, 4, 9):
                for car in (False, True):
                    cp = d_car.data_ptr() if car else 0
                    own = torch.empty((n, case.BH, case.BW, 3), dtype=torch.uint8, device=d.device)
                    e.run_stack(d.data_ptr(), stride, n, own.data_ptr(), cp, balance)
                    for out_fmt in Y.FORMATS:
                        out = torch.empty((n, case.BH * 3 // 2, case.BW), dtype=torch.uint8, device=d.device)
                        e.run_stack(d.data_ptr(), stride, n, out.data_ptr(), cp, balance, out_format=out_fmt)
                        e.ctx.sync()
                        got, mine = out.cpu().numpy(), own.cpu().numpy()
                        assert (got == _yuv(mine, out_fmt)).all(), (case.name, out_fmt, n, balance, car)
                        for s in range(n):
                            w = want(s, balance, car)
                            if w is not None:
                                assert (got[s] == Y.from_bgr(w, out_fmt)).all(), (case.name, out_fmt, n, balance, car, s)
                                n_cmp += 1
            for out_fmt in Y.FORMATS:
                got = e.run(case.sets[:4], case.car, balance, out_format=out_fmt)
                for s in range(4):
                    w = want(s, balance, True)
                    if w is not None:
                        assert (got[s] == Y.from_bgr(w, out_fmt)).all(), (case.name, "run", out_fmt, balance, s)
                        n_cmp += 1
        assert n_cmp > 0
    print(f"{case.name} {case.BW}x{case.BH}: {n_cmp} canvases compared")


def test_fuzz_corpus_has_the_widths_that_pick_a_path():
    """The even canvases of the corpus include BW % 4 == 2 (the byte path) and BW % 4 == 0 (the word path)."""
    even = [c for c in (B.make_case(s) for s in range(B.N_CASES)) if c.BW % 2 == 0 and c.BH % 2 == 0]
    assert {c.BW % 4 for c in even} == {0, 2} and any(c.BW % 16 for c in even)


@pytest.mark.parametrize("balance", [False, True])
def test_graph_replay_of_yuv_canvases(ops, fx, torch, balance):
    """Capture run_stack with an output format on stack A, make an eager call on stack B, replay: A's canvases."""
    g = fx.geometry()
    e, _ = _engine(ops, fx, g, True, calib=fx.calib)
    dev = torch.device("cuda", e.ctx.device)
    n = 3
    car = torch.from_numpy(fx.car()).to(dev)
    frames, _ = _inputs(fx, g, n, "bgr")
    a = np.stack([np.stack(s) for s in frames])
    d_a, d_b = torch.from_numpy(a).to(dev), torch.from_numpy(np.ascontiguousarray(a[::-1]) ^ 0x21).to(dev)
    for out_fmt in Y.FORMATS:
        def call(d, out):
            e.run_stack(d.data_ptr(), g.FW * g.FH * 3, n, out.data_ptr(), car.data_ptr(), balance, out_format=out_fmt)

        want_a, want_b, got = _replay_after_other_stack(torch, e, call, d_a, d_b, (n, g.BH * 3 // 2, g.BW))
        assert (want_a == _yuv(e.run(frames, fx.car(), balance), out_fmt)).all()
        assert (got == want_a).all(), (out_fmt, int((got != want_a).sum()), bool((got == want_b).all()))


def test_alternating_bgr_and_yuv_canvases(ops, fx):
    """One engine, calls alternating between BGR, NV12 and I420 canvases, BALANCE off and on, each checked against the
    oracle: no call depends on state an earlier call in another format left."""
    g = fx.geometry()
    e, masks = _engine(ops, fx, g, True, calib=fx.calib)
    car = fx.car()
    frames, _ = _inputs(fx, g, 3, "bgr")
    want = {b: [_oracle(fx.calib, g, masks, True, b, s, car) for s in frames] for b in (False, True)}
    for out_fmt, balance, sets in (("bgr", False, [0, 1]), ("nv12", True, [2, 0]), ("bgr", True, [1, 2]),
                                   ("i420", False, [0, 2]), ("nv12", False, [1, 0]), ("bgr", False, [2, 1]),
                                   ("i420", True, [1, 2]), ("bgr", True, [0, 1])):
        got = e.run([frames[s] for s in sets], car, balance, out_format=out_fmt)
        for i, s in enumerate(sets):
            w = want[balance][s] if out_fmt == "bgr" else Y.from_bgr(want[balance][s], out_fmt)
            assert (got[i] == w).all(), (out_fmt, balance, s)


def test_bevgenerator_out_format(fx):
    """BevGenerator.run_batch and run_cuda with out_format (blend, BALANCE, car) at the fixture geometry."""
    import torch
    from cameracalibration_b200.SurroundBirdEyeView import surroundBEV as S
    from oracle import restate as R
    from tests.helpers import NAMES
    g = fx.geometry()
    bev = S.BevGenerator(blend=True, balance=True, calib=fx.calib)
    masks = [R.blend_mask(n, g.BW, g.BH, g.CW, g.CH) for n in NAMES]
    car = fx.car()
    frames, _ = _inputs(fx, g, 2, "bgr")
    want = [_oracle(fx.calib, g, masks, True, True, s, car) for s in frames]
    for out_fmt in Y.FORMATS:
        got = bev.run_batch(frames, car, out_format=out_fmt)
        d = torch.from_numpy(np.stack([np.stack(s) for s in frames])).cuda()
        got_d = bev.run_cuda(d, torch.from_numpy(car).cuda(), out_format=out_fmt).cpu().numpy()
        for b in range(2):
            w = Y.from_bgr(want[b], out_fmt)
            assert (got[b] == w).all() and (got_d[b] == w).all(), (out_fmt, b)


def test_refusals(ops, fx, torch):
    from cameracalibration_b200 import _lib as L
    g = fx.geometry(640, 512, 500, 500)
    e, _ = _engine(ops, fx, g, False)
    dev = torch.device("cuda", e.ctx.device)
    frames = fx.frames(640, 512)
    with pytest.raises(L.BevkError, match="out_format"):
        e.run([frames], out_format="yuyv")
    lib, h, V = e.ctx.lib, e.ctx.h, ctypes.c_void_p
    d = torch.zeros((4, 512, 640, 3), dtype=torch.uint8, device=dev)
    out = torch.zeros((1, 500, 500, 3), dtype=torch.uint8, device=dev)
    both = L.FLAG_OUT_NV12 | L.FLAG_OUT_I420
    hp = (V * 4)(*[f.ctypes.data for f in frames])
    table = (V * 4)(*[d[i].data_ptr() for i in range(4)])
    a, b = ctypes.c_int64(), ctypes.c_int64()
    # both output flags: an argument error on every entry point that takes them
    assert lib.bevk_bev_run_stack(h, V(d.data_ptr()), 640 * 512 * 3, 1, None, both, V(out.data_ptr())) == -1
    assert lib.bevk_bev_run_frames(h, table, 1, None, both, V(out.data_ptr())) == -1
    assert lib.bevk_bev_run(h, hp, 640 * 3, 1, None, both, L.vptr(np.zeros((500, 500, 3), np.uint8))) == -1
    assert lib.bevk_bev_host_copy_bytes(h, both, ctypes.byref(a), ctypes.byref(b)) == -1
    assert "exclusive" in lib.bevk_last_error().decode()
    # every entry point with flags other than run / run_device / run_frames / run_stack / host_copy_bytes refuses them
    sizes = (ctypes.c_uint64 * 4)(1, 1, 1, 1)
    streams = np.zeros(1 << 16, np.uint8)
    ssz = (ctypes.c_uint64 * 1)()
    n_own = ctypes.c_int()
    for flag in (L.FLAG_OUT_NV12, L.FLAG_OUT_I420, L.FLAG_OUT_NV12 | L.FLAG_BALANCE):
        rcs = {
            "run_jpeg": lib.bevk_bev_run_jpeg(h, hp, sizes, 1, None, flag, L.vptr(streams)),
            "run_to_jpeg": lib.bevk_bev_run_to_jpeg(h, hp, 640 * 3, 1, None, flag, 95, L.vptr(streams), streams.size, ssz),
            "frames_to_jpeg": lib.bevk_bev_frames_to_jpeg(h, table, 1, None, flag, 95, L.vptr(streams), streams.size, ssz),
            "run_sharded": lib.bevk_bev_run_sharded(h, V(d.data_ptr()), 640 * 512 * 3, 1, None, flag, V(out.data_ptr())),
            "run_scattered": lib.bevk_bev_run_scattered(h, V(d.data_ptr()), 640 * 512 * 3, 1, None, flag, V(out.data_ptr()),
                                                        ctypes.byref(n_own)),
        }
        assert all(rc == -4 for rc in rcs.values()), (flag, rcs)
        assert "BGR canvases only" in lib.bevk_last_error().decode()
    e.ctx.sync()
    # odd canvases: cv2 refuses them, and so do the Python layer and the C ABI
    go = fx.geometry(640, 512, 501, 500)
    eo, _ = _engine(ops, fx, go, False)
    with pytest.raises(L.BevkError, match="even"):
        eo.run([frames], out_format="nv12")
    with pytest.raises(L.BevkError, match="even"):
        eo.host_copy_bytes(out_format="i420")
    for flag in (L.FLAG_OUT_NV12, L.FLAG_OUT_I420):
        assert lib.bevk_bev_run_stack(eo.ctx.h, V(d.data_ptr()), 640 * 512 * 3, 1, None, flag, V(out.data_ptr())) == -4
        assert lib.bevk_bev_run_device(eo.ctx.h, V(d.data_ptr()), 1, None, flag, V(out.data_ptr())) == -4
        assert lib.bevk_bev_run_frames(eo.ctx.h, table, 1, None, flag, V(out.data_ptr())) == -4
        assert lib.bevk_bev_host_copy_bytes(eo.ctx.h, flag, ctypes.byref(a), ctypes.byref(b)) == -4
        assert lib.bevk_bev_run(eo.ctx.h, hp, 640 * 3, 1, None, flag, L.vptr(np.zeros((500, 501, 3), np.uint8))) == -4
