"""BEV canvases from YUV 4:2:0 frames given as separate, pitched planes on the GPU (bevk_bev_run_yuv_planes: a surface
pool at one frame stride; bevk_bev_run_yuv_surfaces: a table of plane addresses; BevEngine.run_cuda_planes).

Every YUV corpus case in both formats, laid out as decoder surfaces (tests/yuv_planes.py): pitches FW, FW + 1, FW + 16 and
a power of two; chroma directly after Y, after 8 / 16 padding rows, before Y, in a separate allocation, and (I420) U and
V apart; odd bases and frame strides; pool and scattered surfaces.  Batches 1, 3, 4, 7, 9, car on and off, BALANCE on
the 4-camera cases and every canvas format.  Each canvas is compared byte for byte with the cv2 oracle (cv2's conversion
of the frames, the BGR oracle, then cv2.cvtColor(COLOR_BGR2YUV_I420) for YUV canvases); sentinels on both sides of the
output must survive; the padding between planes holds one poison value in one call and another in the next, with the
same results.  As in test_gpu_yuv_fuzz, consecutive checked calls on one engine take frame-sets 0.. and 1.. in turn, so
that no check can pass on an earlier call's copy stack."""
import ctypes

import cv2
import numpy as np
import pytest

from tests import bev_cases as B
from tests import yuv_frames as Y
from tests import yuv_planes as P
from tests.test_gpu_bev_fuzz import Want, _engines, ops, torch  # noqa: F401  (module fixtures)
from tests.test_gpu_yuv_fuzz import BATCHES, CASES, _Pools, _render, _yuv_stack

pytestmark = pytest.mark.gpu
V = ctypes.c_void_p
LAYOUTS = [   # (pitch, chroma placement, base, extra stride bytes, scattered)
    ("dense", "after", 0, 0, False),
    ("odd", "pad8", 1, 3, False),
    ("pad16", "pad16", 0, 16, False),
    ("pow2", "before", 3, 1, False),
    ("odd", "separate", 1, 0, True),
    ("pad16", "apart", 0, 5, False),
]


def _as_out(bgr, ofmt):
    if ofmt == "bgr":
        return bgr
    i420 = cv2.cvtColor(bgr, cv2.COLOR_BGR2YUV_I420)
    return i420 if ofmt == "i420" else Y.i420_to_nv12(i420)


def _flags(L, fmt, balance, ofmt):
    return ((L.FLAG_BALANCE if balance else 0) | (L.FLAG_NV12 if fmt == "nv12" else L.FLAG_I420) |
            {"bgr": 0, "nv12": L.FLAG_OUT_NV12, "i420": L.FLAG_OUT_I420}[ofmt])


def _planes_call(torch, e, s, d_arena, frames, d_car, flags, ofmt, entry, off=16):
    """One call on frames (indices into the surfaces s, frame-set major) into a buffer with 0xA5 sentinels: `off` bytes
    before the output and a whole canvas after it.  entry: "pool" or "table".  Returns (return code, canvases or None,
    the whole buffer)."""
    n = len(frames) // e.n_cam
    shape = e._canvas_shape(n, {"bgr": 0, "nv12": 1, "i420": 1}[ofmt])
    cb = int(np.prod(shape[1:]))
    buf = torch.full((off + (n + 1) * cb,), 0xA5, dtype=torch.uint8, device=d_arena.device)
    base = d_arena.data_ptr()
    pitch = (ctypes.c_int64 * 3)(*[int(p) for p in s.pitch])
    npl = s.off.shape[1]
    if entry == "pool":
        y0 = int(s.off[frames[0], 0])
        offs = [int(s.off[frames[0], p]) - y0 for p in range(npl)] + [0] * (3 - npl)
        assert all(int(s.off[f, p]) == int(s.off[frames[0], p]) + j * s.stride for j, f in enumerate(frames) for p in range(npl))
        rc = e.ctx.lib.bevk_bev_run_yuv_planes(e.ctx.h, V(base + y0), s.stride, (ctypes.c_int64 * 3)(*offs), pitch,
                                               n, V(d_car), flags, V(buf.data_ptr() + off))
    else:
        tab = (V * (3 * len(frames)))()
        for i, f in enumerate(frames):
            for p in range(3):
                tab[3 * i + p] = base + int(s.off[f, min(p, npl - 1)])
        rc = e.ctx.lib.bevk_bev_run_yuv_surfaces(e.ctx.h, tab, pitch, n, V(d_car), flags, V(buf.data_ptr() + off))
    e.ctx.sync()
    h = buf.cpu().numpy()
    if rc != 0:
        return rc, None, h
    assert (h[:off] == 0xA5).all() and (h[off + n * cb:] == 0xA5).all(), "bytes written outside the output"
    return rc, h[off:off + n * cb].reshape(shape), h


@pytest.mark.parametrize("fmt", Y.FORMATS)
@pytest.mark.parametrize("name", CASES)
def test_yuv_planes_case_both_entry_points(ops, torch, name, fmt):
    """One YUV corpus case in one format: every surface layout through the pool and the table entry point, batches 1, 3,
    4, 7, 9, car on and off, BALANCE on the 4-camera cases, BGR and YUV canvases; the padding poisoned differently in
    alternate calls.  Then the canvases of 9 frame-sets also against the same engine's dense run_stack render."""
    from cameracalibration_b200 import _lib as L
    case = B.yuv_bgr_case(name, fmt)
    want = Want(case)
    path = "tma" if case.FW % 16 == 0 else "gather"
    balances = (False, True) if case.NC == 4 else (False,)
    outs = ("bgr", "nv12", "i420") if case.BW % 2 == 0 and case.BH % 2 == 0 else ("bgr",)
    frames = [f for fs in case.yuv for f in fs]
    car_t = torch.from_numpy(case.car).cuda()
    k, n_cmp = 0, 0
    with _engines(ops) as make:
        e = make(case)
        pick = _Pools()
        for lay in LAYOUTS:
            s = P.build(frames, fmt, *lay[:4], scatter=lay[4])
            rng = np.random.default_rng(s.arena.size)
            d = [torch.from_numpy(s.poisoned(v)).cuda() for v in (0xA5, rng.integers(0, 256, int(s.pad.sum()), dtype=np.uint8))]
            first = None
            for n in BATCHES:
                for balance in balances:
                    car = k % 2 == 1
                    ofmt = outs[k % len(outs)]
                    entry = "table" if s.stride is None or k % 3 == 2 else "pool"
                    sets = pick(n)
                    idx = [si * case.NC + c for si in sets for c in range(case.NC)]
                    flags = _flags(L, fmt, balance, ofmt)
                    rc, got, _ = _planes_call(torch, e, s, d[k % 2], idx, car_t.data_ptr() if car else 0, flags, ofmt, entry)
                    assert rc == 0, (lay, entry, L.load().bevk_last_error())
                    assert e.last_path() == path, (lay, entry, n)
                    for i, si in enumerate(sets):
                        w = want(si, balance, car)
                        if w is not None:
                            assert (got[i] == _as_out(w, ofmt)).all(), (name, fmt, lay, entry, n, balance, car, ofmt, si)
                            n_cmp += 1
                    if first is None:   # the same call with the other poison in the padding
                        rc2, again, _ = _planes_call(torch, e, s, d[(k + 1) % 2], idx, car_t.data_ptr() if car else 0, flags,
                                                     ofmt, entry)
                        assert rc2 == 0 and (again == got).all(), (lay, "padding reached the canvas")
                        first = True
                    k += 1
        # the dense run_stack render of the same 9 frame-sets, with the car
        s = P.build(frames, fmt, "pow2", "pad8", 1, 3)
        d = torch.from_numpy(s.arena).cuda()
        for balance in balances:
            sets = pick(9)
            idx = [si * case.NC + c for si in sets for c in range(case.NC)]
            _, got, _ = _planes_call(torch, e, s, d, idx, car_t.data_ptr(), _flags(L, fmt, balance, "bgr"), "bgr", "pool")
            dd, base, stride = _yuv_stack(torch, case, sets, True)
            ref = _render(torch, e, dd, stride, 9, case.car, balance, pixel_format=fmt, base=base)
            assert (got == ref).all(), (name, fmt, balance, int((got != ref).sum()))
    assert n_cmp > 0
    print(f"{name} {fmt}: {n_cmp} canvases compared")


def _fixture_engine(ops, fx, FW, FH):
    from tests.test_gpu_tma import _engine
    g = fx.geometry(FW, FH, 1000, 1000)
    e, _ = _engine(ops, fx, g, True)
    return e, g


@pytest.mark.parametrize("fmt", Y.FORMATS)
def test_run_cuda_planes_on_a_decoder_pool_and_on_tensor_lists(ops, torch, fx, fmt):
    """run_cuda_planes at 1920 x 1080 on torch views of one uint8[B*4][1088 + 544][2048] surface pool (NV12: the UV rows
    after the 1088-row coded height; I420: U and V side by side in those rows) and on lists of separate tensors per
    plane: the same canvases as run_cuda on the dense frames, with BALANCE and the car, BGR and NV12 canvases."""
    e, g = _fixture_engine(ops, fx, 1920, 1080)
    try:
        bgr = fx.frames(1920, 1080)
        B_, nc = 3, 4
        dense = np.stack([np.stack([Y.from_bgr(np.roll(f, 31 * b, axis=1), fmt) for f in bgr]) for b in range(B_)])
        d_dense = torch.from_numpy(dense).cuda()
        car = torch.from_numpy(fx.car(1000, 1000)).cuda()
        pool = torch.full((B_ * nc, 1088 + 544, 2048), 0xA5, dtype=torch.uint8, device="cuda").view(B_, nc, 1632, 2048)
        planes = [P.split(dense[b, c], fmt) for b in range(B_) for c in range(nc)]
        y = pool[:, :, :1080, :1920]
        y.copy_(torch.from_numpy(np.stack([p[0] for p in planes]).reshape(B_, nc, 1080, 1920)))
        if fmt == "nv12":
            views = [y, pool[:, :, 1088:1088 + 540, :1920]]
        else:
            views = [y, pool[:, :, 1088:1088 + 540, :960], pool[:, :, 1088:1088 + 540, 1024:1024 + 960]]
        for k in range(1, len(views)):
            views[k].copy_(torch.from_numpy(np.stack([p[k] for p in planes]).reshape(views[k].shape)))
        sep = [[tuple(torch.from_numpy(np.ascontiguousarray(p)).cuda() for p in planes[b * nc + c]) for c in range(nc)]
               for b in range(B_)]
        for ofmt in ("bgr", "nv12"):
            ref = e.run_cuda(d_dense, car, True, pixel_format=fmt, out_format=ofmt)
            torch.cuda.synchronize()
            ref = ref.cpu().numpy()
            got = e.run_cuda_planes(*views, pixel_format=fmt, car=car, balance=True, out_format=ofmt)
            torch.cuda.synchronize()
            assert e.last_path() == "tma"
            assert (got.cpu().numpy() == ref).all(), (fmt, ofmt, "pool")
            got = e.run_cuda_planes(sep, pixel_format=fmt, car=car, balance=True, out_format=ofmt)
            torch.cuda.synchronize()
            assert (got.cpu().numpy() == ref).all(), (fmt, ofmt, "tensor lists")
        # the dense render itself against the BGR render of the cvtColor frames
        d_bgr = torch.from_numpy(np.stack([np.stack([Y.to_bgr(f, fmt) for f in fs]) for fs in dense])).cuda()
        want = e.run_cuda(d_bgr, car, True).cpu().numpy()
        got = e.run_cuda_planes(*views, pixel_format=fmt, car=car, balance=True)
        torch.cuda.synchronize()
        assert (got.cpu().numpy() == want).all(), fmt
    finally:
        e.ctx.close()


@pytest.mark.parametrize("fmt", Y.FORMATS)
def test_graph_replay_of_planes_calls(ops, torch, fx, fmt):
    """A graph captured from a pool call renders what the surfaces hold at replay: new contents written into the same
    surfaces are rendered.  A table call captured after an eager call with the same table needs no upload inside the
    capture; a later call with another table renders the other surfaces."""
    from cameracalibration_b200 import _lib as L
    e, g = _fixture_engine(ops, fx, 640, 512)
    try:
        bgr = fx.frames(640, 512)
        fa = [Y.from_bgr(f, fmt) for f in bgr]
        fb = [Y.from_bgr(np.roll(f, 57, axis=0), fmt) for f in bgr]
        sa, sb = P.build(fa, fmt, "pow2", "pad8", 1, 3), P.build(fb, fmt, "pow2", "pad8", 1, 3)
        sc = P.build(fb, fmt, "odd", "separate", 0, 0, scatter=True)
        d_a, d_b, d_c = (torch.from_numpy(s.arena).cuda() for s in (sa, sb, sc))
        flags = _flags(L, fmt, True, "bgr")
        idx = list(range(4))
        _, want_a, _ = _planes_call(torch, e, sa, d_a, idx, 0, flags, "bgr", "pool")
        _, want_b, _ = _planes_call(torch, e, sb, d_b, idx, 0, flags, "bgr", "pool")
        assert (want_a != want_b).any()
        for entry, s in (("pool", sa), ("table", sa)):
            d_run = torch.from_numpy(sa.arena).cuda()
            _planes_call(torch, e, s, d_run, idx, 0, flags, "bgr", entry)   # eager: every buffer (and the table) exists
            out = torch.zeros((1, 1000, 1000, 3), dtype=torch.uint8, device="cuda")
            pitch = (ctypes.c_int64 * 3)(*[int(p) for p in s.pitch])
            base = d_run.data_ptr()
            torch.cuda.synchronize()
            with e.ctx.graph_capture() as gr:
                if entry == "pool":
                    y0, stride, offs = s.pool()
                    L.check(e.ctx.lib.bevk_bev_run_yuv_planes(e.ctx.h, V(base + y0), stride, (ctypes.c_int64 * 3)(*offs), pitch, 1,
                                                              None, flags, V(out.data_ptr())))
                else:
                    tab = (V * 12)(*[base + int(s.off[i, min(p, s.off.shape[1] - 1)]) for i in range(4) for p in range(3)])
                    L.check(e.ctx.lib.bevk_bev_run_yuv_surfaces(e.ctx.h, tab, pitch, 1, None, flags, V(out.data_ptr())))
            try:
                gr.launch()
                e.ctx.sync()
                assert (out.cpu().numpy() == want_a).all(), (entry, "replay")
                d_run.copy_(torch.from_numpy(sb.arena).cuda())   # new surface contents at the same addresses
                torch.cuda.synchronize()
                gr.launch()
                e.ctx.sync()
                assert (out.cpu().numpy() == want_b).all(), (entry, "replay after new contents")
            finally:
                gr.destroy()
        _, got, _ = _planes_call(torch, e, sc, d_c, idx, 0, flags, "bgr", "table")   # another table: uploaded again
        assert (got == want_b).all()
    finally:
        e.ctx.close()


def test_refusals(ops, torch, fx):
    """Refused with a message and nothing written: no YUV flag or both, a pitch below its plane's row bytes (each plane),
    a null plane, batch x cameras over 65535, odd frame sizes."""
    from cameracalibration_b200 import _lib as L
    e, g = _fixture_engine(ops, fx, 640, 512)
    lib, h = e.ctx.lib, e.ctx.h
    try:
        d = torch.full((4 << 20,), 7, dtype=torch.uint8, device="cuda")
        out = torch.full((1000 * 1000 * 3 + 64,), 0xA5, dtype=torch.uint8, device="cuda")
        o = V(out.data_ptr())
        I64 = ctypes.c_int64 * 3
        fs = 640 * 512 * 3 // 2
        nv12 = (I64(0, 640 * 512, 0), I64(640, 640, 0))
        i420 = (I64(0, 640 * 512, 640 * 512 * 5 // 4), I64(640, 320, 320))
        tab = (V * 12)(*[d.data_ptr() + i * fs + q for i in range(4) for q in (0, 640 * 512, 640 * 512 * 5 // 4)])

        def pool(flags, offs, pitch, batch=1, base=d.data_ptr()):
            return lib.bevk_bev_run_yuv_planes(h, V(base), fs, offs, pitch, batch, None, flags, o)

        def table(flags, pitch, t=tab, batch=1):
            return lib.bevk_bev_run_yuv_surfaces(h, t, pitch, batch, None, flags, o)

        assert pool(0, *nv12) == -1 and table(0, nv12[1]) == -1
        assert pool(L.FLAG_BALANCE, *nv12) == -1
        both = L.FLAG_NV12 | L.FLAG_I420
        assert pool(both, *nv12) == -1 and table(both, nv12[1]) == -1
        for p in range(2):
            bad = I64(*nv12[1]); bad[p] -= 1
            assert pool(L.FLAG_NV12, nv12[0], bad) == -1 and table(L.FLAG_NV12, bad) == -1, p
        for p in range(3):
            bad = I64(*i420[1]); bad[p] -= 1
            assert pool(L.FLAG_I420, i420[0], bad) == -1 and table(L.FLAG_I420, bad) == -1, p
        assert pool(L.FLAG_NV12, *nv12, base=0) == -1
        for p in range(3):
            t = (V * 12)(*tab); t[3 * 2 + p] = None
            assert table(L.FLAG_I420, i420[1], t) == -1, p
        assert pool(L.FLAG_NV12, *nv12, batch=16384) == -1 and table(L.FLAG_NV12, nv12[1], batch=16384) == -1
        assert "65535" in lib.bevk_last_error().decode()
        assert lib.bevk_bev_run_yuv_planes(h, V(d.data_ptr()), fs, None, nv12[1], 1, None, L.FLAG_NV12, o) == -1
        assert lib.bevk_bev_run_yuv_surfaces(h, None, nv12[1], 1, None, L.FLAG_NV12, o) == -1
        e.ctx.sync()
        assert (out.cpu().numpy() == 0xA5).all(), "a refused call wrote"
        t = (V * 12)(*tab); t[3 * 2 + 2] = None   # NV12 does not read plane 2
        assert table(L.FLAG_NV12, nv12[1], t) == 0
        e.ctx.sync()
    finally:
        e.ctx.close()
    eo, _ = _fixture_engine(ops, fx, 641, 512)
    try:
        out = torch.full((1000 * 1000 * 3,), 0xA5, dtype=torch.uint8, device="cuda")
        d = torch.zeros(4 << 20, dtype=torch.uint8, device="cuda")
        for flag in (L.FLAG_NV12, L.FLAG_I420):
            rc = eo.ctx.lib.bevk_bev_run_yuv_planes(eo.ctx.h, V(d.data_ptr()), 642 * 512 * 2, (ctypes.c_int64 * 3)(0, 642 * 512, 642 * 640),
                                                    (ctypes.c_int64 * 3)(642, 642, 642), 1, None, flag, V(out.data_ptr()))
            assert rc == -4 and "even" in eo.ctx.lib.bevk_last_error().decode(), flag
        eo.ctx.sync()
        assert (out.cpu().numpy() == 0xA5).all()
    finally:
        eo.ctx.close()
