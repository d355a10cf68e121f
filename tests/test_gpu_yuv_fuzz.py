"""GPU fuzz of the NV12 / I420 render on the YUV corpus of tests/bev_cases.py (yuv_corpus: the even-sized fuzz corpus
cases and a supplement with FW % 4 == 2, FW % 16 != 0, FW % 32 == 16, FH % 4 == 2, 1-8 cameras, int16-extreme and edge
taps, bright frames): k_vsum_yuv, k_yuv_spans, the page-locked windows (k_fetch_yuv) and the pageable DMA rectangles,
then k_bev_tma or k_bev on the converted copy stack.  Every case runs in both formats through run_stack (dense, and at
an odd base and odd stride), run_cuda, and run on pageable, page-locked and row-padded host frames.  Each canvas is
compared byte for byte with the cv2 / NumPy oracle of cv2.cvtColor of every frame; the run_stack canvases of 9 frame-sets
also with the same engine's BGR render of the cvtColor frames.  Every render must have run k_bev_tma exactly when the
copy stack's pitch is 16-byte friendly (FW % 16 == 0).

The YUV pre-pass writes only the sampled spans into the copy stack, which every call of a context shares; the rest keeps
an earlier call's bytes.  So that no check can pass by reading an earlier call's conversion, consecutive checked calls on
one engine take frame-sets 0.. and 1.. in turn (no frame-set returns at the frame index the previous call gave it), and
a call in the other YUV format and a BGR BALANCE call, on the frame-sets in reverse order, overwrite the copy stack in
between.  tests/test_host_yuv.py pins the same rule on the CPU."""
import numpy as np
import pytest

from oracle import restate as R
from tests import bev_cases as B
from tests import yuv_frames as Y
from tests.helpers import NAMES
from tests.test_gpu_bev_fuzz import Want, _engines, _env, _render, ops, torch  # noqa: F401  (module fixtures)

pytestmark = pytest.mark.gpu
BATCHES = (1, 3, 4, 7, 9)   # NB=1; NB=4 whole; NB=4 with tails of 3 and 1
CASES = [c.name for c in B.yuv_corpus()]


class _Pools:
    """Frame-sets of the checked calls on one engine: 0..n-1, then 1..n, in turn."""

    def __init__(self):
        self.calls = 0

    def __call__(self, n):
        s = self.calls % 2
        self.calls += 1
        return list(range(s, s + n))


def _yuv_stack(torch, case, order, odd):
    """The YUV frame-sets `order` as one device stack: dense, or at byte 1 of the buffer with a frame stride of frame
    bytes + 3 (odd) and 0xFF padding.  Returns (buffer, byte offset of the first frame, stride)."""
    fb = case.FW * case.FH * 3 // 2
    stride, base = (fb + 3, 1) if odd else (fb, 0)
    host = np.full(base + len(order) * case.NC * stride, 0xFF, np.uint8)
    for i, f in enumerate(f for s in order for f in case.yuv[s]):
        host[base + i * stride:base + i * stride + fb] = f.reshape(-1)
    return torch.from_numpy(host).cuda(), base, stride


def _bgr_stack(torch, case, order):
    """The BGR frame-sets `order` of a case as one device stack at a 16-byte stride."""
    fb = case.FW * case.FH * 3
    stride = (fb + 15) // 16 * 16
    host = np.zeros((len(order) * case.NC, stride), np.uint8)
    host[:, :fb] = np.stack([f.reshape(-1) for s in order for f in case.sets[s]])
    return torch.from_numpy(host.reshape(-1)).cuda(), stride


def _host_yuv(case, alloc, pad):
    """Every YUV frame-set as host arrays from alloc(shape), rows FW + pad bytes apart (views of the first FW bytes)."""
    rows = case.FH * 3 // 2
    out = []
    for fs in case.yuv:
        row = []
        for f in fs:
            p = alloc((rows, case.FW + pad))[:, :case.FW]
            p[...] = f
            row.append(p)
        out.append(row)
    return out


@pytest.mark.parametrize("fmt", Y.FORMATS)
@pytest.mark.parametrize("name", CASES)
def test_yuv_fuzz_case_every_entry_point(ops, torch, name, fmt):
    """One YUV corpus case in one format through every entry point that takes YUV frames: run_stack on a dense stack and
    on one at an odd base and stride (batches 1, 3, 4, 7, 9; car on and off; BALANCE on the 4-camera cases), run_cuda
    on one [batch][NC][FH*3/2][FW] array, run on pageable frames (BEVK_BANDS 1 / 3 / 8 x BEVK_CHUNK 1 / 3, 7 frame-sets),
    page-locked ones (BEVK_ZEROCOPY 1 / 0) and frames with padded rows (FW + 16, FW + 2), pageable and page-locked."""
    from cameracalibration_b200 import _lib as L
    case = B.yuv_bgr_case(name, fmt)
    other = "i420" if fmt == "nv12" else "nv12"
    other_case = B.yuv_bgr_case(name, other)
    want, want_other = Want(case), Want(other_case)
    path = "tma" if case.FW % 16 == 0 else "gather"
    balances = (False, True) if case.NC == 4 else (False,)
    rev = list(range(B.N_YUV_SETS))[::-1]
    n_cmp = 0
    with _engines(ops) as make:
        e = make(case)
        pick = _Pools()
        d_rev, base_rev, stride_rev = _yuv_stack(torch, case, rev, False)
        db_rev, sb_rev = _bgr_stack(torch, other_case, rev)

        def overwrite():
            """The copy stack rewritten on other frames: the other YUV format, then (4 cameras) a BGR BALANCE call."""
            got = _render(torch, e, d_rev, stride_rev, 9, case.car, False, pixel_format=other, base=base_rev)
            assert e.last_path() == path, other
            n = want_other.check(got, False, True, f"{other} run_stack", rev)
            if case.NC == 4:
                got = _render(torch, e, db_rev, sb_rev, 9, case.car, True)
                assert e.last_path() == path, "bgr"
                n += want_other.check(got, True, True, "bgr BALANCE run_stack", rev)
            return n

        # run_stack: a dense stack, then one at an odd base address and an odd frame stride
        for odd in (False, True):
            d, base, stride = _yuv_stack(torch, case, range(B.N_YUV_SETS), odd)
            what = "odd stack" if odd else "dense stack"
            for balance in balances:
                for n in BATCHES:
                    for car in (None, case.car):
                        sets = pick(n)
                        got = _render(torch, e, d, stride, n, car, balance, pixel_format=fmt,
                                      base=base + sets[0] * case.NC * stride)
                        assert e.last_path() == path, (what, n, balance)
                        n_cmp += want.check(got, balance, car is not None, f"run_stack {what} batch {n}", sets)
                        if n == 9 and car is not None:   # the same engine's render of the cvtColor frames
                            db, sb = _bgr_stack(torch, case, sets)
                            ref = _render(torch, e, db, sb, n, car, balance)
                            assert (got == ref).all(), (what, balance, int((got != ref).sum()))
            n_cmp += overwrite()
        # run_cuda on one [batch][NC][FH*3/2][FW] array, with the car
        car_t = torch.from_numpy(case.car).cuda()
        for balance in balances:
            sets = pick(7)
            d = torch.from_numpy(np.stack([np.stack(case.yuv[s]) for s in sets])).cuda()
            out = e.run_cuda(d, car_t, balance, pixel_format=fmt)
            torch.cuda.synchronize()
            assert e.last_path() == path, ("run_cuda", balance)
            n_cmp += want.check(out.cpu().numpy(), balance, True, "run_cuda", sets)
        n_cmp += overwrite()
        # pageable host frames through the chunk pipeline (ragged last chunks), each band count's DMA rectangles
        dense = _host_yuv(case, lambda shape: np.zeros(shape, np.uint8), 0)
        for bands in ("1", "3", "8"):
            eb, pb = make(case, {"BEVK_BANDS": bands}), _Pools()
            for chunk in ("1", "3"):
                for balance in balances:
                    sets = pb(7)
                    with _env({"BEVK_CHUNK": chunk}):
                        got = eb.run([dense[s] for s in sets], case.car, balance, pixel_format=fmt)
                    assert eb.last_path() == path, (bands, chunk, balance)
                    if not balance:
                        assert eb.last_h2d_bytes() == 7 * eb.host_copy_bytes(False, fmt)[0], (bands, chunk)
                    n_cmp += want.check(got, balance, True, f"run pageable bands {bands} chunk {chunk}", sets)
        # page-locked host frames: the SMs fetch the windows (zero-copy) or DMA rectangles move them
        pinned = _host_yuv(case, L.pinned_empty, 0)
        ez, pz = make(case, {"BEVK_ZEROCOPY": "0"}), _Pools()
        for eng, pk, what in ((e, pick, "zero-copy"), (ez, pz, "no zero-copy")):
            for balance in balances:
                sets = pk(7)
                got = eng.run([pinned[s] for s in sets], None, balance, pixel_format=fmt)
                assert eng.last_path() == path, (what, balance)
                n_cmp += want.check(got, balance, False, f"run page-locked {what}", sets)
        n_cmp += overwrite()
        # padded rows: FW + 16 (page-locked: zero-copy when FW % 16 == 0) and FW + 2, pageable and page-locked
        for pad in (16, 2):
            for what, alloc in (("pageable", lambda shape: np.zeros(shape, np.uint8)), ("page-locked", L.pinned_empty)):
                frames = _host_yuv(case, alloc, pad)
                for balance in balances:
                    sets = pick(7)
                    got = e.run([frames[s] for s in sets], case.car, balance, pixel_format=fmt)
                    assert e.last_path() == path, (pad, what, balance)
                    n_cmp += want.check(got, balance, True, f"run {what} rows FW + {pad}", sets)
    assert n_cmp > 0
    print(f"{name} {fmt}: {n_cmp} canvases compared")


@pytest.mark.parametrize("fmt", Y.FORMATS)
def test_bevgenerator_yuv_at_the_fixture_geometry(fx, fmt):
    """BevGenerator.run_batch and run_cuda with pixel_format (blend, BALANCE, car) at 1280x1024 -> 1000^2 with the
    reference's calibration: cv2.cvtColor of every frame, then the reference's call sequence (RefBev)."""
    import torch
    from cameracalibration_b200.SurroundBirdEyeView import surroundBEV as S
    from tests.test_gpu_yuv import _oracle, _sets
    g = fx.geometry()
    bev = S.BevGenerator(blend=True, balance=True, calib=fx.calib)
    masks = [R.blend_mask(n, g.BW, g.BH, g.CW, g.CH) for n in NAMES]
    car = fx.car()
    yuv, bgr = _sets(fx, g, 2, fmt)
    want = [_oracle(fx.calib, g, masks, True, True, s, car) for s in bgr]
    got = bev.run_batch(yuv, car, pixel_format=fmt)
    # the second call presents the frame-sets in the other order
    d = torch.from_numpy(np.stack([np.stack(s) for s in yuv[::-1]])).cuda()
    got_d = bev.run_cuda(d, torch.from_numpy(car).cuda(), pixel_format=fmt)
    torch.cuda.synchronize()
    got_d = got_d.cpu().numpy()
    for b in range(2):
        assert (got[b] == want[b]).all(), (fmt, "run_batch", b, int((got[b] != want[b]).sum()))
        assert (got_d[1 - b] == want[b]).all(), (fmt, "run_cuda", b, int((got_d[1 - b] != want[b]).sum()))
