"""GPU fuzz of the fused BEV kernels (k_bev_tma, k_bev) on the seeded corpus of tests/bev_cases.py: arbitrary maps given
through set_maps (random local, int16-extreme, smooth fisheye + tilted homographies), 1-8 cameras, binary / weighted /
all-255 / overlapping masks with bright frames (saturating adds), empty and single-pixel masks, both interpolations,
frame widths for each kernel path, canvases below 32 px and ragged.  Every canvas is compared byte for byte with the
cv2 / NumPy oracle of bev_cases (or, for the alignment regressions, with the same frames' aligned render), never with
itself; every 16-byte friendly stack must have run the TMA kernel.

tests/test_host_bev_fuzz.py shows on the CPU which plan features (multi-pass and GATHER items, saturating items, FULL
items, both orientations, empty and edge tiles) this corpus reaches at each configuration used here."""
import os
from contextlib import contextmanager

import cv2
import numpy as np
import pytest

from tests import bev_cases as B

pytestmark = pytest.mark.gpu
BATCHES = (1, 3, 4, 7, 9)   # NB=1; NB=4 whole; NB=4 with tails of 3 and 1


@pytest.fixture(scope="module")
def ops():
    from cameracalibration_b200 import ops as o
    return o


@pytest.fixture(scope="module")
def torch():
    import torch as t
    return t


@contextmanager
def _env(env):
    """Set tuning variables for the duration of the block, then restore them."""
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


@contextmanager
def _engines(ops):
    """make(case, env) -> finalized BevEngine (env: variables bevk_bev_finalize reads); every context closed afterwards."""
    made = []

    def make(case, env=None):
        e = ops.BevEngine(case.NC, (case.FW, case.FH), (case.BW, case.BH))
        made.append(e)
        for k, ((m1, m2), mk) in enumerate(zip(case.maps, case.masks)):
            e.set_maps(k, m1, m2)
            e.set_mask(k, mk)
        if case.nearest:
            e.set_interpolation(ops.INTER_NEAREST)
        with _env(env or {}):
            e.finalize()
        return e
    try:
        yield make
    finally:
        for e in made:
            e.ctx.close()


class Want:
    """Oracle canvases of one case, computed once per (frame-set, balance, car)."""

    def __init__(self, case):
        self.case, self.memo = case, {}

    def __call__(self, s, balance, car):
        k = (s, balance, car)
        if k not in self.memo:
            self.memo[k] = B.oracle(self.case, s, balance, car)
        return self.memo[k]

    def check(self, got, balance, car, what, sets=None):
        """got[i] against the oracle of frame-set sets[i] (default: i)."""
        compared = 0
        for i in range(got.shape[0]):
            s = i if sets is None else sets[i]
            w = self(s, balance, car)
            if w is None:          # BALANCE of a canvas with a zero channel mean: the reference divides by zero
                continue
            assert (got[i] == w).all(), (self.case.name, what, s, balance, car, int((got[i] != w).sum()))
            compared += 1
        assert compared > 0, (self.case.name, what, "no frame-set has a defined oracle")
        return compared


def _stack(torch, case, n, pad):
    """Frame-sets 0..n-1 as one device stack; pad: frames at a stride padded to a multiple of 16 bytes, padding 0xFF."""
    fb = case.FW * case.FH * 3
    stride = (fb + 48 + 15) // 16 * 16 if pad else fb
    host = np.full((n * case.NC, stride), 0xFF, np.uint8)
    host[:, :fb] = np.stack([np.stack(s) for s in case.sets[:n]]).reshape(n * case.NC, fb)
    return torch.from_numpy(host.reshape(-1)).cuda(), stride


def _render(torch, e, d, stride, n, car, balance, off=16, car_off=0, pixel_format="bgr", base=0):
    """run_stack of the frames at byte `base` of d into a buffer with 0xA5 sentinels: `off` bytes before the output and
    a whole canvas after it.  The car (if any) is placed at byte `car_off` of its own buffer."""
    cb = e.BW * e.BH * 3
    buf = torch.full((off + (n + 1) * cb,), 0xA5, dtype=torch.uint8, device=d.device)
    cptr = 0
    if car is not None:
        cbuf = torch.zeros(cb + 16, dtype=torch.uint8, device=d.device)
        cbuf[car_off:car_off + cb] = torch.from_numpy(car.reshape(-1)).to(d.device)
        cptr = cbuf.data_ptr() + car_off
    e.run_stack(d.data_ptr() + base, stride, n, buf.data_ptr() + off, cptr, balance, pixel_format=pixel_format)
    e.ctx.sync()
    h = buf.cpu().numpy()
    assert (h[:off] == 0xA5).all() and (h[off + n * cb:] == 0xA5).all(), "bytes written outside the output"
    return h[off:off + n * cb].reshape(n, e.BH, e.BW, 3)


def _frame_views(torch, case, n, gaps):
    """Frame-sets 0..n-1 as a list (batch) of lists (camera) of device views into one buffer, 16-byte aligned, at a padded
    stride; gaps: every other frame 16 bytes further on, so that the frames form no stack."""
    fb = case.FW * case.FH * 3
    step = (fb + 32 + 15) // 16 * 16
    buf = torch.zeros(n * case.NC * step + 64, dtype=torch.uint8, device="cuda")
    frames = []
    for b, fs in enumerate(case.sets[:n]):
        row = []
        for k, f in enumerate(fs):
            i = b * case.NC + k
            o = i * step + (16 if gaps and i % 2 else 0)
            v = buf[o:o + fb]
            v.copy_(torch.from_numpy(f.reshape(-1)).cuda())
            row.append(v.view(case.FH, case.FW, 3))
        frames.append(row)
    return frames, buf


def _path(case):
    return "tma" if case.tma_friendly else "gather"


@pytest.mark.parametrize("seed", range(B.N_CASES))
def test_fuzz_case_every_entry_point(ops, torch, seed):
    """One corpus case through run_stack (batches 1, 3, 4, 7, 9; car on and off; BALANCE on the 4-camera cases; padded
    and dense stacks), run on pageable frames (BEVK_BANDS 1 / 3 / 8 x BEVK_CHUNK 1 / 3) and page-locked ones (BEVK_ZEROCOPY
    1 / 0), run_cuda with a pointer table, BEVK_TMA=0, BEVK_NB=8, BEVK_TMA_BACKOFF, and camera ranges composed with the
    saturating sum.  The host entry points stage frames in a stack of their own: the TMA kernel serves them too."""
    from cameracalibration_b200 import _lib as L
    case = B.make_case(seed)
    want = Want(case)
    balances = (False, True) if case.NC == 4 else (False,)
    n_cmp = 0
    with _engines(ops) as make:
        e = make(case)
        assert (e.tma_plan_info()["items"] > 0) == case.tma_friendly
        d_pad, s_pad = _stack(torch, case, 9, True)
        for balance in balances:
            for n in BATCHES:
                for car in (None, case.car):
                    got = _render(torch, e, d_pad, s_pad, n, car, balance)
                    assert e.last_path() == _path(case), (case.name, n)
                    n_cmp += want.check(got, balance, car is not None, f"run_stack batch {n}")
        if (case.FW * case.FH * 3) % 4 == 0:    # a stack's frame stride must be a multiple of 4
            d_dense, s_dense = _stack(torch, case, 9, False)
            got = _render(torch, e, d_dense, s_dense, 9, case.car, False)
            assert e.last_path() == _path(case)
            n_cmp += want.check(got, False, True, "dense stack")
        # host entry points on 7 frame-sets (chunks of 1 and 3: ragged last chunks)
        sets = case.sets[:7]
        pinned = []
        for fs in sets:
            row = []
            for f in fs:
                p = L.pinned_empty(f.shape)
                p[...] = f
                row.append(p)
            pinned.append(row)
        for bands in ("1", "3", "8"):
            eb = make(case, {"BEVK_BANDS": bands})
            for chunk in ("1", "3"):
                for balance in balances:
                    with _env({"BEVK_CHUNK": chunk}):
                        got = eb.run(sets, case.car, balance)
                    assert eb.last_path() == _path(case), (bands, chunk, balance)
                    n_cmp += want.check(got, balance, True, f"run pageable bands {bands} chunk {chunk}")
        ez = make(case, {"BEVK_ZEROCOPY": "0"})
        for eng, what in ((e, "zero-copy"), (ez, "no zero-copy")):
            for balance in balances:
                got = eng.run(pinned, None, balance)
                assert eng.last_path() == _path(case), (what, balance)
                n_cmp += want.check(got, balance, False, f"run page-locked {what}")
        # run_cuda with a pointer table that is no stack (alternating gaps): the gather kernel -- except with BALANCE,
        # which renders from the balanced frame copies, themselves a stack
        frames, _keep = _frame_views(torch, case, 7, gaps=True)
        car_t = torch.from_numpy(case.car).cuda()
        for balance in balances:
            out = e.run_cuda(frames, car_t, balance)
            torch.cuda.synchronize()
            assert e.last_path() == (_path(case) if balance else "gather"), balance
            n_cmp += want.check(out.cpu().numpy(), balance, True, "run_cuda pointer table")
        # the gather kernel only, NB=8 units (k_bev<*, 8>), and a producer that sleeps between polls of a full ring
        for env, n, path in (({"BEVK_TMA": "0"}, 7, "gather"), ({"BEVK_NB": "8"}, 9, "gather"),
                             ({"BEVK_TMA_BACKOFF": "200"}, 9, _path(case))):
            eg = make(case, env)
            for balance in balances:
                got = _render(torch, eg, d_pad, s_pad, n, case.car, balance)
                assert eg.last_path() == path, env
                n_cmp += want.check(got, balance, True, str(env))
        # camera ranges (ragged, some skipping a tile's first camera) composed with the saturating sum
        if case.NC >= 2:
            NC, cb = case.NC, case.BW * case.BH * 3
            cuts = sorted({1, NC // 2, NC - 1} - {0, NC})
            for ranges in ([(0, 1), (1, NC)], [(1, NC), (0, 1)], [(a, b) for a, b in zip([0] + cuts, cuts + [NC])],
                           [(k, k + 1) for k in range(NC)][::-1]):
                parts = []
                for lo, hi in ranges:
                    p = torch.empty((7, case.BH, case.BW, 3), dtype=torch.uint8, device="cuda")
                    e.run_stack_cams(d_pad.data_ptr(), s_pad, 7, lo, hi, p.data_ptr())
                    assert e.last_path() == _path(case)
                    parts.append(p)
                out = torch.empty_like(parts[0])
                e.sat_sum_device([p.data_ptr() for p in parts], 7 * cb, out.data_ptr())
                e.ctx.sync()
                n_cmp += want.check(out.cpu().numpy(), False, False, f"camera ranges {ranges}")
    print(f"{case.name}: {n_cmp} canvases compared")


@pytest.mark.parametrize("name", ["smooth4", "extreme1"])
def test_fuzz_camera_sharded_render_and_compose(ops, torch, name):
    """ShardedBev(..., 'cameras', connect=False): every rank's slabs rendered on this GPU and composed (with the car) for
    worlds of 2, 3 and 8 -- more ranks than cameras, and (smooth4) a camera whose mask is empty."""
    from cameracalibration_b200.sharding import ShardedBev
    case = B.case_by_name(name)
    want = Want(case)
    with _engines(ops) as make:
        e = make(case)
        d = torch.from_numpy(np.stack([np.stack(s) for s in case.sets[:5]])).cuda()
        car = torch.from_numpy(case.car).cuda()
        for world in (2, 3, 8):
            sh = ShardedBev(e, "cameras", rank=0, world=world, connect=False)
            slabs = sh.slab_buffer(5)
            for r in range(world):
                sh.render_slabs(d, r, slabs)
            out = torch.empty((5, case.BH, case.BW, 3), dtype=torch.uint8, device="cuda")
            sh.compose(slabs, out, car)
            torch.cuda.synchronize()
            assert want.check(out.cpu().numpy(), False, True, f"world {world}") == 5


@pytest.mark.parametrize("mm", B.MAX_MULTS)
@pytest.mark.parametrize("cfg", B.tma_configs(), ids=lambda c: "x".join(map(str, c)))
def test_fuzz_every_tma_configuration(ops, torch, cfg, mm):
    """Every BEVK_TMA_CONFIGS instantiation with BEVK_TMA_MAXMULT 1 / 2 / 4 on a smooth minified, a random-local and an
    int16-extreme case, BALANCE off (batch 7: a tail of 3) and on (batch 9: a tail of 1), with the car."""
    fs, slots, _ctas, eg = cfg
    with _engines(ops) as make:
        for name in B.CONFIG_CASES:
            case = B.case_by_name(name)
            want = Want(case)
            e = make(case, {"BEVK_TMA_CFG": f"{fs},{slots},{eg}", "BEVK_TMA_MAXMULT": str(mm)})
            d, stride = _stack(torch, case, 9, True)
            for balance, n in ((False, 7), (True, 9)):
                got = _render(torch, e, d, stride, n, case.car, balance)
                assert e.last_path() == "tma", (name, cfg, mm)
                want.check(got, balance, True, f"cfg {cfg} maxmult {mm}")
    # a configuration that was not built is refused, not replaced by the default
    from cameracalibration_b200 import _lib as L
    with _engines(ops) as make:
        with pytest.raises(L.BevkError, match="BEVK_TMA_CFG"):
            make(B.case_by_name(B.CONFIG_CASES[0]), {"BEVK_TMA_CFG": "1000,2,4"})


@pytest.mark.parametrize("name,env,path", [
    ("smooth4", {}, "tma"),                         # k_bev_tma: interior (row-wise) and generic write-outs
    ("smooth4", {"BEVK_TMA": "0"}, "gather"),       # k_bev on the same frames
    ("local3", {}, "gather"),                       # k_bev: a frame pitch that allows no TMA plan
])
def test_unaligned_output_and_car(ops, torch, name, env, path):
    """Output at byte offsets 1, 2, 3 of a larger buffer and the car at offset 1: run_stack (plain and BALANCE, which
    ends in k_gain) and run_cuda(out=...), through both kernels.  The canvas pitch and size are multiples of 4, so only
    the pointers decide between word and byte stores.  Each result equals the aligned render and the oracle, and the
    sentinels around the output stay untouched."""
    case = B.case_by_name(name)
    want = Want(case)
    cb = case.BW * case.BH * 3
    assert (case.BW * 3) % 4 == 0 and cb % 4 == 0, "an aligned output must take the 32-bit write-out"
    n = 5
    with _engines(ops) as make:
        e = make(case, env)
        d, stride = _stack(torch, case, n, True)
        for balance in (False, True):
            aligned = _render(torch, e, d, stride, n, case.car, balance)
            want.check(aligned, balance, True, "aligned")
            for off in (1, 2, 3):
                for car_off in (0, 1):
                    got = _render(torch, e, d, stride, n, case.car, balance, off=16 + off, car_off=car_off)
                    assert e.last_path() == path
                    assert (got == aligned).all(), (name, balance, off, car_off, int((got != aligned).sum()))
        frames, _keep = _frame_views(torch, case, n, gaps=False)   # a stack at a 16-byte stride: as run_stack above
        for off in (1, 2, 3):
            buf = torch.full((16 + off + (n + 1) * cb,), 0xA5, dtype=torch.uint8, device="cuda")
            cbuf = torch.zeros(cb + 1, dtype=torch.uint8, device="cuda")
            cbuf[1:] = torch.from_numpy(case.car.reshape(-1)).cuda()
            out = buf[16 + off:16 + off + n * cb].view(n, case.BH, case.BW, 3)
            e.run_cuda(frames, cbuf[1:].view(case.BH, case.BW, 3), False, out=out)
            torch.cuda.synchronize()
            assert e.last_path() == path
            h = buf.cpu().numpy()
            assert (h[:16 + off] == 0xA5).all() and (h[16 + off + n * cb:] == 0xA5).all(), off
            want.check(out.cpu().numpy(), False, True, f"run_cuda out offset {off}")


def test_wide_canvases(ops, torch):
    """Tile origins travel to k_bev_tma's consumers as x | y << 16: a 65536-px wide canvas (last tile at 65504) renders
    like cv2.remap through the TMA kernel; a wider one is refused by bevk_bev_configure."""
    from cameracalibration_b200 import _lib as L
    with pytest.raises(L.BevkError, match="65536"):
        ops.BevEngine(1, (64, 40), (65600, 40))
    with pytest.raises(L.BevkError, match="65536"):
        ops.BevEngine(1, (64, 40), (40, 65600))
    FW, FH, BW, BH = 64, 40, 65536, 40
    rng = np.random.default_rng(77)
    yy, xx = np.mgrid[0:BH, 0:BW]
    m1 = np.stack([xx % FW, yy], -1).astype(np.int16)           # wrapped identity: every tile samples the same frame
    m2 = rng.integers(0, 1024, (BH, BW)).astype(np.uint16)
    mask = np.full((BH, BW), 255, np.uint8)
    frames = [rng.integers(0, 256, (FH, FW, 3), dtype=np.uint8) for _ in range(4)]
    case = B.Case("wide", "local", FW, FH, BW, BH, False, [(m1, m2)], [mask], [[f] for f in frames])
    # cv2.remap takes destinations narrower than 32767 px: the oracle in column blocks (the map is per pixel)
    want = [np.concatenate([cv2.remap(f, np.ascontiguousarray(m1[:, x:x + 16384]), np.ascontiguousarray(m2[:, x:x + 16384]),
                                      cv2.INTER_LINEAR) for x in range(0, BW, 16384)], 1) for f in frames]
    with _engines(ops) as make:
        e = make(case)
        d, stride = _stack(torch, case, 4, True)
        for n in (1, 4):
            got = _render(torch, e, d, stride, n, None, False)
            assert e.last_path() == "tma"
            for s in range(n):
                assert (got[s] == want[s]).all(), (n, s, np.nonzero((got[s] != want[s]).any(axis=(0, 2)))[0][:8].tolist())
