"""GPU fuzz of the device JPEG encoder (bevk_jpeg_enc.cuh, jpeg_enqueue / enc_chunks in bevk_api.cu) against
cv2.imencode, byte for byte: the seeded corpus of tests/jpeg_cases.py through ops.jpeg_encode and bevk_jpeg_encode, one
context reused across calls that change size, quality and batch, more than 2^32 entropy bits in one call,
Undistorter.cuda_to_jpeg at every undistorted-width class mod 16 with the chunked pipeline at several chunk sizes, and
BEV-to-JPEG with colour balance (k_gain over the batch, then the encoder) on canvases so small that one CTA's 128
blocks span up to 23 images.

These run the device's decomposition of the work -- k_jpeg_dc's dummy-block DCs across MCUs, the batch-wide bit-offset
scan, atomicOr on the words neighbouring blocks share, the pad written by each image's last block, 0xFF counts per
128-byte chunk, stream compaction and the two-slot chunk pipeline -- which tests/test_host_jpeg_fuzz.py's serial host
build of the same stages never does."""
import ctypes
import os
from contextlib import contextmanager

import cv2
import numpy as np
import pytest

from oracle import cv2_path as C
from tests import bev_cases as B
from tests import calib_cases as CC
from tests import jpeg_cases as J

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
def _env(env):
    """Set (or, for None, unset) variables for the duration of the block, then restore them."""
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


def _device_images(torch, case):
    """(what ops.jpeg_encode takes, device pointer, image stride, row stride, buffer kept alive) of the case's images in
    its layout; "numpy" passes the host array to ops.jpeg_encode and a dense upload to bevk_jpeg_encode."""
    imgs = case.images
    n, H, W, _ = imgs.shape
    dense = torch.from_numpy(imgs).cuda()
    if case.layout in ("dense", "numpy"):
        return (imgs if case.layout == "numpy" else dense), dense.data_ptr(), H * W * 3, W * 3, dense
    pitch, istride, off = 3 * W, 3 * W * H, 0
    if case.layout == "pitch":
        pitch = 3 * W + 13
        istride = H * pitch
    elif case.layout == "stride":
        istride = 3 * W * H + 37
    elif case.layout.startswith("offset"):
        off = int(case.layout[-1])
    else:                                                   # "view": a crop of a larger canvas, rows and images padded
        pitch = 3 * (W + 5) + 1
        istride = (H + 3) * pitch + 11
        off = pitch + 3 * 2 + 1
    base = torch.full((off + n * istride + 64,), 0x5A, dtype=torch.uint8, device="cuda")
    view = torch.as_strided(base, (n, H, W, 3), (istride, pitch, 3, 1), off)
    view.copy_(dense)
    return view, base.data_ptr() + off, istride, pitch, base


def _direct(L, ctx, ptr, istride, pitch, n, W, H, q, want, what):
    """bevk_jpeg_encode into a buffer of exactly the streams' total, followed by 0xA5 sentinels."""
    total = sum(len(s) for s in want)
    buf = np.full(total + 4096, 0xA5, np.uint8)
    sizes = (ctypes.c_uint64 * n)()
    rc = ctx.lib.bevk_jpeg_encode(ctx.h, ctypes.c_void_p(ptr), istride, pitch, n, W, H, q, L.vptr(buf), total, sizes)
    assert rc == 0, (what, ctx.lib.bevk_last_error().decode())
    assert list(sizes) == [len(s) for s in want], what
    assert buf[:total].tobytes() == b"".join(want), what
    assert (buf[total:] == 0xA5).all(), (what, "bytes written past the streams")


def _first_diff(got, want):
    for i, (g, w) in enumerate(zip(got, want)):
        if g != w:
            k = next((j for j in range(min(len(g), len(w))) if g[j] != w[j]), min(len(g), len(w)))
            return f"image {i}: sizes {len(g)} / {len(w)}, first differing byte {k}"
    return "lengths differ" if len(got) != len(want) else "equal"


def test_corpus_through_jpeg_encode_and_direct_call(torch, ops, L):
    """Every corpus case through ops.jpeg_encode (its own layout read in place, or NumPy) and bevk_jpeg_encode on the
    same device images, all on one context."""
    n_img = 0
    with _context(L) as ctx:
        for c in J.corpus():
            want = list(J.streams(c.name))
            arg, ptr, istride, pitch, _keep = _device_images(torch, c)
            got = ops.jpeg_encode(arg, c.quality, ctx=ctx)
            assert got == want, (c.name, c.layout, c.quality, _first_diff(got, want))
            _direct(L, ctx, ptr, istride, pitch, c.n, c.W, c.H, c.quality, want, c.name)
            n_img += c.n
    print(f"{n_img} images compared")


def test_context_reuse_across_sizes_qualities_and_batches(ops, L):
    """One context, calls in a fixed order: large -> small -> large in n and in size, quality changes at one size, and
    width changes at an equal block count (17x16 -> 32x16 -> 16x32, 12 blocks each) -- the (w, h, q) header and table
    cache, scratch growth, and 0xFF chunk counts left behind by bigger earlier calls."""
    rng = np.random.default_rng(9)
    seq = [(9, 200, 120, 100, "noise"), (1, 16, 16, 50, "flat"), (130, 16, 16, 90, "noise"), (3, 17, 16, 75, "noise"),
           (3, 32, 16, 75, "noise"), (3, 32, 16, 20, "noise"), (3, 32, 16, 20, "gradient"), (3, 16, 32, 20, "noise"),
           (2, 640, 480, 100, "noise"), (5, 9, 9, 100, "flat"), (40, 48, 16, 100, "noise"), (1, 640, 480, 95, "gradient"),
           (64, 17, 16, 100, "noise"), (1, 1, 1, 0, "noise"), (7, 37, 23, 101, "checker")]
    with _context(L) as ctx:
        for k, (n, W, H, q, content) in enumerate(seq):
            imgs = np.stack([J.CONTENTS[content](rng, H, W) for _ in range(n)])
            want = [J.encode(i, q) for i in imgs]
            got = ops.jpeg_encode(imgs, q, ctx=ctx)
            assert got == want, (k, n, W, H, q, _first_diff(got, want))


def test_more_than_2_32_entropy_bits_in_one_call(torch, ops, L):
    """17 noise images of 4096x4096 at q100 (3 distinct ones, cycled) in one call: the batch's bit offsets pass 2^32,
    which only the 64-bit offs / image_bits arithmetic survives."""
    free, _ = torch.cuda.mem_get_info()
    if free < 12 << 30:
        pytest.skip(f"needs 12 GB of free device memory, {free / 2**30:.1f} GB free (the GPU is shared)")
    rng = np.random.default_rng(4096)
    distinct = np.stack([rng.integers(0, 256, (4096, 4096, 3), dtype=np.uint8) for _ in range(3)])
    want = [J.encode(d, 100) for d in distinct]
    idx = [i % 3 for i in range(17)]
    bits = sum(8 * len(J.entropy_segment(want[i])) - 7 for i in idx)
    assert bits > 2 ** 32, bits
    with _context(L) as ctx:
        d = torch.from_numpy(distinct).cuda()[idx]
        got = ops.jpeg_encode(d, 100, ctx=ctx)
        del d
    assert len(got) == 17
    for i, g in enumerate(got):
        assert g == want[idx[i]], (i, len(g), len(want[idx[i]]))
    torch.cuda.empty_cache()


def _und_cameras():
    """(calibration case, undistorted width, height) per class of the undistorted width mod 16: the smallest case of the
    corpus in that class, or -- for classes the corpus lacks -- its smallest fisheye case at a width moved into it."""
    best = {}
    for c in CC.corpus():
        r = c.UW % 16
        if r not in best or c.UW * c.UH < best[r].UW * best[r].UH:
            best[r] = c
    fish = min((c for c in CC.corpus() if c.fisheye), key=lambda c: c.UW * c.UH)
    return [(best[r], best[r].UW, best[r].UH) if r in best else (fish, fish.UW - fish.UW % 16 + 16 + r, fish.UH)
            for r in range(16)]


def test_undistorter_cuda_to_jpeg_chunks(torch, ops):
    """Undistorter.cuda_to_jpeg on one camera per UW % 16 class, batches 1, 7 and 17, with BEVK_JPEG_CHUNK unset (8),
    1, 3 and 0 (the whole batch): the two-slot pipeline with ragged last chunks, against cv2.imencode(cv2.remap(...))."""
    n_cmp = 0
    for k, (c, UW, UH) in enumerate(_und_cameras()):
        q = (95, 100, 75, 50, 90, 5, 99, 85)[k % 8]
        u = ops.Undistorter(c.K, c.D if c.fisheye else c.d5, c.P, (UW, UH), model="fisheye" if c.fisheye else "pinhole",
                            fused=bool(k % 2))
        fr = CC.frames(c.name, 3, 17)
        maps = CC.cv2_maps(c.name) if (UW, UH) == (c.UW, c.UH) else C.undistort_maps(c.K, c.D.reshape(4, 1), c.P, UW, UH)
        want = [J.encode(cv2.remap(f, *maps, cv2.INTER_LINEAR), q) for f in fr]
        d = torch.from_numpy(fr).cuda()
        for chunk in (None, "1", "3", "0"):
            with _env({"BEVK_JPEG_CHUNK": chunk}):
                for n in (1, 7, 17):
                    got = u.cuda_to_jpeg(d[:n], quality=q)
                    assert got == want[:n], (c.name, UW, UH, chunk, n, _first_diff(got, want[:n]))
                    n_cmp += n
        u.close()
    print(f"{n_cmp} streams compared")


# tiny canvases: 6, 12, 12 and 54 blocks, so that one CTA's 128 blocks of k_jpeg_blocks touch up to 23 images
_GAIN_CANVASES = (((16, 16), "local", 95), ((24, 16), "extreme", 100), ((17, 9), "local", 50), ((40, 40), "local", 75))


def _gain_case(i, BW, BH, kind, n_sets):
    rng = np.random.default_rng(500 + i)
    FW, FH = 64, 40
    maps = B._maps(rng, kind, 4, FW, FH, BW, BH)
    masks = B._masks(rng, 4, BW, BH, i)
    sets = B._frames(rng, 4, FW, FH, i % 2 == 1, n_sets)
    car = rng.integers(0, 256, (BH, BW, 3), dtype=np.uint8)
    car[rng.integers(0, 2, (BH, BW)) == 0] = 0
    return B.Case(f"gain{i}_{BW}x{BH}", kind, FW, FH, BW, BH, False, maps, masks, sets, car)


def test_bev_to_jpeg_balance_tiny_canvases(torch, ops):
    """BALANCE, car on and off, batches 64 and 129, through BevEngine.cuda_to_jpeg (BEVK_JPEG_CHUNK 0 and the default
    8) and run_to_jpeg: k_gain over a batch of tiny canvases, then the encoder, whose CTAs span many of them.  Every
    stream equals cv2.imencode of the balanced canvas of the bev_cases oracle.  Frame-sets
    whose balance is undefined (a zero channel mean) are skipped; most must be compared."""
    n_cmp = n_skip = 0
    for i, ((BW, BH), kind, q) in enumerate(_GAIN_CANVASES):
        case = _gain_case(i, BW, BH, kind, 129)
        memo = {}

        def want(s, car):
            if (s, car) not in memo:
                w = B.oracle(case, s, True, car)
                memo[(s, car)] = None if w is None else J.encode(w, q)
            return memo[(s, car)]

        e = ops.BevEngine(4, (case.FW, case.FH), (BW, BH))
        for k, ((m1, m2), mk) in enumerate(zip(case.maps, case.masks)):
            e.set_maps(k, m1, m2)
            e.set_mask(k, mk)
        e.finalize()
        frames = torch.from_numpy(np.stack([np.stack(s) for s in case.sets])).cuda()
        car_d = torch.from_numpy(case.car).cuda()
        for n in (64, 129):
            for car in (False, True):
                runs = [("cuda_to_jpeg chunk 0", {"BEVK_JPEG_CHUNK": "0"}, lambda: e.cuda_to_jpeg(frames[:n], q, car_d if car else None, True)),
                        ("cuda_to_jpeg default", {"BEVK_JPEG_CHUNK": None}, lambda: e.cuda_to_jpeg(frames[:n], q, car_d if car else None, True)),
                        ("run_to_jpeg", {}, lambda: e.run_to_jpeg(case.sets[:n], q, case.car if car else None, True))]
                for what, env, run in runs:
                    with _env(env):
                        got = run()
                    assert len(got) == n, (case.name, what)
                    for s in range(n):
                        w = want(s, car)
                        if w is None:
                            n_skip += 1
                            continue
                        assert got[s] == w, (case.name, what, n, car, s, len(got[s]), len(w))
                        n_cmp += 1
        e.ctx.close()
    assert n_cmp > 10 * n_skip, (n_cmp, n_skip)
    print(f"{n_cmp} streams compared, {n_skip} frame-sets without a defined oracle")
