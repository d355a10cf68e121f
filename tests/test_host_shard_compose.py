"""The camera-sharded BALANCE arithmetic on the CPU.  tests/host/shard_compose.cu drives the per-thread body of
k_compose_slabs<UNIT, BAL> (compose_column, bevk_shard.cuh) over the device's grid, and k_delta's body
(gathered_deltas) over world blocks of V sums.

  * compose: random slabs and rectangles for worlds 1-8, both UNIT paths, with and without BAL.  UNIT 1 takes slab edges
    at every byte phase and an unaligned output; UNIT 8 takes the 8-byte aligned edges the real geometry has.  The
    canvas must be NumPy's saturating sum (+ the car without BAL), and BAL's channel sums the exact sums of the raw
    canvas, with bright slabs that saturate where they overlap.
  * delta: the offsets from world blocks -- each camera's V sum in the block of the rank that owns it (shard_block),
    zero elsewhere -- must equal lum_deltas on the merged sums, and the oracle's luminance_offsets on frames.
nvcc compiles the harness; only host code runs."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

from cameracalibration_b200.build import GENCODE
from cameracalibration_b200.sharding import camera_range
from oracle import restate as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    nvcc = next((c for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc") if c and os.path.exists(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("host_shard_compose") / "shard_compose"
    build = subprocess.run([nvcc, "-O2", "-std=c++17", "--fmad=false", "-Xcompiler", "-ffp-contract=off", *GENCODE, "-o", str(out),
                            os.path.join(ROOT, "tests", "host", "shard_compose.cu")], capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stdout + build.stderr
    return str(out)


def _run(exe, tmp_path, mode, blob):
    (tmp_path / "in.bin").write_bytes(blob)
    r = subprocess.run([exe, mode, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr[-2000:])
    return (tmp_path / "out.bin").read_bytes()


def _rect(rng, BW, BH, step):
    """A slab rectangle whose x edges are multiples of `step` pixels (8: the 8-byte aligned edges of UNIT 8), sometimes
    empty, sometimes the whole canvas."""
    k = rng.integers(0, 8)
    if k == 0:
        return 0, 0, 0, 0
    if k == 1:
        return 0, 0, BW, BH
    xs = sorted(rng.choice(np.arange(0, BW + 1, step), 2, replace=False))
    y0 = int(rng.integers(0, BH))
    return int(xs[0]), y0, int(xs[1]), int(rng.integers(y0 + 1, BH + 1))


def _compose_case(rng, unit, bal, world, edge_phase=None):
    BW = 8 * int(rng.integers(1, 12)) if unit == 8 else int(rng.integers(1, 70))
    BH = int(rng.integers(1, 13))
    batch = int(rng.integers(1, 4))
    rects = [_rect(rng, BW, BH, 8 if unit == 8 else 1) for _ in range(world)]
    if edge_phase is not None:                       # one slab's left edge at byte phase edge_phase (mod 8)
        x0 = next(x for x in range(BW) if (3 * x) % 8 == edge_phase) if BW > 8 else 0
        rects[0] = (x0, 0, BW, BH)
    need = max([(x1 - x0) * (y1 - y0) * 3 for x0, y0, x1, y1 in rects] + [8])
    slab_bytes = (need + 7) // 8 * 8 + 8 * int(rng.integers(0, 3))
    rank_stride = (batch + int(rng.integers(0, 2))) * slab_bytes
    bright = rng.integers(0, 2)
    slabs = rng.integers(100 if bright else 0, 256, (world, rank_stride), dtype=np.uint8)
    has_car = int(rng.integers(0, 2))
    car = rng.integers(0, 256, (BH, BW, 3), dtype=np.uint8) if has_car else None
    off = 0 if unit == 8 else int(rng.integers(0, 8))
    want = np.zeros((batch, BH, BW * 3), np.int32)
    for r, (x0, y0, x1, y1) in enumerate(rects):
        if x1 <= x0 or y1 <= y0:
            continue
        pitch = (x1 - x0) * 3
        for b in range(batch):
            blk = slabs[r, b * slab_bytes: b * slab_bytes + pitch * (y1 - y0)].reshape(y1 - y0, pitch)
            want[b, y0:y1, 3 * x0:3 * x1] = np.minimum(want[b, y0:y1, 3 * x0:3 * x1] + blk, 255)
    want = want.reshape(batch, BH, BW, 3)
    sums = want.reshape(batch, -1, 3).sum(axis=1).astype(np.uint64) if bal else None
    if car is not None and not bal:
        want = np.minimum(want + car, 255)
    rec = struct.pack("<8i", unit, int(bal), world, batch, BW, BH, has_car, off) + struct.pack("<2q", slab_bytes, rank_stride)
    rec += np.asarray(rects, np.int32).tobytes() + slabs.tobytes() + (car.tobytes() if car is not None else b"")
    return rec, dict(batch=batch, BW=BW, BH=BH, want=want.astype(np.uint8), sums=sums, rects=rects, unit=unit)


@pytest.mark.parametrize("unit", [8, 1])
@pytest.mark.parametrize("bal", [False, True])
def test_compose_body_against_numpy(exe, tmp_path, unit, bal):
    rng = np.random.default_rng(7 + unit + 100 * bal)
    cases = []
    for world in range(1, 9):
        for phase in range(8):
            cases.append(_compose_case(rng, unit, bal, world, edge_phase=phase if unit == 1 else None))
    raw, p = _run(exe, tmp_path, "compose", b"".join(r for r, _ in cases)), 0
    saturated = 0
    for _, c in cases:
        n = c["batch"] * c["BH"] * c["BW"] * 3
        got = np.frombuffer(raw[p:p + n], np.uint8).reshape(c["want"].shape)
        p += n
        assert (got == c["want"]).all(), {k: v for k, v in c.items() if k not in ("want", "sums")}
        if bal:
            s = np.frombuffer(raw[p:p + 24 * c["batch"]], np.uint64).reshape(c["batch"], 3)
            p += 24 * c["batch"]
            assert (s == c["sums"]).all(), (s, c["sums"])
        saturated += int((c["want"] == 255).sum())
    assert p == len(raw) and saturated > 0
    if unit == 1:   # slab left edges fell at every byte phase
        assert {(3 * c["rects"][0][0]) % 8 for _, c in cases if c["BW"] > 8} == set(range(8))


def _delta_record(world, batch, n_cam, npix, vs):
    """vs: uint64 [batch][n_cam] V sums -> the world blocks camera-sharded ranks exchange."""
    blocks = np.zeros((world, batch, n_cam), np.uint64)
    for r in range(world):
        lo, hi = camera_range(n_cam, r, world)
        blocks[r, :, lo:hi] = vs[:, lo:hi]
    return struct.pack("<3id", world, batch, n_cam, npix) + blocks.tobytes()


def _deltas(raw, recs):
    p, out = 0, []
    for batch, n_cam in recs:
        n = batch * n_cam * 4
        got = np.frombuffer(raw[p:p + n], np.int32).reshape(batch, n_cam)
        merged = np.frombuffer(raw[p + n:p + 2 * n], np.int32).reshape(batch, n_cam)
        p += 2 * n
        out.append((got, merged))
    assert p == len(raw)
    return out


def test_gathered_deltas_equal_merged_lum_deltas(exe, tmp_path):
    rng = np.random.default_rng(11)
    blob, recs = [], []
    for i in range(200):
        world, n_cam, batch = int(rng.integers(1, 9)), int(rng.integers(1, 9)), int(rng.integers(1, 6))
        npix = float(rng.integers(1, 1 << 22))
        top = int(npix) * 255 if i % 3 else 1 << 40          # realistic sums, and huge ones: the adds must stay exact
        vs = rng.integers(0, top + 1, (batch, n_cam), dtype=np.uint64)
        blob.append(_delta_record(world, batch, n_cam, npix, vs))
        recs.append((batch, n_cam))
    for got, merged in _deltas(_run(exe, tmp_path, "delta", b"".join(blob)), recs):
        assert (got == merged).all()


def test_gathered_deltas_equal_oracle_on_frames(exe, tmp_path):
    rng = np.random.default_rng(12)
    blob, recs, want = [], [], []
    for i in range(40):
        world, n_cam, batch = int(rng.integers(1, 9)), int(rng.integers(1, 9)), int(rng.integers(1, 4))
        FW, FH = int(rng.integers(3, 60)), int(rng.integers(2, 40))
        sets = [[rng.integers(int(rng.integers(0, 200)), 256, (FH, FW, 3), dtype=np.uint8) for _ in range(n_cam)] for _ in range(batch)]
        vs = np.array([[np.maximum(np.maximum(f[..., 0], f[..., 1]), f[..., 2]).astype(np.uint64).sum() for f in s] for s in sets], np.uint64)
        blob.append(_delta_record(world, batch, n_cam, float(FW * FH), vs))
        recs.append((batch, n_cam))
        want.append(np.array([R.luminance_offsets(s)[0] for s in sets], np.int32))
    for (got, merged), w in zip(_deltas(_run(exe, tmp_path, "delta", b"".join(blob)), recs), want):
        assert (got == w).all() and (merged == w).all(), (got, w)
