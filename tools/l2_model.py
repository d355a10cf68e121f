#!/usr/bin/env python
"""Model of k_bev_tma's DRAM traffic per step at the bench geometry, for several unit orders (CPU only, no GPU).

    python tools/l2_model.py [--batch 32] [--l2-mb 50] [--jobs 4]

Builds the bench plan on the host: the fixture calibration rescaled as bench.synthetic_calibration does, the blend masks
of the reference, LUT planes through the host form of k_warp_maps (tests/host/kernel_math.cu `bevmaps`), then
tools/l2_model.cu compiles the product plan (build_tma_plan, FS 7936, 4 groups, max-mult 4) in each order and replays
the step's sectors through an LRU (its header lists the simplifications).  Every number printed is MODELLED, not measured.
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (label, order mode, k, hints): modes and hints as l2_model.cu's candidate_order and Lru read them
CANDIDATES = [
    ("cost (tile-major)", 0, 1, 0),
    ("hilbert", 1, 0, 0),
    ("hilbert, cheapest 10 % last (default)", 1, 10, 0),
    ("hilbert, cheapest 25 % last", 1, 25, 0),
    ("blocks 16, cost-sorted", 2, 16, 0),
    ("windows 4", 3, 4, 0),
    ("windows 16", 3, 16, 0),
    ("windows 64", 3, 64, 0),
    ("cost + LUT evict_last", 0, 1, 1),
    ("cost + LUT last, stores first", 0, 1, 3),
    ("cost + all hints (src first)", 0, 1, 7),
    ("default + LUT last, stores first", 1, 10, 3),
]


def nvcc():
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise SystemExit("nvcc not found")


def build(tmp):
    from cameracalibration_b200.build import GENCODE
    exes = {}
    for name, src in (("kernel_math", "tests/host/kernel_math.cu"), ("l2_model", "tools/l2_model.cu")):
        out = os.path.join(tmp, name)
        r = subprocess.run([nvcc(), "-O2", "-std=c++17", "--fmad=false", "-Xcompiler", "-ffp-contract=off", *GENCODE, "-o", out,
                            os.path.join(ROOT, src)], capture_output=True, text=True)
        if r.returncode:
            raise SystemExit(r.stdout + r.stderr)
        exes[name] = out
    return exes


def bench_input(exe, tmp, FW=1920, FH=1080, BW=1000, BH=1000):
    import bench
    from oracle import restate as R
    calib = bench.synthetic_calibration(FW, FH, BW, BH)
    CW, CH = int(250 * BW / 1000), int(400 * BH / 1000)
    blob = [np.array([4, FW, FH, BW, BH, 0], np.int32).tobytes()]
    for n in bench.NAMES:
        K, D, H = calib[n]
        P = bench.dst_matrix(K, FW, FH)
        vals = list(np.asarray(K).ravel()) + list(np.asarray(D, np.float64).ravel()[:4]) + list(P.ravel()) + list(np.asarray(H).ravel())
        out = os.path.join(tmp, f"lut_{n}.bin")
        r = subprocess.run([exe, "bevmaps", str(FW * 2), str(FH * 2), str(BW), str(BH), out],
                           input=" ".join(float(v).hex() for v in vals), capture_output=True, text=True)
        if r.returncode:
            raise SystemExit(r.stderr)
        blob += [open(out, "rb").read(), np.ascontiguousarray(R.blend_mask(n, BW, BH, CW, CH), np.uint8).tobytes()]
    path = os.path.join(tmp, "in.bin")
    with open(path, "wb") as f:
        f.write(b"".join(blob))
    return path


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--l2-mb", type=float, default=50.0)
    ap.add_argument("--ctas", type=int, default=264)
    ap.add_argument("--promotion", type=int, default=128)
    ap.add_argument("--jobs", type=int, default=4)
    ap.add_argument("--json", action="store_true", help="one JSON line per candidate instead of the table")
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        exes = build(tmp)
        inp = bench_input(exes["kernel_math"], tmp)

        def one(c):
            label, mode, k, hints = c
            r = subprocess.run([exes["l2_model"], inp, str(a.batch), str(mode), str(k), str(a.l2_mb), str(a.ctas),
                                str(a.promotion), str(hints)], capture_output=True, text=True)
            if r.returncode:
                raise SystemExit(f"{label}: {r.returncode} {r.stderr}")
            return dict(json.loads(r.stdout), label=label)

        with ThreadPoolExecutor(a.jobs) as pool:
            rows = list(pool.map(one, CANDIDATES))
    if a.json:
        for r in rows:
            print(json.dumps(r))
        return
    mb = 1e6
    print(f"k_bev_tma step model: batch {a.batch}, L2 {a.l2_mb:g} MB (one LRU), {a.ctas} CTAs, TMA L2 promotion {a.promotion} B "
          f"(MODELLED, not measured)")
    print(f"per step: sum of box bytes {rows[0]['box_bytes'] / mb:.1f} MB, box-sector union {rows[0]['box_union_bytes'] / mb:.1f} MB, "
          f"sampled sectors {rows[0]['sampled_bytes'] / mb:.1f} MB, LUT {rows[0]['lut_bytes'] / mb:.1f} MB")
    hdr = f"{'order':38s} {'src MB':>8s} {'LUT MB':>8s} {'write MB':>9s} {'total MB':>9s} {'src/union':>9s} {'spread':>7s}"
    print(hdr)
    print("-" * len(hdr))
    for r in rows:
        tot = r["dram_read_src"] + r["dram_read_lut"] + r["dram_write"]
        print(f"{r['label']:38s} {r['dram_read_src'] / mb:8.1f} {r['dram_read_lut'] / mb:8.1f} {r['dram_write'] / mb:9.1f} "
              f"{tot / mb:9.1f} {r['dram_read_src'] / max(1, r['box_union_bytes']):9.2f} {100 * r['finish_spread']:6.1f}%")


if __name__ == "__main__":
    main()
