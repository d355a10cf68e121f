#!/usr/bin/env python
"""cv2.resize and cv2.warpAffine on the device (ops.resize / ops.warp_affine on CUDA arrays: bevk_resize_stack,
bevk_warp_affine_stack) against cv2 over all host cores, on the same inputs.  One JSON line, with the card's name, power
limit and SM clock read in the same run.

    workloads  batch 32 of 1280x1024x3 frames: LINEAR to 640x480 and to 2560x2048, AREA to 640x512 (whole 2x2 cells) and
               to 427x341 (fractional cells); batch 32 of 1000x1000x3 BEV canvases: LINEAR to 500x500; warpAffine
               translate (CenterImage.translate's matrix) of a batch of 32 1280x1024x3 frames
    kernel     CUDA events around --reps calls, after a warm-up; per batch, per frame, and the bytes the call must move
               (source frames read once + destination written) per second, as a share of the H100 SXM's 3.35 TB/s
               data-sheet HBM3 bandwidth
    cv2        the same 32 frames, one frame per host core at a time (cv2.setNumThreads(1)); its outputs are compared
               byte for byte with the device's from the timed run

    python tools/bench_resize_affine.py [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM_BPS = 3.35e12


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def _frames(n, w, h):
    from tests.helpers import Fixtures
    fx = Fixtures()
    base = [cv2.resize(f, (w, h), interpolation=cv2.INTER_AREA) if f.shape[:2] != (h, w) else f for f in fx.frames()]
    rng = np.random.default_rng(5)
    return np.stack([np.clip(base[i % 4].astype(np.int16) + rng.integers(-3, 4, (h, w, 3)), 0, 255).astype(np.uint8)
                     for i in range(n)])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    import torch
    from cameracalibration_b200 import _lib as L
    from cameracalibration_b200 import ops
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU form")
    ctx = L.Context(0)
    dev = torch.device("cuda", 0)
    cams = _frames(32, 1280, 1024)
    bev = _frames(32, 1000, 1000)
    M = np.float32([[1, 0, 640 - 600], [0, 1, 512 - 530]])
    work = [("resize_linear_640x480", cams, lambda f: cv2.resize(f, (640, 480)),
             lambda d, o: ops.resize(d, (640, 480), ctx=ctx, out=o), (640, 480)),
            ("resize_linear_2560x2048", cams, lambda f: cv2.resize(f, (2560, 2048)),
             lambda d, o: ops.resize(d, (2560, 2048), ctx=ctx, out=o), (2560, 2048)),
            ("resize_area_640x512", cams, lambda f: cv2.resize(f, (640, 512), interpolation=cv2.INTER_AREA),
             lambda d, o: ops.resize(d, (640, 512), interpolation=cv2.INTER_AREA, ctx=ctx, out=o), (640, 512)),
            ("resize_area_427x341", cams, lambda f: cv2.resize(f, (427, 341), interpolation=cv2.INTER_AREA),
             lambda d, o: ops.resize(d, (427, 341), interpolation=cv2.INTER_AREA, ctx=ctx, out=o), (427, 341)),
            ("resize_bev_linear_500x500", bev, lambda f: cv2.resize(f, (500, 500)),
             lambda d, o: ops.resize(d, (500, 500), ctx=ctx, out=o), (500, 500)),
            ("warp_affine_translate_1280x1024", cams, lambda f: cv2.warpAffine(f, M, (1280, 1024)),
             lambda d, o: ops.warp_affine(d, M, (1280, 1024), ctx=ctx, out=o), (1280, 1024))]
    res = {"card": _card(), "batch": 32, "reps": args.reps, "workloads": {}}
    cv2.setNumThreads(1)
    cores = os.cpu_count() or 1
    for name, frames, host, call, (dw, dh) in work:
        n = frames.shape[0]
        d = torch.from_numpy(frames).to(dev)
        o = torch.empty((n, dh, dw, 3), dtype=torch.uint8, device=dev)
        for _ in range(3):
            call(d, o)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            call(d, o)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.reps
        got = o.cpu().numpy()
        t0 = time.perf_counter()
        with ThreadPoolExecutor(cores) as ex:
            want = list(ex.map(host, list(frames)))
        cpu_ms = (time.perf_counter() - t0) * 1e3
        same = all((g == w).all() for g, w in zip(got, want))
        moved = frames.nbytes + got.nbytes
        res["workloads"][name] = dict(kernel_ms_per_batch=round(ms, 4), kernel_us_per_frame=round(ms * 1e3 / n, 2),
                                      bytes_per_batch=int(moved), achieved_GBps=round(moved / (ms * 1e-3) / 1e9, 1),
                                      share_of_hbm_datasheet=round(moved / (ms * 1e-3) / HBM_BPS, 3),
                                      cv2_ms_per_batch=round(cpu_ms, 2), cv2_threads=cores, byte_identical=bool(same))
        if not same:
            raise SystemExit(f"{name}: device output differs from cv2")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
