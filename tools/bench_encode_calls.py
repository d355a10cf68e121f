#!/usr/bin/env python
"""Whole-call wall time of the device encoders' Python entry points on 32 device-resident 1000x1000 BEV canvases (the
bench workload's output): what a caller waits for, from the call to the streams in host memory as ``bytes``.  One JSON
line with the card's name and power limit read in the same run, and a digest of every call's streams, so that two
builds (BEVK_LIB_PATH) can be compared on time and bytes.

    jpeg             ops.jpeg_encode(canvases, 95)
    jpeg_progressive ops.jpeg_encode_params(canvases, [IMWRITE_JPEG_PROGRESSIVE, 1], 95)
    png              ops.png_encode(canvases)                                   cv2's defaults
    png_level9       ops.png_encode(canvases, [IMWRITE_PNG_COMPRESSION, 9])     zlib's hash-chain parse
    bev_to_jpeg      BevEngine.cuda_to_jpeg(frame-sets, 95)                     render + encode, chunks of 8 canvases

Each figure is the median host-clock time of --iters calls after --warmup (every call ends in a synchronise).

    python tools/bench_encode_calls.py [--iters 20] [--warmup 3]
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    from oracle import cv2_path as C
    from oracle import restate as R
    from tests.helpers import NAMES, Fixtures
    from cameracalibration_b200 import _lib as L
    from cameracalibration_b200 import ops
    fx = Fixtures()
    g = fx.geometry()
    e = ops.BevEngine(4, (g.FW, g.FH), (g.BW, g.BH))
    for i, n in enumerate(NAMES):
        K, D, H = fx.calib[n]
        e.set_camera(i, K, D, C.dst_camera_matrix(K, g.FW, g.FH, g.FS, g.SS), (int(g.FW * g.SS), int(g.FH * g.SS)), H)
        e.set_mask(i, R.blend_mask(n, g.BW, g.BH, g.CW, g.CH))
    e.finalize()
    frames = torch.from_numpy(np.stack([np.stack(fx.perturbed_frames(g.FW, g.FH, b)) for b in range(32)])).cuda()
    car = torch.from_numpy(fx.car()).cuda()
    canvases = e.run_cuda(frames, car=car)
    torch.cuda.synchronize()
    ctx = L.Context(canvases.device.index or 0)
    calls = {
        "jpeg": lambda: ops.jpeg_encode(canvases, 95, ctx=ctx),
        "jpeg_progressive": lambda: ops.jpeg_encode_params(canvases, [cv2.IMWRITE_JPEG_PROGRESSIVE, 1], 95, ctx=ctx),
        "png": lambda: ops.png_encode(canvases, ctx=ctx),
        "png_level9": lambda: ops.png_encode(canvases, ctx=ctx, params=[cv2.IMWRITE_PNG_COMPRESSION, 9]),
        "bev_to_jpeg": lambda: e.cuda_to_jpeg(frames, 95, car),
    }
    res = {}
    for name, call in calls.items():
        for _ in range(a.warmup):
            streams = call()
        t = []
        for _ in range(a.iters):
            t0 = time.perf_counter()
            call()
            t.append(time.perf_counter() - t0)
        res[name] = {"call_ms": float(np.median(t)) * 1e3, "spread_ms": [float(min(t)) * 1e3, float(max(t)) * 1e3],
                     "stream_bytes": sum(map(len, streams)), "sha256": hashlib.sha256(b"".join(streams)).hexdigest()[:16]}
    print(json.dumps({"tool": "bench_encode_calls", "card": _card(), "lib": L.LIB_PATH, "images": 32,
                      "width": g.BW, "height": g.BH, "iters": a.iters, "results": res}))


if __name__ == "__main__":
    main()
