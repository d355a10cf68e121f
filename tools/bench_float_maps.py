#!/usr/bin/env python
"""What following cv2's float maps costs the undistortion on the device: the cv2.stereoRectify pair of
tests/float_map_cases.py (1280x720, 5-coefficient pinholes, R1 / R2), batches of 1 and 128 device frames, 3 channels,
INTER_LINEAR.  Slots: CV_16SC2 map-resident and fused, CV_32FC1 and CV_32FC2 map-resident (8 map bytes per pixel
instead of 6), CV_32FC1 fused; plus ops.remap with device CV_32FC1 maps (bevk_remap_f32_stack).  Per frame from CUDA
events around repeated calls (about 0.2 s per point after a warm-up), the configurations alternated over --rounds
rounds and the best round kept.  cv2.remap with CV_32FC1 maps over the host cores (cv2's own threads) is timed with a
host clock on the same frames.  One JSON line, with the card's name and power limit read in the same run.

    python tools/bench_float_maps.py [--batches 1,128] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

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


def _per_frame_ms(torch, call, n):
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 1
    while True:
        e0.record()
        for _ in range(reps):
            call()
        e1.record()
        e1.synchronize()
        total = e0.elapsed_time(e1)
        if total > 200 or reps >= 4096:
            return total / reps / n
        reps *= 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,128")
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import cv2
    import torch
    from cameracalibration_b200 import _lib as L
    from cameracalibration_b200 import ops
    from tests import float_map_cases as FC
    batches = [int(b) for b in a.batches.split(",")]
    cams = [FC.case_by_name("stereo_left"), FC.case_by_name("stereo_right")]
    W, H = cams[0].W, cams[0].H
    rng = np.random.default_rng(0)
    nmax = max(batches)
    host = rng.integers(0, 256, (nmax, H, W, 3), dtype=np.uint8)
    frames = torch.from_numpy(host).cuda()
    out = torch.empty((nmax, H, W, 3), dtype=torch.uint8, device="cuda")
    slots = {"16SC2/map": (ops.CV_16SC2, False), "16SC2/fused": (ops.CV_16SC2, True), "32FC1/map": (ops.CV_32FC1, False),
             "32FC2/map": (ops.CV_32FC2, False), "32FC1/fused": (ops.CV_32FC1, True)}
    calls = {}
    for c in cams:
        side = c.name.split("_")[-1]
        ctx = L.Context(0)   # one per camera: a context has 8 undistorter slots
        for key, (t, fused) in slots.items():
            u = ops.Undistorter(c.K, c.D, c.P, (W, H), "pinhole", fused=fused, ctx=ctx, R=c.R, m1type=t)
            for n in batches:
                calls[f"{side}/{key}/n{n}"] = (lambda u=u, n=n: u.cuda(frames[:n], out=out[:n]), n, u)
        mx, my = cv2.initUndistortRectifyMap(c.K, c.D, c.R, c.P, (W, H), cv2.CV_32FC1)
        dx, dy = torch.from_numpy(mx).cuda(), torch.from_numpy(my).cuda()
        for n in batches:
            calls[f"{side}/remap_32FC1_device_maps/n{n}"] = (
                lambda n=n, dx=dx, dy=dy, ctx=ctx: ops.remap(frames[:n], dx, dy, cv2.INTER_LINEAR, ctx=ctx, out=out[:n]), n, None)
    best = {}
    for _ in range(a.rounds):   # alternate the configurations; keep each one's best round
        for key, (call, n, _) in calls.items():
            ms = _per_frame_ms(torch, call, n)
            best[key] = min(best.get(key, float("inf")), ms)
    res = {"card": _card(), "frame": f"{W}x{H}x3", "gather_ms_per_frame": {k: round(v, 5) for k, v in best.items()}}
    # cv2.remap with CV_32FC1 maps on the host cores, over the same frames
    cpu = {}
    for c in cams:
        mx, my = cv2.initUndistortRectifyMap(c.K, c.D, c.R, c.P, (W, H), cv2.CV_32FC1)
        n = min(nmax, 32)
        cv2.remap(host[0], mx, my, cv2.INTER_LINEAR)
        t = time.perf_counter()
        for i in range(n):
            cv2.remap(host[i], mx, my, cv2.INTER_LINEAR)
        cpu[c.name.split("_")[-1]] = round((time.perf_counter() - t) * 1e3 / n, 4)
    res["cv2_remap_32FC1_ms_per_frame"] = cpu
    res["cv2_threads"] = cv2.getNumThreads()
    res["host_cpus"] = os.cpu_count()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
