#!/usr/bin/env python
"""What cv2's wider lens models cost the undistortion on the device: fisheye-4, pinhole-5, rational-8, thin-prism-12 and
tilted-14 cameras (the reference's front camera K; seeded mild D), map-resident and fused slots, 1280x1024 frames ->
1280x1024 and -> 2560x2048, batches 1 and 128, 3 channels, INTER_LINEAR.  Per frame from CUDA events around repeated
Undistorter.cuda calls (about 0.2 s per point after a warm-up); plus the map build (bevk_undistorter_set_rectify of a
map-resident slot) and bevk_bev_set_camera_model, host clock around the call and a device synchronise; and the map build
of the fisheye and of the rational-8 pinhole rotated by a stereo-rectification-sized R (0.05 rad), whose rays are walked
row by row first (k_walk_rays).
One JSON line, with the card's name and power limit read in the same run.

    python tools/bench_lens_models.py [--batches 1,128] [--sizes 1280x1024,2560x2048]
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
FW, FH = 1280, 1024
CAMERAS = ("fisheye4", "pinhole5", "rational8", "thinprism12", "tilted14")


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def _camera(name, dst):
    """(model, K, D, P) of the named camera for undistorted size dst."""
    from oracle import cv2_path as C
    from tests.helpers import Fixtures
    from tests import lens_cases as LC
    K, D4, _ = Fixtures().calib["front"]
    P = C.dst_camera_matrix(K, FW, FH, 1, dst[0] / FW)
    if name == "fisheye4":
        return "fisheye", K, np.asarray(D4, np.float64).ravel(), P
    n = int("".join(ch for ch in name if ch.isdigit()))
    return "pinhole", K, LC._pinhole_D(np.random.default_rng(n), n, False), P


def _per_frame_ms(torch, u, frames, out, n):
    for _ in range(3):
        u.cuda(frames[:n], out=out[:n])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps, total = 1, 0.0
    while True:
        e0.record()
        for _ in range(reps):
            u.cuda(frames[:n], out=out[:n])
        e1.record()
        e1.synchronize()
        total = e0.elapsed_time(e1)
        if total > 200 or reps >= 4096:
            return total / reps / n
        reps *= 2


def _setup_ms(ctx, fn, times=5):
    ctx.sync()
    best = float("inf")
    for _ in range(times):
        t = time.perf_counter()
        fn()
        ctx.sync()
        best = min(best, (time.perf_counter() - t) * 1e3)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,128")
    ap.add_argument("--sizes", default="1280x1024,2560x2048")
    a = ap.parse_args()
    import torch
    from cameracalibration_b200 import _lib as L
    from cameracalibration_b200 import ops
    batches = [int(b) for b in a.batches.split(",")]
    sizes = [tuple(int(v) for v in s.split("x")) for s in a.sizes.split(",")]
    res = {"card": _card(), "gather_ms_per_frame": {}, "map_build_ms": {}, "bev_set_camera_ms": {}, "walked_map_build_ms": {}}
    import cv2
    R = cv2.Rodrigues(np.array([0.03, -0.02, 0.035]))[0]
    rng = np.random.default_rng(0)
    frames = torch.from_numpy(rng.integers(0, 256, (max(batches), FH, FW, 3), dtype=np.uint8)).cuda()
    ctx = L.Context(0)
    for dst in sizes:
        out = torch.empty((max(batches), dst[1], dst[0], 3), dtype=torch.uint8, device="cuda")
        for cam in CAMERAS:
            model, K, D, P = _camera(cam, dst)
            for fused in (False, True):
                u = ops.Undistorter(K, D, P, dst, model=model, fused=fused, ctx=ctx, R=np.eye(3))
                for n in batches:
                    key = f"{cam}/{dst[0]}x{dst[1]}/{'fused' if fused else 'map'}/n{n}"
                    res["gather_ms_per_frame"][key] = round(_per_frame_ms(torch, u, frames, out, n), 5)
                if not fused:
                    res["map_build_ms"][f"{cam}/{dst[0]}x{dst[1]}"] = round(_setup_ms(
                        ctx, lambda: ops.Undistorter(K, D, P, dst, model=model, ctx=ctx, slot=7, R=np.eye(3)).close()), 3)
                u.close()
            eng = ops.BevEngine(1, (FW, FH), (1000, 1000), ctx=ctx)
            H = np.array([[0.5, 0, 10], [0, 0.5, 10], [0, 1e-4, 1.0]])
            res["bev_set_camera_ms"][f"{cam}/{dst[0]}x{dst[1]}"] = round(_setup_ms(
                ctx, lambda: eng.set_camera(0, K, D, P, dst, H, model=model)), 3)
        for cam in ("fisheye4", "rational8"):
            model, K, D, P = _camera(cam, dst)
            res["walked_map_build_ms"][f"{cam}/{dst[0]}x{dst[1]}"] = round(_setup_ms(
                ctx, lambda: ops.Undistorter(K, D, P, dst, model=model, ctx=ctx, slot=7, R=R).close()), 3)
        del out
    print(json.dumps(res))


if __name__ == "__main__":
    main()
