#!/usr/bin/env python
"""What cv2's point functions cost on the device: ops.undistort_points (5-coefficient pinhole with R and P, cv2's 5
iterations), ops.fisheye_undistort_points (cv2's default COUNT | EPS, 10, 1e-8), ops.project_points,
ops.fisheye_distort_points and ops.perspective_transform on device-resident points, at 1 M and 16 M points, float32 (and
float64 for the two pinhole calls).  Per call from CUDA events around repeated calls after a warm-up.  cv2's point
functions are single-threaded loops: each is timed with a host clock on 1 M points (best of 3 after one warm call) and
scaled to the size.  Bytes moved are computed from the shapes (8 or 16
bytes in per 2-D point, 12 or 24 per 3-D point, 8 or 16 out).  One JSON line, with the card's name and power limit read
in the same run.

    python tools/bench_points.py [--sizes 1048576,16777216] [--out results.json]
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


def _ms(torch, call):
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
        torch.cuda.synchronize()
        t = e0.elapsed_time(e1)
        if t > 200 or reps >= 4096:
            return t / reps
        reps *= 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1048576,16777216")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import cv2
    import torch
    from cameracalibration_b200 import ops
    from tests import points_cases as PC
    K, D5, Df = PC.K, np.array([-0.3, 0.12, 1e-3, -2e-3, -0.02]), PC.D_FISH
    rv, tv = np.array([0.3, -0.2, 0.1]), np.array([0.1, 0.2, 0.5])
    calls = {
        "undistort_points": (2, True, lambda p: ops.undistort_points(p, K, D5, R=PC.R_MAT, P=PC.P_NEW),
                             lambda p: cv2.undistortPoints(p, K, D5, R=PC.R_MAT, P=PC.P_NEW)),
        "fisheye_undistort_points": (2, False, lambda p: ops.fisheye_undistort_points(p, K, Df, P=PC.P_NEW),
                                     lambda p: cv2.fisheye.undistortPoints(p, K, Df, P=PC.P_NEW)),
        "project_points": (3, True, lambda p: ops.project_points(p, rv, tv, K, D5)[0],
                           lambda p: cv2.projectPoints(p, rv, tv, K, D5)[0]),
        "fisheye_distort_points": (2, False, lambda p: ops.fisheye_distort_points(p, K, Df),
                                   lambda p: cv2.fisheye.distortPoints(p, K, Df)),
        "perspective_transform": (2, False, lambda p: ops.perspective_transform(p, PC.H),
                                  lambda p: cv2.perspectiveTransform(p, PC.H)),
    }
    rng = np.random.default_rng(0)
    res = {"card": _card(), "cv2": cv2.__version__ + ", one host thread per call", "results": []}
    for name, (k, f64, dev, ref) in calls.items():
        for dt in (np.float32, np.float64) if f64 else (np.float32,):
            host = (rng.uniform(0, 640, (1 << 20, 1, k)) + ([0, 0, 2] if k == 3 else 0)).astype(dt)
            ref(host)
            cv2_ms_1m = float("inf")
            for _ in range(3):
                t0 = time.perf_counter()
                ref(host)
                cv2_ms_1m = min(cv2_ms_1m, (time.perf_counter() - t0) * 1e3)
            for n in (int(s) for s in a.sizes.split(",")):
                pts = torch.from_numpy(np.resize(host, (n, 1, k))).cuda()
                ms = _ms(torch, lambda: dev(pts))
                nbytes = n * np.dtype(dt).itemsize * (k + 2)
                res["results"].append({"op": name, "dtype": np.dtype(dt).name, "n": n, "device_ms": round(ms, 4),
                                       "GB_per_s": round(nbytes / ms / 1e6, 1),
                                       "cv2_host_ms_scaled": round(cv2_ms_1m * n / (1 << 20), 2)})
                del pts
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
