"""Device time per frame of the gathers under each cv2 border mode, batches of 128 CUDA frames: 1920x1080 rectification
through a map-resident CV_16SC2 Undistorter slot at 8UC3 LINEAR (word path), 8UC1 LINEAR, 8UC3 CUBIC and 32FC1 LINEAR,
and a zoomed-out warpAffine of 8UC3 LINEAR frames in which most pixels fall outside the source (warpPerspective has no
device-batch form).  BORDER_TRANSPARENT writes into the destination in place; 32F LINEAR under it is refused and skipped.
Each case also times cv2 on the host cores over one frame, and checks the device result against it.  Prints one JSON line
per case and the card's name and power limit, read in the same run; --out writes them all.

    python tools/bench_remap_border.py [--reps 10] [--out results.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

W, H, N = 1920, 1080, 128
MODES = {"constant": 0, "replicate": 1, "reflect": 2, "wrap": 3, "reflect_101": 4, "transparent": 5}


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import cv2
    import torch
    from cameracalibration_b200 import ops
    K = np.array([[1000.0, 0, 961.5], [0, 1002.0, 538.25], [0, 0, 1]])
    D = np.array([-0.28, 0.09, 0.001, -0.0005, -0.012])
    P = K.copy()
    P[0, 0] *= 0.6   # zoomed out: the frame's edges and the border both show
    P[1, 1] *= 0.6
    u = ops.Undistorter(K, D, P, (W, H), model="pinhole")
    m1, m2 = u.maps()
    M = np.array([[0.4, 0.05, 700.0], [-0.05, 0.4, 400.0]])   # a quarter-size image in the middle of the canvas
    cases = [("rectify", "8uc3", np.uint8, 3, cv2.INTER_LINEAR), ("rectify", "8uc1", np.uint8, 1, cv2.INTER_LINEAR),
             ("rectify", "8uc3", np.uint8, 3, cv2.INTER_CUBIC), ("rectify", "32fc1", np.float32, 1, cv2.INTER_LINEAR),
             ("warp_affine_out", "8uc3", np.uint8, 3, cv2.INTER_LINEAR)]
    rows, info = [], card()
    print(json.dumps({"card": info}))
    rng = np.random.default_rng(0)
    for what, tname, dt, ch, inter in cases:
        base = rng.integers(0, 256, (H, W, ch)).astype(dt)
        frames = torch.from_numpy(base).cuda().expand(N, H, W, ch).contiguous()
        out = torch.zeros_like(frames)
        host = base if ch > 1 else base[..., 0]
        for mname, mode in MODES.items():
            if mode == 5 and dt == np.float32 and inter == cv2.INTER_LINEAR:
                continue
            bv = (40, 80, 120, 0)
            if what == "rectify":
                dev = lambda: u.cuda(frames, out, interpolation=inter, borderMode=mode, borderValue=bv)
                ref = lambda d: cv2.remap(host, m1, m2, inter, dst=d, borderMode=mode, borderValue=bv)
            else:
                dev = lambda: ops.warp_affine_border(frames, M, (W, H), inter, borderMode=mode, borderValue=bv, out=out)
                ref = lambda d: cv2.warpAffine(host, M, (W, H), dst=d, flags=inter, borderMode=mode, borderValue=bv)
            out.zero_()
            dev()                                  # warm-up: module load
            torch.cuda.synchronize()
            path = ops.last_path()
            want = ref(np.zeros_like(host)).reshape(H, W, ch)
            assert (out[0].cpu().numpy() == want).all() and (out[-1].cpu().numpy() == want).all(), (what, tname, mname)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.reps):
                dev()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / args.reps
            d = np.zeros_like(host)
            ref(d)                                 # warm-up: cv2's first call
            t0 = time.perf_counter()
            for _ in range(3):
                ref(d)
            host_ms = (time.perf_counter() - t0) / 3 * 1e3
            row = dict(case=what, type=tname, interp=inter, border=mname, batch=N, us_per_frame=round(ms / N * 1e3, 2),
                       cv2_host_ms_per_frame=round(host_ms, 3), path=path, card=info)
            rows.append(row)
            print(json.dumps(row), flush=True)
        del frames, out
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": info, "cv2": cv2.__version__, "host_cores": os.cpu_count(), "reps": args.reps, "rows": rows}, f,
                      indent=1)


if __name__ == "__main__":
    main()
