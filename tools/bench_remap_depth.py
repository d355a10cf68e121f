"""Device time of 1920x1080 rectification at 8U, 16U and 32F (1 and 3 channels), batches of 1 and 128, through a
map-resident (CV_16SC2) and a fused Undistorter slot, INTER_LINEAR; and cv2.remap on the host cores over the same
frames.  Achieved bytes per second count the algorithmic bytes: the map (6 bytes per pixel, read once per GATHER_NB
frames; none when fused), the destination, and the source frames once.  Prints one JSON line per case and the card's
name and power limit, read in the same run; --out writes them all, with the run's card, cv2 version and host cores.
At n = 1 the events bracket whole calls, so they measure the Python and launch overhead of a call more than the kernel.

    python tools/bench_remap_depth.py [--reps 20] [--out results.json]
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

W, H = 1920, 1080
GATHER_NB = 8
DTYPES = {"8u": np.uint8, "16u": np.uint16, "32f": np.float32}


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import cv2
    import torch
    from cameracalibration_b200 import ops
    K = np.array([[1000.0, 0, 961.5], [0, 1002.0, 538.25], [0, 0, 1]])
    D = np.array([-0.28, 0.09, 0.001, -0.0005, -0.012])
    P = K.copy()
    P[0, 0] *= 0.8
    P[1, 1] *= 0.8
    slots = {fused: ops.Undistorter(K, D, P, (W, H), model="pinhole", fused=fused) for fused in (False, True)}
    m1, m2 = slots[False].maps()
    rows, info = [], card()
    print(json.dumps({"card": info}))
    rng = np.random.default_rng(0)
    for dname, dt in DTYPES.items():
        es = np.dtype(dt).itemsize
        for ch in (1, 3):
            base = rng.integers(0, 256, (H, W, ch)).astype(dt)
            cv2.remap(base if ch > 1 else base[..., 0], m1, m2, cv2.INTER_LINEAR)   # warm-up: cv2's first call
            t0 = time.perf_counter()
            for _ in range(3):
                cv2.remap(base if ch > 1 else base[..., 0], m1, m2, cv2.INTER_LINEAR)
            host_ms = (time.perf_counter() - t0) / 3 * 1e3
            for n in (1, 128):
                frames = torch.from_numpy(base).cuda().expand(n, H, W, ch).contiguous()
                out = torch.empty_like(frames)
                for fused, u in slots.items():
                    u.cuda(frames, out)                        # warm-up: module load
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.reps):
                        u.cuda(frames, out)
                    e1.record()
                    torch.cuda.synchronize()
                    ms = e0.elapsed_time(e1) / args.reps
                    want = cv2.remap(base if ch > 1 else base[..., 0], m1, m2, cv2.INTER_LINEAR).reshape(H, W, ch)
                    assert (out[0].cpu().numpy() == want).all() and (out[-1].cpu().numpy() == want).all(), (dname, ch, n, fused)
                    px = W * H
                    nbytes = (0 if fused else 6 * px * -(-n // GATHER_NB)) + 2 * n * px * ch * es
                    row = dict(depth=dname, channels=ch, batch=n, slot="fused" if fused else "map", ms_per_call=round(ms, 4),
                               ms_per_frame=round(ms / n, 5), gb_per_s=round(nbytes / ms / 1e6, 1),
                               cv2_host_ms_per_frame=round(host_ms, 3), path=u.last_path(), card=info)
                    rows.append(row)
                    print(json.dumps(row), flush=True)
                del frames, out
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": info, "cv2": cv2.__version__, "host_cores": os.cpu_count(), "reps": args.reps, "rows": rows}, f,
                      indent=1)


if __name__ == "__main__":
    main()
