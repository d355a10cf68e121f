#!/usr/bin/env python
"""Undistortion with INTER_LINEAR, INTER_CUBIC and INTER_LANCZOS4 (Undistorter.cuda, bevk_undistort_stack_interp) on the
fisheye front camera of the reference, against cv2.remap with the same interpolation over all host cores.  One JSON
line, with the card's name and power limit read in the same run.

    sizes    1280x1024 -> 1280x1024 (Tools/undistort.py's default) and the fixture frames resized to 1920x1080 ->
             1920x1080
    kernel   map and fused slots, batches 1 and 128.  Kernel time from CUDA events around a CUDA graph of --reps calls,
             replayed until about 0.2 s have passed; per frame and frames/s.  The last frame of each batch is checked
             against cv2.remap.
    cv2      cv2.remap of 32 frames through cv2's maps, one frame per host core at a time (cv2.setNumThreads(1)).

    python tools/bench_remap_interp.py [--reps 10]
"""
import argparse
import ctypes
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
INTERS = {"linear": cv2.INTER_LINEAR, "cubic": cv2.INTER_CUBIC, "lanczos4": cv2.INTER_LANCZOS4}


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def _setup(size):
    """The front camera's K scaled to `size`, P for the same size (FOCAL_SCALE 1), cv2's maps, 8 distinct frames."""
    from oracle import cv2_path as C
    from tests.helpers import Fixtures
    fx = Fixtures()
    K, D, _ = fx.calib["front"]
    W, H = size
    K = np.diag([W / 1280, H / 1024, 1.0]) @ K
    P = C.dst_camera_matrix(K, W, H, 1, 1)
    frames = [fx.perturbed_frames(W, H, b)[b % 4] for b in range(8)]
    return K, D, P, C.undistort_maps(K, D, P, W, H), frames


def _kernel(size, fused, inter, batches, reps, K, D, P, maps, distinct):
    import torch
    from cameracalibration_b200 import _lib as L
    from cameracalibration_b200 import ops
    W, H = size
    u = ops.Undistorter(K, D, P, size, fused=fused, ctx=L.Context(0))
    nmax = max(batches)
    frames = torch.from_numpy(np.stack([distinct[i % len(distinct)] for i in range(nmax)])).cuda()
    out = torch.empty((nmax, H, W, 3), dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    res = []
    for n in batches:
        call = lambda: L.check(u.ctx.lib.bevk_undistort_stack_interp(u.ctx.h, u.slot, ctypes.c_void_p(frames.data_ptr()), W * H * 3,
                                                                     W, H, W * 3, 3, n, ctypes.c_void_p(out.data_ptr()), W * H * 3,
                                                                     W, H, W * 3, inter))
        with u.ctx.on_stream(s.cuda_stream):
            call()
            path = u.last_path()
            s.synchronize()
            with u.ctx.graph_capture() as g:
                for _ in range(reps):
                    call()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            g.launch()
            e0.record(s)
            g.launch()
            e1.record(s)
            e1.synchronize()
            launches = max(3, int(200.0 / max(e0.elapsed_time(e1), 1e-3)))
            e0.record(s)
            g.launch(launches)
            e1.record(s)
            e1.synchronize()
            ms = e0.elapsed_time(e1) / (launches * reps)
            g.destroy()
        last = out[n - 1].cpu().numpy()
        exact = bool((last == cv2.remap(distinct[(n - 1) % len(distinct)], maps[0], maps[1], inter)).all())
        res.append({"slot": "fused" if fused else "map", "batch": n, "path": path, "kernel_ms_per_call": ms,
                    "kernel_ms_per_frame": ms / n, "frames_per_s": n / ms * 1e3, "last_frame_equals_cv2": exact})
    u.close()
    return res


def _cv2(inter, maps, distinct, n=32):
    cores = os.cpu_count() or 1
    cv2.setNumThreads(1)
    work = [distinct[i % len(distinct)] for i in range(n)]
    f = lambda img: cv2.remap(img, maps[0], maps[1], inter)
    with ThreadPoolExecutor(cores) as pool:
        list(pool.map(f, work))                    # warm-up
        t0 = time.perf_counter()
        list(pool.map(f, work))
        dt = time.perf_counter() - t0
    return {"frames_per_s": n / dt, "host_threads": cores}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    res = {"tool": "bench_remap_interp", "card": _card(), "runs": []}
    for size in ((1280, 1024), (1920, 1080)):
        K, D, P, maps, distinct = _setup(size)
        for name, inter in INTERS.items():
            kern = []
            for fused in (False, True):
                kern += _kernel(size, fused, inter, (1, 128), a.reps, K, D, P, maps, distinct)
            res["runs"].append({"size": f"{size[0]}x{size[1]}", "interpolation": name, "kernel": kern,
                                "cv2_remap_all_cores": _cv2(inter, maps, distinct)})
    res["card_after"] = _card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
