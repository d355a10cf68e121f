#!/usr/bin/env python
"""Device JPEG encoder (bevk_jpeg_encode) against cv2.imencode on the host, for the two workloads it serves.  One JSON
line with the card's name and power limit read in the same run.

    canvases  32 device-resident 1000x1000 BEV canvases (the bench workload's output), quality 95
    frames    8 undistorted 2560x2048 frames (Camera geometry, SIZE_SCALE 2), quality 100

Per workload: kernel time (CUDA events around the encoder's kernels, averaged over --iters calls after --warmup), the
whole bevk_jpeg_encode call (wall clock; it ends in a synchronise after the streams reached host memory), and
cv2.imencode of the same images on one host thread and over all cores (one image per thread).  Every GPU stream is
checked byte for byte against cv2's.

    python tools/bench_jpeg_encode.py [--iters 50] [--warmup 5]
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


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def _workloads():
    from oracle import cv2_path as C
    from oracle import restate as R
    from tests.helpers import NAMES, Fixtures
    from cameracalibration_b200 import ops
    import torch
    fx = Fixtures()
    g = fx.geometry()
    e = ops.BevEngine(4, (g.FW, g.FH), (g.BW, g.BH))
    for i, n in enumerate(NAMES):
        K, D, H = fx.calib[n]
        e.set_camera(i, K, D, C.dst_camera_matrix(K, g.FW, g.FH, g.FS, g.SS), (int(g.FW * g.SS), int(g.FH * g.SS)), H)
        e.set_mask(i, R.blend_mask(n, g.BW, g.BH, g.CW, g.CH))
    e.finalize()
    frames = np.stack([np.stack(fx.perturbed_frames(g.FW, g.FH, b)) for b in range(32)])
    canvases = e.run_cuda(torch.from_numpy(frames).cuda(), car=torch.from_numpy(fx.car()).cuda())
    torch.cuda.synchronize()
    K, D, _ = fx.calib["front"]
    P = C.dst_camera_matrix(K, 1280, 1024, 1, 2)
    u = ops.Undistorter(K, D, P, (2560, 2048))
    und = []
    for b in range(8):
        src = fx.perturbed_frames(1280, 1024, b)[b % 4]
        und.append(u(src))
    return [("canvases_32x1000x1000_q95", canvases, 95), ("undistorted_8x2560x2048_q100", torch.from_numpy(np.stack(und)).cuda(), 100)]


def _bench(name, images, q, iters, warmup):
    from cameracalibration_b200 import _lib as L
    from cameracalibration_b200 import ops
    ctx = L.Context(images.device.index or 0)
    n, h, w, _ = images.shape
    cap = n * ops.jpeg_encode_bound(w, h)
    out = L.pinned_empty((cap,))
    sizes = (ctypes.c_uint64 * n)()
    ms = ctypes.c_float()
    call = lambda: L.check(ctx.lib.bevk_jpeg_encode(ctx.h, ctypes.c_void_p(images.data_ptr()), h * w * 3, w * 3, n, w, h, q,
                                                    L.vptr(out), cap, sizes))
    for _ in range(warmup):
        call()
    kern, wall = [], []
    for _ in range(iters):
        t0 = time.perf_counter()
        call()
        wall.append(time.perf_counter() - t0)
        L.check(ctx.lib.bevk_last_kernel_ms(ctx.h, ctypes.byref(ms)))
        kern.append(ms.value / 1e3)
    host = images.cpu().numpy()
    off, identical = 0, True
    for i in range(n):
        identical &= out[off:off + sizes[i]].tobytes() == cv2.imencode(".jpg", host[i], [cv2.IMWRITE_JPEG_QUALITY, q])[1].tobytes()
        off += sizes[i]
    enc = lambda img: cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q])
    reps = 3
    t0 = time.perf_counter()
    for _ in range(reps):
        for i in range(n):
            enc(host[i])
    one = (time.perf_counter() - t0) / reps
    cores = os.cpu_count() or 1
    with ThreadPoolExecutor(cores) as pool:
        list(pool.map(enc, list(host)))
        t0 = time.perf_counter()
        for _ in range(reps):
            list(pool.map(enc, list(host)))
        allc = (time.perf_counter() - t0) / reps
    in_bytes = n * h * w * 3
    k, wl = float(np.median(kern)), float(np.median(wall))
    return {"workload": name, "images": n, "width": w, "height": h, "quality": q, "stream_bytes": int(sum(sizes)),
            "byte_identical_to_cv2": bool(identical),
            "gpu_kernel_ms": k * 1e3, "gpu_kernel_images_per_s": n / k, "gpu_kernel_input_gbs": in_bytes / k / 1e9,
            "gpu_call_ms": wl * 1e3, "gpu_call_images_per_s": n / wl, "gpu_call_input_gbs": in_bytes / wl / 1e9,
            "cv2_1_thread_images_per_s": n / one, "cv2_1_thread_input_gbs": in_bytes / one / 1e9,
            "cv2_all_cores_images_per_s": n / allc, "cv2_all_cores_input_gbs": in_bytes / allc / 1e9, "host_threads": cores}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    cv2.setNumThreads(1)      # cv2.imencode is single-threaded; the all-core figure uses one image per thread
    res = [_bench(name, imgs, q, a.iters, a.warmup) for name, imgs, q in _workloads()]
    print(json.dumps({"tool": "bench_jpeg_encode", "card": _card(), "results": res}))


if __name__ == "__main__":
    main()
