#!/usr/bin/env python
"""Progressive JPEG on the device (bevk_jpeg_encode_params with IMWRITE_JPEG_PROGRESSIVE) against the device's default
and OPTIMIZE paths and cv2.imencode progressive over all host cores.  One JSON line with the card's name and power limit
read in the same run.

    canvases  32 device-resident 1000x1000 BEV canvases (the bench workload's output)
    frames    8 undistorted 2560x2048 frames (Camera geometry, SIZE_SCALE 2)

both at quality 95.  Per workload and option: kernel time (CUDA events around the encoder's kernels, median of --iters
calls after --warmup), images/s, stream bytes, and cv2.imencode of the same images with the same parameters over all
cores (one image per thread).  Every GPU stream is checked byte for byte against cv2's.

    python tools/bench_jpeg_progressive.py [--iters 30] [--warmup 5]
"""
import argparse
import ctypes
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_jpeg_encode import _card, _workloads   # noqa: E402

OPTIONS = [("default", []), ("optimize", [cv2.IMWRITE_JPEG_OPTIMIZE, 1]), ("progressive", [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])]


def _bench(name, images, q, opt, params, iters, warmup, pool):
    from cameracalibration_b200 import _lib as L
    from cameracalibration_b200 import ops
    ctx = L.Context(images.device.index or 0)
    n, h, w, _ = images.shape
    cap = n * ops.jpeg_encode_params_bound(w, h, params)
    out = L.pinned_empty((cap,))
    sizes = (ctypes.c_uint64 * n)()
    ms = ctypes.c_float()
    arr = (ctypes.c_int * max(len(params), 1))(*params)
    call = lambda: L.check(ctx.lib.bevk_jpeg_encode_params(ctx.h, arr, len(params), ctypes.c_void_p(images.data_ptr()), h * w * 3,
                                                           w * 3, n, w, h, q, L.vptr(out), cap, sizes))
    for _ in range(warmup):
        call()
    kern = []
    for _ in range(iters):
        call()
        L.check(ctx.lib.bevk_last_kernel_ms(ctx.h, ctypes.byref(ms)))
        kern.append(ms.value)
    host = list(images.cpu().numpy())
    enc = lambda img: cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q] + params)[1].tobytes()
    want = list(pool.map(enc, host))
    off, identical = 0, True
    for i in range(n):
        identical &= out[off:off + sizes[i]].tobytes() == want[i]
        off += sizes[i]
    reps = 3
    t0 = time.perf_counter()
    for _ in range(reps):
        list(pool.map(enc, host))
    allc = (time.perf_counter() - t0) / reps
    ctx.close()
    k = float(np.median(kern))
    return {"workload": name, "option": opt, "params": params, "images": n, "quality": q, "stream_bytes": int(sum(sizes)),
            "byte_identical_to_cv2": bool(identical), "gpu_kernel_ms": k,
            "gpu_kernel_ms_min": float(np.min(kern)), "gpu_kernel_ms_max": float(np.max(kern)),
            "gpu_kernel_images_per_s": n / (k / 1e3), "cv2_all_cores_images_per_s": n / allc}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    cv2.setNumThreads(1)
    cores = os.cpu_count() or 1
    res = []
    with ThreadPoolExecutor(cores) as pool:
        for name, imgs, _q in _workloads():
            name = name.rsplit("_q", 1)[0] + "_q95"
            res += [_bench(name, imgs, 95, opt, params, a.iters, a.warmup, pool) for opt, params in OPTIONS]
    print(json.dumps({"tool": "bench_jpeg_progressive", "card": _card(), "host_threads": cores, "results": res}))


if __name__ == "__main__":
    main()
