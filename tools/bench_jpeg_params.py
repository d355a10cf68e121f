#!/usr/bin/env python
"""Device JPEG encoder under cv2.imwrite's JPEG parameters (bevk_jpeg_set_params) against cv2.imencode with the same
parameters over all host cores.  One JSON line with the card's name and power limit read in the same run.

    canvases  32 device-resident 1000x1000 BEV canvases (the bench workload's output)
    frames    8 undistorted 2560x2048 frames (Camera geometry, SIZE_SCALE 2)

both at quality 95, under: the default (4:2:0), 4:4:4, 4:2:2, OPTIMIZE, 4:4:4 + OPTIMIZE, one restart interval per
MCU row, and LUMA_QUALITY 90 / CHROMA_QUALITY 70 (which cv2 writes as 4:4:4).  Per workload and option: kernel time
(CUDA events around the encoder's kernels, median of --iters calls after --warmup), images/s, stream bytes, and
cv2.imencode of the same images over all cores (one image per thread); per workload the added kernel time of the
optimised tables (OPTIMIZE against the default).  Every GPU stream is checked byte for byte against cv2's.

    python tools/bench_jpeg_params.py [--iters 30] [--warmup 5]
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

S444 = [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, 0x111111]
OPT = [cv2.IMWRITE_JPEG_OPTIMIZE, 1]


def options(width):
    return [("default", []), ("444", S444), ("422", [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, 0x211111]), ("optimize", OPT),
            ("444_optimize", S444 + OPT), ("rst_per_mcu_row", [cv2.IMWRITE_JPEG_RST_INTERVAL, -(-width // 16)]),
            ("luma90_chroma70", [cv2.IMWRITE_JPEG_LUMA_QUALITY, 90, cv2.IMWRITE_JPEG_CHROMA_QUALITY, 70])]


def _bench(name, images, q, opt, params, iters, warmup, pool):
    from cameracalibration_b200 import _lib as L
    from cameracalibration_b200 import ops
    ctx = L.Context(images.device.index or 0)
    n, h, w, _ = images.shape
    cap = n * ops.jpeg_encode_bound(w, h, params)
    out = L.pinned_empty((cap,))
    sizes = (ctypes.c_uint64 * n)()
    ms = ctypes.c_float()
    ops.jpeg_set_params(ctx, params)
    call = lambda: L.check(ctx.lib.bevk_jpeg_encode(ctx.h, ctypes.c_void_p(images.data_ptr()), h * w * 3, w * 3, n, w, h, q,
                                                    L.vptr(out), cap, sizes))
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
    res, added = [], {}
    with ThreadPoolExecutor(cores) as pool:
        for name, imgs, _q in _workloads():
            name = name.rsplit("_q", 1)[0] + "_q95"
            rows = [_bench(name, imgs, 95, opt, params, a.iters, a.warmup, pool) for opt, params in options(imgs.shape[2])]
            ms = {r["option"]: r["gpu_kernel_ms"] for r in rows}
            added[name] = {"optimize_added_kernel_ms": ms["optimize"] - ms["default"],
                           "444_optimize_added_kernel_ms": ms["444_optimize"] - ms["444"]}
            res += rows
    print(json.dumps({"tool": "bench_jpeg_params", "card": _card(), "host_threads": cores, "results": res,
                      "optimize_cost": added}))


if __name__ == "__main__":
    main()
