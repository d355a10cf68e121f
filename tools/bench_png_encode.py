#!/usr/bin/env python
"""Device PNG encoder (bevk_png_encode) against cv2.imencode('.png') over all host cores.  One JSON line with the card's
name and power limit read in the same run.

    canvases  32 device-resident 1000x1000 BEV canvases (the bench workload's output)
    frames    32 undistorted 1920x1080 frames (the front camera's calibration, 1280x1024 sources)

under cv2's defaults (SUB, level 1, Z_RLE) and IMWRITE_PNG_STRATEGY_HUFFMAN_ONLY.  Per workload and option: kernel time
(bevk_last_kernel_ms, CUDA events around the encoder's kernels; median of --iters calls after --warmup), images/s,
stream bytes, and cv2.imencode of the same images over all cores (one image per thread).  Every GPU stream is checked
byte for byte against cv2's.

    python tools/bench_png_encode.py [--iters 20] [--warmup 3]
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

from bench_jpeg_encode import _card   # noqa: E402


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
    P = C.dst_camera_matrix(K, 1280, 1024, 1, 1.5)
    u = ops.Undistorter(K, D, P, (1920, 1080))
    und = [u(fx.perturbed_frames(1280, 1024, b)[b % 4]) for b in range(32)]
    return [("canvases_32x1000x1000", canvases), ("undistorted_32x1920x1080", torch.from_numpy(np.stack(und)).cuda())]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    from cameracalibration_b200 import _lib as L
    from cameracalibration_b200 import ops
    ctx = L.default_context()
    res = {"card": _card(), "workloads": {}}
    for name, imgs in _workloads():
        host = imgs.cpu().numpy()
        w = {}
        for opt, params in (("default", []), ("huffman_only", [cv2.IMWRITE_PNG_STRATEGY, cv2.IMWRITE_PNG_STRATEGY_HUFFMAN_ONLY])):
            for _ in range(args.warmup):
                ops.png_encode(imgs, ctx=ctx, params=params)
            ms = []
            for _ in range(args.iters):
                got = ops.png_encode(imgs, ctx=ctx, params=params)
                m = ctypes.c_float()
                L.check(ctx.lib.bevk_last_kernel_ms(ctx.h, ctypes.byref(m)))
                ms.append(m.value)
            with ThreadPoolExecutor(os.cpu_count()) as ex:
                t0 = time.perf_counter()
                want = list(ex.map(lambda i: cv2.imencode(".png", i, params)[1].tobytes(), host))
                cpu_s = time.perf_counter() - t0
            kern = float(np.median(ms))
            w[opt] = {"kernel_ms": round(kern, 3), "images_per_s": round(len(host) / kern * 1e3, 1),
                      "bytes": sum(map(len, got)), "cv2_all_cores_ms": round(cpu_s * 1e3, 1), "host_cores": os.cpu_count(),
                      "cv2_images_per_s": round(len(host) / cpu_s, 1), "identical": got == want}
            assert got == want, (name, opt)
        res["workloads"][name] = w
    print(json.dumps(res))


if __name__ == "__main__":
    main()
