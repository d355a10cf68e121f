#!/usr/bin/env python
"""Device PNG encoder (bevk_png_encode_params) against cv2.imencode('.png') over all host cores.  One JSON line with the card's
name and power limit read in the same run.

    canvases  32 device-resident 1000x1000 BEV canvases (the bench workload's output)
    frames    32 undistorted 1920x1080 frames (the front camera's calibration, 1280x1024 sources)
    words     8 synthetic 1000x1000 images strung together from 4 random 64-byte words: the hash-chain parse's
              bad case -- every 3-byte string about 128 times per window and matches of about 85 bytes, mostly below
              nice_match, so the device's search at every position costs about a match length times zlib's search at
              its parse steps

under cv2's defaults (SUB, level 1, Z_RLE), IMWRITE_PNG_STRATEGY_HUFFMAN_ONLY and zlib's hash-chain parse at
[IMWRITE_PNG_COMPRESSION, 6] and [.., 9] (cv2.imwrite's level 9 is what Tools/undistort.py writes by default; --options
picks a subset).  Per workload and option: kernel time
(bevk_last_kernel_ms, CUDA events around the encoder's kernels; median of --iters calls after --warmup), images/s,
stream bytes, and cv2.imencode of the same images over all cores (one image per thread).  Every GPU stream is checked
byte for byte against cv2's.

    python tools/bench_png_encode.py [--iters 20] [--warmup 3] [--options default,huffman_only,level6,level9]
                                     [--workloads canvases,frames,words]
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


def _words(n=8, side=1000, nwords=4, wlen=64, seed=17):
    import torch
    rng = np.random.default_rng(seed)
    words = rng.integers(0, 256, (nwords, wlen), dtype=np.uint8)
    per = 3 * side * side
    imgs = [words[rng.integers(0, nwords, per // wlen + 1)].reshape(-1)[:per].reshape(side, side, 3) for _ in range(n)]
    return torch.from_numpy(np.stack(imgs)).cuda()


def _workloads(which):
    out = []
    if "words" in which:
        out.append(("words_8x1000x1000", _words()))
    if not {"canvases", "frames"} & set(which):
        return out
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
    if "canvases" in which:
        out.append(("canvases_32x1000x1000", canvases))
    if "frames" in which:
        out.append(("undistorted_32x1920x1080", torch.from_numpy(np.stack(und)).cuda()))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--options", default="default,huffman_only,level6,level9")
    ap.add_argument("--workloads", default="canvases,frames,words")
    args = ap.parse_args()
    options = {"default": [], "huffman_only": [cv2.IMWRITE_PNG_STRATEGY, cv2.IMWRITE_PNG_STRATEGY_HUFFMAN_ONLY],
               "level6": [cv2.IMWRITE_PNG_COMPRESSION, 6], "level9": [cv2.IMWRITE_PNG_COMPRESSION, 9]}
    from cameracalibration_b200 import _lib as L
    from cameracalibration_b200 import ops
    ctx = L.default_context()
    res = {"card": _card(), "workloads": {}}
    for name, imgs in _workloads(args.workloads.split(",")):
        host = imgs.cpu().numpy()
        w = {}
        for opt in args.options.split(","):
            params = options[opt]
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
