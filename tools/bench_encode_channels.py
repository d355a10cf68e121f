#!/usr/bin/env python
"""Grey and BGRA images through the device encoders (ops.imencode: bevk_jpeg_encode_channels / bevk_png_encode_channels)
against cv2.imencode over all host cores.  One JSON line with the card's name and power limit read in the same run.

    grey   32 device-resident grey 1280x1024 frames (the reference's camera frame size): the fixture camera frames
           converted with cv2.COLOR_BGR2GRAY
    bgra   32 device-resident BGRA 1000x1000 images: BEV-sized, the fixture frames resized with an alpha ramp

each at JPEG q95, progressive JPEG, PNG defaults and PNG level 9.  Per workload and option: kernel time
(bevk_last_kernel_ms, CUDA events around the encoder's kernels; median of --iters calls after --warmup), images/s, stream
bytes, and cv2.imencode of the same images over all cores (one image per thread).  Every GPU stream is checked byte for
byte against cv2's.

    python tools/bench_encode_channels.py [--iters 20] [--warmup 3] [--options jpeg,progressive,png,png9]
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

OPTIONS = {"jpeg": (".jpg", []), "progressive": (".jpg", [cv2.IMWRITE_JPEG_PROGRESSIVE, 1]), "png": (".png", []),
           "png9": (".png", [cv2.IMWRITE_PNG_COMPRESSION, 9])}


def _workloads():
    import torch
    from tests.helpers import Fixtures
    fx = Fixtures()
    grey, bgra = [], []
    ramp = np.tile(np.linspace(0, 255, 1000, dtype=np.uint8), (1000, 1))[..., None]
    for b in range(32):
        frames = fx.perturbed_frames(1280, 1024, b)
        grey.append(cv2.cvtColor(frames[b % 4], cv2.COLOR_BGR2GRAY)[..., None])
        bgra.append(np.concatenate([cv2.resize(frames[(b + 1) % 4], (1000, 1000), interpolation=cv2.INTER_AREA), ramp], -1))
    return [("grey_32x1280x1024", torch.from_numpy(np.stack(grey)).cuda()),
            ("bgra_32x1000x1000", torch.from_numpy(np.stack(bgra)).cuda())]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--options", default=",".join(OPTIONS))
    args = ap.parse_args()
    from cameracalibration_b200 import _lib as L
    from cameracalibration_b200 import ops
    ctx = L.default_context()
    res = {"card": _card(), "workloads": {}}
    for name, imgs in _workloads():
        host = imgs.cpu().numpy()
        host = host[..., 0] if host.shape[-1] == 1 else host
        w = {}
        for opt in args.options.split(","):
            ext, params = OPTIONS[opt]
            for _ in range(args.warmup):
                ops.imencode(ext, imgs, params, ctx=ctx)
            ms = []
            for _ in range(args.iters):
                got = ops.imencode(ext, imgs, params, ctx=ctx)
                m = ctypes.c_float()
                L.check(ctx.lib.bevk_last_kernel_ms(ctx.h, ctypes.byref(m)))
                ms.append(m.value)
            with ThreadPoolExecutor(os.cpu_count()) as ex:
                t0 = time.perf_counter()
                want = list(ex.map(lambda i: cv2.imencode(ext, i, params)[1].tobytes(), host))
                cpu_s = time.perf_counter() - t0
            kern = float(np.median(ms))
            w[opt] = {"kernel_ms": round(kern, 3), "kernel_ms_min": round(min(ms), 3), "kernel_ms_max": round(max(ms), 3),
                      "images_per_s": round(len(host) / kern * 1e3, 1), "bytes": sum(map(len, got)),
                      "cv2_all_cores_ms": round(cpu_s * 1e3, 1), "host_cores": os.cpu_count(),
                      "cv2_images_per_s": round(len(host) / cpu_s, 1), "identical": got == want}
            assert got == want, (name, opt)
        res["workloads"][name] = w
    print(json.dumps(res))


if __name__ == "__main__":
    main()
