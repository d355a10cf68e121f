#!/usr/bin/env python
"""Surround-view frame-sets straight to JPEG (bevk_bev_run_to_jpeg / bevk_bev_frames_to_jpeg) against the two-step paths
they replace.  One JSON line with the card's name and power limit read in the same run.

Workloads: the bench workload (32 x 4 x 1920x1080 -> 1000x1000, blend) and cfg3 (1920x1080 -> 1200x1200, blend +
balance), quality 95.  Per workload:
  host     frame-sets/s of BevEngine.run_to_jpeg on page-locked and on pageable host frames; of run() + cv2.imencode
           over all host cores (one canvas per thread); of the reference's cv2 path + cv2.imencode (one frame-set per
           thread, all cores, on a sample)
  device   frame-sets/s of BevEngine.cuda_to_jpeg on a device frame stack, in chunks of 8 canvases (the default: chunks
           that stay in the 50 MB L2) and the whole batch at once (BEVK_JPEG_CHUNK=0), against run_stack + ops.jpeg_encode
  d2h      bytes per frame-set that come back: the streams and their sizes, against the canvas
  kernels  (balance only) kernel ms per step of cuda_to_jpeg from torch.profiler, and the kernels it launches
Every stream is checked byte for byte against cv2.imencode of the canvas run() returns, and on the sample against the
reference's cv2 path (``files_byte_identical``).

    python tools/bench_bev_jpeg.py [--iters 20] [--warmup 3] [--ref-sample 8]
"""
import argparse
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

Q = 95


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def _median_s(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    t = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return float(np.median(t))


def _kernel_ms(fn, steps):
    """Kernel time per step (ms) from torch.profiler's CUDA activities, and the kernel names seen."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    tot, names = 0.0, {}
    for e in prof.events():
        if str(e.device_type).endswith("CUDA") and not e.name.startswith(("Memcpy", "Memset")):
            us = getattr(e, "device_time", None) or getattr(e, "cuda_time", 0.0)
            tot += us
            short = e.name.split("<")[0].split("(")[0].replace("void ", "").split("::")[-1]
            names[short] = names.get(short, 0.0) + us / 1e3 / steps
    return tot / 1e3 / steps, {k: round(v, 4) for k, v in sorted(names.items(), key=lambda kv: -kv[1])}


def _enc(img):
    return cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, Q])[1].tobytes()


def _workload(name, w, iters, warmup, ref_sample, pool):
    import torch
    import bench as B
    from cameracalibration_b200 import _lib as L
    from cameracalibration_b200 import ops
    from oracle import cv2_path as C
    from tests.helpers import Fixtures
    eng, calib, masks, g = B.build_engine(w, 0)
    n, bal = w["batch"], w["balance"]
    host = B.synthetic_frames(w["FW"], w["FH"], w["n_cam"], n, seed=7)
    pinned = L.pinned_empty(host.shape)
    pinned[...] = host
    sets_pageable = [[host[b, c] for c in range(w["n_cam"])] for b in range(n)]
    sets_pinned = [[pinned[b, c] for c in range(w["n_cam"])] for b in range(n)]
    car = Fixtures().car(w["BW"], w["BH"])
    car_d = torch.from_numpy(car).cuda()
    d = torch.from_numpy(host).cuda()
    res = {"workload": name, "frame_sets": n, "frame": [w["FW"], w["FH"]], "canvas": [w["BW"], w["BH"]], "blend": w["blend"],
           "balance": bal, "quality": Q}

    canvases = np.array(eng.run(sets_pageable, car, bal))
    want = list(pool.map(_enc, list(canvases)))
    got = {"pinned": eng.run_to_jpeg(sets_pinned, Q, car, bal), "pageable": eng.run_to_jpeg(sets_pageable, Q, car, bal),
           "device": eng.cuda_to_jpeg(d, Q, car_d, bal)}
    identical = all(v == want for v in got.values())
    # the reference's cv2 path on a sample of frame-sets, one per thread
    ref = C.RefBev(calib, C.Geometry(FW=g.FW, FH=g.FH, BW=g.BW, BH=g.BH, CW=g.CW, CH=g.CH), w["blend"], bal, masks=masks)
    sample = list(range(min(ref_sample, n)))
    ref_job = lambda b: _enc(ref(*sets_pageable[b], car))
    t0 = time.perf_counter()
    ref_streams = list(pool.map(ref_job, sample))
    ref_s = time.perf_counter() - t0
    files_identical = identical and all(ref_streams[i] == want[b] for i, b in enumerate(sample))

    fs = lambda s: n / s
    res["host_run_to_jpeg_pinned_frame_sets_per_s"] = fs(_median_s(lambda: eng.run_to_jpeg(sets_pinned, Q, car, bal), iters, warmup))
    res["host_run_to_jpeg_pageable_frame_sets_per_s"] = fs(_median_s(lambda: eng.run_to_jpeg(sets_pageable, Q, car, bal), iters, warmup))
    res["host_run_pinned_plus_cv2_all_cores_frame_sets_per_s"] = fs(_median_s(
        lambda: list(pool.map(_enc, list(eng.run(sets_pinned, car, bal)))), max(3, iters // 4), 1))
    res["reference_cv2_path_plus_imencode_all_cores_frame_sets_per_s"] = len(sample) / ref_s
    res["reference_sample"] = len(sample)

    out = torch.empty((n, g.BH, g.BW, 3), dtype=torch.uint8, device="cuda")
    fb = w["FW"] * w["FH"] * 3

    def two_step():
        eng.run_stack(d.data_ptr(), fb, n, out.data_ptr(), car_d.data_ptr(), bal)
        return ops.jpeg_encode(out, Q, ctx=eng.ctx)

    assert two_step() == want
    res["device_cuda_to_jpeg_chunks_of_8_frame_sets_per_s"] = fs(_median_s(lambda: eng.cuda_to_jpeg(d, Q, car_d, bal), iters, warmup))
    os.environ["BEVK_JPEG_CHUNK"] = "0"
    try:
        assert eng.cuda_to_jpeg(d, Q, car_d, bal) == want
        res["device_cuda_to_jpeg_whole_batch_frame_sets_per_s"] = fs(_median_s(lambda: eng.cuda_to_jpeg(d, Q, car_d, bal), iters, warmup))
    finally:
        del os.environ["BEVK_JPEG_CHUNK"]
    res["device_run_stack_plus_jpeg_encode_frame_sets_per_s"] = fs(_median_s(two_step, iters, warmup))

    res["d2h_bytes_per_frame_set_jpeg"] = (sum(len(s) for s in want) + 8 * n) / n
    res["d2h_bytes_per_frame_set_canvas"] = g.BW * g.BH * 3
    res["h2d_bytes_per_frame_set"] = eng.host_copy_bytes(bal)[0]

    if bal:
        res["kernel_ms_per_step"], res["kernels"] = _kernel_ms(lambda: eng.cuda_to_jpeg(d, Q, car_d, True), 10)
    res["byte_identical_to_cv2"] = bool(identical)
    res["files_byte_identical"] = bool(files_identical)
    eng.ctx.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ref-sample", type=int, default=8)
    a = ap.parse_args()
    import bench as B
    cv2.setNumThreads(1)      # cv2.imencode / remap per thread; the all-core figures use one image per thread
    cores = os.cpu_count() or 1
    with ThreadPoolExecutor(cores) as pool:
        res = [_workload("bench", dict(B.WORKLOAD), a.iters, a.warmup, a.ref_sample, pool),
               _workload("cfg3", {**B.WORKLOAD, **B.ALT_WORKLOADS["cfg3"]}, a.iters, a.warmup, a.ref_sample, pool)]
    print(json.dumps({"tool": "bench_bev_jpeg", "card": _card(), "host_threads": cores, "results": res}))


if __name__ == "__main__":
    main()
