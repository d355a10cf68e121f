#!/usr/bin/env python
"""BEV canvases written as NV12 / I420 (out_format, BEVK_FLAG_OUT_*) against BGR canvases, in one process.  One JSON line
with the card's name and power limit read in the same run, and the library that ran (BEVK_LIB_PATH selects an A/B
build, e.g. one compiled with -DBEVK_YUV_OUT_CHUNK=0).

Workloads: the bench workload (32 x 4 x 1920x1080 -> 1000x1000, blend) and cfg3 (1920x1080 -> 1200x1200, blend +
balance).  Per workload:
  device   ms per step of run_stack on a device BGR frame stack with BGR, NV12 and I420 canvases (CUDA events, median of
           blocks that alternate the three), and the kernel ms per step from torch.profiler, per kernel; the conversion
           pass (k_canvas_yuv) with the bytes it moves (3 read + 1.5 written per canvas pixel) per second
  host     frame-sets/s of BevEngine.run from page-locked NV12 frames: NV12 canvases, BGR canvases, and BGR canvases
           followed by host cv2.cvtColor(COLOR_BGR2YUV_I420) over all cores; bytes per frame-set each way
Every YUV canvas is checked against cvtColor of the BGR canvas (``byte_identical``).

    python tools/bench_yuv_out.py [--iters 10] [--warmup 2]
"""
import argparse
import json
import os
import sys
from concurrent.futures import ThreadPoolExecutor

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_yuv import _card, _kernel_ms, _median_s, _step_ms  # noqa: E402


def _workload(name, w, iters, warmup, pool):
    import torch
    import bench as B
    from cameracalibration_b200 import _lib as L
    from tests.yuv_frames import from_bgr, to_bgr
    eng, calib, masks, g = B.build_engine(w, 0)
    n, nc, bal = w["batch"], w["n_cam"], w["balance"]
    FW, FH, BW, BH = w["FW"], w["FH"], g.BW, g.BH
    bgr = B.synthetic_frames(FW, FH, nc, n, seed=7)
    nv12 = np.stack([np.stack([from_bgr(bgr[b, c], "nv12") for c in range(nc)]) for b in range(n)])
    pin_nv12 = L.pinned_empty(nv12.shape)
    pin_nv12[...] = nv12
    sets = lambda a: [[a[b, c] for c in range(nc)] for b in range(n)]
    res = {"workload": name, "frame_sets": n, "frame": [FW, FH], "canvas": [BW, BH], "blend": w["blend"], "balance": bal}

    d_bgr = torch.from_numpy(bgr).cuda()
    outs = {"bgr": torch.empty((n, BH, BW, 3), dtype=torch.uint8, device="cuda")}
    for f in ("nv12", "i420"):
        outs[f] = torch.empty((n, BH * 3 // 2, BW), dtype=torch.uint8, device="cuda")
    run = {f: (lambda f=f: eng.run_stack(d_bgr.data_ptr(), FW * FH * 3, n, outs[f].data_ptr(), 0, bal, out_format=f))
           for f in outs}
    for f in outs:
        run[f]()
    torch.cuda.synchronize()
    ok = all((outs[f].cpu().numpy() == np.stack([from_bgr(c, f) for c in outs["bgr"].cpu().numpy()])).all()
             for f in ("nv12", "i420"))
    host_bgr = np.array(eng.run(sets(pin_nv12), None, bal, pixel_format="nv12"))
    host_nv12 = np.array(eng.run(sets(pin_nv12), None, bal, pixel_format="nv12", out_format="nv12"))
    ok = ok and bool((host_nv12 == np.stack([from_bgr(c, "nv12") for c in host_bgr])).all())
    res["byte_identical"] = bool(ok)

    with eng.ctx.on_stream(torch.cuda.current_stream().cuda_stream):   # the events and the renders on one stream
        ms = _step_ms(torch, [run[f] for f in outs], iters, 20)
    for f, m in zip(outs, ms):
        res[f"device_ms_per_step_{f}_out"] = m
        res[f"device_frame_sets_per_s_{f}_out"] = n / m * 1e3
    conv_bytes = n * BW * BH * 4.5
    for f in outs:
        tot, names = _kernel_ms(run[f], 10)
        res[f"kernel_ms_per_step_{f}_out"], res[f"kernels_{f}_out"] = tot, names
        if f != "bgr":
            k = names.get("k_canvas_yuv", 0.0)
            res[f"k_canvas_yuv_ms_{f}"] = k
            res[f"k_canvas_yuv_tb_per_s_{f}"] = conv_bytes / (k * 1e-3) / 1e12 if k else None

    def bgr_then_cvt():
        out = eng.run(sets(pin_nv12), None, bal, pixel_format="nv12")
        return list(pool.map(lambda c: cv2.cvtColor(c, cv2.COLOR_BGR2YUV_I420), list(out)))

    host = {}
    for _ in range(2):   # alternate the paths so that drift in the host or the link hits them alike
        for key, fn in (("nv12_in_nv12_out", lambda: eng.run(sets(pin_nv12), None, bal, pixel_format="nv12", out_format="nv12")),
                        ("nv12_in_bgr_out", lambda: eng.run(sets(pin_nv12), None, bal, pixel_format="nv12")),
                        ("nv12_in_bgr_out_host_cvtcolor_i420", bgr_then_cvt)):
            host.setdefault(key, []).append(_median_s(fn, max(2, iters // 2), warmup))
            res[f"h2d_bytes_per_frame_set_{key}"] = eng.last_h2d_bytes() / n
    for key, v in host.items():
        res[f"host_frame_sets_per_s_{key}"] = n / float(np.median(v))
    res["d2h_bytes_per_frame_set_bgr_out"] = eng.host_copy_bytes(bal, "nv12")[1]
    res["d2h_bytes_per_frame_set_nv12_out"] = eng.host_copy_bytes(bal, "nv12", "nv12")[1]
    eng.ctx.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import bench as B
    from cameracalibration_b200 import _lib as L
    cv2.setNumThreads(1)      # cvtColor one canvas per thread in the host-conversion figure
    cores = os.cpu_count() or 1
    card = _card()
    with ThreadPoolExecutor(cores) as pool:
        res = [_workload("bench", dict(B.WORKLOAD), a.iters, a.warmup, pool),
               _workload("cfg3", {**B.WORKLOAD, **B.ALT_WORKLOADS["cfg3"]}, a.iters, a.warmup, pool)]
    print(json.dumps({"tool": "bench_yuv_out", "card": card, "lib": os.path.basename(L.LIB_PATH), "host_threads": cores,
                      "results": res}))


if __name__ == "__main__":
    main()
