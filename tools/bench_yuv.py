#!/usr/bin/env python
"""BEV renders from NV12 frames (BEVK_FLAG_NV12) and packed 4:2:2 frames (BEVK_FLAG_YUYV / _UYVY) against BGR frames,
the formats alternating in one process.  One JSON line with the card's name and power limit read in the same run.

Workloads: the bench workload (32 x 4 x 1920x1080 -> 1000x1000, blend) and cfg3 (1920x1080 -> 1200x1200, blend +
balance).  Per workload:
  device   ms per step of run_stack on a device frame stack, NV12 against BGR (CUDA events, median of blocks that
           alternate the two), and in a separate run the kernel ms per step from torch.profiler, per kernel (the NV12
           conversion pass is k_yuv_spans)
  host     frame-sets/s of BevEngine.run from page-locked and from pageable host frames, NV12 against BGR, and against
           host cv2.cvtColor(COLOR_YUV2BGR_NV12) over all cores followed by the BGR run
  h2d      host->device bytes per frame-set each of those moves
The YUYV and UYVY rows (keys ending in _yuyv / _uyvy) measure the same, their host conversion being
cv2.cvtColor(COLOR_YUV2BGR_YUY2 / _UYVY).  Every NV12 canvas is checked against the BGR render of the cvtColor output
(``byte_identical``), and every 4:2:2 one likewise (``byte_identical_yuyv`` / ``_uyvy``).

    python tools/bench_yuv.py [--iters 10] [--warmup 2]
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
    """Kernel ms per step from torch.profiler's CUDA activities: total and per kernel name."""
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


def _step_ms(torch, fns, iters, steps):
    """Median ms per step of each fn, measured in blocks of `steps` calls that alternate between the fns."""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for f in fns:
        f()
    torch.cuda.synchronize()
    t = [[] for _ in fns]
    for _ in range(iters):
        for i, f in enumerate(fns):
            ev[0].record()
            for _ in range(steps):
                f()
            ev[1].record()
            ev[1].synchronize()
            t[i].append(ev[0].elapsed_time(ev[1]) / steps)
    return [float(np.median(x)) for x in t]


def _workload(name, w, iters, warmup, pool):
    import torch
    import bench as B
    from cameracalibration_b200 import _lib as L
    eng, calib, masks, g = B.build_engine(w, 0)
    n, nc, bal = w["batch"], w["n_cam"], w["balance"]
    FW, FH = w["FW"], w["FH"]
    bgr = B.synthetic_frames(FW, FH, nc, n, seed=7)
    # NV12 frames: the BGR frames through cv2's I420 encoder, planes interleaved; the BGR the engine compares with is
    # what cv2.cvtColor makes of them
    from tests.yuv_frames import from_bgr, to_bgr
    nv12 = np.stack([np.stack([from_bgr(bgr[b, c], "nv12") for c in range(nc)]) for b in range(n)])
    bgr = np.stack([np.stack([to_bgr(nv12[b, c], "nv12") for c in range(nc)]) for b in range(n)])
    # packed 4:2:2 frames (YUYV, UYVY): the BGR frames as a camera delivers them, chroma averaged over pixel pairs; the
    # BGR their canvases are compared with is cv2.cvtColor(COLOR_YUV2BGR_YUY2 / _UYVY) of them
    from tests import yuv422_frames as Y2
    packed = {f: np.stack([np.stack([Y2.from_bgr(bgr[b, c], f) for c in range(nc)]) for b in range(n)]) for f in Y2.FORMATS}
    bgr422 = {f: np.stack([np.stack([Y2.to_bgr(a[b, c], f) for c in range(nc)]) for b in range(n)]) for f, a in packed.items()}
    pin_bgr, pin_nv12 = L.pinned_empty(bgr.shape), L.pinned_empty(nv12.shape)
    pin_bgr[...], pin_nv12[...] = bgr, nv12
    pin422 = {}
    for f, a in packed.items():
        pin422[f] = L.pinned_empty(a.shape)
        pin422[f][...] = a
    sets = lambda a: [[a[b, c] for c in range(nc)] for b in range(n)]
    res = {"workload": name, "frame_sets": n, "frame": [FW, FH], "canvas": [g.BW, g.BH], "blend": w["blend"], "balance": bal}

    want = np.array(eng.run(sets(bgr), None, bal))
    got = {"pinned": np.array(eng.run(sets(pin_nv12), None, bal, pixel_format="nv12")),
           "pageable": np.array(eng.run(sets(nv12), None, bal, pixel_format="nv12"))}
    d_bgr, d_nv12 = torch.from_numpy(bgr).cuda(), torch.from_numpy(nv12).cuda()
    got["device"] = eng.run_cuda(d_nv12, None, bal, pixel_format="nv12").cpu().numpy()
    res["byte_identical"] = bool(all((v == want).all() for v in got.values()))
    d422 = {f: torch.from_numpy(a).cuda() for f, a in packed.items()}
    for f in Y2.FORMATS:
        want = np.array(eng.run(sets(bgr422[f]), None, bal))
        got = [np.array(eng.run(sets(pin422[f]), None, bal, pixel_format=f)),
               np.array(eng.run(sets(packed[f]), None, bal, pixel_format=f)),
               eng.run_cuda(d422[f], None, bal, pixel_format=f).cpu().numpy()]
        res[f"byte_identical_{f}"] = bool(all((v == want).all() for v in got))

    out = torch.empty((n, g.BH, g.BW, 3), dtype=torch.uint8, device="cuda")
    run_bgr = lambda: eng.run_stack(d_bgr.data_ptr(), FW * FH * 3, n, out.data_ptr(), 0, bal)
    run_nv12 = lambda: eng.run_stack(d_nv12.data_ptr(), FW * FH * 3 // 2, n, out.data_ptr(), 0, bal, pixel_format="nv12")
    run_422 = {f: (lambda f=f: eng.run_stack(d422[f].data_ptr(), FW * FH * 2, n, out.data_ptr(), 0, bal, pixel_format=f))
               for f in Y2.FORMATS}
    with eng.ctx.on_stream(torch.cuda.current_stream().cuda_stream):   # the events and the renders on one stream
        ms_bgr, ms_nv12, *ms_422 = _step_ms(torch, [run_bgr, run_nv12] + [run_422[f] for f in Y2.FORMATS], iters, 20)
    res["device_ms_per_step_bgr"], res["device_ms_per_step_nv12"] = ms_bgr, ms_nv12
    res["device_frame_sets_per_s_bgr"], res["device_frame_sets_per_s_nv12"] = n / ms_bgr * 1e3, n / ms_nv12 * 1e3
    for f, ms in zip(Y2.FORMATS, ms_422):
        res[f"device_ms_per_step_{f}"], res[f"device_frame_sets_per_s_{f}"] = ms, n / ms * 1e3
    res["kernel_ms_per_step_bgr"], res["kernels_bgr"] = _kernel_ms(run_bgr, 10)
    res["kernel_ms_per_step_nv12"], res["kernels_nv12"] = _kernel_ms(run_nv12, 10)
    for f in Y2.FORMATS:
        res[f"kernel_ms_per_step_{f}"], res[f"kernels_{f}"] = _kernel_ms(run_422[f], 10)

    fs = lambda s: n / s

    def cvt_then_run(a, conv_fn):
        conv = list(pool.map(conv_fn, [a[b, c] for b in range(n) for c in range(nc)]))
        return eng.run([conv[b * nc:(b + 1) * nc] for b in range(n)], None, bal)

    # alternate the paths so that drift in the host or the link hits them alike
    host = {}
    paths = [("pinned_bgr", lambda: eng.run(sets(pin_bgr), None, bal)),
             ("pinned_nv12", lambda: eng.run(sets(pin_nv12), None, bal, pixel_format="nv12")),
             ("pageable_bgr", lambda: eng.run(sets(bgr), None, bal)),
             ("pageable_nv12", lambda: eng.run(sets(nv12), None, bal, pixel_format="nv12")),
             ("pinned_nv12_host_cvtcolor_then_bgr", lambda: cvt_then_run(pin_nv12, lambda f: to_bgr(f, "nv12")))]
    for f in Y2.FORMATS:
        paths += [(f"pinned_{f}", lambda f=f: eng.run(sets(pin422[f]), None, bal, pixel_format=f)),
                  (f"pageable_{f}", lambda f=f: eng.run(sets(packed[f]), None, bal, pixel_format=f)),
                  (f"pinned_{f}_host_cvtcolor_then_bgr", lambda f=f: cvt_then_run(pin422[f], lambda x: Y2.to_bgr(x, f)))]
    for _ in range(2):
        for key, fn in paths:
            host.setdefault(key, []).append(_median_s(fn, max(2, iters // 2), warmup))
            if not key.endswith("_host_cvtcolor_then_bgr"):
                res[f"h2d_bytes_per_frame_set_{key}"] = eng.last_h2d_bytes() / n
    for key, v in host.items():
        res[f"host_frame_sets_per_s_{key}"] = fs(float(np.median(v)))
    res["h2d_bytes_per_frame_set_plan_pageable_bgr"] = eng.host_copy_bytes(bal)[0]
    res["h2d_bytes_per_frame_set_plan_pageable_nv12"] = eng.host_copy_bytes(bal, "nv12")[0]
    for f in Y2.FORMATS:
        res[f"h2d_bytes_per_frame_set_plan_pageable_{f}"] = eng.host_copy_bytes(bal, f)[0]
    eng.ctx.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import bench as B
    cv2.setNumThreads(1)      # cvtColor one frame per thread in the host-conversion figure
    cores = os.cpu_count() or 1
    card = _card()
    with ThreadPoolExecutor(cores) as pool:
        res = [_workload("bench", dict(B.WORKLOAD), a.iters, a.warmup, pool),
               _workload("cfg3", {**B.WORKLOAD, **B.ALT_WORKLOADS["cfg3"]}, a.iters, a.warmup, pool)]
    print(json.dumps({"tool": "bench_yuv", "card": card, "host_threads": cores, "results": res}))


if __name__ == "__main__":
    main()
