#!/usr/bin/env python
"""BEV renders from NV12 decoder surfaces (pitch 2048, chroma after the 1088-row coded height of a 1080p surface, one
uint8[n * n_cam][1088 + 544][2048] pool) straight through bevk_bev_run_yuv_planes, against what a caller had to do before:
repack every surface into cv2's dense single buffer with torch and call run_stack(nv12); and against run_stack(nv12) on
frames that already are dense.  One JSON line with the card's name, power limit and SM clocks read in the same run.

Workloads: the bench workload (32 x 4 x 1920x1080 -> 1000x1000, blend) and cfg3 (1920x1080 -> 1200x1200, blend +
balance).  Per workload: ms per step of each path (CUDA events, median of blocks that alternate the three), kernel ms per
step per kernel (torch.profiler; the repack shows as torch's copy kernels), and whether the three paths give the same
canvases (``byte_identical``).

    python tools/bench_yuv_planes.py [--iters 10]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_yuv import _kernel_ms, _step_ms   # noqa: E402

PITCH, CODED_H = 2048, 1088


def _card():
    try:
        q = "name,power.limit,clocks.sm,clocks.max.sm"
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return {"query": q, "value": out[0] if out else "unknown"}
    except Exception as e:   # noqa: BLE001
        return {"query": "", "value": f"unknown ({e})"}


def _workload(name, w, iters):
    import torch
    import bench as B
    from tests.yuv_frames import from_bgr
    eng, _, _, g = B.build_engine(w, 0)
    n, nc, bal = w["batch"], w["n_cam"], w["balance"]
    FW, FH = w["FW"], w["FH"]
    assert (FW, FH) == (1920, 1080)
    bgr = B.synthetic_frames(FW, FH, nc, n, seed=7)
    nv12 = np.stack([np.stack([from_bgr(bgr[b, c], "nv12") for c in range(nc)]) for b in range(n)])
    d_dense = torch.from_numpy(nv12).cuda()
    pool = torch.full((n, nc, CODED_H * 3 // 2, PITCH), 0x80, dtype=torch.uint8, device="cuda")
    y, uv = pool[:, :, :FH, :FW], pool[:, :, CODED_H:CODED_H + FH // 2, :FW]
    y.copy_(d_dense[:, :, :FH])
    uv.copy_(d_dense[:, :, FH:])
    repacked = torch.empty_like(d_dense)
    out = torch.empty((n, g.BH, g.BW, 3), dtype=torch.uint8, device="cuda")
    res = {"workload": name, "frame_sets": n, "frame": [FW, FH], "canvas": [g.BW, g.BH], "blend": w["blend"], "balance": bal,
           "surface": {"pitch": PITCH, "chroma_row": CODED_H}}

    def planes():
        eng.run_cuda_planes(y, uv, pixel_format="nv12", balance=bal, out=out, stream=torch.cuda.current_stream().cuda_stream)

    def repack_then_stack():
        repacked[:, :, :FH].copy_(y)
        repacked[:, :, FH:].copy_(uv)
        eng.run_stack(repacked.data_ptr(), FW * FH * 3 // 2, n, out.data_ptr(), 0, bal, pixel_format="nv12")

    def dense():
        eng.run_stack(d_dense.data_ptr(), FW * FH * 3 // 2, n, out.data_ptr(), 0, bal, pixel_format="nv12")

    fns = {"planes": planes, "repack_then_run_stack": repack_then_stack, "dense_run_stack": dense}
    canv = {}
    with eng.ctx.on_stream(torch.cuda.current_stream().cuda_stream):   # the events, the copies and the renders on one stream
        for k, f in fns.items():
            out.fill_(0)
            f()
            torch.cuda.synchronize()
            canv[k] = out.cpu().numpy()
        res["byte_identical"] = bool(all((v == canv["dense_run_stack"]).all() for v in canv.values()))
        ms = _step_ms(torch, list(fns.values()), iters, 20)
        for k, m in zip(fns, ms):
            res[f"ms_per_step_{k}"] = m
            res[f"frame_sets_per_s_{k}"] = n / m * 1e3
        for k, f in fns.items():
            res[f"kernel_ms_per_step_{k}"], res[f"kernels_{k}"] = _kernel_ms(f, 10)
    eng.ctx.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    import bench as B
    card = _card()
    res = [_workload("bench", dict(B.WORKLOAD), a.iters),
           _workload("cfg3", {**B.WORKLOAD, **B.ALT_WORKLOADS["cfg3"]}, a.iters)]
    print(json.dumps({"tool": "bench_yuv_planes", "card": card, "results": res, "card_after": _card()}))


if __name__ == "__main__":
    main()
