#!/usr/bin/env python
"""Batched device undistortion (bevk_undistort_stack, Undistorter.cuda / cuda_to_jpeg) on the fisheye front camera of
the reference.  One JSON line, with the card's name and power limit read in the same run.

    kernel   map and fused slots, 1280x1024 frames -> 1280x1024 (Tools/undistort.py's default) and -> 2560x2048 (BEV's
             SIZE_SCALE 2), batches 1, 8, 32, 128.  Kernel time from CUDA events around a CUDA graph of --reps calls,
             replayed until about 0.2 s have passed; per frame, frames/s, and the algorithmic bytes -- the map (6 B/px,
             read once per group of --nb frames; none for fused slots) + the 32-byte source sectors the taps touch + the
             destination -- as GB/s and as a share of the H100 SXM data-sheet 3.35 TB/s.
    jpeg     Undistorter.cuda_to_jpeg of 32 device frames (map slot, 1280x1024) at q95 and q100, against Undistorter.jpeg
             per host image and cv2.remap + cv2.imencode over all host cores; every device stream is checked against cv2.
    --n1-vs DIR  the single-frame gather that bevk_undistort launches (torch.profiler kernel time), this tree against
             the built source tree DIR (e.g. a checkout of the parent commit), alternating, in subprocesses.

    python tools/bench_undistort_stack.py [--nb 8] [--n1-vs path/to/other/tree] [--skip-jpeg]
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
HBM_PEAK = 3.35e12          # H100 SXM data sheet, bytes/s
FW, FH = 1280, 1024


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def _camera(dst):
    from oracle import cv2_path as C
    from tests.helpers import Fixtures
    fx = Fixtures()
    K, D, _ = fx.calib["front"]
    P = C.dst_camera_matrix(K, FW, FH, 1, dst[0] / FW)
    return fx, K, D, P, C.undistort_maps(K, D, P, *dst)


def _frames(fx, n):
    distinct = [fx.perturbed_frames(FW, FH, b)[b % 4] for b in range(min(n, 8))]
    return np.stack([distinct[i % len(distinct)] for i in range(n)])


def _sector_bytes(maps):
    """32-byte sectors of one dense 1280x1024x3 frame that the four taps of every output pixel touch."""
    m = maps[0].reshape(-1, 2).astype(np.int64)
    secs = []
    for dy in (0, 1):
        y = m[:, 1] + dy
        for dx in (0, 1):
            x = m[:, 0] + dx
            v = (x >= 0) & (x < FW) & (y >= 0) & (y < FH)
            a = y[v] * FW * 3 + 3 * x[v]
            secs += [a // 32, (a + 2) // 32]
    return int(np.unique(np.concatenate(secs)).size) * 32


def _kernel(dst, fused, batches, reps, nb):
    import torch
    from cameracalibration_b200 import _lib as L
    from cameracalibration_b200 import ops
    fx, K, D, P, maps = _camera(dst)
    u = ops.Undistorter(K, D, P, dst, fused=fused, ctx=L.Context(0))
    frames = torch.from_numpy(_frames(fx, max(batches))).cuda()
    out = torch.empty((max(batches), dst[1], dst[0], 3), dtype=torch.uint8, device="cuda")
    src_sec, dst_bytes, map_bytes = _sector_bytes(maps), dst[0] * dst[1] * 3, 0 if fused else dst[0] * dst[1] * 6
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    res = []
    for n in batches:
        call = lambda: L.check(u.ctx.lib.bevk_undistort_stack(u.ctx.h, u.slot, ctypes.c_void_p(frames.data_ptr()), FW * FH * 3, FW, FH,
                                                              FW * 3, 3, n, ctypes.c_void_p(out.data_ptr()), dst[0] * dst[1] * 3,
                                                              dst[0], dst[1], dst[0] * 3, ops.INTER_LINEAR))
        with u.ctx.on_stream(s.cuda_stream):
            call()
            path = u.last_path()
            s.synchronize()
            with u.ctx.graph_capture() as g:
                for _ in range(reps):
                    call()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            g.launch()
            e0.record(s)
            g.launch()
            e1.record(s)
            e1.synchronize()
            launches = max(3, int(200.0 / max(e0.elapsed_time(e1), 1e-3)))
            e0.record(s)
            g.launch(launches)
            e1.record(s)
            e1.synchronize()
            ms = e0.elapsed_time(e1) / (launches * reps)
            g.destroy()
        host = out[n - 1].cpu().numpy()
        exact = bool((host == cv2.remap(frames[n - 1].cpu().numpy(), maps[0], maps[1], cv2.INTER_LINEAR)).all())
        algo = map_bytes * -(-n // nb) + n * (src_sec + dst_bytes)
        res.append({"slot": "fused" if fused else "map", "dst": f"{dst[0]}x{dst[1]}", "batch": n, "path": path,
                    "kernel_ms_per_call": ms, "kernel_ms_per_frame": ms / n, "frames_per_s": n / ms * 1e3,
                    "algorithmic_bytes": algo, "achieved_gbs": algo / ms / 1e6, "share_of_3p35_tbs": algo / ms / 1e-3 / HBM_PEAK,
                    "last_frame_equals_cv2": exact})
    u.close()
    return res


def _jpeg(n=32):
    import torch
    from cameracalibration_b200 import ops
    fx, K, D, P, maps = _camera((FW, FH))
    u = ops.Undistorter(K, D, P, (FW, FH))
    host = _frames(fx, n)
    frames = torch.from_numpy(host).cuda()
    cores = os.cpu_count() or 1
    cv2.setNumThreads(1)
    res = []
    for q in (95, 100):
        streams = u.cuda_to_jpeg(frames, q)
        t = []
        for _ in range(5):
            t0 = time.perf_counter()
            u.cuda_to_jpeg(frames, q)
            t.append(time.perf_counter() - t0)
        dev = n / float(np.median(t))
        t0 = time.perf_counter()
        for i in range(n):
            u.jpeg(host[i], q)
        per_image = n / (time.perf_counter() - t0)
        enc = lambda img: cv2.imencode(".jpg", cv2.remap(img, maps[0], maps[1], cv2.INTER_LINEAR), [cv2.IMWRITE_JPEG_QUALITY, q])[1]
        with ThreadPoolExecutor(cores) as pool:
            want = [w.tobytes() for w in pool.map(enc, list(host))]
            t0 = time.perf_counter()
            list(pool.map(enc, list(host)))
            cpu = n / (time.perf_counter() - t0)
        res.append({"quality": q, "frames": n, "cuda_to_jpeg_frames_per_s": dev, "undistorter_jpeg_per_image_frames_per_s": per_image,
                    "cv2_remap_imencode_all_cores_frames_per_s": cpu, "host_threads": cores,
                    "byte_identical_to_cv2": streams == want, "stream_bytes": sum(len(s) for s in streams)})
    u.close()
    return res


def _n1_profile(iters=30):
    """Device time of the gather kernel bevk_undistort launches for one host frame (works with any library version)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from cameracalibration_b200 import ops
    res = {}
    for dst in ((FW, FH), (2 * FW, 2 * FH)):
        fx, K, D, P, _ = _camera(dst)
        frame = _frames(fx, 1)[0]
        for fused in (False, True):
            u = ops.Undistorter(K, D, P, dst, fused=fused)
            out = np.empty((dst[1], dst[0], 3), np.uint8)
            for _ in range(3):
                u(frame, out=out)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(iters):
                    u(frame, out=out)
            ks = [e for e in prof.events() if "k_gather" in e.name]
            res[f"{'fused' if fused else 'map'}_{dst[0]}x{dst[1]}_us"] = sum(e.device_time for e in ks) / max(1, len(ks))
            u.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nb", type=int, default=8, help="frames per thread the library was built with (BEVK_GATHER_NB), for the bytes")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--n1-vs", default=None)
    ap.add_argument("--n1-profile", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--root", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--skip-jpeg", action="store_true")
    a = ap.parse_args()
    if a.n1_profile:
        if a.root:                       # the other tree's package, library and fixtures
            sys.path.insert(0, os.path.abspath(a.root))
        print(json.dumps(_n1_profile()))
        return
    card = _card()
    kern = []
    for dst in ((FW, FH), (2 * FW, 2 * FH)):
        for fused in (False, True):
            kern += _kernel(dst, fused, (1, 8, 32, 128), a.reps, a.nb)
    res = {"tool": "bench_undistort_stack", "card": card, "lib": os.environ.get("BEVK_LIB_PATH", "in-tree"), "nb": a.nb, "kernel": kern}
    if not a.skip_jpeg:
        res["jpeg"] = _jpeg()
    if a.n1_vs:
        runs = []
        for rnd in range(2):
            for name, root in (("this", ROOT), ("other", a.n1_vs)):
                env = dict(os.environ)
                env.pop("BEVK_LIB_PATH", None)
                r = subprocess.run([sys.executable, os.path.abspath(__file__), "--n1-profile", "--root", os.path.abspath(root)],
                                   capture_output=True, text=True, env=env, timeout=900)
                runs.append({"lib": name, "round": rnd, **(json.loads(r.stdout.strip().splitlines()[-1]) if r.returncode == 0
                                                          else {"error": r.stderr[-500:]})})
        res["n1_single_frame_gather"] = {"other": a.n1_vs, "runs": runs}
    res["card_after"] = _card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
