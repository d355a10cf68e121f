#!/usr/bin/env python
"""BALANCE under the 'cameras' sharding policy, BASELINE cfg3 (32 frame-sets of 4 x 1920x1080 -> 1200x1200, blend +
balance).  One JSON line, with the card's name and power limit read in the same run.

    one GPU (default)
        single       run_stack(balance=True): the single-GPU BALANCE render
        world4_bal   the world-4 decomposition emulated on this GPU: every rank's V sums (bevk_shard_vsum), every rank's
                     balanced slabs (bevk_shard_render_balanced), then ONE compose with colour balance
                     (bevk_shard_compose_balanced: k_compose_slabs<.., true> + k_gain)
        world4_plain the same without balance (bevk_shard_render x 4 + bevk_shard_compose), for comparison
        compose_plain / compose_bal   the compose alone, without and with the channel sums + k_gain
        Milliseconds per step from CUDA events over --steps calls after --warmup, arms alternated over --rounds rounds
        (median).  The world-4 canvases must equal the single-GPU ones byte for byte.
    --profile    per-kernel device time of single and world4_bal from torch.profiler, in a separate run.
    --tree DIR   import the package from DIR instead (e.g. a built checkout of another commit); only the arms that DIR's
                 library has run (compose_plain / world4_plain need nothing new).
    --nccl       under torchrun with >= 2 processes: ShardedBev.render(balance=True) and render_scattered(balance=True)
                 over NCCL, frame-sets/s and NVLink bytes per step (the V-sum exchange included); every canvas is
                 checked against the single-GPU render on the same rank.

    python tools/bench_shard_balance.py [--profile] [--tree DIR] [--only compose_plain,world4_plain]
    torchrun --nproc-per-node 2 tools/bench_shard_balance.py --nccl
"""
import argparse
import json
import os
import statistics
import subprocess
import sys


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def _setup(device, batch):
    import torch
    import bench
    w = dict(bench.WORKLOAD, **bench.ALT_WORKLOADS["cfg3"])
    w["batch"] = batch
    eng, _, _, g = bench.build_engine(w, device)
    dev = torch.device("cuda", device)
    host = bench.synthetic_frames(w["FW"], w["FH"], w["n_cam"], batch, seed=1000)
    d_frames = torch.from_numpy(host).to(dev)
    stream = torch.cuda.Stream(device=dev)
    eng.ctx.set_stream(stream.cuda_stream)
    return w, eng, d_frames, stream


def _timed(torch, stream, fn, steps, warmup):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(steps):
        fn()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / steps


def one_gpu(a):
    import torch
    from cameracalibration_b200.sharding import ShardedBev
    w, eng, d, stream = _setup(0, a.batch)
    nb, s = w["batch"], stream.cuda_stream
    fb = w["FW"] * w["FH"] * 3
    out_single = torch.empty((nb, w["BH"], w["BW"], 3), dtype=torch.uint8, device="cuda")
    out_w4 = torch.empty_like(out_single)
    sh = ShardedBev(eng, "cameras", rank=0, world=4, connect=False)
    slabs = sh.slab_buffer(nb)
    has_bal = hasattr(sh, "vsum_buffer")
    vs = sh.vsum_buffer(nb) if has_bal else None
    torch.cuda.synchronize()

    def single():
        eng.run_stack(d.data_ptr(), fb, nb, out_single.data_ptr(), 0, True)

    def w4_ranks(balance):
        if balance:
            for r in range(4):
                sh.vsums(d, r, vs, stream=s)
        for r in range(4):
            if balance:
                sh.render_slabs(d, r, slabs, stream=s, vsums=vs)
            else:
                sh.render_slabs(d, r, slabs, stream=s)

    def world4_bal():
        w4_ranks(True)
        sh.compose(slabs, out_w4, stream=s, balance=True)

    def world4_plain():
        w4_ranks(False)
        sh.compose(slabs, out_w4, stream=s)

    def compose_plain():
        sh.compose(slabs, out_w4, stream=s)

    def compose_bal():
        sh.compose(slabs, out_w4, stream=s, balance=True)

    arms = {"single": single, "world4_plain": world4_plain, "compose_plain": compose_plain}
    if has_bal:
        arms.update(world4_bal=world4_bal, compose_bal=compose_bal)
    if a.only:
        arms = {k: v for k, v in arms.items() if k in a.only.split(",")}
    line = {"tool": "bench_shard_balance", "card": _card(), "workload": f"cfg3: {nb} frame-sets x 4 cams {w['FW']}x{w['FH']} -> "
            f"{w['BW']}x{w['BH']}, blend + balance", "tree": os.path.abspath(a.tree or "."), "steps": a.steps, "rounds": a.rounds}
    if has_bal and (not a.only or "world4_bal" in arms):
        single(); world4_bal()
        torch.cuda.synchronize()
        line["world4_equal_single"] = bool(torch.equal(out_single, out_w4))
    times = {k: [] for k in arms}
    for _ in range(a.rounds):
        for k, fn in arms.items():
            with torch.cuda.stream(stream):
                times[k].append(_timed(torch, stream, fn, a.steps, a.warmup))
    line["ms_per_step"] = {k: round(statistics.median(v), 4) for k, v in times.items()}
    line["ms_per_step_all"] = {k: [round(x, 4) for x in v] for k, v in times.items()}
    line["frame_sets_per_s"] = {k: round(nb / (statistics.median(v) / 1e3), 1) for k, v in times.items() if not k.startswith("compose")}
    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        split = {}
        for k in [x for x in ("single", "world4_bal") if x in arms]:
            for _ in range(a.warmup):
                arms[k]()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as p:
                for _ in range(a.steps):
                    arms[k]()
                torch.cuda.synchronize()
            per = {}
            for ev in p.key_averages():
                if ev.device_type.name == "CUDA" and ev.self_device_time_total > 0:
                    per[ev.key[:90]] = round(ev.self_device_time_total / a.steps / 1e3, 4)   # ms per step
            split[k] = dict(sorted(per.items(), key=lambda kv: -kv[1]))
        line["kernel_ms_per_step"] = split
    print(json.dumps(line))


def nccl(a):
    import torch
    import torch.distributed as dist
    from cameracalibration_b200.sharding import ShardedBev
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    try:
        w, eng, d, stream = _setup(local, a.batch)
        nb, s = w["batch"], stream.cuda_stream
        fb = w["FW"] * w["FH"] * 3
        want = torch.empty((nb, w["BH"], w["BW"], 3), dtype=torch.uint8, device="cuda")
        eng.run_stack(d.data_ptr(), fb, nb, want.data_ptr(), 0, True)
        torch.cuda.synchronize()
        sh = ShardedBev(eng, "cameras")
        out = torch.empty_like(want)
        own = torch.empty(((nb + world - 1) // world, w["BH"], w["BW"], 3), dtype=torch.uint8, device="cuda")
        res = {}
        for name, fn in (("allgather", lambda: sh.render(d, out, None, True, stream=s)),
                         ("p2p", lambda: sh.render_scattered(d, own, None, stream=s, balance=True))):
            fn()
            torch.cuda.synchronize()
            if name == "allgather":
                ok = bool(torch.equal(out, want))
            else:
                mine = sh.own_frame_sets(nb)
                ok = all(torch.equal(own[i], want[b]) for i, b in enumerate(mine))
            dist.barrier()
            ms = _timed(torch, stream, fn, a.steps, a.warmup)
            dist.barrier()
            res[name] = {"ms_per_step": round(ms, 4), "frame_sets_per_s": round(nb / (ms / 1e3), 1), "equal_single": ok,
                         "link_bytes_per_step": sh.link_bytes(),
                         "vsum_bytes_per_step": nb * w["n_cam"] * 8 * (world - 1)}
        allres = [None] * world
        dist.all_gather_object(allres, res)
        if rank == 0:
            print(json.dumps({"tool": "bench_shard_balance", "mode": "nccl", "card": _card(), "world": world,
                              "workload": f"cfg3: {nb} frame-sets x 4 cams, blend + balance", "per_rank": allres}))
    finally:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--nccl", action="store_true")
    ap.add_argument("--tree", default=None)
    ap.add_argument("--only", default=None, help="comma-separated arms")
    a = ap.parse_args()
    root = os.path.abspath(a.tree) if a.tree else os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    nccl(a) if a.nccl else one_gpu(a)


if __name__ == "__main__":
    main()
