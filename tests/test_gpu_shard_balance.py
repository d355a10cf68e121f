"""GPU tests of BALANCE under the 'cameras' sharding policy: each rank sums V over its own cameras' frames, the ranks
exchange those sums ([world][batch][n_cam] uint64), each rank luminance-balances and renders its own cameras, and the
compose takes the channel sums of the raw canvas for the colour balance (k_compose_slabs<.., true>, then k_gain).
Every canvas must be byte-identical to the single-GPU BALANCE render and to the cv2 oracle.

  * one GPU emulates every world size through the one-GPU halves (ShardedBev.vsums / render_slabs(vsums=...) /
    compose(balance=True)), with foreign cameras' frames poisoned, on the reference's data and on the fuzz corpus;
  * the peer-store kernel variant runs with a world of one;
  * with >= 2 GPUs, two processes over NCCL run ShardedBev.render and render_scattered with balance=True."""
import ctypes
import os

import numpy as np
import pytest

from oracle import cv2_path as C
from tests import bev_cases as B
from tests.helpers import h16
from tests.test_gpu_shard import _engine, _free_port

pytestmark = pytest.mark.gpu
WORLDS = (2, 3, 4, 8)


def _sets(fx):
    F = fx.frames()
    return [F, [np.ascontiguousarray(f[::-1]) for f in F], [np.ascontiguousarray(np.roll(f, 31, axis=1)) for f in F]]


def _poisoned(host, lo, hi):
    """The stack a rank owning cameras [lo, hi) holds: every other camera's frames overwritten with 0xAB."""
    mine = host.copy()
    mine[:, :lo] = 0xAB
    mine[:, hi:] = 0xAB
    return mine


def _emulate(torch, sh, frames_of_rank, batch, car, out):
    """Every rank's BALANCE work on this GPU (ΣV blocks, then balanced slabs), then one compose."""
    vs = sh.vsum_buffer(batch)
    for r in range(sh.world):
        sh.vsums(frames_of_rank(r), r, vs)
    slabs = sh.slab_buffer(batch)
    for r in range(sh.world):
        sh.render_slabs(frames_of_rank(r), r, slabs, vsums=vs)
    sh.compose(slabs, out, car, balance=True)
    return vs


@pytest.mark.parametrize("blend", [False, True])
def test_every_world_size_on_one_gpu(fx, blend):
    import torch
    from cameracalibration_b200.sharding import ShardedBev, camera_range
    g = fx.geometry()
    e, masks = _engine(fx, g, blend, calib=fx.calib)
    dev = torch.device("cuda", e.ctx.device)
    sets = _sets(fx)
    host = np.stack([np.stack(s) for s in sets])
    d_all = torch.from_numpy(host).to(dev)
    car = torch.from_numpy(fx.car()).to(dev)
    ref = C.RefBev(fx.calib, g, blend, True, masks=masks)
    gold = fx.gold["native"][f"blend{int(blend)}_balance1"]
    for c in (None, car):
        full = torch.empty((3, g.BH, g.BW, 3), dtype=torch.uint8, device=dev)
        e.run_stack(d_all.data_ptr(), g.FH * g.FW * 3, 3, full.data_ptr(), 0 if c is None else c.data_ptr(), balance=True)
        e.ctx.sync()
        full = full.cpu().numpy()
        assert h16(full[0]) == gold["nocar" if c is None else "car"]
        for i in (1, 2):
            assert (full[i] == ref(*sets[i], fx.car() if c is not None else None)).all(), i
        for world in WORLDS:
            sh = ShardedBev(e, "cameras", rank=0, world=world, connect=False)
            out = torch.empty((3, g.BH, g.BW, 3), dtype=torch.uint8, device=dev)
            vs = _emulate(torch, sh, lambda r: d_all, 3, c, out)
            torch.cuda.synchronize()
            assert (out.cpu().numpy() == full).all(), (world, c is not None)
            # block r holds ΣV of rank r's cameras only
            v = vs.cpu().numpy()
            for r in range(world):
                lo, hi = camera_range(4, r, world)
                assert (v[r][:, :lo] == 0).all() and (v[r][:, hi:] == 0).all() and (v[r][:, lo:hi] > 0).all()


def test_foreign_frames_are_never_read(fx):
    import torch
    from cameracalibration_b200.sharding import ShardedBev
    g = fx.geometry()
    e, _ = _engine(fx, g, True, calib=fx.calib)
    dev = torch.device("cuda", e.ctx.device)
    host = np.stack([np.stack(s) for s in _sets(fx)])
    d_all = torch.from_numpy(host).to(dev)
    car = torch.from_numpy(fx.car()).to(dev)
    full = torch.empty((3, g.BH, g.BW, 3), dtype=torch.uint8, device=dev)
    e.run_stack(d_all.data_ptr(), g.FH * g.FW * 3, 3, full.data_ptr(), car.data_ptr(), balance=True)
    e.ctx.sync()
    full = full.cpu().numpy()
    for world in WORLDS:
        sh = ShardedBev(e, "cameras", rank=0, world=world, connect=False)
        mine = [torch.from_numpy(_poisoned(host, *sh.info(r)[:2])).to(dev) for r in range(world)]
        out = torch.empty((3, g.BH, g.BW, 3), dtype=torch.uint8, device=dev)
        _emulate(torch, sh, lambda r: mine[r], 3, car, out)
        torch.cuda.synchronize()
        assert (out.cpu().numpy() == full).all(), world
        del mine


def _case_engine(ops, case):
    e = ops.BevEngine(case.NC, (case.FW, case.FH), (case.BW, case.BH))
    for k, ((m1, m2), mk) in enumerate(zip(case.maps, case.masks)):
        e.set_maps(k, m1, m2)
        e.set_mask(k, mk)
    if case.nearest:
        e.set_interpolation(ops.INTER_NEAREST)
    e.finalize()
    return e


def _emulate_stack(e, sh, d, stride, n, car, out):
    """_emulate through the C ABI, for frame stacks whose stride is padded (frames of odd byte size)."""
    import torch
    from cameracalibration_b200 import _lib as L
    lib, h, V = e.ctx.lib, e.ctx.h, ctypes.c_void_p
    vs, slabs = sh.vsum_buffer(n), sh.slab_buffer(n)
    torch.cuda.synchronize()                 # torch zeroed them on its stream; the calls below run on the ctx stream
    for r in range(sh.world):
        L.check(lib.bevk_shard_vsum(h, V(d.data_ptr()), stride, n, r, V(vs.data_ptr())))
    for r in range(sh.world):
        L.check(lib.bevk_shard_render_balanced(h, V(d.data_ptr()), stride, n, r, V(vs.data_ptr()), V(slabs.data_ptr())))
    L.check(lib.bevk_shard_compose_balanced(h, V(slabs.data_ptr()), n, V(car.data_ptr()), V(out.data_ptr())))


def test_fuzz_corpus_worlds_2_and_3():
    """The 4-camera cases (FW % 32 luminance row tails, saturating seams, every kernel path) through worlds 2 and 3,
    batches 1 and 5, with the car; both compose paths (BW % 8 == 0 and not).  Frames sit in a stack whose stride is
    padded to 16 bytes with 0xFF."""
    import torch
    from cameracalibration_b200 import ops
    from cameracalibration_b200.sharding import ShardedBev
    compared, wide, narrow = 0, 0, 0
    for case in (c for c in B.corpus() if c.NC == 4):
        e = _case_engine(ops, case)
        try:
            car = torch.from_numpy(case.car).cuda()
            fb = case.FW * case.FH * 3
            stride = (fb + 15) // 16 * 16
            for n in (1, 5):
                want = [B.oracle(case, s, True, True) for s in range(n)]
                if all(w is None for w in want):
                    continue
                host = np.full((n * 4, stride), 0xFF, np.uint8)
                host[:, :fb] = np.stack([np.stack(s) for s in case.sets[:n]]).reshape(n * 4, fb)
                d = torch.from_numpy(host).cuda()
                torch.cuda.synchronize()
                for world in (2, 3):
                    sh = ShardedBev(e, "cameras", rank=0, world=world, connect=False)
                    out = torch.empty((n, case.BH, case.BW, 3), dtype=torch.uint8, device="cuda")
                    torch.cuda.synchronize()
                    _emulate_stack(e, sh, d, stride, n, car, out)
                    e.ctx.sync()
                    got = out.cpu().numpy()
                    for s, w in enumerate(want):
                        if w is None:
                            continue
                        assert (got[s] == w).all(), (case.name, n, world, s)
                        compared += 1
                        wide += case.BW % 8 == 0
                        narrow += case.BW % 8 != 0
        finally:
            e.ctx.close()
    assert compared > 0 and wide > 0 and narrow > 0, (compared, wide, narrow)


def test_peer_store_variant_with_balance_on_one_gpu(fx):
    """bevk_bev_run_scattered with BALANCE and a world of one: the ΣV exchange is skipped, the peer-store render reads
    the balanced copies, and the owner colour-balances its canvases.  Batch 6, with and without the car."""
    import torch
    from cameracalibration_b200 import _lib as L
    g = fx.geometry()
    e, _ = _engine(fx, g, True, calib=fx.calib)
    dev = torch.device("cuda", e.ctx.device)
    F = fx.frames()
    sets = [[np.ascontiguousarray(np.roll(f, 17 * i + 3 * c, axis=1)) for c, f in enumerate(F)] for i in range(6)]
    d_all = torch.from_numpy(np.stack([np.stack(s) for s in sets])).to(dev)
    car = torch.from_numpy(fx.car()).to(dev)
    lib, h = e.ctx.lib, e.ctx.h
    L.check(lib.bevk_shard_configure(h, L.SHARD_CAMERAS, 0, 1))
    handle = (ctypes.c_uint8 * 64)()
    L.check(lib.bevk_shard_prepare(h, 6, handle))
    L.check(lib.bevk_shard_attach(h, bytes(handle)))
    for c in (None, car):
        full = torch.empty((6, g.BH, g.BW, 3), dtype=torch.uint8, device=dev)
        e.run_stack(d_all.data_ptr(), g.FH * g.FW * 3, 6, full.data_ptr(), 0 if c is None else c.data_ptr(), balance=True)
        own = torch.zeros((6, g.BH, g.BW, 3), dtype=torch.uint8, device=dev)
        n_own = ctypes.c_int()
        L.check(lib.bevk_bev_run_scattered(h, ctypes.c_void_p(d_all.data_ptr()), g.FH * g.FW * 3, 6,
                                           ctypes.c_void_p(0 if c is None else c.data_ptr()), L.FLAG_BALANCE,
                                           ctypes.c_void_p(own.data_ptr()), ctypes.byref(n_own)))
        e.ctx.sync()
        assert n_own.value == 6 and e.last_path() == "tma"
        assert (own.cpu().numpy() == full.cpu().numpy()).all()


def test_byte_compose_on_unaligned_output_with_saturating_seams(fx):
    """Canvas 998 px wide (BW % 8 != 0) into an output at byte offset 1: the byte path of the compose and of k_gain.
    Plain masks overlap on their seams, and bright frames make those sums saturate; the channel sums must stay exact."""
    import cv2
    import torch
    from cameracalibration_b200.sharding import ShardedBev
    g = fx.geometry(FW=640, FH=512, BW=998, BH=500)
    e, masks = _engine(fx, g, False)
    dev = torch.device("cuda", e.ctx.device)
    F = [cv2.add(f, 90) for f in fx.frames(640, 512)]
    sets = [F, [np.ascontiguousarray(f[:, ::-1]) for f in F]]
    d_all = torch.from_numpy(np.stack([np.stack(s) for s in sets])).to(dev)
    car = torch.from_numpy(fx.car(998, 500)).to(dev)
    cb = g.BW * g.BH * 3
    full = torch.empty((2, g.BH, g.BW, 3), dtype=torch.uint8, device=dev)
    e.run_stack(d_all.data_ptr(), g.FH * g.FW * 3, 2, full.data_ptr(), car.data_ptr(), balance=True)
    e.ctx.sync()
    full = full.cpu().numpy()
    ref = C.RefBev(fx.scaled_calib(g), g, False, True, masks=masks)
    assert (full[0] == ref(*sets[0], fx.car(998, 500))).all()
    # saturating seams: where two plain masks overlap, the compose of the bright frames hits 255
    overlap = (np.stack(masks) != 0).sum(axis=0) > 1
    raw = torch.empty((2, g.BH, g.BW, 3), dtype=torch.uint8, device=dev)
    e.run_stack(d_all.data_ptr(), g.FH * g.FW * 3, 2, raw.data_ptr())
    e.ctx.sync()
    assert (raw.cpu().numpy()[0][overlap] == 255).any()
    for world in (2, 4):
        sh = ShardedBev(e, "cameras", rank=0, world=world, connect=False)
        buf = torch.full((2 * cb + 17,), 0xA5, dtype=torch.uint8, device=dev)
        out = buf[1:1 + 2 * cb].view(2, g.BH, g.BW, 3)
        _emulate(torch, sh, lambda r: d_all, 2, car, out)
        torch.cuda.synchronize()
        b = buf.cpu().numpy()
        assert (b[1:1 + 2 * cb].reshape(full.shape) == full).all(), world
        assert b[0] == 0xA5 and (b[1 + 2 * cb:] == 0xA5).all()


def test_stream_ordering_and_graph_replay(fx):
    import torch
    from cameracalibration_b200 import _lib as L
    from cameracalibration_b200.sharding import ShardedBev
    g = fx.geometry()
    e, _ = _engine(fx, g, True, calib=fx.calib)
    dev = torch.device("cuda", e.ctx.device)
    host = np.stack([np.stack(s) for s in _sets(fx)])
    d_src = torch.from_numpy(host).to(dev)
    car = torch.from_numpy(fx.car()).to(dev)
    sh = ShardedBev(e, "cameras", rank=0, world=3, connect=False)
    direct = torch.empty((3, g.BH, g.BW, 3), dtype=torch.uint8, device=dev)
    _emulate(torch, sh, lambda r: d_src, 3, car, direct)
    torch.cuda.synchronize()
    direct = direct.cpu().numpy()
    # on a side stream, after the kernel that produced the frames
    side = torch.cuda.Stream(device=dev)
    out = torch.zeros((3, g.BH, g.BW, 3), dtype=torch.uint8, device=dev)
    with torch.cuda.stream(side):
        d_in = (d_src.to(torch.int16) * 1).to(torch.uint8)      # frames produced by torch kernels on `side`
        _emulate(torch, sh, lambda r: d_in, 3, car, out)
        got = out.clone()
    side.synchronize()
    assert (got.cpu().numpy() == direct).all()
    # the same sequence captured into a CUDA graph, replayed twice
    lib, h = e.ctx.lib, e.ctx.h
    e.ctx.sync()
    vs, slabs = sh.vsum_buffer(3), sh.slab_buffer(3)
    out = torch.zeros((3, g.BH, g.BW, 3), dtype=torch.uint8, device=dev)
    stride = g.FH * g.FW * 3

    def seq():
        for r in range(3):
            L.check(lib.bevk_shard_vsum(h, ctypes.c_void_p(d_src.data_ptr()), stride, 3, r, ctypes.c_void_p(vs.data_ptr())))
        for r in range(3):
            L.check(lib.bevk_shard_render_balanced(h, ctypes.c_void_p(d_src.data_ptr()), stride, 3, r, ctypes.c_void_p(vs.data_ptr()),
                                                   ctypes.c_void_p(slabs.data_ptr())))
        L.check(lib.bevk_shard_compose_balanced(h, ctypes.c_void_p(slabs.data_ptr()), 3, ctypes.c_void_p(car.data_ptr()),
                                                ctypes.c_void_p(out.data_ptr())))
    torch.cuda.synchronize()
    seq()
    e.ctx.sync()
    assert (out.cpu().numpy() == direct).all()
    with e.ctx.graph_capture() as gr:
        seq()
    try:
        for rep in range(2):
            out.zero_(); vs.zero_(); slabs.zero_()
            torch.cuda.synchronize()
            gr.launch()
            e.ctx.sync()
            assert (out.cpu().numpy() == direct).all(), rep
    finally:
        gr.destroy()


def test_argument_errors(fx):
    import torch
    from cameracalibration_b200 import _lib as L
    from cameracalibration_b200 import ops
    from cameracalibration_b200.sharding import ShardedBev
    g = fx.geometry(FW=128, FH=64, BW=96, BH=96)
    e, _ = _engine(fx, g, True)
    lib, h = e.ctx.lib, e.ctx.h
    dev = torch.device("cuda", e.ctx.device)
    stride = g.FH * g.FW * 3
    frames = torch.zeros((2, 4, g.FH, g.FW, 3), dtype=torch.uint8, device=dev)
    fp = ctypes.c_void_p(frames.data_ptr())
    sh = ShardedBev(e, "cameras", rank=0, world=2, connect=False)
    vs, slabs = sh.vsum_buffer(2), sh.slab_buffer(2)
    vp, sp = vs.data_ptr(), slabs.data_ptr()
    out = torch.empty((2, g.BH, g.BW, 3), dtype=torch.uint8, device=dev)
    e.ctx.sync()
    n0 = e.ctx.launches

    def refused(rc, msg):
        assert rc != 0 and msg in lib.bevk_last_error().decode(), lib.bevk_last_error().decode()

    V = lambda p: ctypes.c_void_p(p)
    refused(lib.bevk_shard_vsum(h, fp, stride, 2, 0, None), "V-sum buffer")
    refused(lib.bevk_shard_vsum(h, fp, stride, 2, 0, V(vp + 4)), "8-byte aligned")
    refused(lib.bevk_shard_vsum(h, fp, stride, 2, 2, V(vp)), "rank 2 out of range")
    refused(lib.bevk_shard_vsum(h, fp, stride, 0, 0, V(vp)), "batch 0")
    refused(lib.bevk_shard_vsum(h, fp, stride, 16384, 0, V(vp)), "65535 frames")
    refused(lib.bevk_shard_render_balanced(h, fp, stride, 2, 0, None, V(sp)), "V-sum buffer")
    refused(lib.bevk_shard_render_balanced(h, fp, stride, 2, 0, V(vp + 4), V(sp)), "8-byte aligned")
    refused(lib.bevk_shard_render_balanced(h, fp, stride, 2, 0, V(vp), V(sp + 8)), "16-byte aligned")
    refused(lib.bevk_shard_render_balanced(h, fp, stride, 2, -1, V(vp), V(sp)), "out of range")
    refused(lib.bevk_shard_render_balanced(h, fp, stride, 16384, 0, V(vp), V(sp)), "65535 frames")
    refused(lib.bevk_shard_compose_balanced(h, None, 2, None, V(out.data_ptr())), "null")
    refused(lib.bevk_shard_compose_balanced(h, V(sp), 2, None, None), "null")
    refused(lib.bevk_shard_compose_balanced(h, V(sp), 16384, None, V(out.data_ptr())), "65535 frames")
    refused(lib.bevk_shard_compose_balanced(h, V(sp), 0, None, V(out.data_ptr())), "batch 0")
    with pytest.raises(L.BevkError, match="8-byte integers"):
        sh.vsums(frames, 0, torch.zeros((2, 2, 4), dtype=torch.int32, device=dev))
    with pytest.raises(L.BevkError, match="shape"):
        sh.render_slabs(frames, 0, slabs, vsums=torch.zeros((2, 3, 4), dtype=torch.int64, device=dev))
    # a single-GPU engine refuses batch x n_cam > 65535 under BALANCE before it enqueues anything
    big = 16384
    with pytest.raises(L.BevkError, match="65535 frames"):
        e.run_stack(frames.data_ptr(), stride, big, out.data_ptr(), 0, balance=True)
    assert e.ctx.launches == n0
    # configure and finalize come first
    e2 = ops.BevEngine(4, (g.FW, g.FH), (g.BW, g.BH))
    try:
        refused(lib.bevk_shard_vsum(e2.ctx.h, fp, stride, 2, 0, V(vp)), "bevk_shard_configure not called")
        L.check(lib.bevk_shard_configure(e2.ctx.h, L.SHARD_CAMERAS, 0, 2))
        refused(lib.bevk_shard_vsum(e2.ctx.h, fp, stride, 2, 0, V(vp)), "bevk_bev_finalize not called")
        refused(lib.bevk_shard_render_balanced(e2.ctx.h, fp, stride, 2, 0, V(vp), V(sp)), "bevk_bev_finalize not called")
        refused(lib.bevk_shard_compose_balanced(e2.ctx.h, V(sp), 2, None, V(out.data_ptr())), "bevk_bev_finalize not called")
    finally:
        e2.ctx.close()


def _nccl_balance_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), LOCAL_RANK=str(rank))
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from cameracalibration_b200.sharding import ShardedBev
        from tests.helpers import Fixtures
        fx = Fixtures()
        g = fx.geometry()
        res = {}
        for blend in (False, True):
            e, masks = _engine(fx, g, blend, calib=fx.calib, device=rank)
            dev = torch.device("cuda", rank)
            F = fx.frames()
            sets = [F, [np.ascontiguousarray(f[::-1]) for f in F], F, F, [np.ascontiguousarray(np.roll(f, 31, axis=1)) for f in F]]
            host = np.stack([np.stack(s) for s in sets])
            lo, hi = ShardedBev(e, "cameras", connect=False).my_cameras()
            d_mine = torch.from_numpy(_poisoned(host, lo, hi)).to(dev)
            car = torch.from_numpy(fx.car()).to(dev)
            sh = ShardedBev(e, "cameras")
            ref = C.RefBev(fx.calib, g, blend, True, masks=masks)
            out = torch.empty((5, g.BH, g.BW, 3), dtype=torch.uint8, device=dev)
            stream = torch.cuda.Stream(device=dev)
            with torch.cuda.stream(stream):
                d_in = d_mine.clone()
                sh.render(d_in, out, car, balance=True)
                got = out.clone()
            stream.synchronize()
            got = got.cpu().numpy()
            ok = all((got[i] == ref(*sets[i], fx.car())).all() for i in (0, 1, 4))
            slab_bytes = sh.info()[3]
            want_link = 5 * slab_bytes * (world - 1) + 5 * 4 * 8 * (world - 1)
            res[f"cameras_blend{int(blend)}"] = (ok, sh.link_bytes() == want_link, sh.link_bytes())
            own = sh.own_frame_sets(5)
            out_own = torch.zeros((3, g.BH, g.BW, 3), dtype=torch.uint8, device=dev)
            okp, vs_bytes = True, 5 * 4 * 8 * (world - 1)
            for step in range(3):
                d_in = d_mine.roll(step, 0).contiguous()
                torch.cuda.synchronize()
                n_own = sh.render_scattered(d_in, out_own, car, balance=True)
                torch.cuda.synchronize()
                want = [ref(*sets[(b - step) % 5], fx.car()) for b in own]
                okp &= n_own == len(own) and all((out_own[i].cpu().numpy() == want[i]).all() for i in range(n_own))
                okp &= sh.link_bytes() == (5 - n_own) * slab_bytes + vs_bytes
            res[f"p2p_blend{int(blend)}"] = (bool(okp), sh.link_bytes() > vs_bytes, sh.link_bytes())
        q.put((rank, res))
    finally:
        dist.destroy_process_group()


def test_balance_world2_nccl(fx):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_nccl_balance_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=600) for _ in procs)
    for p in procs:
        p.join(60)
    for r in (0, 1):
        for key, val in res[r].items():
            assert val[0] and val[1], (r, key, val)
