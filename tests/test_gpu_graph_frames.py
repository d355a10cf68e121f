"""A CUDA graph captured from a frame-stack call keeps reading the stack it was captured with.

Every case: render stack A eagerly, capture the same call into a graph, make one eager call on another stack B (same
shape, other contents), replay the graph, and require A's eager canvases byte for byte.  The kernels take a stack as
(base, stride) by value, so nothing an eager call leaves in the context can redirect a replay.  The cases are the paths
that read the source stack outside k_bev_tma's tensor maps:
  * run_stack with BALANCE: k_vsum and k_lum_spans read the frames, k_bev_tma reads the balanced copies;
  * run_stack on a stack whose stride is a multiple of 4 but not of 16: the k_bev fallback;
  * the camera-sharded BALANCE halves (bevk_shard_vsum / _render_balanced / _compose_balanced) for a world of 2."""
import ctypes

import numpy as np
import pytest

from tests.test_gpu_tma import _engine

pytestmark = pytest.mark.gpu


def _stacks(torch, dev, fx, batch, stride):
    """Stacks A and B on the device, frame i at base + i * stride (padding bytes 0xFF), with different contents."""
    F = fx.frames()
    fb = F[0].nbytes
    a = np.stack([np.stack([np.roll(f, 17 * b + 5 * c, axis=1) for c, f in enumerate(F)]) for b in range(batch)])
    out = []
    for frames in (a, a ^ 0x35):
        host = np.full((frames.shape[0] * frames.shape[1], stride), 0xFF, np.uint8)
        host[:, :fb] = frames.reshape(-1, fb)
        out.append(torch.from_numpy(host).to(dev))
    return out


def _replay_after_other_stack(torch, e, call, d_a, d_b, shape):
    """call(d_frames, d_out) enqueues on the ctx stream.  Returns (A's eager canvases, B's, the replay's)."""
    dev = d_a.device

    def eager(d):
        out = torch.zeros(shape, dtype=torch.uint8, device=dev)
        torch.cuda.synchronize()
        call(d, out)
        e.ctx.sync()
        return out.cpu().numpy()

    want_b = eager(d_b)
    want_a = eager(d_a)              # last eager call before the capture: everything A needs exists
    out = torch.zeros(shape, dtype=torch.uint8, device=dev)
    other = torch.zeros(shape, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()
    with e.ctx.graph_capture() as gr:
        call(d_a, out)
    try:
        call(d_b, other)             # one eager call on the other stack between capture and replay
        e.ctx.sync()
        gr.launch()
        e.ctx.sync()
        got = out.cpu().numpy()
    finally:
        gr.destroy()
    assert (want_a != want_b).any()
    assert (other.cpu().numpy() == want_b).all()
    return want_a, want_b, got


@pytest.mark.parametrize("pad, balance, path", [(0, True, "tma"), (4, False, "gather")])
def test_run_stack_replay_reads_the_captured_stack(fx, pad, balance, path):
    import torch
    from cameracalibration_b200 import ops
    g = fx.geometry()
    e, _ = _engine(ops, fx, g, True, calib=fx.calib)
    dev = torch.device("cuda", e.ctx.device)
    n, stride = 5, g.FH * g.FW * 3 + pad
    d_a, d_b = _stacks(torch, dev, fx, n, stride)
    car = torch.from_numpy(fx.car()).to(dev)

    def call(d, out):
        e.run_stack(d.data_ptr(), stride, n, out.data_ptr(), car.data_ptr(), balance)

    want_a, want_b, got = _replay_after_other_stack(torch, e, call, d_a, d_b, (n, g.BH, g.BW, 3))
    assert e.last_path() == path
    assert (got == want_a).all(), (f"replay differs from A's canvases in {int((got != want_a).sum())} bytes; "
                                   f"it equals B's: {bool((got == want_b).all())}")


def test_sharded_balance_replay_reads_the_captured_stack(fx):
    import torch
    from cameracalibration_b200 import _lib as L
    from cameracalibration_b200 import ops
    from cameracalibration_b200.sharding import ShardedBev
    g = fx.geometry()
    e, _ = _engine(ops, fx, g, True, calib=fx.calib)
    dev = torch.device("cuda", e.ctx.device)
    n, stride = 3, g.FH * g.FW * 3
    d_a, d_b = _stacks(torch, dev, fx, n, stride)
    car = torch.from_numpy(fx.car()).to(dev)
    sh = ShardedBev(e, "cameras", rank=0, world=2, connect=False)
    vs, slabs = sh.vsum_buffer(n), sh.slab_buffer(n)
    lib, h, V = e.ctx.lib, e.ctx.h, ctypes.c_void_p

    def call(d, out):
        for r in range(2):
            L.check(lib.bevk_shard_vsum(h, V(d.data_ptr()), stride, n, r, V(vs.data_ptr())))
        for r in range(2):
            L.check(lib.bevk_shard_render_balanced(h, V(d.data_ptr()), stride, n, r, V(vs.data_ptr()), V(slabs.data_ptr())))
        L.check(lib.bevk_shard_compose_balanced(h, V(slabs.data_ptr()), n, V(car.data_ptr()), V(out.data_ptr())))

    want_a, want_b, got = _replay_after_other_stack(torch, e, call, d_a, d_b, (n, g.BH, g.BW, 3))
    full = torch.empty((n, g.BH, g.BW, 3), dtype=torch.uint8, device=dev)
    e.run_stack(d_a.data_ptr(), stride, n, full.data_ptr(), car.data_ptr(), True)
    e.ctx.sync()
    assert (want_a == full.cpu().numpy()).all()
    assert (got == want_a).all(), (f"replay differs from A's canvases in {int((got != want_a).sum())} bytes; "
                                   f"it equals B's: {bool((got == want_b).all())}")
