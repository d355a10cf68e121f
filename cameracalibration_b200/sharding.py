"""Multi-GPU sharding of the BEV path: one process per GPU.

The reference is single-process (SURVEY 2.1: no collective anywhere); the path shards two ways, both implemented in
libbevk.so (bevk_shard_* / bevk_bev_run_sharded, include/bevk.h) so that a binding without torch can use them too:

  * frame-sets per GPU ("frames"): every rank renders its own block of frame-sets with a full replica of the plan.
    No data-path collective.
  * cameras per GPU ("cameras"): rank r renders cameras [lo_r, hi_r) of every frame-set into a SLAB (the tile-aligned
    bounding box of the union of their masks: 0.9-1.2 MB per frame-set at 1000x1000 instead of the 3 MB canvas), ONE
    ncclAllGather moves the slabs over NVLink, and every rank composes them with the saturating sum.  Exact, because
    the reference's cv2.add chain (surroundBEV.py:316-320) is order-independent.  With balance=True each rank first
    sums V over its own cameras' frames and one all-gather of those uint64 sums ([world][batch][n_cam]) gives every
    rank every camera's luminance offset (luminance_balance needs all V means before the warp); each rank balances
    and renders its own cameras, and colour balance runs on the composed canvases.  Every step is exact in integers,
    so the canvases are byte-identical to the single-GPU render.
    The same policy with the exchange FUSED into the render kernel: ShardedBev.render_scattered -- frame-set b is owned
    by rank b % world, the fused kernel's write-out stores each slab straight into the owner's memory over NVLink (CUDA
    IPC peer mapping), a 4-byte all-gather is the step barrier, each rank composes the canvases it owns.

ShardedBev is a thin caller: it carries the NCCL unique id between the ranks with torch.distributed (any backend) and
points the engine at torch's current stream for the duration of a call, so that frames produced by torch kernels,
the render, the collective and the consumer of ``out`` are ordered on ONE stream.

The pure partition functions below are what the world_size-2 gloo tests exercise on CPU; libbevk.so uses the same rule
(bevk_shard.cuh: shard_block), and the GPU tests compare the two.
"""
from __future__ import annotations

import ctypes as C


def block_range(n_items: int, rank: int, world: int) -> tuple[int, int]:
    """Contiguous block partition of n_items over world ranks; the first n_items % world ranks
    get one extra item.  Returns [lo, hi)."""
    if world < 1 or not (0 <= rank < world):
        raise ValueError(f"rank {rank} outside world {world}")
    base, extra = divmod(n_items, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def camera_range(n_cam: int, rank: int, world: int) -> tuple[int, int]:
    """Cameras of one rank.  With more ranks than cameras the trailing ranks get an empty range
    (they still join the all-gather, with an empty slab)."""
    return block_range(n_cam, rank, world)


def slab_rect(masks, lo: int, hi: int, tile: int = 32):
    """Tile-aligned bounding box (x0, y0, x1, y1) of the union of masks[lo:hi], clipped to the canvas; (0, 0, 0, 0)
    when empty.  NumPy statement of bevk_shard.cuh:slab_rect."""
    import numpy as np
    if hi <= lo:
        return 0, 0, 0, 0
    u = np.zeros_like(np.asarray(masks[lo]), dtype=bool)
    for m in masks[lo:hi]:
        u |= np.asarray(m) != 0
    if not u.any():
        return 0, 0, 0, 0
    ys, xs = np.nonzero(u.any(axis=1))[0], np.nonzero(u.any(axis=0))[0]
    BH, BW = u.shape
    x0, y0 = int(xs[0]) // tile * tile, int(ys[0]) // tile * tile
    x1 = min(BW, (int(xs[-1]) + tile) // tile * tile)
    y1 = min(BH, (int(ys[-1]) + tile) // tile * tile)
    return x0, y0, x1, y1


class ShardedBev:
    """Drives a BevEngine under a multi-process launch.  Tensors are CUDA arrays (torch or anything with
    ``__cuda_array_interface__``); the engine only sees their device pointers."""

    def __init__(self, engine, policy: str = "frames", group=None, rank: int | None = None, world: int | None = None,
                 connect: bool = True):
        from . import _lib as L
        if policy not in ("frames", "cameras"):
            raise ValueError("policy must be 'frames' or 'cameras'")
        self.e, self.policy, self.group = engine, policy, group
        if rank is None or world is None:
            import torch.distributed as dist
            on = dist.is_available() and dist.is_initialized()
            rank = dist.get_rank(group) if on else 0
            world = dist.get_world_size(group) if on else 1
        self.rank, self.world = int(rank), int(world)
        if not engine.finalized:
            engine.finalize()
        lib, h = engine.ctx.lib, engine.ctx.h
        L.check(lib.bevk_shard_configure(h, L.SHARD_CAMERAS if policy == "cameras" else L.SHARD_FRAMES, self.rank, self.world))
        if policy == "cameras" and self.world > 1 and connect:   # connect=False: geometry / render_slabs / compose only
            self._connect()

    def _connect(self):
        """NCCL unique id: made on rank 0, carried to the others as a tensor broadcast (works on gloo and nccl)."""
        import torch
        import torch.distributed as dist
        from . import _lib as L
        lib, h = self.e.ctx.lib, self.e.ctx.h
        buf = (C.c_uint8 * 128)()
        if self.rank == 0:
            L.check(lib.bevk_shard_unique_id(buf, 128))
        backend = dist.get_backend(self.group)
        dev = torch.device("cuda", self.e.ctx.device) if backend == "nccl" else torch.device("cpu")
        t = torch.tensor(list(buf), dtype=torch.uint8, device=dev)
        dist.broadcast(t, src=dist.get_global_rank(self.group, 0) if self.group is not None else 0, group=self.group)
        raw = bytes(t.cpu().tolist())
        L.check(lib.bevk_shard_connect(h, raw, 128))

    def my_frame_sets(self, n_sets: int):
        return block_range(n_sets, self.rank, self.world)

    def my_cameras(self):
        return camera_range(self.e.n_cam, self.rank, self.world)

    def info(self, rank: int | None = None):
        """(cam_lo, cam_hi, (x0, y0, x1, y1), slab_bytes) of `rank` as libbevk.so computed them."""
        from . import _lib as L
        lo, hi, sb = C.c_int(), C.c_int(), C.c_int64()
        rect = (C.c_int32 * 4)()
        L.check(self.e.ctx.lib.bevk_shard_info(self.e.ctx.h, self.rank if rank is None else rank, C.byref(lo), C.byref(hi), rect, C.byref(sb)))
        return lo.value, hi.value, tuple(rect), sb.value

    def render(self, frames, out, car=None, balance: bool = False, stream: int | None = None):
        """frames: uint8 CUDA array [batch][n_cam][FH][FW][3] (a frame stack; with policy 'cameras' every rank passes
        the same batch and only its own cameras' frames are read).  out: uint8 CUDA array [batch][BH][BW][3].
        ``stream``: raw CUDA stream handle; default torch's current stream.  Only enqueues; returns ``out``."""
        from . import _lib as L
        from .ops import _cuda_ptr
        e = self.e
        base, shape = _cuda_ptr(frames, None)
        if len(shape) != 5 or tuple(shape[1:]) != (e.n_cam, e.FH, e.FW, 3):
            raise L.BevkError(f"frames must be uint8[batch][{e.n_cam}][{e.FH}][{e.FW}][3], got {tuple(shape)}")
        batch = shape[0]
        d_out = _cuda_ptr(out, (batch, e.BH, e.BW, 3))[0]
        d_car = _cuda_ptr(car, (e.BH, e.BW, 3))[0] if car is not None else None
        if stream is None:
            stream = _torch_current_stream(e.ctx.device)
        with e.ctx.on_stream(stream):
            L.check(e.ctx.lib.bevk_bev_run_sharded(e.ctx.h, C.c_void_p(base), e.FH * e.FW * 3, batch, C.c_void_p(d_car),
                                                   L.FLAG_BALANCE if balance else 0, C.c_void_p(d_out)))
        return out

    def slab_buffer(self, batch: int):
        """torch uint8 CUDA tensor [world][batch][slab_bytes] for render_slabs / compose."""
        import torch
        return torch.zeros((self.world, batch, self.info()[3]), dtype=torch.uint8, device=torch.device("cuda", self.e.ctx.device))

    def vsum_buffer(self, batch: int):
        """torch int64 CUDA tensor [world][batch][n_cam], zeroed, for vsums / render_slabs(vsums=...).  The library
        treats it as uint64; a V sum stays far below 2**63."""
        import torch
        return torch.zeros((self.world, batch, self.e.n_cam), dtype=torch.int64, device=torch.device("cuda", self.e.ctx.device))

    def vsums(self, frames, as_rank: int, buf, stream: int | None = None):
        """The first BALANCE step of the 'cameras' policy on its own: the V sums of rank `as_rank`'s own cameras into
        buf[as_rank] (zero in the other cameras' columns).  Every block must be filled (an all-gather, or every rank
        on one GPU) before render_slabs(vsums=buf)."""
        from . import _lib as L
        from .ops import _cuda_ptr
        e = self.e
        base, shape = _cuda_ptr(frames, None)
        d_buf = _vsum_ptr(buf, (self.world, shape[0], e.n_cam))
        with e.ctx.on_stream(_torch_current_stream(e.ctx.device) if stream is None else stream):
            L.check(e.ctx.lib.bevk_shard_vsum(e.ctx.h, C.c_void_p(base), e.FH * e.FW * 3, shape[0], int(as_rank), C.c_void_p(d_buf)))

    def render_slabs(self, frames, as_rank: int, slabs, stream: int | None = None, vsums=None):
        """The render half of the 'cameras' policy on its own: the slabs of rank `as_rank` into slabs[as_rank].
        ``vsums``: the filled vsum_buffer -- render the luminance-balanced slabs (then compose with balance=True)."""
        from . import _lib as L
        from .ops import _cuda_ptr
        e = self.e
        base, shape = _cuda_ptr(frames, None)
        d_slabs = _cuda_ptr(slabs, (self.world, shape[0], self.info()[3]))[0]
        with e.ctx.on_stream(_torch_current_stream(e.ctx.device) if stream is None else stream):
            if vsums is None:
                L.check(e.ctx.lib.bevk_shard_render(e.ctx.h, C.c_void_p(base), e.FH * e.FW * 3, shape[0], int(as_rank), C.c_void_p(d_slabs)))
            else:
                d_vs = _vsum_ptr(vsums, (self.world, shape[0], e.n_cam))
                L.check(e.ctx.lib.bevk_shard_render_balanced(e.ctx.h, C.c_void_p(base), e.FH * e.FW * 3, shape[0], int(as_rank),
                                                             C.c_void_p(d_vs), C.c_void_p(d_slabs)))

    def compose(self, slabs, out, car=None, stream: int | None = None, balance: bool = False):
        """The compose half: slabs[world][batch][slab_bytes] (+ car) -> out[batch][BH][BW][3].  balance=True: colour
        balance of the composed canvases before the car (slabs rendered with vsums=...)."""
        from . import _lib as L
        from .ops import _cuda_ptr
        e = self.e
        d_slabs, shape = _cuda_ptr(slabs, None)
        d_out = _cuda_ptr(out, (shape[1], e.BH, e.BW, 3))[0]
        d_car = _cuda_ptr(car, (e.BH, e.BW, 3))[0] if car is not None else None
        fn = e.ctx.lib.bevk_shard_compose_balanced if balance else e.ctx.lib.bevk_shard_compose
        with e.ctx.on_stream(_torch_current_stream(e.ctx.device) if stream is None else stream):
            L.check(fn(e.ctx.h, C.c_void_p(d_slabs), shape[1], C.c_void_p(d_car), C.c_void_p(d_out)))
        return out

    def own_frame_sets(self, batch: int):
        """Frame-sets of a batch whose canvases render_scattered() leaves on this rank: rank, rank + world, ..."""
        return list(range(self.rank, batch, self.world))

    def _prepare_peers(self, batch: int):
        """Size the peer-store receive buffers for `batch` and map every rank's buffer into this process (CUDA IPC):
        the 64-byte handles travel with one all_gather."""
        import torch
        import torch.distributed as dist
        from . import _lib as L
        lib, h = self.e.ctx.lib, self.e.ctx.h
        mine = (C.c_uint8 * 64)()
        L.check(lib.bevk_shard_prepare(h, int(batch), mine))
        backend = dist.get_backend(self.group)
        dev = torch.device("cuda", self.e.ctx.device) if backend == "nccl" else torch.device("cpu")
        t = torch.tensor(list(mine), dtype=torch.uint8, device=dev)
        allh = [torch.empty_like(t) for _ in range(self.world)]
        dist.all_gather(allh, t, group=self.group)
        raw = b"".join(bytes(x.cpu().tolist()) for x in allh)
        L.check(lib.bevk_shard_attach(h, raw))
        dist.barrier(group=self.group)      # nobody stores into a peer before every peer has mapped and zeroed its buffer
        self._peers_for = batch

    def render_scattered(self, frames, out_own, car=None, stream: int | None = None, balance: bool = False):
        """Policy 'cameras' with peer stores (bevk_bev_run_scattered): every rank renders its cameras' slabs of ALL
        frame-sets of ``frames`` ([batch][n_cam][FH][FW][3]; only its own cameras' frames are read), the fused kernel
        stores each slab straight into the memory of the rank that OWNS the frame-set (b % world) over NVLink, and each
        rank composes its own canvases into ``out_own`` ([ceil(batch / world)][BH][BW][3]; the first
        len(own_frame_sets(batch)) entries are valid).  balance=True: the V-sum all-gather first, colour balance of the
        owned canvases last.  Returns the number of canvases written."""
        from . import _lib as L
        from .ops import _cuda_ptr
        e = self.e
        base, shape = _cuda_ptr(frames, None)
        if len(shape) != 5 or tuple(shape[1:]) != (e.n_cam, e.FH, e.FW, 3):
            raise L.BevkError(f"frames must be uint8[batch][{e.n_cam}][{e.FH}][{e.FW}][3], got {tuple(shape)}")
        batch = shape[0]
        if getattr(self, "_peers_for", None) != batch:
            self._prepare_peers(batch)
        own_max = (batch + self.world - 1) // self.world
        d_out = _cuda_ptr(out_own, (own_max, e.BH, e.BW, 3))[0]
        d_car = _cuda_ptr(car, (e.BH, e.BW, 3))[0] if car is not None else None
        n_own = C.c_int()
        if stream is None:
            stream = _torch_current_stream(e.ctx.device)
        with e.ctx.on_stream(stream):
            L.check(e.ctx.lib.bevk_bev_run_scattered(e.ctx.h, C.c_void_p(base), e.FH * e.FW * 3, batch, C.c_void_p(d_car),
                                                     L.FLAG_BALANCE if balance else 0, C.c_void_p(d_out), C.byref(n_own)))
        return n_own.value

    def link_bytes(self) -> int:
        """Bytes this rank received (render) or stored into its peers (render_scattered) over NVLink in the last call,
        the V sums of balance=True included."""
        return int(self.e.ctx.lib.bevk_shard_last_link_bytes(self.e.ctx.h))


def _vsum_ptr(buf, shape):
    """Device pointer of a V-sum buffer: a C-contiguous 8-byte integer CUDA array of `shape` (vsum_buffer's)."""
    from . import _lib as L
    cai = getattr(buf, "__cuda_array_interface__", None)
    if cai is None:
        raise L.BevkError("V-sum buffer must expose __cuda_array_interface__")
    if cai["typestr"] not in ("<i8", "<u8"):
        raise L.BevkError(f"V-sum buffer must hold 8-byte integers, got {cai['typestr']}")
    if tuple(cai["shape"]) != tuple(shape):
        raise L.BevkError(f"V-sum buffer shape {tuple(cai['shape'])} != {tuple(shape)}")
    if cai.get("strides") is not None:
        want, acc = [], 8
        for n in reversed(shape):
            want.insert(0, acc)
            acc *= n
        if any(n > 1 and s != w for n, s, w in zip(shape, cai["strides"], want)):
            raise L.BevkError("V-sum buffer must be C-contiguous")
    return cai["data"][0]


def _torch_current_stream(device: int):
    """torch's current stream on `device` as a raw handle, or None (= the ctx's own stream) without torch."""
    try:
        import torch
        if torch.cuda.is_available():
            return torch.cuda.current_stream(device).cuda_stream
    except Exception:
        pass
    return None
