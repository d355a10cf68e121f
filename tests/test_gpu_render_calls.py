"""Every BEV render entry point under every flag set it accepts, and the refusals of those it does not: how many kernels
each call enqueues (bevk_launch_count), which fused kernel it ran (bevk_bev_last_path), whether bevk_last_kernel_ms
reports a window afterwards, and that its canvases equal bevk_bev_run_stack's on the same frames.

The rig is the fixture cameras at 640 x 512 with a 400 x 400 canvas and 5 frame-sets: the host pipeline then runs two
chunks (4 + 1 frame-sets), and the fused kernels run both 4-frame-set and 1-frame-set work units.  Flag sets: none,
BALANCE and OUT_NV12 for BGR frames; NV12 and YUYV frames; NV12 frames with OUT_I420 and BALANCE."""
import ctypes as C

import cv2
import numpy as np
import pytest

from oracle import cv2_path as CV
from oracle import restate as R
from tests import yuv422_frames as Y422
from tests import yuv_frames as Y420
from tests.helpers import NAMES

pytestmark = pytest.mark.gpu
V = C.c_void_p
N, NC = 5, 4
ARG, UNSUP = -1, -4
BAL, NV12, I420, YUYV, OUT_NV12, OUT_I420 = 1, 2, 4, 32, 8, 16
YUV_IN = NV12 | I420 | YUYV | 64
BGR_FLAGS = (0, BAL, OUT_NV12)
ALL_FLAGS = BGR_FLAGS + (NV12, YUYV, NV12 | OUT_I420 | BAL)
YUV_FLAGS = (NV12, YUYV, NV12 | OUT_I420 | BAL)
QUALITY = 90


def render_launches(flags):
    """Kernels of one whole-canvas render: the fused kernel; with BALANCE the V sums, the deltas and the balanced (for
    YUV: converted) copies, for YUV frames without BALANCE the converted copies; k_gain or k_canvas_yuv last."""
    n = 1
    if flags & BAL:
        n += 3
    elif flags & YUV_IN:
        n += 1
    if flags & (BAL | OUT_NV12 | OUT_I420):
        n += 1
    return n


def gather_path(flags):
    """The fused kernel of a frame table: k_bev, but BALANCE and YUV renders read the copy stack of their pre-pass with
    k_bev_tma."""
    return 2 if flags & (BAL | YUV_IN) else 1


class Rig:
    def __init__(self, fx):
        import torch
        from cameracalibration_b200 import _lib as L
        from cameracalibration_b200 import ops
        self.torch, self.L = torch, L
        g = fx.geometry(640, 512, 400, 400)
        self.g = g
        calib = fx.scaled_calib(g)
        e = ops.BevEngine(NC, (g.FW, g.FH), (g.BW, g.BH), ctx=L.Context(0))
        for i, n in enumerate(NAMES):
            K, D, H = calib[n]
            e.set_camera(i, K, D, CV.dst_camera_matrix(K, g.FW, g.FH, g.FS, g.SS), (int(g.FW * g.SS), int(g.FH * g.SS)), H)
            e.set_mask(i, R.blend_mask(n, g.BW, g.BH, g.CW, g.CH))
        e.finalize()
        assert e.tma_plan_info()["items"] > 0, "the rig needs the TMA-staged kernel"
        self.e, self.lib, self.h = e, e.ctx.lib, e.ctx.h
        self.dev = torch.device("cuda", e.ctx.device)
        F = fx.frames(g.FW, g.FH)
        sets = [[np.ascontiguousarray(np.roll(f, 23 * b + 5 * k, axis=1)) for k, f in enumerate(F)] for b in range(N)]
        self.host = {0: [f for s in sets for f in s]}
        self.host[NV12] = [Y420.from_bgr(f, "nv12") for f in self.host[0]]
        self.host[YUYV] = [Y422.from_bgr(f, "yuyv") for f in self.host[0]]
        self.stack = {k: torch.from_numpy(np.stack(v)).to(self.dev) for k, v in self.host.items()}
        self.car_host = np.ascontiguousarray(fx.car(g.BW, g.BH))
        self.car = torch.from_numpy(self.car_host).to(self.dev)
        self.refs = {}

    def fmt(self, flags):
        return NV12 if flags & NV12 else YUYV if flags & YUYV else 0

    def stride(self, flags):
        return self.stack[self.fmt(flags)][0].numel()

    def ptrs(self, flags, order=None):
        s = self.stack[self.fmt(flags)]
        order = range(N * NC) if order is None else order
        return [s.data_ptr() + i * self.stride(flags) for i in order]

    def shape(self, flags, n=N):
        return (n, self.g.BH * 3 // 2, self.g.BW) if flags & (OUT_NV12 | OUT_I420) else (n, self.g.BH, self.g.BW, 3)

    def out(self, flags, n=N):
        return self.torch.zeros(self.shape(flags, n), dtype=self.torch.uint8, device=self.dev)

    def ref(self, flags, car=True):
        """bevk_bev_run_stack's canvases of the rig's frames under flags."""
        key = (flags, car)
        if key not in self.refs:
            o = self.out(flags)
            self.L.check(self.lib.bevk_bev_run_stack(self.h, V(self.stack[self.fmt(flags)].data_ptr()), self.stride(flags), N,
                                                     V(self.car.data_ptr() if car else 0), flags, V(o.data_ptr())))
            self.e.ctx.sync()
            self.refs[key] = o.cpu().numpy()
        return self.refs[key]

    def timed(self):
        ms = C.c_float()
        return self.lib.bevk_last_kernel_ms(self.h, C.byref(ms)) == 0

    def launches(self):
        return int(self.lib.bevk_launch_count(self.h))

    def path(self):
        return int(self.lib.bevk_bev_last_path(self.h))

    def error(self):
        return self.lib.bevk_last_error().decode()

    def slab_bytes(self):
        sb = C.c_int64()
        self.L.check(self.lib.bevk_shard_info(self.h, 0, None, None, None, C.byref(sb)))
        return sb.value

    def jpeg_encode(self, canvases, n):
        """(launches, streams) of bevk_jpeg_encode over the first n canvases (a device tensor)."""
        bound = C.c_uint64()
        self.L.check(self.lib.bevk_jpeg_encode_bound(self.g.BW, self.g.BH, C.byref(bound)))
        cap = bound.value * n
        out, sizes = np.zeros(cap, np.uint8), (C.c_uint64 * n)()
        l0 = self.launches()
        self.L.check(self.lib.bevk_jpeg_encode(self.h, V(canvases.data_ptr()), self.g.BW * self.g.BH * 3, self.g.BW * 3, n,
                                               self.g.BW, self.g.BH, QUALITY, V(out.ctypes.data), cap, sizes))
        return self.launches() - l0, _split(out, sizes)


def _split(buf, sizes):
    out, o = [], 0
    for s in sizes:
        out.append(bytes(buf[o:o + s]))
        o += s
    return out


@pytest.fixture(scope="module")
def rig(fx):
    r = Rig(fx)
    yield r
    r.e.ctx.close()


def _host_array(ptrs, T=V):
    return (T * len(ptrs))(*ptrs)


# Each call returns (rc, canvases, a function that returns the canvases bevk_bev_run_stack makes of the same frames (or None),
# kernels expected, fused kernel expected (1 k_bev, 2 k_bev_tma, None: no render), timed afterwards).  batch overrides N
# for the refusals.

def call_run_device(r, flags, batch=N):
    tab = r.torch.tensor(r.ptrs(flags), dtype=r.torch.int64, device=r.dev)
    o = r.out(flags)
    rc = r.lib.bevk_bev_run_device(r.h, V(tab.data_ptr()), batch, V(r.car.data_ptr()), flags, V(o.data_ptr()))
    r.e.ctx.sync()
    return rc, o, lambda: r.ref(flags), render_launches(flags), gather_path(flags), True


def call_run_frames(r, flags, batch=N):
    o = r.out(flags)
    rc = r.lib.bevk_bev_run_frames(r.h, _host_array(r.ptrs(flags)), batch, V(r.car.data_ptr()), flags, V(o.data_ptr()))
    return rc, o, lambda: r.ref(flags), render_launches(flags), 2, True


def call_run_frames_table(r, flags, batch=N):
    """A table that is not a frame stack (frame-sets in reverse order): the cached device table and k_bev."""
    order = [b * NC + k for b in reversed(range(N)) for k in range(NC)]
    o = r.out(flags)
    rc = r.lib.bevk_bev_run_frames(r.h, _host_array(r.ptrs(flags, order)), batch, V(r.car.data_ptr()), flags, V(o.data_ptr()))
    return rc, o, lambda: r.ref(flags)[::-1], render_launches(flags), gather_path(flags), True


def call_run_stack(r, flags, batch=N):
    o = r.out(flags)
    rc = r.lib.bevk_bev_run_stack(r.h, V(r.stack[r.fmt(flags)].data_ptr()), r.stride(flags), batch, V(r.car.data_ptr()), flags,
                                  V(o.data_ptr()))
    return rc, o, lambda: r.ref(flags), render_launches(flags), 2, True


def _planes(r, flags):
    fw, fh = r.g.FW, r.g.FH
    if r.fmt(flags) == YUYV:
        return [0, 0, 0], [2 * fw, 0, 0], 1
    return [0, fw * fh, 0], [fw, fw, 0], 2


def call_yuv_planes(r, flags, batch=N):
    offs, pitch, _ = _planes(r, flags)
    s = r.stack[r.fmt(flags)] if r.fmt(flags) else r.stack[NV12]
    o = r.out(flags)
    rc = r.lib.bevk_bev_run_yuv_planes(r.h, V(s.data_ptr()), s[0].numel(), _host_array(offs, C.c_int64),
                                       _host_array(pitch, C.c_int64), batch, V(r.car.data_ptr()), flags, V(o.data_ptr()))
    return rc, o, lambda: r.ref(flags) if r.fmt(flags) else None, render_launches(flags), 2, True


def call_yuv_surfaces(r, flags, batch=N):
    offs, pitch, np_ = _planes(r, flags)
    tab = []
    for p in r.ptrs(flags if r.fmt(flags) else NV12):
        tab += [p + offs[q] if q < np_ else 0 for q in range(3)]
    o = r.out(flags)
    rc = r.lib.bevk_bev_run_yuv_surfaces(r.h, _host_array(tab), _host_array(pitch, C.c_int64), batch, V(r.car.data_ptr()), flags,
                                         V(o.data_ptr()))
    return rc, o, lambda: r.ref(flags) if r.fmt(flags) else None, render_launches(flags), 2, True


def call_stack_cams(r, cams, batch=N):
    o = r.out(0)
    rc = r.lib.bevk_bev_run_stack_cams(r.h, V(r.stack[0].data_ptr()), r.stride(0), batch, cams[0], cams[1], V(o.data_ptr()))
    return rc, o, lambda: r.ref(0, car=False) if cams == (0, NC) else None, 1, 2, True


def call_device_cams(r, cams, batch=N):
    tab = r.torch.tensor(r.ptrs(0), dtype=r.torch.int64, device=r.dev)
    o = r.out(0)
    rc = r.lib.bevk_bev_run_device_cams(r.h, V(tab.data_ptr()), batch, cams[0], cams[1], V(o.data_ptr()))
    r.e.ctx.sync()
    return rc, o, lambda: r.ref(0, car=False) if cams == (0, NC) else None, 1, 1, True


def call_run_sharded_frames(r, flags, batch=N):
    r.L.check(r.lib.bevk_shard_configure(r.h, r.L.SHARD_FRAMES, 1, 2))
    o = r.out(flags)
    rc = r.lib.bevk_bev_run_sharded(r.h, V(r.stack[0].data_ptr()), r.stride(0), batch, V(r.car.data_ptr()), flags, V(o.data_ptr()))
    return rc, o, lambda: r.ref(flags), render_launches(flags), 2, True


def call_run_sharded_cameras1(r, flags, batch=N):
    r.L.check(r.lib.bevk_shard_configure(r.h, r.L.SHARD_CAMERAS, 0, 1))
    o = r.out(flags)
    rc = r.lib.bevk_bev_run_sharded(r.h, V(r.stack[0].data_ptr()), r.stride(0), batch, V(r.car.data_ptr()), flags, V(o.data_ptr()))
    return rc, o, lambda: r.ref(flags), render_launches(flags), 2, True


def call_run_sharded_cameras2(r, flags, batch=N):
    r.L.check(r.lib.bevk_shard_configure(r.h, r.L.SHARD_CAMERAS, 0, 2))
    o = r.out(flags)
    rc = r.lib.bevk_bev_run_sharded(r.h, V(r.stack[0].data_ptr()), r.stride(0), batch, V(r.car.data_ptr()), flags, V(o.data_ptr()))
    return rc, o, None, None, None, None


def call_scattered(r, flags, batch=N):
    """A world of one: the peer-store kernel writes into this rank's own receive buffer (no NCCL)."""
    r.L.check(r.lib.bevk_shard_configure(r.h, r.L.SHARD_CAMERAS, 0, 1))
    handle = (C.c_uint8 * 64)()
    r.L.check(r.lib.bevk_shard_prepare(r.h, N, handle))
    r.L.check(r.lib.bevk_shard_attach(r.h, bytes(handle)))
    o, n_own = r.out(flags), C.c_int()
    rc = r.lib.bevk_bev_run_scattered(r.h, V(r.stack[0].data_ptr()), r.stride(0), batch, V(r.car.data_ptr()), flags, V(o.data_ptr()),
                                      C.byref(n_own))
    assert rc != 0 or n_own.value == N
    # V sums, deltas and balanced copies with BALANCE; the render; the compose, then k_gain with BALANCE
    return rc, o, lambda: r.ref(flags), 6 if flags & BAL else 2, 2, False


def call_bev_run(r, flags, batch=N):
    """Host frames (pageable: DMA copies, no fetch kernel) in chunks of 4 and 1 frame-sets."""
    frames = r.host[r.fmt(flags)]
    o = np.zeros(r.shape(flags), np.uint8)
    rc = r.lib.bevk_bev_run(r.h, _host_array([f.ctypes.data for f in frames]), frames[0].strides[0], batch, V(r.car_host.ctypes.data),
                            flags, V(o.ctypes.data))
    return rc, o, lambda: r.ref(flags), 2 * render_launches(flags), 2, False


def call_bev_run_jpeg(r, flags, batch=N):
    streams = [cv2.imencode(".jpg", f, [cv2.IMWRITE_JPEG_QUALITY, 95])[1].tobytes() for f in r.host[0]]
    bufs = [np.frombuffer(s, np.uint8) for s in streams]
    sizes = _host_array([len(s) for s in streams], C.c_uint64)
    o = np.zeros(r.shape(flags), np.uint8)
    rc = r.lib.bevk_bev_run_jpeg(r.h, _host_array([b.ctypes.data for b in bufs]), sizes, batch, V(r.car_host.ctypes.data), flags,
                                 V(o.ctypes.data))
    if rc == UNSUP and "nvJPEG" in r.error():
        pytest.skip("nvJPEG is not available")

    def ref():   # the same streams decoded into a stack of our own, rendered by bevk_bev_run_stack
        d = r.torch.zeros_like(r.stack[0])
        r.L.check(r.lib.bevk_jpeg_decode(r.h, _host_array([b.ctypes.data for b in bufs]), sizes, N * NC, r.g.FW, r.g.FH,
                                         V(d.data_ptr()), r.stride(0)))
        ro = r.out(flags)
        r.L.check(r.lib.bevk_bev_run_stack(r.h, V(d.data_ptr()), r.stride(0), N, V(r.car.data_ptr()), flags, V(ro.data_ptr())))
        r.e.ctx.sync()
        return ro.cpu().numpy()
    return rc, o, ref, render_launches(flags), 2, False


def _to_jpeg_result(r, flags, rc, out, sizes, chunks):
    ref = r.torch.from_numpy(np.ascontiguousarray(r.ref(flags))).to(r.dev)
    enc = 0
    for b0, nb in chunks:
        enc += r.jpeg_encode(ref[b0:], nb)[0]
    want = r.jpeg_encode(ref, N)[1]
    got = _split(out, sizes) if rc == 0 else None
    return rc, got, want, sum(render_launches(flags) for _ in chunks) + enc, 2, True


def call_run_to_jpeg(r, flags, batch=N):
    frames = r.host[0]
    bound = C.c_uint64()
    r.L.check(r.lib.bevk_jpeg_encode_bound(r.g.BW, r.g.BH, C.byref(bound)))
    cap = bound.value * N
    out, sizes = np.zeros(cap, np.uint8), (C.c_uint64 * N)()
    rc = r.lib.bevk_bev_run_to_jpeg(r.h, _host_array([f.ctypes.data for f in frames]), frames[0].strides[0], batch,
                                    V(r.car_host.ctypes.data), flags, QUALITY, V(out.ctypes.data), cap, sizes)
    return rc, out, sizes, [(0, 4), (4, 1)]


def call_frames_to_jpeg(r, flags, batch=N):
    bound = C.c_uint64()
    r.L.check(r.lib.bevk_jpeg_encode_bound(r.g.BW, r.g.BH, C.byref(bound)))
    cap = bound.value * N
    out, sizes = np.zeros(cap, np.uint8), (C.c_uint64 * N)()
    rc = r.lib.bevk_bev_frames_to_jpeg(r.h, _host_array(r.ptrs(0)), batch, V(r.car.data_ptr()), flags, QUALITY, V(out.ctypes.data),
                                       cap, sizes)
    return rc, out, sizes, [(0, N)]


CALLS = {
    "run_device": (call_run_device, BGR_FLAGS), "run_frames": (call_run_frames, BGR_FLAGS),
    "run_frames_table": (call_run_frames_table, BGR_FLAGS), "run_stack": (call_run_stack, ALL_FLAGS),
    "yuv_planes": (call_yuv_planes, YUV_FLAGS), "yuv_surfaces": (call_yuv_surfaces, YUV_FLAGS),
    "stack_cams": (call_stack_cams, ((0, NC), (1, 3))), "device_cams": (call_device_cams, ((0, NC), (1, 3))),
    "run_sharded_frames": (call_run_sharded_frames, (0, BAL)), "run_sharded_cameras1": (call_run_sharded_cameras1, (0, BAL)),
    "scattered": (call_scattered, (0, BAL)), "bev_run": (call_bev_run, ALL_FLAGS), "bev_run_jpeg": (call_bev_run_jpeg, (0, BAL)),
    "run_to_jpeg": (call_run_to_jpeg, (0, BAL)), "frames_to_jpeg": (call_frames_to_jpeg, (0, BAL)),
}
ACCEPTED = [(name, f) for name, (_, fl) in CALLS.items() for f in fl]


@pytest.mark.parametrize("name,flags", ACCEPTED, ids=[f"{n}-{f}" for n, f in ACCEPTED])
def test_accepted_call(rig, name, flags):
    fn = CALLS[name][0]
    rig.ref(flags if isinstance(flags, int) else 0)   # the reference renders come before the counted call
    l0 = rig.launches()
    res = fn(rig, flags)
    launched = rig.launches() - l0
    rig.e.ctx.sync()
    rc = res[0]
    assert rc == 0, rig.error()
    path, timed = rig.path(), rig.timed()
    if name.endswith("to_jpeg"):
        rc, got, want, kernels, want_path, want_timed = _to_jpeg_result(rig, flags, *res)
        assert got == want
    else:
        _, out, want, kernels, want_path, want_timed = res
        want = want()
        if want is not None:
            assert ((out.cpu().numpy() if hasattr(out, "cpu") else out) == want).all()
    assert launched == kernels
    assert path == want_path
    assert timed == want_timed


def test_shard_halves(rig):
    """bevk_shard_render / _compose over a world of two on one GPU, and the BALANCE halves: the renders are timed, the
    V sums and the composes leave the timing state as it was."""
    torch, lib, h, L = rig.torch, rig.lib, rig.h, rig.L
    L.check(lib.bevk_shard_configure(h, L.SHARD_CAMERAS, 0, 2))
    sb = rig.slab_bytes()
    slabs = torch.zeros(2 * N * sb, dtype=torch.uint8, device=rig.dev)
    vs = torch.zeros(2 * N * NC, dtype=torch.int64, device=rig.dev)
    fp, stride = V(rig.stack[0].data_ptr()), rig.stride(0)

    def counted(fn, *args):
        l0 = rig.launches()
        L.check(fn(h, *args))
        rig.e.ctx.sync()
        return rig.launches() - l0

    for bal in (False, True):
        want = rig.ref(BAL if bal else 0)
        for r in range(2 if bal else 0):   # every rank's V sums come before any balanced render
            before = rig.timed()
            assert counted(lib.bevk_shard_vsum, fp, stride, N, r, V(vs.data_ptr())) == 1
            assert rig.timed() == before
        for r in range(2):
            if bal:
                # deltas from the exchanged sums, the balanced copies, the render
                assert counted(lib.bevk_shard_render_balanced, fp, stride, N, r, V(vs.data_ptr()), V(slabs.data_ptr())) == 3
            else:
                assert counted(lib.bevk_shard_render, fp, stride, N, r, V(slabs.data_ptr())) == 1
            assert rig.path() == 2 and rig.timed()
        out = rig.out(0)
        compose = lib.bevk_shard_compose_balanced if bal else lib.bevk_shard_compose
        assert counted(compose, V(slabs.data_ptr()), N, V(rig.car.data_ptr()), V(out.data_ptr())) == (2 if bal else 1)
        assert rig.timed()
        assert (out.cpu().numpy() == want).all(), f"balance {bal}"
    # bevk_sat_sum_device leaves the timing state alone too
    parts = (V * 2)(rig.stack[0].data_ptr(), rig.stack[0].data_ptr())
    o = torch.zeros(64, dtype=torch.uint8, device=rig.dev)
    before = rig.timed()
    assert counted(lib.bevk_sat_sum_device, parts, 2, 64, None, V(o.data_ptr())) == 1
    assert rig.timed() == before


REFUSED = [
    ("run_device", NV12, N, UNSUP, "BGR frames only"), ("run_device", YUYV, N, UNSUP, "BGR frames only"),
    ("run_frames", NV12, N, UNSUP, "BGR frames only"), ("run_frames", YUYV | OUT_NV12, N, UNSUP, "BGR frames only"),
    ("run_stack", NV12 | I420, N, ARG, "exclusive"), ("run_stack", OUT_NV12 | OUT_I420, N, ARG, "exclusive"),
    ("run_stack", 0, 0, ARG, "65535"), ("run_stack", BAL, 16384, ARG, "65535"), ("run_stack", NV12, 16384, ARG, "65535"),
    ("yuv_planes", 0, N, ARG, "YUV planes need"), ("yuv_planes", BAL, N, ARG, "YUV planes need"),
    ("yuv_planes", NV12, 16384, ARG, "65535"), ("yuv_surfaces", 0, N, ARG, "YUV planes need"),
    ("yuv_surfaces", YUYV, 16384, ARG, "65535"),
    ("run_sharded_frames", OUT_NV12, N, UNSUP, "BGR canvases only"),
    ("run_sharded_frames", NV12 | OUT_NV12, N, UNSUP, "BGR frames only"),
    ("run_sharded_cameras2", 0, N, ARG, "bevk_shard_connect"), ("run_sharded_cameras2", BAL, 16384, ARG, "65535"),
    ("scattered", NV12, N, UNSUP, "BGR frames only"), ("scattered", OUT_I420, N, UNSUP, "BGR canvases only"),
    ("bev_run", NV12 | YUYV, N, ARG, "exclusive"), ("bev_run", OUT_NV12 | OUT_I420, N, ARG, "exclusive"),
    ("bev_run_jpeg", NV12, N, UNSUP, "BGR frames only"), ("bev_run_jpeg", OUT_NV12, N, UNSUP, "BGR canvases only"),
    ("run_to_jpeg", NV12, N, UNSUP, "BGR frames only"), ("run_to_jpeg", OUT_NV12, N, UNSUP, "BGR canvases only"),
    ("frames_to_jpeg", YUYV, N, UNSUP, "BGR frames only"), ("frames_to_jpeg", OUT_I420, N, UNSUP, "BGR canvases only"),
]
CAM_CALLS = {"run_sharded_cameras2": call_run_sharded_cameras2}


@pytest.mark.parametrize("name,flags,batch,code,fragment", REFUSED,
                         ids=[f"{n}-{f}-{b}" for n, f, b, _, _ in REFUSED])
def test_refused_call(rig, name, flags, batch, code, fragment):
    fn = CAM_CALLS.get(name) or CALLS[name][0]
    l0 = rig.launches()
    rc = fn(rig, flags, batch)[0]
    assert rc == code and fragment in rig.error(), (rc, rig.error())
    assert rig.launches() == l0
