"""ctypes binding of libbevk.so (include/bevk.h).  There is no CPU fallback: if the
shared library is missing or no CUDA device is present, the calls raise."""
from __future__ import annotations

import ctypes as C
import os
import weakref

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("BEVK_LIB_PATH") or os.path.join(_HERE, "libbevk.so")   # BEVK_LIB_PATH: A/B builds

INTER_NEAREST, INTER_LINEAR = 0, 1
MAPS_UNDISTORT, MAPS_BEV = 0, 1
MODEL_FISHEYE, MODEL_PINHOLE = 0, 1
FLAG_BALANCE = 1
FLAG_NV12, FLAG_I420 = 2, 4          # YUV 4:2:0 frames (cv2's single-buffer layout), bevk_bev_run / _run_stack only
FLAG_YUYV, FLAG_UYVY = 32, 64        # packed YUV 4:2:2 frames uint8[FH][FW][2] (cv2's COLOR_YUV2BGR_YUY2 / _UYVY input)
PIXEL_FORMATS = {"bgr": 0, "nv12": FLAG_NV12, "i420": FLAG_I420, "yuyv": FLAG_YUYV, "uyvy": FLAG_UYVY}
PACKED_FORMATS = (FLAG_YUYV, FLAG_UYVY)
FLAG_OUT_NV12, FLAG_OUT_I420 = 8, 16  # YUV 4:2:0 canvases uint8[BH*3/2][BW] (cv2.cvtColor(COLOR_BGR2YUV_I420) layout)
OUT_FORMATS = {"bgr": 0, "nv12": FLAG_OUT_NV12, "i420": FLAG_OUT_I420}
SHARD_FRAMES, SHARD_CAMERAS = 0, 1
MAX_CAMERAS = 8

_p = C.c_void_p
_dp = C.POINTER(C.c_double)
# name -> (restype, argtypes); mirrors include/bevk.h one to one
SIGNATURES = {
    "bevk_version": (C.c_int, []),
    "bevk_last_error": (C.c_char_p, []),
    "bevk_ctx_create": (C.c_int, [C.c_int, C.POINTER(_p)]),
    "bevk_ctx_destroy": (C.c_int, [_p]),
    "bevk_ctx_set_stream": (C.c_int, [_p, _p]),
    "bevk_ctx_sync": (C.c_int, [_p]),
    "bevk_device_pci_bus_id": (C.c_int, [C.c_int, C.c_char_p, C.c_int]),
    "bevk_host_alloc": (C.c_int, [C.c_uint64, C.POINTER(_p)]),
    "bevk_host_free": (C.c_int, [_p]),
    "bevk_undistort_map": (C.c_int, [_p, C.c_int, _dp, _dp, C.c_int, _dp, C.c_int, C.c_int, _p, _p]),
    "bevk_remap": (C.c_int, [_p, _p, C.c_int, C.c_int, C.c_int64, C.c_int, _p, _p, C.c_int, C.c_int, _p, C.c_int64, C.c_int]),
    "bevk_undistorter_set": (C.c_int, [_p, C.c_int, C.c_int, _dp, _dp, C.c_int, _dp, C.c_int, C.c_int, C.c_int]),
    "bevk_undistorter_maps": (C.c_int, [_p, C.c_int, _p, _p]),
    "bevk_undistort": (C.c_int, [_p, C.c_int, _p, C.c_int, C.c_int, C.c_int64, C.c_int, _p, C.c_int, C.c_int, C.c_int64, C.c_int]),
    "bevk_undistort_stack": (C.c_int, [_p, C.c_int, _p, C.c_int64, C.c_int, C.c_int, C.c_int64, C.c_int, C.c_int, _p, C.c_int64,
                                       C.c_int, C.c_int, C.c_int64, C.c_int]),
    "bevk_undistort_last_path": (C.c_int, [_p]),
    "bevk_warp_perspective":(C.c_int, [_p, _p, C.c_int, C.c_int, C.c_int64, C.c_int, _dp, _p, C.c_int, C.c_int, C.c_int64, C.c_int]),
    "bevk_warp_maps": (C.c_int, [_p, _p, _p, C.c_int, C.c_int, _dp, C.c_int, C.c_int, _p, _p]),
    "bevk_bev_configure": (C.c_int, [_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "bevk_bev_set_camera": (C.c_int, [_p, C.c_int, _dp, _dp, _dp, C.c_int, C.c_int, _dp]),
    "bevk_bev_set_maps": (C.c_int, [_p, C.c_int, _p, _p]),
    "bevk_bev_get_maps": (C.c_int, [_p, C.c_int, _p, _p]),
    "bevk_bev_set_interpolation": (C.c_int, [_p, C.c_int]),
    "bevk_bev_set_mask": (C.c_int, [_p, C.c_int, _p]),
    "bevk_blend_masks": (C.c_int, [_p, _p, _p, C.c_int, C.c_int, _p]),
    "bevk_bev_finalize": (C.c_int, [_p]),
    "bevk_bev_run": (C.c_int, [_p, C.POINTER(_p), C.c_int64, C.c_int, _p, C.c_int, _p]),
    "bevk_bev_run_device": (C.c_int, [_p, _p, C.c_int, _p, C.c_int, _p]),
    "bevk_bev_run_frames": (C.c_int, [_p, _p, C.c_int, _p, C.c_int, _p]),
    "bevk_bev_run_stack": (C.c_int, [_p, _p, C.c_int64, C.c_int, _p, C.c_int, _p]),
    "bevk_bev_run_yuv_planes": (C.c_int, [_p, _p, C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_int, _p, C.c_int,
                                          _p]),
    "bevk_bev_run_yuv_surfaces": (C.c_int, [_p, C.POINTER(_p), C.POINTER(C.c_int64), C.c_int, _p, C.c_int, _p]),
    "bevk_bev_run_device_cams": (C.c_int, [_p, _p, C.c_int, C.c_int, C.c_int, _p]),
    "bevk_bev_run_stack_cams": (C.c_int, [_p, _p, C.c_int64, C.c_int, C.c_int, C.c_int, _p]),
    "bevk_sat_sum_device": (C.c_int, [_p, C.POINTER(_p), C.c_int, C.c_uint64, _p, _p]),
    "bevk_apply_mask": (C.c_int, [_p, _p, _p, C.c_int, C.c_int, C.c_int, _p]),
    "bevk_color_balance": (C.c_int, [_p, _p, C.c_int, C.c_int, _p]),
    "bevk_luminance_balance": (C.c_int, [_p, C.POINTER(_p), C.c_int, C.c_int, C.c_int, C.POINTER(_p)]),
    "bevk_bev_plan_info": (C.c_int, [_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "bevk_bev_host_copy_bytes": (C.c_int, [_p, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "bevk_bev_last_h2d_bytes": (C.c_int64, [_p]),
    "bevk_bev_last_path": (C.c_int, [_p]),
    "bevk_bev_tma_plan_info": (C.c_int, [_p] + [C.POINTER(C.c_int64)] * 5),
    "bevk_shard_configure": (C.c_int, [_p, C.c_int, C.c_int, C.c_int]),
    "bevk_shard_unique_id": (C.c_int, [_p, C.c_int]),
    "bevk_shard_connect": (C.c_int, [_p, _p, C.c_int]),
    "bevk_shard_info": (C.c_int, [_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int32), C.POINTER(C.c_int64)]),
    "bevk_bev_run_sharded": (C.c_int, [_p, _p, C.c_int64, C.c_int, _p, C.c_int, _p]),
    "bevk_shard_prepare": (C.c_int, [_p, C.c_int, _p]),
    "bevk_shard_attach": (C.c_int, [_p, _p]),
    "bevk_bev_run_scattered": (C.c_int, [_p, _p, C.c_int64, C.c_int, _p, C.c_int, _p, C.POINTER(C.c_int)]),
    "bevk_shard_last_link_bytes": (C.c_int64, [_p]),
    "bevk_shard_render": (C.c_int, [_p, _p, C.c_int64, C.c_int, C.c_int, _p]),
    "bevk_shard_compose": (C.c_int, [_p, _p, C.c_int, _p, _p]),
    "bevk_shard_vsum": (C.c_int, [_p, _p, C.c_int64, C.c_int, C.c_int, _p]),
    "bevk_shard_render_balanced": (C.c_int, [_p, _p, C.c_int64, C.c_int, C.c_int, _p, _p]),
    "bevk_shard_compose_balanced": (C.c_int, [_p, _p, C.c_int, _p, _p]),
    "bevk_jpeg_decode": (C.c_int, [_p, C.POINTER(_p), C.POINTER(C.c_uint64), C.c_int, C.c_int, C.c_int, _p, C.c_int64]),
    "bevk_bev_run_jpeg": (C.c_int, [_p, C.POINTER(_p), C.POINTER(C.c_uint64), C.c_int, _p, C.c_int, _p]),
    "bevk_jpeg_encode_bound": (C.c_int, [C.c_int, C.c_int, C.POINTER(C.c_uint64)]),
    "bevk_jpeg_set_params": (C.c_int, [_p, C.POINTER(C.c_int), C.c_int]),
    "bevk_jpeg_encode_bound_params": (C.c_int, [C.c_int, C.c_int, C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_uint64)]),
    "bevk_png_set_params": (C.c_int, [_p, C.POINTER(C.c_int), C.c_int]),
    "bevk_png_encode_bound": (C.c_int, [C.c_int, C.c_int, C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_uint64)]),
    "bevk_png_encode": (C.c_int, [_p, _p, C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_int, _p, C.c_uint64,
                                  C.POINTER(C.c_uint64)]),
    "bevk_png_encode_params": (C.c_int, [_p, C.POINTER(C.c_int), C.c_int, _p, C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_int,
                                         _p, C.c_uint64, C.POINTER(C.c_uint64)]),
    "bevk_jpeg_encode": (C.c_int, [_p, _p, C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int, _p, C.c_uint64,
                                   C.POINTER(C.c_uint64)]),
    "bevk_undistort_jpeg": (C.c_int, [_p, C.c_int, _p, C.c_int, C.c_int, C.c_int64, C.c_int, C.c_int, _p, C.c_uint64,
                                      C.POINTER(C.c_uint64)]),
    "bevk_undistort_stack_jpeg": (C.c_int, [_p, C.c_int, _p, C.c_int64, C.c_int, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_int, _p,
                                            C.c_uint64, C.POINTER(C.c_uint64)]),
    "bevk_bev_run_to_jpeg":(C.c_int, [_p, C.POINTER(_p), C.c_int64, C.c_int, _p, C.c_int, C.c_int, _p, C.c_uint64,
                                       C.POINTER(C.c_uint64)]),
    "bevk_bev_frames_to_jpeg": (C.c_int, [_p, C.POINTER(_p), C.c_int, _p, C.c_int, C.c_int, _p, C.c_uint64, C.POINTER(C.c_uint64)]),
    "bevk_graph_begin": (C.c_int, [_p]),
    "bevk_graph_end": (C.c_int, [_p, C.POINTER(C.c_int)]),
    "bevk_graph_launch": (C.c_int, [_p, C.c_int, C.c_int]),
    "bevk_graph_destroy": (C.c_int, [_p, C.c_int]),
    "bevk_launch_count": (C.c_int64, [_p]),
    "bevk_last_kernel_ms": (C.c_int, [_p, C.POINTER(C.c_float)]),
}

_lib = None


def load() -> C.CDLL:
    """dlopen libbevk.so and type every export.  Raises if the library was not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -m cameracalibration_b200.build` "
                "(nvcc, sm_90a).  cameracalibration_b200 has no CPU fallback.")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
        _lib = lib
    return _lib


class BevkError(Exception):
    pass


def check(rc: int):
    if rc != 0:
        raise BevkError(f"libbevk error {rc}: {load().bevk_last_error().decode()}")


def dptr(a) -> _dp:
    """float64 C-contiguous view -> double*; keeps the array alive via the returned object."""
    arr = np.ascontiguousarray(np.asarray(a, dtype=np.float64).reshape(-1))
    p = arr.ctypes.data_as(_dp)
    p._keep = arr
    return p


def vptr(a: np.ndarray) -> _p:
    return C.c_void_p(a.ctypes.data)


def image_view(img: np.ndarray):
    """(array to pass, w, h, row stride, channels) for a uint8 HxW or HxWxC image.  Rows
    must be internally contiguous; otherwise a contiguous copy is made."""
    if img.dtype != np.uint8:
        raise BevkError("images must be uint8")
    if img.ndim == 2:
        ch = 1
    elif img.ndim == 3 and img.shape[2] in (1, 3, 4):
        ch = img.shape[2]
    else:
        raise BevkError(f"unsupported image shape {img.shape}")
    h, w = img.shape[:2]
    ok = img.strides[1] == ch and (img.ndim == 2 or img.strides[2] == 1) and img.strides[0] >= w * ch
    if not ok:
        img = np.ascontiguousarray(img)
    return img, w, h, img.strides[0], ch


class Context:
    """Owner of a bevk_ctx (one per thread)."""

    def __init__(self, device: int = 0):
        self.lib = load()
        h = _p()
        check(self.lib.bevk_ctx_create(int(device), C.byref(h)))
        self.h = h
        self.device = device
        self._stream = None

    def close(self):
        if getattr(self, "h", None):
            self.lib.bevk_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    _UNSET = object()

    def set_stream(self, stream_ptr: int | None):
        """None -> the ctx's own stream; 0 (torch's default stream handle) -> the legacy
        default stream (cudaStreamLegacy); anything else -> that cudaStream_t."""
        if stream_ptr is None:
            ptr = 0
        else:
            ptr = 1 if stream_ptr == 0 else stream_ptr
        check(self.lib.bevk_ctx_set_stream(self.h, _p(ptr)))
        self._stream = stream_ptr

    def on_stream(self, stream_ptr: int | None):
        """``with ctx.on_stream(s): ...`` -- run the calls inside on stream ``s`` (same values as set_stream) and put
        the previous stream back afterwards."""
        return _StreamScope(self, stream_ptr)

    def sync(self):
        check(self.lib.bevk_ctx_sync(self.h))

    def graph_capture(self):
        """``with ctx.graph_capture() as g: <device-pointer calls>`` -> g.launch(times).  The calls inside the block are
        recorded into a CUDA graph instead of executed (run them once before, so every buffer exists)."""
        return _GraphCapture(self)

    @property
    def launches(self) -> int:
        return int(self.lib.bevk_launch_count(self.h))


class _StreamScope:
    def __init__(self, ctx, stream_ptr):
        self.ctx, self.want = ctx, stream_ptr

    def __enter__(self):
        self.prev = getattr(self.ctx, "_stream", None)
        if self.want != self.prev:
            self.ctx.set_stream(self.want)
        return self.ctx

    def __exit__(self, et, ev, tb):
        if self.want != self.prev:
            self.ctx.set_stream(self.prev)
        return False


class _GraphCapture:
    def __init__(self, ctx: Context):
        self.ctx, self.id = ctx, None

    def __enter__(self):
        check(self.ctx.lib.bevk_graph_begin(self.ctx.h))
        return self

    def __exit__(self, et, ev, tb):
        gid = C.c_int(-1)
        rc = self.ctx.lib.bevk_graph_end(self.ctx.h, C.byref(gid))
        if et is None:
            check(rc)
            self.id = gid.value
        return False

    def launch(self, times: int = 1):
        if self.id is None:
            raise BevkError("graph capture did not complete")
        check(self.ctx.lib.bevk_graph_launch(self.ctx.h, self.id, int(times)))

    def destroy(self):
        if self.id is not None and getattr(self.ctx, "h", None):
            check(self.ctx.lib.bevk_graph_destroy(self.ctx.h, self.id))
            self.id = None


_default_ctx: dict[int, Context] = {}


def default_context(device: int | None = None) -> Context:
    if device is None:
        device = int(os.environ.get("BEVK_DEVICE", os.environ.get("LOCAL_RANK", "0")))
    if device not in _default_ctx:
        _default_ctx[device] = Context(device)
    return _default_ctx[device]


def _free_pinned(addr: int):
    try:
        if _lib is not None:
            _lib.bevk_host_free(_p(addr))
    except Exception:
        pass


def pinned_empty(shape, dtype=np.uint8) -> np.ndarray:
    """numpy array backed by page-locked host memory (full-rate PCIe copies).  The allocation is returned with
    bevk_host_free when the array and every view of it have been garbage-collected."""
    lib = load()
    n = int(np.prod(shape)) * np.dtype(dtype).itemsize
    p = _p()
    check(lib.bevk_host_alloc(n, C.byref(p)))
    buf = (C.c_uint8 * max(n, 1)).from_address(p.value)
    weakref.finalize(buf, _free_pinned, p.value)     # numpy keeps `buf` alive as the base of the array and its views
    return np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)


class PinnedPool:
    """Recycling allocator of page-locked result arrays.  The reference returns a freshly allocated ndarray from every
    call (the caller owns it); a pageable result makes the driver stage the device->host copy through its own bounce
    buffer.  get(shape) hands out a page-locked array instead; when the caller drops it (and every view of it), the
    buffer goes back to the pool rather than to cudaFreeHost, so a steady stream of calls allocates nothing."""

    def __init__(self, keep: int = 8):
        self.keep, self.free = keep, {}

    def get(self, shape, dtype=np.uint8) -> np.ndarray:
        n = int(np.prod(shape)) * np.dtype(dtype).itemsize
        stack = self.free.setdefault(n, [])
        if stack:
            buf, addr = stack.pop()
        else:
            p = _p()
            check(load().bevk_host_alloc(n, C.byref(p)))
            addr = p.value
            buf = (C.c_uint8 * max(n, 1)).from_address(addr)
        flat = np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape)))
        weakref.finalize(flat, self._give_back, n, buf, addr)    # every view (reshape, out[0], slices) has `flat` as its base
        return flat.reshape(shape)

    def _give_back(self, n, buf, addr):
        stack = self.free.setdefault(n, [])
        if len(stack) < self.keep:
            stack.append((buf, addr))
        else:
            _free_pinned(addr)
