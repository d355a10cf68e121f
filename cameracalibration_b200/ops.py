"""NumPy-facing wrappers of the C ABI, one per OpenCV call the reference makes on the
hot path.  Signatures follow the cv2 functions they replace; all pixel work happens in
libbevk.so on the GPU."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib as L

INTER_NEAREST, INTER_LINEAR, INTER_CUBIC, INTER_AREA, INTER_LANCZOS4 = (
    L.INTER_NEAREST, L.INTER_LINEAR, L.INTER_CUBIC, L.INTER_AREA, L.INTER_LANCZOS4)
_INTERPOLATIONS = (INTER_NEAREST, INTER_LINEAR, INTER_CUBIC, INTER_AREA, INTER_LANCZOS4)
CV_16SC2, CV_32FC1, CV_32FC2 = L.CV_16SC2, L.CV_32FC1, L.CV_32FC2
_MAP_TYPES = (CV_16SC2, CV_32FC1, CV_32FC2)

# cv2's border modes (cv2.BORDER_*), for remap, warp_perspective, warp_affine and Undistorter
BORDER_CONSTANT, BORDER_REPLICATE, BORDER_REFLECT, BORDER_WRAP, BORDER_REFLECT_101, BORDER_TRANSPARENT = 0, 1, 2, 3, 4, 5


def _interp(flag: int) -> int:
    if flag not in _INTERPOLATIONS:
        raise L.BevkError(f"interpolation {flag} is not supported (cv2's INTER_NEAREST, _LINEAR, _CUBIC, _AREA or "
                          "_LANCZOS4)")
    return flag


def fisheye_init_undistort_rectify_map(K, D, P, size, ctx: L.Context | None = None, R=None, m1type: int = CV_16SC2):
    """cv2.fisheye.initUndistortRectifyMap(K, D, R, P, size, m1type); R=None is eye(3).  m1type: CV_16SC2 (int16[h][w][2]
    and uint16[h][w]) or CV_32FC1 (float32[h][w] x and y planes); cv2 refuses CV_32FC2 for the fisheye, and so does this."""
    return _undistort_map(L.MODEL_FISHEYE, K, D, P, size, ctx, R, m1type)


def init_undistort_rectify_map(K, D, P, size, ctx: L.Context | None = None, R=None, m1type: int = CV_16SC2):
    """cv2.initUndistortRectifyMap(K, D, R, P, size, m1type) with D of 4, 5, 8, 12 or 14 coefficients (rational,
    thin-prism and tilted models); R=None is eye(3).  m1type: CV_16SC2, CV_32FC1 (float32 x and y planes) or CV_32FC2
    (float32[h][w][2] and None)."""
    return _undistort_map(L.MODEL_PINHOLE, K, D, P, size, ctx, R, m1type)


def _rotation(R):
    """double* of a 3x3 rectification rotation, or None (NULL: the identity)."""
    if R is None:
        return None
    r = np.asarray(R, np.float64)
    if r.shape != (3, 3):
        raise L.BevkError(f"R must be a 3x3 matrix, got shape {r.shape}")
    return L.dptr(r)


def _map_type(m1type):
    if m1type not in _MAP_TYPES:
        raise L.BevkError(f"m1type {m1type} is not a map type (cv2's CV_16SC2, CV_32FC1 or CV_32FC2)")
    return int(m1type)


def _float_maps(m1type, h, w):
    """Empty host maps of a float type: CV_32FC1's two planes, or CV_32FC2's pairs and None."""
    if m1type == CV_32FC2:
        return np.empty((h, w, 2), np.float32), None
    return np.empty((h, w), np.float32), np.empty((h, w), np.float32)


def _undistort_map(model, K, D, P, size, ctx, R=None, m1type=CV_16SC2):
    ctx = ctx or L.default_context()
    w, h = int(size[0]), int(size[1])
    d = np.asarray(D, np.float64).reshape(-1)
    if _map_type(m1type) != CV_16SC2:
        m1, m2 = _float_maps(m1type, h, w)
        L.check(ctx.lib.bevk_undistort_rectify_map_f32(ctx.h, model, L.dptr(K), L.dptr(d), int(d.size), _rotation(R),
                                                       L.dptr(P), w, h, int(m1type), L.vptr(m1),
                                                       None if m2 is None else L.vptr(m2)))
        return m1, m2
    m1 = np.empty((h, w, 2), np.int16)
    m2 = np.empty((h, w), np.uint16)
    if R is None:
        L.check(ctx.lib.bevk_undistort_map(ctx.h, model, L.dptr(K), L.dptr(d), int(d.size), L.dptr(P), w, h,
                                           L.vptr(m1), L.vptr(m2)))
    else:
        L.check(ctx.lib.bevk_undistort_rectify_map(ctx.h, model, L.dptr(K), L.dptr(d), int(d.size), _rotation(R), L.dptr(P),
                                                   w, h, L.vptr(m1), L.vptr(m2)))
    return m1, m2


def _out(shape, out, dtype=np.uint8):
    """cv2-style optional destination (e.g. a page-locked array from pinned_empty for full-rate D2H)."""
    if out is None:
        return np.empty(shape, dtype)
    if out.dtype != dtype or out.shape != tuple(shape) or not out.flags.c_contiguous:
        raise L.BevkError(f"out must be a C-contiguous {np.dtype(dtype).name} array of shape {tuple(shape)}")
    return out


def _cuda_ptr(arr, shape):
    """(device pointer, shape) of a uint8 C-contiguous array exposing ``__cuda_array_interface__``."""
    iface = getattr(arr, "__cuda_array_interface__", None)
    if iface is None:
        raise L.BevkError("expected a CUDA array (an object with __cuda_array_interface__)")
    got = tuple(iface["shape"])
    if iface["typestr"] not in ("|u1", "<u1", "=u1"):
        raise L.BevkError(f"CUDA array must be uint8, got typestr {iface['typestr']}")
    if shape is not None and got != tuple(shape):
        raise L.BevkError(f"CUDA array must have shape {tuple(shape)}, got {got}")
    strides = iface.get("strides")
    if strides is not None:
        dense, step = [], 1
        for n in reversed(got):
            dense.append(step)
            step *= n
        if any(n > 1 and s != d for n, s, d in zip(got, strides, reversed(dense))):
            raise L.BevkError("CUDA array must be C-contiguous")
    ptr = iface["data"][0]
    if not ptr:
        raise L.BevkError("CUDA array has a null data pointer")
    return int(ptr), got


def _cuda_plane(arr, shape, what):
    """(device pointer, byte strides) of a uint8 CUDA array of the given shape whose last axis is dense (pixels within a
    row); the other axes may have any non-negative stride (pitched rows, views of a larger pool)."""
    iface = getattr(arr, "__cuda_array_interface__", None)
    if iface is None:
        raise L.BevkError(f"{what}: expected a CUDA array (an object with __cuda_array_interface__)")
    got = tuple(iface["shape"])
    if iface["typestr"] not in ("|u1", "<u1", "=u1"):
        raise L.BevkError(f"{what} must be uint8, got typestr {iface['typestr']}")
    if got != tuple(shape):
        raise L.BevkError(f"{what} must have shape {tuple(shape)}, got {got}")
    strides = iface.get("strides")
    if strides is None:
        strides, step = [], 1
        for n in reversed(got):
            strides.insert(0, step)
            step *= n
    strides = [int(s) for s in strides]
    if got[-1] > 1 and strides[-1] != 1:
        raise L.BevkError(f"{what}: pixels within a row must be dense")
    if any(s < 0 for s in strides):
        raise L.BevkError(f"{what}: negative strides are not supported")
    ptr = iface["data"][0]
    if not ptr:
        raise L.BevkError(f"{what} has a null data pointer")
    return int(ptr), strides[:-1]


def jpeg_decode(jpegs, width: int, height: int, out=None, ctx: L.Context | None = None):
    """Decode JPEG byte strings on the GPU (nvJPEG) into a uint8 CUDA frame stack [n][height][width][3] (BGR, what
    cv2.imread's layout is).  ``out``: a CUDA array of that shape; default a new torch tensor.  Enqueued on the ctx
    stream; returns ``out``."""
    ctx = ctx or L.default_context()
    n = len(jpegs)
    if out is None:
        import torch
        out = torch.empty((n, height, width, 3), dtype=torch.uint8, device=torch.device("cuda", ctx.device))
    d_out = _cuda_ptr(out, (n, height, width, 3))[0]
    keep = [(C.c_char * len(x)).from_buffer_copy(bytes(x)) for x in jpegs]
    ptrs = (C.c_void_p * n)(*[C.addressof(k) for k in keep])
    sizes = (C.c_uint64 * n)(*[len(x) for x in jpegs])
    L.check(ctx.lib.bevk_jpeg_decode(ctx.h, ptrs, sizes, n, int(width), int(height), C.c_void_p(d_out), width * height * 3))
    return out


def _jpeg_params(params):
    """(ctypes int array, n) of a cv2.imwrite JPEG parameter list without the IMWRITE_JPEG_QUALITY pair; None is []."""
    p = [] if params is None else [int(v) for v in params]
    return (C.c_int * max(len(p), 1))(*p), len(p)


def jpeg_set_params(ctx: L.Context, params=None):
    """Apply cv2.imwrite's JPEG (key, value) pairs (keys 2..7, cv2.IMWRITE_JPEG_*) to ctx's encoding calls; None or []
    restores cv2's defaults.  The wrappers below call it on every call, so no call inherits another's params."""
    arr, n = _jpeg_params(params)
    L.check(ctx.lib.bevk_jpeg_set_params(ctx.h, arr, n))


def jpeg_encode_bound(width: int, height: int, params=None) -> int:
    """Largest JPEG stream bevk_jpeg_encode can produce for a width x height image under params (cv2.imwrite's JPEG
    pairs without IMWRITE_JPEG_QUALITY; None: cv2's defaults)."""
    n = C.c_uint64()
    if params is None:
        L.check(L.load().bevk_jpeg_encode_bound(int(width), int(height), C.byref(n)))
    else:
        arr, k = _jpeg_params(params)
        L.check(L.load().bevk_jpeg_encode_bound_params(int(width), int(height), arr, k, C.byref(n)))
    return n.value


# the image gathers' sources beyond uint8: dtype -> cv2 depth (CV_16U, CV_16S, CV_32F), and their CUDA typestrs
_WIDE = {np.dtype(np.uint16): 2, np.dtype(np.int16): 3, np.dtype(np.float32): 5}
_WIDE_TYPESTRS = {"<u2": np.uint16, "<i2": np.int16, "<f4": np.float32}


def _cuda_dtype(arr):
    """The NumPy dtype of a CUDA array's elements as the image calls read them (uint8 for any 1-byte unsigned typestr)."""
    ts = arr.__cuda_array_interface__["typestr"]
    return np.dtype(_WIDE_TYPESTRS.get(ts, np.uint8))


def _cuda_images(arr, what, wide=False):
    """(device pointer, rank, n, h, w, channels, image stride, row stride) of a uint8 CUDA array [H][W], [H][W][C] or
    [N][H][W][C] (C in 1, 3, 4) whose pixels are dense (C-byte pixels, 1-byte channels); rows and images may be padded.
    wide: the image gathers' uint16, int16 and float32 arrays too (strides in bytes, dense C-element pixels)."""
    iface = getattr(arr, "__cuda_array_interface__", None)
    if iface is None:
        raise L.BevkError(f"{what} must be a CUDA array (an object with __cuda_array_interface__), got {type(arr).__name__}")
    shape = tuple(iface["shape"])
    es, dtypes = 1, "uint8, uint16, int16 or float32" if wide else "uint8"
    if wide and iface["typestr"] in _WIDE_TYPESTRS:
        es = np.dtype(_WIDE_TYPESTRS[iface["typestr"]]).itemsize
    elif iface["typestr"] not in ("|u1", "<u1", "=u1"):
        raise L.BevkError(f"{what} must be {dtypes}, got typestr {iface['typestr']}")
    rank = len(shape)
    if rank not in (2, 3, 4) or (rank > 2 and shape[-1] not in (1, 3, 4)):
        kind = "uint8" if not wide else f"({dtypes}) "
        raise L.BevkError(f"{what} must be {kind}[H][W], [H][W][C] or [N][H][W][C] with C in 1, 3, 4, got shape {shape}")
    strides = iface.get("strides")
    if strides is None:
        strides = tuple(es * int(np.prod(shape[i + 1:])) for i in range(rank))
    strides = tuple(int(s) for s in strides)
    if rank == 2:
        shape, strides = shape + (1,), strides + (es,)
    if rank != 4:
        shape, strides = (1,) + shape, (0,) + strides
    n, h, w, ch = shape
    if (ch > 1 and strides[3] != es) or (w > 1 and strides[2] != ch * es):
        raise L.BevkError(f"{what} must have dense pixels (strides {ch * es} and {es} along width and channels)")
    ptr = iface["data"][0]
    if not ptr:
        raise L.BevkError(f"{what} has a null data pointer")
    row = strides[1] if h > 1 else w * ch * es
    img = strides[0] if n > 1 else h * row
    return int(ptr), rank, n, h, w, ch, img, row


def _split(out, sizes):
    """The streams an encoding call wrote back to back into out, one ``bytes`` each."""
    res, off = [], 0
    for s in sizes:
        res.append(out[off:off + s].tobytes())
        off += s
    return res


def _encode(what, images, ctx, bound, call, channels=False):
    """The body of the encoding wrappers over uint8[H][W][3] or [N][H][W][3] BGR images: CUDA arrays
    (``__cuda_array_interface__``) are read in place, NumPy input is uploaded once.  bound(w, h): the largest stream of one
    image; call((ptr, image stride, row stride, n, w, h), out, capacity, sizes): the C call, run on torch's current
    stream.  channels: take [H][W] and [H][W][C] / [N][H][W][C] with C in 1, 3, 4 instead, with bound(w, h, C) and
    call((ptr, image stride, row stride, C, n, w, h), ...)."""
    from .sharding import _torch_current_stream
    keep = images
    if not hasattr(images, "__cuda_array_interface__"):
        a = np.asarray(images)
        if channels:
            if a.dtype != np.uint8 or a.ndim not in (2, 3, 4) or (a.ndim > 2 and a.shape[-1] not in (1, 3, 4)):
                raise L.BevkError(f"{what} takes uint8[H][W], [H][W][C] or [N][H][W][C] images with C in 1, 3, 4, "
                                  f"got {a.dtype} {a.shape}")
        elif a.dtype != np.uint8 or a.ndim not in (3, 4) or a.shape[-1] != 3:
            raise L.BevkError(f"{what} takes uint8[H][W][3] or uint8[N][H][W][3] BGR images, got {a.dtype} {a.shape}")
        import torch
        keep = torch.from_numpy(np.ascontiguousarray(a)).to(torch.device("cuda", ctx.device))
    ptr, rank, n, h, w, ch, img_stride, row_stride = _cuda_images(keep, what)
    if not channels and (ch != 3 or rank == 2):
        raise L.BevkError(f"{what} takes uint8[H][W][3] or uint8[N][H][W][3] BGR images")
    if n < 1:
        return []
    cap = n * (bound(w, h, ch) if channels else bound(w, h))
    out = np.empty(cap, np.uint8)          # pages are only touched where streams land
    sizes = (C.c_uint64 * n)()
    img = (C.c_void_p(ptr), img_stride, row_stride) + ((ch,) if channels else ()) + (n, w, h)
    with ctx.on_stream(_torch_current_stream(ctx.device)):
        L.check(call(img, L.vptr(out), cap, sizes))
    return _split(out, sizes)


def jpeg_encode(images, quality: int = 95, ctx: L.Context | None = None, params=None) -> list[bytes]:
    """cv2.imencode('.jpg', img, [cv2.IMWRITE_JPEG_QUALITY, quality] + params) on the GPU, byte for byte, for one
    uint8[H][W][3] BGR image or a batch uint8[N][H][W][3].  params: cv2.imwrite's other JPEG pairs
    (IMWRITE_JPEG_SAMPLING_FACTOR, _LUMA_QUALITY, _CHROMA_QUALITY, _OPTIMIZE, _RST_INTERVAL; see bevk_jpeg_set_params),
    None for cv2's defaults.
    CUDA arrays (``__cuda_array_interface__``, e.g. the torch canvases of BevEngine.run_cuda) are read in place, on
    torch's current stream; NumPy input is uploaded once.  Returns one ``bytes`` per image -- what cv2.imwrite would
    write to a .jpg file."""
    ctx = ctx or L.default_context()
    jpeg_set_params(ctx, params)
    return _encode("jpeg_encode", images, ctx, lambda w, h: jpeg_encode_bound(w, h, params),
                   lambda img, out, cap, sizes: ctx.lib.bevk_jpeg_encode(ctx.h, *img, int(quality), out, cap, sizes))


def jpeg_encode_params_bound(width: int, height: int, params=None) -> int:
    """Largest JPEG stream jpeg_encode_params can produce for a width x height image under params."""
    n = C.c_uint64()
    arr, k = _jpeg_params(params)
    L.check(L.load().bevk_jpeg_encode_params_bound(int(width), int(height), arr, k, C.byref(n)))
    return n.value


def jpeg_encode_params(images, params, quality: int = 95, ctx: L.Context | None = None) -> list[bytes]:
    """cv2.imencode('.jpg', img, [cv2.IMWRITE_JPEG_QUALITY, quality] + params) on the GPU, byte for byte, with the
    parameter list given per call (bevk_jpeg_encode_params): jpeg_encode's keys plus IMWRITE_JPEG_PROGRESSIVE, read as
    cv2 4.13 reads it.  Takes the same images as jpeg_encode (NumPy, or CUDA arrays read in place on torch's current
    stream); the ctx's jpeg_set_params list is left as it was.  Returns one ``bytes`` per image."""
    ctx = ctx or L.default_context()
    arr, k = _jpeg_params(params)
    return _encode("jpeg_encode_params", images, ctx, lambda w, h: jpeg_encode_params_bound(w, h, params),
                   lambda img, out, cap, sizes: ctx.lib.bevk_jpeg_encode_params(ctx.h, arr, k, *img, int(quality), out, cap,
                                                                                sizes))


def png_set_params(ctx: L.Context, params=None):
    """Apply cv2.imwrite's PNG (key, value) pairs (keys 16..20, cv2.IMWRITE_PNG_*) to ctx's PNG encoding; None or []
    restores cv2's defaults.  The list applies to bevk_png_encode; png_encode takes its own list per call."""
    arr, n = _jpeg_params(params)
    L.check(ctx.lib.bevk_png_set_params(ctx.h, arr, n))


def png_encode_bound(width: int, height: int, params=None) -> int:
    """Largest PNG stream bevk_png_encode can produce for a width x height image under params (cv2.imwrite's PNG
    pairs; None: cv2's defaults)."""
    n = C.c_uint64()
    arr, k = _jpeg_params(params)
    L.check(L.load().bevk_png_encode_bound(int(width), int(height), arr, k, C.byref(n)))
    return n.value


def png_encode(images, ctx: L.Context | None = None, params=None) -> list[bytes]:
    """cv2.imencode('.png', img, params) on the GPU, byte for byte, for one uint8[H][W][3] BGR image or a batch
    uint8[N][H][W][3].  params: cv2.imwrite's PNG pairs (see bevk_png_encode_params), None for cv2's defaults; the
    RLE / HUFFMAN_ONLY strategies at any level and zlib's hash-chain parse at levels 4..9 (cv2.imwrite's
    [IMWRITE_PNG_COMPRESSION, 9] among them).  Level 0, levels 1..3 under the hash-chain strategies, BILEVEL and
    ZLIBBUFFER_SIZE raise BevkError.  The ctx's png_set_params list is left as it was.
    CUDA arrays (``__cuda_array_interface__``) are read in place, on torch's current stream; NumPy input is uploaded
    once.  Returns one ``bytes`` per image -- what cv2.imwrite would write to a .png file."""
    ctx = ctx or L.default_context()
    arr, k = _jpeg_params(params)
    return _encode("png_encode", images, ctx, png_encode_bound,   # the bound holds under every list
                   lambda img, out, cap, sizes: ctx.lib.bevk_png_encode_params(ctx.h, arr, k, *img, out, cap, sizes))


JPEG_EXTS = (".jpg", ".jpeg", ".jpe")


def imencode_bound(ext: str, width: int, height: int, channels: int = 3, params=None) -> int:
    """Largest stream imencode can produce for one width x height image of `channels` channels under params."""
    ext = str(ext).lower()
    n = C.c_uint64()
    if ext in JPEG_EXTS:
        _, arr, k = _imencode_jpeg_params(params)
        L.check(L.load().bevk_jpeg_encode_channels_bound(int(width), int(height), int(channels), arr, k, C.byref(n)))
    elif ext == ".png":
        L.check(L.load().bevk_png_encode_channels_bound(int(width), int(height), int(channels), C.byref(n)))
    else:
        raise L.BevkError(f"imencode: extension {ext!r} is not one the device encoders write (.jpg, .jpeg, .jpe, .png)")
    return n.value


def _imencode_jpeg_params(params):
    """(quality, ctypes array, n) of a whole cv2 JPEG list: IMWRITE_JPEG_QUALITY pairs become the quality (the last one
    wins, as in cv2; 95 without one), the other pairs stay in order."""
    p = [] if params is None else [int(v) for v in params]
    if len(p) % 2:
        raise L.BevkError(f"imencode: params must be (key, value) pairs, got {len(p)} ints")
    quality, rest = 95, []
    for key, value in zip(p[::2], p[1::2]):
        if key == 1:   # cv2.IMWRITE_JPEG_QUALITY
            quality = value
        else:
            rest += [key, value]
    arr, k = _jpeg_params(rest)
    return quality, arr, k


def imencode(ext: str, images, params=None, ctx: L.Context | None = None) -> list[bytes]:
    """cv2.imencode(ext, img, params) on the GPU, byte for byte, for grey, BGR and BGRA images: one stream per image.
    ext: ".jpg", ".jpeg", ".jpe" or ".png" (others raise BevkError).  images: uint8[H][W], [H][W][C] or [N][H][W][C] with
    C in 1 (grey), 3 (BGR), 4 (BGRA; JPEG drops alpha as cv2 does, PNG stores RGBA); a grey batch is [N][H][W][1].
    CUDA arrays (``__cuda_array_interface__``, e.g. the output of Undistorter.cuda) are read in place on torch's current
    stream; NumPy input is uploaded once.  params: cv2's whole list for the format, read as cv2 4.13 reads it --
    IMWRITE_JPEG_QUALITY (default 95) with the other IMWRITE_JPEG_* keys, PROGRESSIVE included, or the IMWRITE_PNG_*
    keys with png_encode's refusals (level 0, levels 1..3 under the hash-chain strategies, BILEVEL, ZLIBBUFFER_SIZE)."""
    ctx = ctx or L.default_context()
    ext = str(ext).lower()
    if ext in JPEG_EXTS:
        quality, arr, k = _imencode_jpeg_params(params)
        return _encode("imencode", images, ctx, lambda w, h, ch: imencode_bound(ext, w, h, ch, params),
                       lambda img, out, cap, sizes: ctx.lib.bevk_jpeg_encode_channels(ctx.h, arr, k, *img, int(quality),
                                                                                      out, cap, sizes),
                       channels=True)
    if ext == ".png":
        arr, k = _jpeg_params(params)
        return _encode("imencode", images, ctx, lambda w, h, ch: imencode_bound(ext, w, h, ch),
                       lambda img, out, cap, sizes: ctx.lib.bevk_png_encode_channels(ctx.h, arr, k, *img, out, cap, sizes),
                       channels=True)
    raise L.BevkError(f"imencode: extension {ext!r} is not one the device encoders write (.jpg, .jpeg, .jpe, .png)")


def remap(src: np.ndarray, map1: np.ndarray, map2: np.ndarray | None, interpolation: int = INTER_LINEAR,
          ctx: L.Context | None = None, out: np.ndarray | None = None, borderMode: int = BORDER_CONSTANT,
          borderValue=0) -> np.ndarray:
    """cv2.remap with CV_16SC2 (+CV_16UC1) maps.  interpolation: INTER_NEAREST, INTER_LINEAR,
    INTER_CUBIC, INTER_AREA (read as INTER_LINEAR, as cv2.remap reads it) or INTER_LANCZOS4; all but NEAREST need map2.
    The result is byte-identical to cv2.remap's.

    float32 maps (CV_32FC1: map1, map2 float32[h][w]; CV_32FC2: map1 float32[h][w][2], map2 None) give cv2.remap's bytes
    for float maps.  With them src may also be a CUDA array ([H][W], [H][W][C] or a batch [N][H][W][C], rows and images
    may be padded), read in place on torch's current stream, with the maps NumPy or CUDA arrays; the result then stays
    on the device (``out``, default a new torch tensor).

    src may be uint8, uint16, int16 or float32 (CUDA typestr <u2, <i2, <f4); the result has src's dtype and cv2's bits
    at that depth (DESIGN.md section 2).

    borderMode, borderValue: cv2's, bit for bit (BORDER_CONSTANT, _REPLICATE, _REFLECT, _WRAP, _REFLECT_101 and
    _TRANSPARENT; a number v means (v, 0, 0, 0)).  BORDER_TRANSPARENT writes into ``out``, which it needs; LINEAR under it
    at float32, which cv2 sums another way, raises BevkError (include/bevk.h has the rules)."""
    border = _border(borderMode, borderValue, out)
    ctx = ctx or L.default_context()
    if _is_float32(map1):
        return _remap_f32(src, map1, map2, interpolation, ctx, out, border)
    m1 = np.ascontiguousarray(map1, np.int16)
    if m1.ndim != 3 or m1.shape[2] != 2:
        raise L.BevkError("map1 must be int16[h][w][2] (CV_16SC2)")
    dh, dw = m1.shape[:2]
    m2 = None if map2 is None else np.ascontiguousarray(map2, np.uint16)
    if m2 is not None and m2.shape != (dh, dw):
        raise L.BevkError("map2 must be uint16[h][w] (CV_16UC1)")
    return _host_image(src, dw, dh, out, lambda f, s, d, dstride: f(
        ctx.h, *s, L.vptr(m1), None if m2 is None else L.vptr(m2), dw, dh, d, dstride, _interp(interpolation)), ctx.lib, "bevk_remap",
        border)


def _is_float32(a) -> bool:
    iface = getattr(a, "__cuda_array_interface__", None)
    if iface is not None:
        return iface["typestr"] == "<f4"
    return getattr(a, "dtype", None) == np.float32


def _float_map_shapes(map1, map2):
    """(dh, dw) of a float map pair: CV_32FC1 planes [h][w] + [h][w], or CV_32FC2 [h][w][2] + None."""
    s1 = _shape(map1)
    if map2 is None:
        if len(s1) != 3 or s1[2] != 2:
            raise L.BevkError(f"a float map1 without map2 must be float32[h][w][2] (CV_32FC2), got shape {s1}")
    elif len(s1) != 2 or _shape(map2) != s1 or not _is_float32(map2):
        raise L.BevkError(f"float maps must be float32[h][w] planes (CV_32FC1) or float32[h][w][2] and None (CV_32FC2); "
                          f"got shapes {s1} and {_shape(map2)}")
    return s1[0], s1[1]


def _shape(a):
    iface = getattr(a, "__cuda_array_interface__", None)
    return tuple(iface["shape"]) if iface is not None else np.shape(a)


def _cuda_dense(arr, typestr, what):
    """Device pointer of a C-contiguous CUDA array of the given typestr."""
    iface = arr.__cuda_array_interface__
    if iface["typestr"] != typestr:
        raise L.BevkError(f"{what} must have typestr {typestr}, got {iface['typestr']}")
    shape, strides = tuple(iface["shape"]), iface.get("strides")
    if strides is not None:
        step = np.dtype(typestr).itemsize
        for n, st in zip(reversed(shape), reversed(strides)):
            if n > 1 and st != step:
                raise L.BevkError(f"{what} must be C-contiguous")
            step *= n
    if not iface["data"][0]:
        raise L.BevkError(f"{what} has a null data pointer")
    return C.c_void_p(int(iface["data"][0]))


def _device_maps(maps, dtypes, ctx):
    """Device pointers of maps (None stays None) given as CUDA arrays of the given dtypes, or as NumPy arrays, which are
    uploaded on torch's current stream and returned with the pointers so that they outlive the call that reads them."""
    import torch
    ptrs, keep = [], []
    for m, dt in zip(maps, dtypes):
        if m is None:
            ptrs.append(None)
            continue
        if not hasattr(m, "__cuda_array_interface__"):
            m = torch.from_numpy(np.ascontiguousarray(m, dt)).to(torch.device("cuda", ctx.device))
            keep.append(m)
        ptrs.append(_cuda_dense(m, np.dtype(dt).str, "map"))
    return ptrs, keep


def _remap_f32(src, map1, map2, interpolation, ctx, out, border=None):
    dh, dw = _float_map_shapes(map1, map2)
    if hasattr(src, "__cuda_array_interface__"):
        (m1, m2), keep = _device_maps((map1, map2), (np.float32, np.float32), ctx)
        return _device_images(src, dw, dh, out, ctx, "remap", lambda f, s, d: f(
            ctx.h, *s, m1, m2, *d, _interp(interpolation)), name="bevk_remap_f32_stack", border=border)
    if hasattr(map1, "__cuda_array_interface__") or hasattr(map2, "__cuda_array_interface__"):
        raise L.BevkError("remap: CUDA maps need a CUDA source image")
    m1 = np.ascontiguousarray(map1, np.float32)
    m2 = None if map2 is None else np.ascontiguousarray(map2, np.float32)
    return _host_image(src, dw, dh, out, lambda f, s, d, dstride: f(
        ctx.h, *s, L.vptr(m1), None if m2 is None else L.vptr(m2), dw, dh, d, dstride, _interp(interpolation)), ctx.lib,
        "bevk_remap_f32", border)


def convert_maps(map1, map2, dstmap1type: int, nninterpolation: bool = False, ctx: L.Context | None = None):
    """cv2.convertMaps(map1, map2, dstmap1type, nninterpolation=...) between CV_16SC2 (int16[h][w][2] with a uint16[h][w]
    map2 or None), CV_32FC1 (float32[h][w] planes) and CV_32FC2 (float32[h][w][2], map2 None), bit for bit.  Returns
    (map1, map2) with map2 None for CV_32FC2 and for CV_16SC2 with nninterpolation.  NumPy maps come back as NumPy
    arrays; CUDA arrays are converted in place on torch's current stream into new torch tensors.  Converting a type
    to itself raises BevkError."""
    ctx = ctx or L.default_context()
    dst = _map_type(dstmap1type)
    s1 = _shape(map1)
    if len(s1) == 3 and s1[2] == 2 and not _is_float32(map1):
        src = CV_16SC2
        if map2 is not None and _shape(map2) != s1[:2]:
            raise L.BevkError(f"map2 of a CV_16SC2 map1 must be uint16{list(s1[:2])} or None")
    else:
        src = CV_32FC2 if map2 is None else CV_32FC1
        _float_map_shapes(map1, map2)
    h, w = s1[0], s1[1]
    nn = bool(nninterpolation) and dst == CV_16SC2
    shapes = {CV_16SC2: [((h, w, 2), np.int16), None if nn else ((h, w), np.uint16)],
              CV_32FC1: [((h, w), np.float32), ((h, w), np.float32)],
              CV_32FC2: [((h, w, 2), np.float32), None]}[dst]
    want = {CV_16SC2: (np.int16, np.uint16), CV_32FC1: (np.float32, np.float32), CV_32FC2: (np.float32, None)}[src]
    if hasattr(map1, "__cuda_array_interface__"):
        import torch
        dev = torch.device("cuda", ctx.device)
        outs = [None if sd is None else torch.empty(sd[0], dtype=getattr(torch, np.dtype(sd[1]).name), device=dev)
                for sd in shapes]
        (p1, p2), keep = _device_maps((map1, map2), want, ctx)
        from .sharding import _torch_current_stream
        with ctx.on_stream(_torch_current_stream(ctx.device)):
            L.check(ctx.lib.bevk_convert_maps(ctx.h, p1, p2, src, w, h, dst, int(nn),
                                              *[None if o is None else C.c_void_p(o.data_ptr()) for o in outs], 1))
        return outs[0], outs[1]
    m1 = np.ascontiguousarray(map1, want[0])
    m2 = None if map2 is None else np.ascontiguousarray(map2, want[1])
    outs = [None if sd is None else np.empty(*sd) for sd in shapes]
    L.check(ctx.lib.bevk_convert_maps(ctx.h, L.vptr(m1), None if m2 is None else L.vptr(m2), src, w, h, dst, int(nn),
                                      *[None if o is None else L.vptr(o) for o in outs], 0))
    return outs[0], outs[1]


def warp_perspective(src: np.ndarray, H, dsize, flags: int = INTER_LINEAR, ctx: L.Context | None = None,
                     out: np.ndarray | None = None, borderMode: int = BORDER_CONSTANT, borderValue=0):
    """cv2.warpPerspective(src, H, dsize, flags, borderMode=, borderValue=) for uint8, uint16, int16 and float32 images,
    borders as remap() takes them; NEAREST and LINEAR at int16 under BORDER_REPLICATE / BORDER_TRANSPARENT raise
    BevkError (cv2 computes them with another body than cv2.remap's).  flags:
    INTER_NEAREST, INTER_LINEAR, INTER_CUBIC, INTER_AREA (read as INTER_LINEAR, as cv2 reads it) or INTER_LANCZOS4; LINEAR / AREA at
    uint16 with 3 or 4 channels and NEAREST at float32 with 1 or 4 channels raise BevkError (cv2 computes them with
    other bodies than cv2.remap's)."""
    border = _border(borderMode, borderValue, out)
    ctx = ctx or L.default_context()
    dw, dh = int(dsize[0]), int(dsize[1])
    return _host_image(src, dw, dh, out, lambda f, s, d, dstride: f(
        ctx.h, *s, L.dptr(H), d, dw, dh, dstride, _interp(flags)), ctx.lib, "bevk_warp_perspective", border)


INTER_LINEAR_EXACT, INTER_NEAREST_EXACT, WARP_INVERSE_MAP = L.INTER_LINEAR_EXACT, L.INTER_NEAREST_EXACT, L.WARP_INVERSE_MAP


def _border(borderMode, borderValue, out):
    """cv2's borderMode and borderValue as a gather's _border arguments (mode, double[4]), or None for the zero constant
    border, which the _typed and uint8 entry points give.  borderValue follows cv2's Scalar: a number v is (v, 0, 0, 0),
    a sequence gives up to four values.  The library checks the mode (BORDER_ISOLATED and unknown modes raise) and
    converts the values to the image's depth as cv2 does.  BORDER_TRANSPARENT leaves pixels of the destination as they
    were, so it needs ``out``: cv2 leaves them undefined in a new array."""
    vals = np.atleast_1d(np.asarray(borderValue, np.float64)).ravel()
    if vals.size > 4:
        raise L.BevkError(f"borderValue takes up to 4 values (cv2's Scalar), got {vals.size}")
    mode = int(borderMode)
    if mode == BORDER_TRANSPARENT and out is None:
        raise L.BevkError("BORDER_TRANSPARENT needs out=: it writes only some pixels of the destination")
    if mode == BORDER_CONSTANT and not vals.any():
        return None
    v = (C.c_double * 4)(*vals, *[0.0] * (4 - vals.size))
    return mode, v


def _gather_fn(lib, name, dtype, border=None):
    """The library entry point of an image gather: `name` for uint8 images, its _typed sibling (a cv2 type code in place
    of the channel count) for uint16, int16 and float32 ones, and with a border (_border's) its _border sibling, which
    takes the type code at every depth and the border after the _typed arguments."""
    if border is not None:
        fn = getattr(lib, name + "_border")
        return lambda *a: fn(*a, *border)
    return getattr(lib, name) if dtype == np.uint8 else getattr(lib, name + "_typed")


def _type_code(dtype, ch, border):
    """The kind argument of a gather entry point: the channel count for uint8 images without a border, else cv2's type
    code."""
    if dtype == np.uint8:
        return ch if border is None else (ch - 1) << 3
    return _WIDE[dtype] + ((ch - 1) << 3)


def _host_image(src, dw, dh, out, call, lib=None, name=None, border=None):
    """The body of the host forms: src a NumPy image [H][W] or [H][W][C]; out (default a new array) [dh][dw] of the same
    rank and dtype; call(src, dst, dst_stride) with src's (pointer, width, height, stride, channels) and dst's pointer.
    With lib and name (an image gather) src may also be uint16, int16 or float32: call then takes the entry point first
    (_gather_fn), and the channel count becomes the cv2 type code for the _typed sibling.  border: _border's."""
    if name is None:
        img, sw, sh, ss, ch = L.image_view(src)
        out = _out((dh, dw) if src.ndim == 2 else (dh, dw, ch), out)
        L.check(call((L.vptr(img), sw, sh, ss, ch), L.vptr(out), dw * ch))
        return out
    img, sw, sh, ss, ch = L.image_view(src, (np.uint8, *_WIDE))
    out = _out((dh, dw) if src.ndim == 2 else (dh, dw, ch), out, img.dtype)
    kind = _type_code(img.dtype, ch, border)
    L.check(call(_gather_fn(lib, name, img.dtype, border), (L.vptr(img), sw, sh, ss, kind), L.vptr(out),
                 dw * ch * img.itemsize))
    return out


def _device_images(src, dw, dh, out, ctx, what, call, stream=None, name=None, border=None):
    """The body of the device forms: src a uint8 CUDA array [H][W], [H][W][C] or [N][H][W][C] read in place; out
    (default a new torch tensor) of the same rank with dh x dw images; call(src, out) with the (pointer, image stride,
    ...) layouts is run on ``stream`` (default torch's current stream) and only enqueues.  With name (an image gather)
    src may also be uint16, int16 or float32 (typestr <u2, <i2, <f4), out of the same dtype, and call takes the entry
    point first, as _host_image's does (border too)."""
    wide = name is not None
    ptr, rank, n, sh, sw, ch, simg, srow = _cuda_images(src, what, wide)
    dtype = _cuda_dtype(src) if wide else np.dtype(np.uint8)
    shape = {2: (dh, dw), 3: (dh, dw, ch), 4: (n, dh, dw, ch)}[rank]
    if out is None:
        import torch
        out = torch.empty(shape, dtype=getattr(torch, dtype.name), device=torch.device("cuda", ctx.device))
    optr, orank, on, oh, ow, och, oimg, orow = _cuda_images(out, "out", wide)
    if orank != rank or (on, oh, ow, och) != (n, dh, dw, ch) or (wide and _cuda_dtype(out) != dtype):
        raise L.BevkError(f"out must be a {dtype.name} CUDA array of shape {shape}")
    if stream is None:
        from .sharding import _torch_current_stream
        stream = _torch_current_stream(ctx.device)
    kind = _type_code(dtype, ch, border)
    s, d = (C.c_void_p(ptr), simg, sw, sh, srow, kind, n), (C.c_void_p(optr), oimg, dw, dh, orow)
    with ctx.on_stream(stream):
        L.check(call(_gather_fn(ctx.lib, name, dtype, border), s, d) if wide else call(s, d))
    return out


def _image_call(src, dw, dh, out, ctx, what, host, device, name=None, border=None):
    """A CUDA array goes to the device form (_device_images, with ``device``), anything else to the host form
    (_host_image, with ``host``); name: the host entry point of an image gather (its device form is name + "_stack")."""
    if hasattr(src, "__cuda_array_interface__"):
        return _device_images(src, dw, dh, out, ctx, what, device, name=name and name + "_stack", border=border)
    return _host_image(src, dw, dh, out, host, ctx.lib, name, border)


def _src_size(src):
    """(width, height) of a NumPy image or a CUDA array [H][W], [H][W][C] or [N][H][W][C]."""
    if hasattr(src, "__cuda_array_interface__"):
        shape = tuple(src.__cuda_array_interface__["shape"])
        return (shape[1], shape[0]) if len(shape) < 4 else (shape[2], shape[1])
    return src.shape[1], src.shape[0]


def resize_size(ssize, dsize, fx: float = 0, fy: float = 0):
    """cv2.resize's output size: dsize, or when dsize is (0, 0) / None, (round(sw * fx), round(sh * fy))."""
    if dsize is not None and tuple(int(v) for v in dsize) != (0, 0):
        return int(dsize[0]), int(dsize[1])
    if not (fx > 0 and fy > 0):
        raise L.BevkError("resize: dsize (0, 0) needs fx > 0 and fy > 0")
    dw, dh = int(np.rint(ssize[0] * float(fx))), int(np.rint(ssize[1] * float(fy)))   # saturate_cast: half to even
    if dw <= 0 or dh <= 0:
        raise L.BevkError(f"resize: fx {fx}, fy {fy} make an empty image from {ssize}")
    return dw, dh


def resize(src, dsize, fx: float = 0, fy: float = 0, interpolation: int = INTER_LINEAR, ctx: L.Context | None = None,
           out=None):
    """cv2.resize(src, dsize, fx=fx, fy=fy, interpolation=interpolation) for uint8 images, byte for byte: INTER_NEAREST,
    INTER_LINEAR and INTER_AREA (others raise BevkError).  As in cv2, a dsize of (0, 0) takes the size from fx, fy and uses
    them as the scales, which gives other pixels than the dsize form of the same size.
    NumPy input ([H][W] or [H][W][C]) is uploaded, resized and downloaded; a CUDA array ([H][W], [H][W][C] or a batch
    [N][H][W][C], rows and images may be padded) is read in place on torch's current stream and the result stays on the
    device (``out``, default a new torch tensor)."""
    ctx = ctx or L.default_context()
    dw, dh = resize_size(_src_size(src), dsize, fx, fy)
    sx, sy = (float(fx), float(fy)) if dsize is None or tuple(int(v) for v in dsize) == (0, 0) else (0.0, 0.0)
    return _image_call(src, dw, dh, out, ctx, "resize",
                       lambda s, d, ds: ctx.lib.bevk_resize(ctx.h, *s, d, dw, dh, ds, sx, sy, int(interpolation)),
                       lambda s, d: ctx.lib.bevk_resize_stack(ctx.h, *s, *d, sx, sy, int(interpolation)))


def warp_affine(src, M, dsize, flags: int = INTER_LINEAR, borderMode: int = BORDER_CONSTANT, borderValue=0,
                ctx: L.Context | None = None, out=None):
    """cv2.warpAffine(src, M, dsize, flags=flags) for uint8, uint16, int16 and float32 images with a zero
    constant border, bit for bit; NEAREST at int16 and at uint16 with 4 channels raises BevkError (cv2 computes it with
    another body than cv2.remap's).  M: 2x3.
    flags: any interpolation warp_perspective takes, optionally | WARP_INVERSE_MAP.  Other borders raise BevkError:
    warp_affine_border takes them.
    Takes NumPy images and CUDA arrays as resize() does."""
    if borderMode != BORDER_CONSTANT or np.any(np.asarray(borderValue) != 0):
        raise L.BevkError("warp_affine supports BORDER_CONSTANT with value 0 only; warp_affine_border takes cv2's other "
                          "borders")
    return _warp_affine(src, M, dsize, flags, None, ctx, out)


def warp_affine_border(src, M, dsize, flags: int = INTER_LINEAR, borderMode: int = BORDER_CONSTANT, borderValue=0,
                       ctx: L.Context | None = None, out=None):
    """cv2.warpAffine(src, M, dsize, flags=flags, borderMode=borderMode, borderValue=borderValue), bit for bit: warp_affine
    with cv2's border modes and values as remap() takes them.  BORDER_TRANSPARENT writes into ``out``, which it needs."""
    return _warp_affine(src, M, dsize, flags, _border(borderMode, borderValue, out), ctx, out)


def _warp_affine(src, M, dsize, flags, border, ctx, out):
    ctx = ctx or L.default_context()
    m = np.asarray(M, np.float64)
    if m.shape != (2, 3):
        raise L.BevkError(f"M must be 2x3, got shape {m.shape}")
    dw, dh = int(dsize[0]), int(dsize[1])
    return _image_call(src, dw, dh, out, ctx, "warp_affine",
                       lambda f, s, d, ds: f(ctx.h, *s, L.dptr(m), d, dw, dh, ds, int(flags)),
                       lambda f, s, d: f(ctx.h, *s, L.dptr(m), *d, int(flags)), "bevk_warp_affine", border)


_GATHER_PATHS = {4: "word", 1: "byte", 2: "taps", 3: "resize"}


def last_path(ctx: L.Context | None = None) -> str:
    """Which kernel the last gather or resize call of ctx launched: 'word' (k_gather4), 'byte' (k_gather), 'taps'
    (k_gather_taps) or 'resize' (k_resize)."""
    ctx = ctx or L.default_context()
    return _GATHER_PATHS.get(int(ctx.lib.bevk_undistort_last_path(ctx.h)), "none")


def warp_perspective_maps(map1, map2, H, dsize, ctx: L.Context | None = None):
    """cv2.warpPerspective applied to a CV_16SC2 / CV_16UC1 map pair (Camera.get_bev_maps)."""
    ctx = ctx or L.default_context()
    m1 = np.ascontiguousarray(map1, np.int16)
    m2 = np.ascontiguousarray(map2, np.uint16)
    sh, sw = m2.shape
    dw, dh = int(dsize[0]), int(dsize[1])
    o1 = np.empty((dh, dw, 2), np.int16)
    o2 = np.empty((dh, dw), np.uint16)
    L.check(ctx.lib.bevk_warp_maps(ctx.h, L.vptr(m1), L.vptr(m2), sw, sh, L.dptr(H), dw, dh, L.vptr(o1), L.vptr(o2)))
    return o1, o2


def _dense_bgr(img: np.ndarray) -> np.ndarray:
    if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3:
        raise L.BevkError("expected a uint8[h][w][3] BGR image")
    return np.ascontiguousarray(img)


def apply_mask(img: np.ndarray, mask: np.ndarray, blend: bool, ctx: L.Context | None = None) -> np.ndarray:
    """Mask.__call__ (blend=False) / BlendMask.__call__ (blend=True)."""
    ctx = ctx or L.default_context()
    a = _dense_bgr(img)
    m = np.ascontiguousarray(mask, np.uint8)
    if m.shape != a.shape[:2]:
        raise L.BevkError("mask and image sizes differ")
    out = np.empty_like(a)
    L.check(ctx.lib.bevk_apply_mask(ctx.h, L.vptr(a), L.vptr(m), a.shape[1], a.shape[0], int(blend), L.vptr(out)))
    return out


def color_balance(image: np.ndarray, ctx: L.Context | None = None) -> np.ndarray:
    ctx = ctx or L.default_context()
    a = _dense_bgr(image)
    out = np.empty_like(a)
    L.check(ctx.lib.bevk_color_balance(ctx.h, L.vptr(a), a.shape[1], a.shape[0], L.vptr(out)))
    return out


def luminance_balance(images, ctx: L.Context | None = None):
    ctx = ctx or L.default_context()
    imgs = [_dense_bgr(i) for i in images]
    if len({i.shape for i in imgs}) != 1:
        raise L.BevkError("luminance_balance: frames must share one size")
    outs = [np.empty_like(i) for i in imgs]
    n = len(imgs)
    ip = (C.c_void_p * n)(*[i.ctypes.data for i in imgs])
    op = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
    L.check(ctx.lib.bevk_luminance_balance(ctx.h, ip, n, imgs[0].shape[1], imgs[0].shape[0], op))
    return outs


# ---- points: cv2's point functions (bevk_points.cuh), bit for bit.  NumPy points come back as NumPy arrays; CUDA
# points (__cuda_array_interface__) are mapped on torch's current stream into new torch tensors, without a synchronise.
TERM_COUNT, TERM_EPS = 1, 2   # cv2.TermCriteria_COUNT / _EPS
_POINT_DEPTHS = {"<f4": 5, "<f8": 6}


def _points(pts, k, what, flat=True):
    """(pts, n, typestr, out shape) of cv2 points of k elements: [N][1][k] or [1][N][k] (and [N][k] where cv2's pinhole
    functions take it, flat=True, which they return as [N][1][2]); float32 or float64, dense."""
    iface = getattr(pts, "__cuda_array_interface__", None)
    if iface is None:
        pts = np.asarray(pts)
        typestr = pts.dtype.str
        pts = np.ascontiguousarray(pts)
    else:
        typestr = iface["typestr"]
    if typestr not in _POINT_DEPTHS:
        raise L.BevkError(f"{what}: points must be float32 or float64, got {typestr}")
    shape = _shape(pts)
    if len(shape) == 3 and shape[2] == k and 1 in shape[:2]:
        n = shape[0] * shape[1]
        out = (n, 1, 2) if flat else (shape[0], shape[1], 2)
    elif flat and len(shape) == 2 and shape[1] == k:
        n, out = shape[0], (shape[0], 1, 2)
    else:
        raise L.BevkError(f"{what}: points must be [N][1][{k}] or [1][N][{k}]{f' or [N][{k}]' if flat else ''}, got {shape}")
    return pts, n, typestr, out


def _point_call(pts, k, what, flat, call, ctx, out=None):
    """Run call(src, dst, n, depth, on_device) on host or CUDA points; out: an existing destination (in place: pts).
    A NumPy destination must be a writeable C-contiguous float32 / float64 ndarray (the call writes it densely)."""
    ctx = ctx or L.default_context()
    if out is not None and not hasattr(out, "__cuda_array_interface__") and not (
            isinstance(out, np.ndarray) and out.dtype.str in _POINT_DEPTHS and out.flags.c_contiguous
            and out.flags.writeable):
        raise L.BevkError(f"{what}: inplace needs a writeable C-contiguous float32 or float64 array")
    pts, n, typestr, shape = _points(pts, k, what, flat)
    depth = _POINT_DEPTHS[typestr]
    if hasattr(pts, "__cuda_array_interface__"):
        import torch
        from .sharding import _torch_current_stream
        if out is None:
            out = torch.empty(shape, dtype=torch.float32 if depth == 5 else torch.float64, device=torch.device("cuda", ctx.device))
        src = _cuda_dense(pts, typestr, what) if n else None
        dst = _cuda_dense(out, typestr, what) if n else None
        with ctx.on_stream(_torch_current_stream(ctx.device)):
            L.check(call(ctx, src, dst, n, depth, 1))
        return out
    if out is None:
        out = np.empty(shape, np.dtype(typestr))
    L.check(call(ctx, L.vptr(pts) if n else None, L.vptr(out) if n else None, n, depth, 0))
    return out


def _dist(D):
    d = None if D is None else np.asarray(D, np.float64).reshape(-1)
    return (None, 0) if d is None or d.size == 0 else (L.dptr(d), int(d.size))


def _mat3(M, what):
    if M is None:
        return None
    m = np.asarray(M, np.float64)
    if m.shape == (3, 4):   # a projection matrix: its first three columns, as cv2 takes them
        m = m[:, :3]
    if m.shape != (3, 3):
        raise L.BevkError(f"{what} must be 3x3, got shape {m.shape}")
    return L.dptr(m)


def _undistort_points(model, src, K, D, R, P, criteria, ctx, inplace, what):
    typ, count, eps = criteria
    d, nd = _dist(D)
    r, nr = None, 0
    if R is not None:
        rr = np.asarray(R, np.float64)
        if rr.size == 3 and model == L.MODEL_FISHEYE:
            r, nr = L.dptr(rr), 3
        else:
            r, nr = _mat3(rr, "R"), 9
    return _point_call(src, 2, what, model == L.MODEL_PINHOLE, lambda c, s, o, n, dep, dev: c.lib.bevk_undistort_points(
        c.h, model, s, o, n, dep, L.dptr(K), d, nd, r, nr, _mat3(P, "P"), int(typ), int(count), float(eps), dev), ctx,
        src if inplace else None)


def undistort_points(src, cameraMatrix, distCoeffs, dst=None, R=None, P=None, ctx: L.Context | None = None,
                     inplace: bool = False):
    """cv2.undistortPoints(src, cameraMatrix, distCoeffs, R=, P=): D of 0, 4, 5, 8, 12 or 14 coefficients (None: no
    distortion), R 3x3, P 3x3 or 3x4.  Returns [N][1][2] of src's dtype.  inplace=True writes into src ([N][1][2] or
    [1][N][2]) and returns it."""
    return undistort_points_iter(src, cameraMatrix, distCoeffs, R, P, (TERM_COUNT, 5, 0.01), ctx=ctx, inplace=inplace)


def undistort_points_iter(src, cameraMatrix, distCoeffs, R, P, criteria, dst=None, ctx: L.Context | None = None,
                          inplace: bool = False):
    """cv2.undistortPointsIter(src, cameraMatrix, distCoeffs, R, P, criteria) with a COUNT criteria of at most 1000
    iterations; EPS raises BevkError (its reprojection-error stop is not followed)."""
    return _undistort_points(L.MODEL_PINHOLE, src, cameraMatrix, distCoeffs, R, P, criteria, ctx, inplace,
                             "undistort_points")


def fisheye_undistort_points(distorted, K, D, undistorted=None, R=None, P=None, criteria=(TERM_COUNT | TERM_EPS, 10, 1e-8),
                             ctx: L.Context | None = None, inplace: bool = False):
    """cv2.fisheye.undistortPoints(distorted, K, D, R=, P=, criteria=) for float32 points ([N][1][2] or [1][N][2], returned
    in the same shape); R a 3x3 matrix or an rvec.  float64 raises BevkError (cv2's glibc tan is not reproducible)."""
    return _undistort_points(L.MODEL_FISHEYE, distorted, K, D, R, P, criteria, ctx, inplace, "fisheye_undistort_points")


def _project(model, objectPoints, rvec, tvec, K, D, alpha, ctx, what):
    d, nd = _dist(D)
    rv, tv = np.asarray(rvec, np.float64).reshape(-1), np.asarray(tvec, np.float64).reshape(-1)
    if rv.size != 3 or tv.size != 3:
        raise L.BevkError(f"{what}: rvec and tvec must have 3 entries")
    pts = _point_call(objectPoints, 3, what, model == L.MODEL_PINHOLE, lambda c, s, o, n, dep, dev: c.lib.bevk_project_points(
        c.h, model, s, o, n, dep, L.dptr(rv), L.dptr(tv), L.dptr(K), d, nd, float(alpha), dev), ctx)
    return pts, None


def project_points(objectPoints, rvec, tvec, cameraMatrix, distCoeffs, imagePoints=None, jacobian=None, aspectRatio=0,
                   ctx: L.Context | None = None):
    """cv2.projectPoints(objectPoints, rvec, tvec, cameraMatrix, distCoeffs) -> (imagePoints [N][1][2], None): no
    jacobian is computed."""
    if aspectRatio:
        raise L.BevkError("project_points: aspectRatio is only used by cv2's jacobian, which is not computed")
    return _project(L.MODEL_PINHOLE, objectPoints, rvec, tvec, cameraMatrix, distCoeffs, 0., ctx, "project_points")


def fisheye_project_points(objectPoints, rvec, tvec, K, D, imagePoints=None, alpha: float = 0, jacobian=None,
                           ctx: L.Context | None = None):
    """cv2.fisheye.projectPoints(objectPoints, rvec, tvec, K, D, alpha=) -> (imagePoints, None) for float32 points
    [N][1][3] or [1][N][3]; float64 raises BevkError."""
    return _project(L.MODEL_FISHEYE, objectPoints, rvec, tvec, K, D, alpha, ctx, "fisheye_project_points")


def fisheye_distort_points(undistorted, K, D, distorted=None, alpha: float = 0, ctx: L.Context | None = None,
                           inplace: bool = False):
    """cv2.fisheye.distortPoints(undistorted, K, D, alpha=) of float32 normalised points [N][1][2] or [1][N][2]."""
    d, nd = _dist(D)
    return _point_call(undistorted, 2, "fisheye_distort_points", False, lambda c, s, o, n, dep, dev:
                       c.lib.bevk_fisheye_distort_points(c.h, s, o, n, dep, L.dptr(K), d, nd, float(alpha), dev), ctx,
                       undistorted if inplace else None)


def perspective_transform(src, m, dst=None, ctx: L.Context | None = None, inplace: bool = False):
    """cv2.perspectiveTransform(src, m) of float32 or float64 2-D points [N][1][2] or [1][N][2] by a 3x3 m."""
    mm = np.asarray(m, np.float64)
    if mm.shape != (3, 3):
        raise L.BevkError(f"perspective_transform: m must be 3x3 (2-D points), got shape {mm.shape}")
    return _point_call(src, 2, "perspective_transform", False, lambda c, s, o, n, dep, dev:
                       c.lib.bevk_perspective_transform(c.h, s, o, n, dep, L.dptr(mm), dev), ctx, src if inplace else None)


class Undistorter:
    """Device-resident undistortion map (or fused camera model) + per-frame gather.

    D: 4 fisheye coefficients, or 4, 5, 8, 12 or 14 pinhole ones (cv2's rational, thin-prism and tilted models).  R: a
    rectification rotation (cv2.stereoRectify's R1 / R2), None for eye(3).  A fused fisheye whose rotated rays depend on
    the row is refused (BevkError): cv2 walks those rays with running row sums, which only a map-resident slot follows.
    A fused pinhole slot of such a camera keeps the block starts of cv2's sums (3 bytes per pixel of device memory).
    m1type: the maps whose cv2.remap bytes every call gives: CV_16SC2 (default), CV_32FC1 or CV_32FC2 (pinhole only, as
    in cv2).  A map-resident float slot keeps 8 bytes per pixel; a fused one rounds the model's (u, v) to float per pixel.

    A bevk_ctx has 8 undistorter slots.  Each live Undistorter owns one slot of its ctx; the slot returns to the
    pool on close() / garbage collection, and a 9th live object on one ctx raises instead of silently taking over a
    slot another object still uses."""

    def __init__(self, K, D, P, size, model: str = "fisheye", fused: bool = False, ctx: L.Context | None = None,
                 slot: int | None = None, R=None, m1type: int = CV_16SC2):
        self.ctx = ctx or L.default_context()
        self.slot = None
        live = self.ctx.__dict__.setdefault("_und_slots", set())
        if slot is None:
            free = [i for i in range(8) if i not in live]
            if not free and ctx is None:
                # the shared default context is full (e.g. two BevGenerators' cameras): this object gets its own
                self.ctx = L.Context(self.ctx.device)
                live = self.ctx.__dict__.setdefault("_und_slots", set())
                free = [0]
            if not free:
                raise L.BevkError("all 8 undistorter slots of this context are in use: close() an Undistorter "
                                  "(or let it be collected), or give this one its own Context")
            slot = free[0]
        elif not 0 <= int(slot) < 8:
            raise L.BevkError(f"slot {slot} out of range [0, 8)")
        elif slot in live:
            raise L.BevkError(f"undistorter slot {slot} of this context is owned by a live Undistorter")
        self.w, self.h = int(size[0]), int(size[1])
        d = np.asarray(D, np.float64).reshape(-1)
        m = L.MODEL_FISHEYE if model == "fisheye" else L.MODEL_PINHOLE
        self.m1type = _map_type(m1type)
        if self.m1type != CV_16SC2:
            L.check(self.ctx.lib.bevk_undistorter_set_f32(self.ctx.h, slot, m, L.dptr(K), L.dptr(d), int(d.size),
                                                          _rotation(R), L.dptr(P), self.w, self.h, int(fused), self.m1type))
        elif R is None:
            L.check(self.ctx.lib.bevk_undistorter_set(self.ctx.h, slot, m, L.dptr(K), L.dptr(d), int(d.size), L.dptr(P),
                                                      self.w, self.h, int(fused)))
        else:
            L.check(self.ctx.lib.bevk_undistorter_set_rectify(self.ctx.h, slot, m, L.dptr(K), L.dptr(d), int(d.size),
                                                              _rotation(R), L.dptr(P), self.w, self.h, int(fused)))
        self.slot = int(slot)
        live.add(self.slot)

    def close(self):
        if getattr(self, "slot", None) is not None:
            self.ctx.__dict__.get("_und_slots", set()).discard(self.slot)
            self.slot = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _live(self):
        if self.slot is None:
            raise L.BevkError("this Undistorter was closed")

    def maps(self):
        """The maps the slot follows, as cv2.initUndistortRectifyMap builds them with the slot's m1type."""
        self._live()
        if self.m1type != CV_16SC2:
            m1, m2 = _float_maps(self.m1type, self.h, self.w)
            L.check(self.ctx.lib.bevk_undistorter_maps_f32(self.ctx.h, self.slot, L.vptr(m1), None if m2 is None else L.vptr(m2)))
            return m1, m2
        m1 = np.empty((self.h, self.w, 2), np.int16)
        m2 = np.empty((self.h, self.w), np.uint16)
        L.check(self.ctx.lib.bevk_undistorter_maps(self.ctx.h, self.slot, L.vptr(m1), L.vptr(m2)))
        return m1, m2

    def __call__(self, src: np.ndarray, interpolation: int = INTER_LINEAR, out: np.ndarray | None = None,
                 borderMode: int = BORDER_CONSTANT, borderValue=0) -> np.ndarray:
        """cv2.remap(src, map1, map2, interpolation, borderMode=, borderValue=), any of remap()'s interpolations and
        borders.  A CUDA array (e.g. a torch tensor on the GPU) goes to cuda() and
        the result stays on the device; NumPy input is uploaded, undistorted and downloaded in one call."""
        self._live()
        lib, h = self.ctx.lib, self.ctx.h
        if hasattr(src, "__cuda_array_interface__"):
            return self.cuda(src, out, interpolation, borderMode=borderMode, borderValue=borderValue)
        border = _border(borderMode, borderValue, out)
        return _host_image(src, self.w, self.h, out, lambda f, s, d, ds: f(h, self.slot, *s, d, self.w, self.h, ds,
                                                                           _interp(interpolation)), lib, "bevk_undistort",
                           border)

    def jpeg(self, src: np.ndarray, quality: int = 95, interpolation: int = INTER_LINEAR, params=None) -> bytes:
        """The undistorted image as the bytes cv2.imwrite(path, self(src), [IMWRITE_JPEG_QUALITY, quality] + params)
        writes to a .jpg file; the image itself never leaves the GPU.  src: uint8[h][w][3] BGR.  params: cv2.imwrite's
        other JPEG pairs (see jpeg_encode), None for cv2's defaults.  interpolation: as for __call__."""
        self._live()
        img, sw, sh, ss, ch = L.image_view(src)
        if ch != 3 or src.ndim != 3:
            raise L.BevkError("Undistorter.jpeg takes uint8[h][w][3] BGR images")
        bound = jpeg_encode_bound(self.w, self.h, params)
        if getattr(self, "_jpeg_buf", None) is None or self._jpeg_buf.size < bound:
            self._jpeg_buf = np.empty(bound, np.uint8)
        jpeg_set_params(self.ctx, params)
        size = C.c_uint64()
        L.check(self.ctx.lib.bevk_undistort_jpeg(self.ctx.h, self.slot, L.vptr(img), sw, sh, ss, _interp(interpolation),
                                                 int(quality), L.vptr(self._jpeg_buf), self._jpeg_buf.size, C.byref(size)))
        return self._jpeg_buf[:size.value].tobytes()

    def png(self, src: np.ndarray, params=None, interpolation: int = INTER_LINEAR) -> bytes:
        """The undistorted image as the bytes cv2.imwrite(path, self(src), params) writes to a .png file: undistorted
        and encoded on the device (png_encode's params, e.g. [IMWRITE_PNG_COMPRESSION, 9]), only the stream comes back.
        src: uint8[h][w][3] BGR.  interpolation: as for __call__."""
        self._live()
        a = np.asarray(src)
        if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3:
            raise L.BevkError("Undistorter.png takes uint8[h][w][3] BGR images")
        import torch
        d = torch.from_numpy(np.ascontiguousarray(a)).to(torch.device("cuda", self.ctx.device))
        return png_encode(self.cuda(d, interpolation=interpolation), ctx=self.ctx, params=params)[0]

    def cuda(self, frames, out=None, interpolation: int = INTER_LINEAR, stream: int | None = None,
             borderMode: int = BORDER_CONSTANT, borderValue=0):
        """Undistort frames that already live on the GPU: no PCIe in the call.

        frames: a uint8, uint16, int16 or float32 CUDA array (``__cuda_array_interface__``; ``out`` of the same dtype)
        [H][W] (one grey image), [H][W][C] (one image) or
        [N][H][W][C] (a batch; a grey batch is [N][H][W][1]), C in 1, 3, 4.  Pixels must be dense; rows and images may
        be padded.  ``out``: a CUDA array of the matching shape (rows and images may be padded too), default a new torch
        tensor.  ``interpolation``: as for __call__.  Each output pixel's map entry (or camera model) and, for INTER_CUBIC /
        INTER_LANCZOS4, its row of weights are read once for several frames of the batch.  Runs on
        ``stream`` (a raw CUDA stream handle), default torch's current stream, and only enqueues.  Returns ``out``.
        borderMode, borderValue: as remap() takes them; BORDER_TRANSPARENT writes into ``out`` in place."""
        self._live()
        border = _border(borderMode, borderValue, out)
        return _device_images(frames, self.w, self.h, out, self.ctx, "frames", lambda f, s, d: f(
            self.ctx.h, self.slot, *s, *d, _interp(interpolation)), stream, "bevk_undistort_stack_interp", border)

    def cuda_to_jpeg(self, frames, quality: int = 95, interpolation: int = INTER_LINEAR, params=None) -> list[bytes]:
        """cuda() followed by cv2.imencode('.jpg', img, [IMWRITE_JPEG_QUALITY, quality] + params) per frame, with the
        encoder on the GPU: the undistorted images stay in library scratch and only the JPEG streams come back.  frames:
        a uint8 CUDA array [H][W][3] or [N][H][W][3] (BGR) laid out as cuda() takes it.  params and interpolation as in jpeg().  Runs on
        torch's current stream and synchronises.  Returns one ``bytes`` per frame, byte-identical to cv2's."""
        self._live()
        ptr, rank, n, sh, sw, ch, simg, srow = _cuda_images(frames, "frames")
        if ch != 3 or rank == 2:
            raise L.BevkError("Undistorter.cuda_to_jpeg takes uint8[H][W][3] or uint8[N][H][W][3] BGR frames")
        out = np.empty(max(n, 1) * jpeg_encode_bound(self.w, self.h, params), np.uint8)   # pages are only touched where streams land
        sizes = (C.c_uint64 * max(n, 1))()
        jpeg_set_params(self.ctx, params)
        from .sharding import _torch_current_stream
        with self.ctx.on_stream(_torch_current_stream(self.ctx.device)):
            L.check(self.ctx.lib.bevk_undistort_stack_jpeg(self.ctx.h, self.slot, C.c_void_p(ptr), simg, sw, sh, srow, n,
                                                           _interp(interpolation), int(quality), L.vptr(out), out.size, sizes))
        return _split(out, sizes)

    def last_path(self) -> str:
        """Which gather the last call of this ctx launched: 'word' (k_gather4, 4 pixels per thread), 'byte' (k_gather) or
        'taps' (k_gather_taps, INTER_CUBIC / INTER_LANCZOS4)."""
        return last_path(self.ctx)


class BevEngine:
    """The fused surround-BEV engine (bevk_bev_* entry points)."""

    def __init__(self, n_cam: int, frame_size, bev_size, ctx: L.Context | None = None):
        self.ctx = ctx or L.Context(L.default_context().device)   # own ctx: the plan is per-ctx state
        self.n_cam = n_cam
        self.FW, self.FH = int(frame_size[0]), int(frame_size[1])
        self.BW, self.BH = int(bev_size[0]), int(bev_size[1])
        self._point_cams = {}   # cam -> (model, K, D, P, H, inv(H)): what camera_to_canvas / canvas_to_camera chain
        L.check(self.ctx.lib.bevk_bev_configure(self.ctx.h, n_cam, self.FW, self.FH, self.BW, self.BH))
        self.finalized = False

    def set_camera(self, cam: int, K, D, P, und_size, H, model: str = "fisheye"):
        """Camera `cam`'s LUT: cv2.warpPerspective by H of cv2's undistortion maps of (K, D, P) at und_size.  model
        "fisheye" (D: the first 4 coefficients) or "pinhole" (D: 0, 4, 5, 8, 12 or 14 coefficients, as cv2 takes them)."""
        dd = np.asarray(D, np.float64).reshape(-1)
        if model == "fisheye":
            d = np.zeros(4)
            d[:min(4, dd.size)] = dd[:4]
            L.check(self.ctx.lib.bevk_bev_set_camera(self.ctx.h, cam, L.dptr(K), L.dptr(d), L.dptr(P),
                                                     int(und_size[0]), int(und_size[1]), L.dptr(H)))
        elif model == "pinhole":
            L.check(self.ctx.lib.bevk_bev_set_camera_model(self.ctx.h, cam, L.MODEL_PINHOLE, L.dptr(K), L.dptr(dd), int(dd.size),
                                                           L.dptr(P), int(und_size[0]), int(und_size[1]), L.dptr(H)))
        else:
            raise L.BevkError(f'camera model must be "fisheye" or "pinhole", got {model!r}')
        Hd, Hi = np.array(H, np.float64).reshape(3, 3), np.empty((3, 3))
        L.check(self.ctx.lib.bevk_invert3(L.dptr(Hd), Hi.ctypes.data_as(L._dp)))
        self._point_cams[cam] = (model, np.array(K, np.float64), d if model == "fisheye" else dd, np.array(P, np.float64),
                                 Hd, Hi)
        self.finalized = False

    def _point_cam(self, cam):
        if cam not in self._point_cams:
            raise L.BevkError(f"camera {cam} is not set")
        return self._point_cams[cam]

    def camera_to_canvas(self, cam, pts):
        """Camera `cam`'s raw-frame pixels -> canvas pixels, as the chain cv2.perspectiveTransform(
        cv2.fisheye.undistortPoints(pts, K, D, P=P), H) (a pinhole: cv2.undistortPoints) of set_camera's K, D, P, H
        computes them, bit for bit.  pts: float32 [N][1][2] or [1][N][2] (a pinhole also takes float64 and [N][2]),
        NumPy or CUDA; the result has the chain's shape and dtype."""
        model, K, D, P, H, _ = self._point_cam(cam)
        und = (fisheye_undistort_points(pts, K, D, P=P, ctx=self.ctx) if model == "fisheye"
               else undistort_points(pts, K, D, P=P, ctx=self.ctx))
        return perspective_transform(und, H, ctx=self.ctx)

    def canvas_to_camera(self, cam, pts):
        """Canvas pixels -> camera `cam`'s raw-frame pixels, as the chain cv2.fisheye.distortPoints(cv2.undistortPoints(
        cv2.perspectiveTransform(pts, cv2.invert(H)[1]), P, None), K, D) computes them (a pinhole: cv2.projectPoints of
        (x, y, 1) with zero rvec and tvec), bit for bit.  pts: float32 [N][1][2] or [1][N][2] (a pinhole also takes
        float64), NumPy or CUDA; returns [N][1][2]."""
        model, K, D, P, _, Hi = self._point_cam(cam)
        xy = undistort_points(perspective_transform(pts, Hi, ctx=self.ctx), P, None, ctx=self.ctx)
        if model == "fisheye":
            return fisheye_distort_points(xy, K, D, ctx=self.ctx)
        if hasattr(xy, "__cuda_array_interface__"):
            import torch
            xyz = torch.cat([xy, torch.ones_like(xy[..., :1])], -1)
        else:
            xyz = np.concatenate([xy, np.ones_like(xy[..., :1])], -1)
        return project_points(xyz, np.zeros(3), np.zeros(3), K, D, ctx=self.ctx)[0]

    def set_maps(self, cam: int, map1, map2):
        m1 = np.ascontiguousarray(map1, np.int16)
        m2 = np.ascontiguousarray(map2, np.uint16)
        if m1.shape != (self.BH, self.BW, 2) or m2.shape != (self.BH, self.BW):
            raise L.BevkError("BEV maps must match the canvas size")
        L.check(self.ctx.lib.bevk_bev_set_maps(self.ctx.h, cam, L.vptr(m1), L.vptr(m2)))
        self.finalized = False

    def get_maps(self, cam: int):
        m1 = np.empty((self.BH, self.BW, 2), np.int16)
        m2 = np.empty((self.BH, self.BW), np.uint16)
        L.check(self.ctx.lib.bevk_bev_get_maps(self.ctx.h, cam, L.vptr(m1), L.vptr(m2)))
        return m1, m2

    def set_interpolation(self, interpolation: int):
        """INTER_LINEAR (the reference) or INTER_NEAREST for the raw2bev gather; before finalize()."""
        L.check(self.ctx.lib.bevk_bev_set_interpolation(self.ctx.h, _interp(interpolation)))
        self.finalized = False

    def set_mask(self, cam: int, mask: np.ndarray):
        m = np.ascontiguousarray(mask, np.uint8)
        if m.shape != (self.BH, self.BW):
            raise L.BevkError("mask must be uint8[bev_h][bev_w]")
        L.check(self.ctx.lib.bevk_bev_set_mask(self.ctx.h, cam, L.vptr(m)))
        self.finalized = False

    def blend_masks(self, polys: np.ndarray, lines: np.ndarray) -> np.ndarray:
        p = np.ascontiguousarray(polys, np.uint8)
        ln = np.ascontiguousarray(lines, np.int32).reshape(8, 4)
        out = np.empty_like(p)
        L.check(self.ctx.lib.bevk_blend_masks(self.ctx.h, L.vptr(p), L.vptr(ln), self.BW, self.BH, L.vptr(out)))
        return out

    def finalize(self):
        L.check(self.ctx.lib.bevk_bev_finalize(self.ctx.h))
        self.finalized = True

    def plan_info(self):
        a, b, c = C.c_int64(), C.c_int64(), C.c_int64()
        L.check(self.ctx.lib.bevk_bev_plan_info(self.ctx.h, C.byref(a), C.byref(b), C.byref(c)))
        return {"tiles": a.value, "items": b.value, "lut_bytes": c.value}

    def run(self, frame_sets, car: np.ndarray | None = None, balance: bool = False, out: np.ndarray | None = None,
            pixel_format: str = "bgr", out_format: str = "bgr"):
        """frame_sets: list (batch) of lists (n_cam) of uint8[FH][FW][3] arrays.  Returns
        uint8[batch][BH][BW][3].

        pixel_format "nv12" / "i420": every frame is a YUV 4:2:0 buffer uint8[FH*3//2][FW] in cv2's layout (rows may be
        padded); the canvases are those of cv2.cvtColor(frame, COLOR_YUV2BGR_NV12 / _I420) followed by the BGR call.
        The conversion runs on the GPU, and only the bytes the render samples (1.5 per pixel) cross PCIe.

        pixel_format "yuyv" / "uyvy": every frame is a packed YUV 4:2:2 frame uint8[FH][FW][2] as UVC / V4L2 and GMSL
        cameras deliver it (rows may be padded, pixels must be dense); the canvases are those of cv2.cvtColor(frame,
        COLOR_YUV2BGR_YUY2 / _UYVY) followed by the BGR call, with 2 bytes per sampled pixel crossing PCIe.

        out_format "nv12" / "i420": the canvases are returned as YUV 4:2:0, uint8[batch][BH*3//2][BW], each
        cv2.cvtColor(bgr_canvas, COLOR_BGR2YUV_I420) (NV12: its U and V planes interleaved); the conversion runs on the
        GPU, so 1.5 bytes per canvas pixel come back instead of 3."""
        if not self.finalized:
            self.finalize()
        fmt = self._pixel_format(pixel_format)
        ofmt = self._out_format(out_format)
        keep, ptrs, stride, batch = self._host_frames(frame_sets, "run()", fmt)
        shape = self._canvas_shape(batch, ofmt)
        if out is None:   # a fresh array per call, as the reference returns -- page-locked and recycled (PinnedPool)
            if getattr(self, "_pool", None) is None:
                self._pool = L.PinnedPool()
            out = self._pool.get(shape)
        else:
            out = _out(shape, out)
        car, carp = self._host_car(car)
        L.check(self.ctx.lib.bevk_bev_run(self.ctx.h, ptrs, stride, batch, carp,
                                          (L.FLAG_BALANCE if balance else 0) | fmt | ofmt, L.vptr(out)))
        return out

    def _out_format(self, out_format: str) -> int:
        """Flag bits of an out_format argument ("bgr", "nv12", "i420"); YUV 4:2:0 canvases need an even canvas size."""
        ofmt = L.OUT_FORMATS.get(str(out_format).lower())
        if ofmt is None:
            raise L.BevkError(f"out_format must be one of {sorted(L.OUT_FORMATS)}, got {out_format!r}")
        if ofmt and (self.BW % 2 or self.BH % 2):
            raise L.BevkError(f"{out_format} canvases need an even canvas size, this engine's is {self.BW} x {self.BH}")
        return ofmt

    def _canvas_shape(self, batch: int, ofmt: int):
        """Shape of `batch` canvases in the format of out-format flag bits ofmt."""
        return (batch, self.BH * 3 // 2, self.BW) if ofmt else (batch, self.BH, self.BW, 3)

    def _pixel_format(self, pixel_format: str) -> int:
        """Flag bits of a pixel_format argument ("bgr", "nv12", "i420", "yuyv", "uyvy"); YUV 4:2:0 needs an even frame
        size, packed 4:2:2 an even frame width."""
        fmt = L.PIXEL_FORMATS.get(str(pixel_format).lower())
        if fmt is None:
            raise L.BevkError(f"pixel_format must be one of {sorted(L.PIXEL_FORMATS)}, got {pixel_format!r}")
        if fmt in L.PACKED_FORMATS:
            if self.FW % 2:
                raise L.BevkError(f"{pixel_format} frames need an even frame width, this engine's is {self.FW}")
        elif fmt and (self.FW % 2 or self.FH % 2):
            raise L.BevkError(f"{pixel_format} frames need an even frame size, this engine's is {self.FW} x {self.FH}")
        return fmt

    def _yuv_shape(self, fmt: int):
        """Shape of one YUV frame of input flag fmt: uint8[FH*3//2][FW] (4:2:0) or uint8[FH][FW][2] (packed 4:2:2)."""
        return (self.FH, self.FW, 2) if fmt in L.PACKED_FORMATS else (self.FH * 3 // 2, self.FW)

    def _yuv_view(self, f, fmt: int):
        """A host YUV frame as bevk_bev_run reads it: _yuv_shape(fmt) with dense pixels (rows may be padded)."""
        shape = self._yuv_shape(fmt)
        if not isinstance(f, np.ndarray) or f.dtype != np.uint8 or f.shape != shape:
            got = f"{f.dtype} {f.shape}" if isinstance(f, np.ndarray) else type(f).__name__
            kind = "packed YUV 4:2:2" if fmt in L.PACKED_FORMATS else "YUV 4:2:0"
            name = next(k for k, v in L.PIXEL_FORMATS.items() if v == fmt)
            raise L.BevkError(f"{kind} frames (pixel_format {name!r}) must be uint8{list(shape)} arrays, got {got}")
        row = self.FW * (2 if fmt in L.PACKED_FORMATS else 1)
        if any(s != d for s, d in zip(f.strides[1:], np.empty(shape[1:], np.uint8).strides)) or f.strides[0] < row:
            f = np.ascontiguousarray(f)
        return f, f.strides[0]

    def _host_frames(self, frame_sets, what, fmt: int = 0):
        """(arrays to keep alive, host pointer table, row stride, batch) of host frame-sets laid out as run() takes them."""
        batch = len(frame_sets)
        if batch < 1:
            raise L.BevkError(f"{what} needs at least one frame-set")
        keep, ptrs, stride = [], (C.c_void_p * (batch * self.n_cam))(), None
        for b, fs in enumerate(frame_sets):
            if len(fs) != self.n_cam:
                raise L.BevkError(f"frame-set {b} has {len(fs)} frames, expected {self.n_cam}")
            for k, f in enumerate(fs):
                if fmt:
                    img, s = self._yuv_view(f, fmt)
                else:
                    f = self._conform(f)
                    img, w, h, s, ch = L.image_view(f)
                if stride is None:
                    stride = s
                elif s != stride:
                    img = np.ascontiguousarray(img)
                    if img.strides[0] != stride:
                        raise L.BevkError("all frames of a call must share one row stride")
                keep.append(img)
                ptrs[b * self.n_cam + k] = img.ctypes.data
        return keep, ptrs, stride, batch

    def _host_car(self, car):
        """(dense car array or None, its pointer or None)."""
        if car is None:
            return None, None
        car = np.ascontiguousarray(car, np.uint8)
        if car.shape != (self.BH, self.BW, 3):
            raise L.BevkError("car must be uint8[bev_h][bev_w][3]")
        return car, L.vptr(car)

    def _streams(self, batch, params=None):
        """Host buffer for `batch` JPEG streams of a canvas under params (pages are only touched where streams land) and
        sizes[batch]; params are set on the context for the encoding call that follows."""
        out = np.empty(batch * jpeg_encode_bound(self.BW, self.BH, params), np.uint8)
        jpeg_set_params(self.ctx, params)
        return out, (C.c_uint64 * batch)()

    def run_to_jpeg(self, frame_sets, quality: int = 95, car: np.ndarray | None = None, balance: bool = False,
                    params=None) -> list[bytes]:
        """run() followed by cv2.imencode('.jpg', canvas, [IMWRITE_JPEG_QUALITY, quality] + params) per frame-set, with
        the encoder on the GPU: only the JPEG streams come back over PCIe.  frame_sets as in run(); params as in
        ops.jpeg_encode.  Returns one ``bytes`` per frame-set, byte-identical to cv2's."""
        if not self.finalized:
            self.finalize()
        keep, ptrs, stride, batch = self._host_frames(frame_sets, "run_to_jpeg()")
        car, carp = self._host_car(car)
        out, sizes = self._streams(batch, params)
        L.check(self.ctx.lib.bevk_bev_run_to_jpeg(self.ctx.h, ptrs, stride, batch, carp, L.FLAG_BALANCE if balance else 0,
                                                  int(quality), L.vptr(out), out.size, sizes))
        return _split(out, sizes)

    def run_jpeg(self, jpeg_sets, car: np.ndarray | None = None, balance: bool = False, out: np.ndarray | None = None):
        """jpeg_sets: list (batch) of lists (n_cam) of JPEG byte strings (the files cv2.imread would open).  The streams
        are decoded on the GPU (nvJPEG) straight into the frame stack the fused kernel reads: only compressed bytes cross
        PCIe on the way in.  Pixels are nvJPEG's decode (not libjpeg-turbo's); the BEV path on them is bit-exact."""
        if not self.finalized:
            self.finalize()
        batch = len(jpeg_sets)
        if batch < 1:
            raise L.BevkError("run_jpeg() needs at least one frame-set")
        flat = []
        for b, fs in enumerate(jpeg_sets):
            if len(fs) != self.n_cam:
                raise L.BevkError(f"frame-set {b} has {len(fs)} streams, expected {self.n_cam}")
            flat += [bytes(x) if not isinstance(x, (bytes, bytearray)) else x for x in fs]
        keep = [(C.c_char * len(x)).from_buffer_copy(x) if isinstance(x, bytes) else (C.c_char * len(x)).from_buffer(x) for x in flat]
        ptrs = (C.c_void_p * len(flat))(*[C.addressof(k) for k in keep])
        sizes = (C.c_uint64 * len(flat))(*[len(x) for x in flat])
        if out is None:
            if getattr(self, "_pool", None) is None:
                self._pool = L.PinnedPool()
            out = self._pool.get((batch, self.BH, self.BW, 3))
        else:
            out = _out((batch, self.BH, self.BW, 3), out)
        carp = None
        if car is not None:
            car = np.ascontiguousarray(car, np.uint8)
            if car.shape != (self.BH, self.BW, 3):
                raise L.BevkError("car must be uint8[bev_h][bev_w][3]")
            carp = L.vptr(car)
        L.check(self.ctx.lib.bevk_bev_run_jpeg(self.ctx.h, ptrs, sizes, batch, carp, L.FLAG_BALANCE if balance else 0, L.vptr(out)))
        return out

    def host_copy_bytes(self, balance: bool = False, pixel_format: str = "bgr", out_format: str = "bgr"):
        """(host->device, device->host) bytes per frame-set that run() moves over PCIe (pageable frames)."""
        if not self.finalized:
            self.finalize()
        flags = (L.FLAG_BALANCE if balance else 0) | self._pixel_format(pixel_format) | self._out_format(out_format)
        a, b = C.c_int64(), C.c_int64()
        L.check(self.ctx.lib.bevk_bev_host_copy_bytes(self.ctx.h, flags, C.byref(a), C.byref(b)))
        return a.value, b.value

    def last_h2d_bytes(self) -> int:
        """Host->device bytes moved by the last run() call."""
        return int(self.ctx.lib.bevk_bev_last_h2d_bytes(self.ctx.h))

    def _conform(self, f: np.ndarray) -> np.ndarray:
        """The reference never validates frame sizes (cv2.remap samples whatever it is given, zero outside).  The engine's
        LUT is compiled for FW x FH: a SMALLER frame is embedded into an FW x FH zero canvas, which samples identically
        (cv2's BORDER_CONSTANT 0).  A LARGER frame is cropped, which differs from the reference wherever the LUT points
        beyond FW x FH (the reference would sample the extra pixels there, this engine reads zeros)."""
        if f.ndim != 3 or f.shape[2] != 3 or f.dtype != np.uint8:
            raise L.BevkError("frames must be uint8[h][w][3] (BGR)")
        if f.shape[0] == self.FH and f.shape[1] == self.FW:
            return f
        g = np.zeros((self.FH, self.FW, 3), np.uint8)
        h, w = min(self.FH, f.shape[0]), min(self.FW, f.shape[1])
        g[:h, :w] = f[:h, :w]
        return g

    # device-resident entry points (raw device pointers, e.g. torch tensors' data_ptr())
    def run_device(self, d_srcs_ptr: int, batch: int, d_out_ptr: int, d_car_ptr: int = 0, balance: bool = False,
                   out_format: str = "bgr"):
        """out_format "nv12" / "i420": d_out_ptr receives uint8[batch][BH*3//2][BW] YUV 4:2:0 canvases (see run())."""
        if not self.finalized:
            self.finalize()
        flags = (L.FLAG_BALANCE if balance else 0) | self._out_format(out_format)
        L.check(self.ctx.lib.bevk_bev_run_device(self.ctx.h, C.c_void_p(d_srcs_ptr), batch, C.c_void_p(d_car_ptr or None),
                                                 flags, C.c_void_p(d_out_ptr)))

    def run_stack(self, d_frames_ptr: int, frame_stride: int, batch: int, d_out_ptr: int, d_car_ptr: int = 0, balance: bool = False,
                  pixel_format: str = "bgr", out_format: str = "bgr"):
        """Frame stack on the device (frame i at d_frames_ptr + i * frame_stride, i = set * n_cam + camera): the
        TMA-staged kernel when base and stride are 16-byte aligned.  Only enqueues on the ctx stream.  pixel_format
        "nv12" / "i420": dense uint8[FH*3//2][FW] YUV 4:2:0 frames at any base and stride; "yuyv" / "uyvy": dense
        uint8[FH][FW][2] packed 4:2:2 frames at any base and stride (see run()).  out_format "nv12" / "i420":
        d_out_ptr receives uint8[batch][BH*3//2][BW] YUV 4:2:0 canvases (see run())."""
        if not self.finalized:
            self.finalize()
        flags = (L.FLAG_BALANCE if balance else 0) | self._pixel_format(pixel_format) | self._out_format(out_format)
        L.check(self.ctx.lib.bevk_bev_run_stack(self.ctx.h, C.c_void_p(d_frames_ptr), int(frame_stride), batch,
                                                C.c_void_p(d_car_ptr or None), flags, C.c_void_p(d_out_ptr)))

    def run_stack_cams(self, d_frames_ptr: int, frame_stride: int, batch: int, cam_lo: int, cam_hi: int, d_out_ptr: int):
        if not self.finalized:
            self.finalize()
        L.check(self.ctx.lib.bevk_bev_run_stack_cams(self.ctx.h, C.c_void_p(d_frames_ptr), int(frame_stride), batch, cam_lo,
                                                     cam_hi, C.c_void_p(d_out_ptr)))

    def last_path(self) -> str:
        """Which fused kernel the last call launched: 'tma' (k_bev_tma) or 'gather' (k_bev)."""
        return {1: "gather", 2: "tma"}.get(int(self.ctx.lib.bevk_bev_last_path(self.ctx.h)), "none")

    def tma_plan_info(self):
        v = [C.c_int64() for _ in range(5)]
        L.check(self.ctx.lib.bevk_bev_tma_plan_info(self.ctx.h, *[C.byref(x) for x in v]))
        return dict(zip(("items", "shapes", "box_bytes", "tma_entries", "gather_entries"), (x.value for x in v)))

    def run_cuda(self, frames, car=None, balance: bool = False, out=None, stream: int | None = None,
                 pixel_format: str = "bgr", out_format: str = "bgr"):
        """Frames that already live on the GPU (decoder output, torch / CuPy arrays): no PCIe in the call.

        frames: one uint8 CUDA array [batch][n_cam][FH][FW][3], or a list (batch) of lists (n_cam) of uint8
        CUDA arrays [FH][FW][3] -- anything exposing ``__cuda_array_interface__``, C-contiguous, on this
        engine's device.  car / out likewise ([BH][BW][3] / [batch][BH][BW][3]); without ``out`` a torch
        tensor is allocated.  ``stream``: raw CUDA stream handle the work is enqueued on for THIS call; default torch's
        current stream on the engine's device (so that torch kernels that produced ``frames``, this render and whatever
        consumes ``out`` are ordered), or the ctx's own stream when torch is not in use.  The ctx goes back to its previous
        stream afterwards.  The call does not synchronise.  Returns ``out``.

        pixel_format "nv12" / "i420": frames is one C-contiguous uint8 CUDA array [batch][n_cam][FH*3//2][FW] of YUV
        4:2:0 frames in cv2's layout (e.g. NVDEC NV12 surfaces); the result is that of cv2.cvtColor to BGR followed by
        the BGR call, with the conversion done on the GPU.  pixel_format "yuyv" / "uyvy": one C-contiguous uint8 CUDA
        array [batch][n_cam][FH][FW][2] of packed 4:2:2 frames; the result is that of cv2.cvtColor(COLOR_YUV2BGR_YUY2 /
        _UYVY) followed by the BGR call.

        out_format "nv12" / "i420": ``out`` is uint8[batch][BH*3//2][BW], YUV 4:2:0 canvases as run() describes them
        (e.g. for a hardware video encoder's NV12 input)."""
        if not self.finalized:
            self.finalize()
        fmt = self._pixel_format(pixel_format)
        ofmt = self._out_format(out_format)
        if fmt:
            return self._run_cuda_yuv(frames, car, balance, out, stream, fmt, pixel_format, ofmt)
        ptrs = self._cuda_frames(frames)
        batch = len(ptrs) // self.n_cam
        out, d_out = self._cuda_out(out, batch, ofmt)
        d_car = _cuda_ptr(car, (self.BH, self.BW, 3))[0] if car is not None else None
        if stream is None:
            from .sharding import _torch_current_stream
            stream = _torch_current_stream(self.ctx.device)
        table = (C.c_void_p * len(ptrs))(*ptrs)
        with self.ctx.on_stream(stream):
            L.check(self.ctx.lib.bevk_bev_run_frames(self.ctx.h, table, batch, C.c_void_p(d_car),
                                                     (L.FLAG_BALANCE if balance else 0) | ofmt, C.c_void_p(d_out)))
        return out

    def _cuda_out(self, out, batch, ofmt):
        """(out, its device pointer) for `batch` canvases in the format of ofmt: a new torch tensor when out is None."""
        shape = self._canvas_shape(batch, ofmt)
        if out is None:
            import torch
            out = torch.empty(shape, dtype=torch.uint8, device=torch.device("cuda", self.ctx.device))
        return out, _cuda_ptr(out, shape)[0]

    def _run_cuda_yuv(self, frames, car, balance, out, stream, fmt, name, ofmt=0):
        """run_cuda() on a YUV frame stack: bevk_bev_run_stack with a YUV flag."""
        want = (self.n_cam,) + self._yuv_shape(fmt)
        dims = "".join(f"[{n}]" for n in want)
        if not hasattr(frames, "__cuda_array_interface__"):
            raise L.BevkError(f"{name} frames must be one uint8 CUDA array [batch]{dims}")
        base, shape = _cuda_ptr(frames, None)
        if len(shape) != len(want) + 1 or tuple(shape[1:]) != want or shape[0] < 1:
            raise L.BevkError(f"{name} frames must be uint8[batch]{dims}, got {tuple(shape)}")
        batch = shape[0]
        frame_bytes = int(np.prod(want[1:]))
        out, d_out = self._cuda_out(out, batch, ofmt)
        d_car = _cuda_ptr(car, (self.BH, self.BW, 3))[0] if car is not None else None
        if stream is None:
            from .sharding import _torch_current_stream
            stream = _torch_current_stream(self.ctx.device)
        with self.ctx.on_stream(stream):
            L.check(self.ctx.lib.bevk_bev_run_stack(self.ctx.h, C.c_void_p(base), frame_bytes, batch,
                                                    C.c_void_p(d_car), (L.FLAG_BALANCE if balance else 0) | fmt | ofmt,
                                                    C.c_void_p(d_out)))
        return out

    def run_cuda_planes(self, y, c=None, v=None, pixel_format: str = "nv12", car=None, balance: bool = False, out=None,
                        stream: int | None = None, out_format: str = "bgr"):
        """run_cuda() on YUV 4:2:0 frames given plane by plane, as video decoders leave them on the GPU (NVDEC /
        DeepStream surfaces, FFmpeg CUDA frames' data[] and linesize[]): no repack into cv2's single buffer.

        y: uint8 CUDA array [batch][n_cam][FH][FW]; c: [batch][n_cam][FH/2][FW] of interleaved U,V (pixel_format
        "nv12") or [batch][n_cam][FH/2][FW/2] of U ("i420"); v: the V plane like c ("i420" only).  Strided views are
        fine (e.g. slices of one decoder pool): rows may be padded to any pitch, pixels within a row must be dense, and
        each plane has one row pitch for all frames.  Or y is a list (batch) of lists (n_cam) of per-frame plane tuples
        (y, c) / (y, u, v) of 2-D CUDA arrays [rows][cols].  When every plane of every frame lies at one common frame
        stride (a surface pool) the call goes through bevk_bev_run_yuv_planes, otherwise through the plane table of
        bevk_bev_run_yuv_surfaces.  car, balance, out, stream and out_format as in run_cuda(); the result is that of
        run_cuda() on the same frames in cv2's single-buffer layout.  Returns ``out``.

        pixel_format "yuyv" / "uyvy": y is the one packed plane, a strided uint8 CUDA array [batch][n_cam][FH][FW][2]
        (rows padded to any pitch, pixels dense) or a list of lists of per-frame 1-tuples (y,) of [FH][FW][2] arrays; c
        and v must be None.  The result is that of run_cuda() on the same frames packed densely."""
        if not self.finalized:
            self.finalize()
        fmt = self._pixel_format(pixel_format)
        ofmt = self._out_format(out_format)
        if not fmt:
            raise L.BevkError(f"run_cuda_planes takes nv12, i420, yuyv or uyvy frames, not {pixel_format!r}")
        planes, pitch = self._yuv_planes(y, c, v, fmt, pixel_format)
        n = len(planes[0])
        batch = n // self.n_cam
        out, d_out = self._cuda_out(out, batch, ofmt)
        d_car = _cuda_ptr(car, (self.BH, self.BW, 3))[0] if car is not None else None
        if stream is None:
            from .sharding import _torch_current_stream
            stream = _torch_current_stream(self.ctx.device)
        flags = (L.FLAG_BALANCE if balance else 0) | fmt | ofmt
        pitches = (C.c_int64 * 3)(*(pitch + [pitch[-1]] * (3 - len(pitch))))
        strides = {p[i] - p[i - 1] for p in planes for i in range(1, n)}
        with self.ctx.on_stream(stream):
            if len(strides) <= 1:   # a surface pool: plane p of frame i at planes[0][0] + i * stride + offset[p]
                stride = strides.pop() if strides else 0
                offs = [p[0] - planes[0][0] for p in planes]
                offsets = (C.c_int64 * 3)(*(offs + [offs[-1]] * (3 - len(offs))))
                L.check(self.ctx.lib.bevk_bev_run_yuv_planes(self.ctx.h, C.c_void_p(planes[0][0]), stride, offsets, pitches,
                                                             batch, C.c_void_p(d_car), flags, C.c_void_p(d_out)))
            else:
                table = (C.c_void_p * (3 * n))()
                for i in range(n):
                    for k, p in enumerate(planes):
                        table[3 * i + k] = p[i]
                L.check(self.ctx.lib.bevk_bev_run_yuv_surfaces(self.ctx.h, table, pitches, batch, C.c_void_p(d_car), flags,
                                                               C.c_void_p(d_out)))
        return out

    def _yuv_planes(self, y, c, v, fmt, name):
        """([per plane: device address of the plane of every frame, frame-set major], [row pitch per plane]) of the
        frames run_cuda_planes takes."""
        FW, FH, nc = self.FW, self.FH, self.n_cam
        packed = fmt in L.PACKED_FORMATS
        if packed:
            shapes, what = [(FH, FW, 2)], ("packed",)
        elif fmt == L.FLAG_NV12:
            shapes, what = [(FH, FW), (FH // 2, FW)], ("y", "uv")
        else:
            shapes, what = [(FH, FW), (FH // 2, FW // 2), (FH // 2, FW // 2)], ("y", "u", "v")

        def plane(a, shape, k):
            ptr, strides = _cuda_plane(a, shape, f"{name} plane {what[k]}")
            if packed and strides[-1] != 2:
                raise L.BevkError(f"{name} plane {what[k]}: the pixels of a row must be dense (2 bytes apart)")
            return ptr, strides

        if isinstance(y, (list, tuple)):
            if c is not None or v is not None:
                raise L.BevkError("with per-frame plane tuples, pass the list alone")
            frames = []
            for b, fs in enumerate(y):
                if len(fs) != nc:
                    raise L.BevkError(f"frame-set {b} has {len(fs)} frames, expected {nc}")
                frames += list(fs)
            if not frames:
                raise L.BevkError("batch must be >= 1")
            planes, pitch = [[] for _ in shapes], [None] * len(shapes)
            for i, f in enumerate(frames):
                if len(f) != len(shapes):
                    raise L.BevkError(f"{name} frames are {len(shapes)} planes {what}, frame {i} has {len(f)}")
                for k, a in enumerate(f):
                    ptr, strides = plane(a, shapes[k], k)
                    if pitch[k] is None:
                        pitch[k] = strides[0]
                    elif strides[0] != pitch[k]:
                        raise L.BevkError(f"every {what[k]} plane of a call must share one row pitch")
                    planes[k].append(ptr)
            return planes, pitch
        if packed:
            if c is not None or v is not None:
                raise L.BevkError(f"{name} frames are one packed plane: pass y alone (c and v must be None)")
            arrs = [y]
        else:
            arrs = [y, c] if fmt == L.FLAG_NV12 else [y, c, v]
        if any(a is None for a in arrs) or (fmt == L.FLAG_NV12 and v is not None):
            raise L.BevkError(f"{name} frames need the planes {', '.join(what)}")
        planes, pitch, batch = [], [], None
        for k, a in enumerate(arrs):
            iface = getattr(a, "__cuda_array_interface__", None)
            shape = tuple(iface["shape"]) if iface else ()
            if (len(shape) != 2 + len(shapes[k]) or shape[1:] != (nc,) + shapes[k] or shape[0] < 1 or
                    (batch is not None and shape[0] != batch)):
                raise L.BevkError(f"{name} plane {what[k]} must be a uint8 CUDA array [batch][{nc}]"
                                  f"{''.join(f'[{n}]' for n in shapes[k])}, got {shape}")
            batch = shape[0]
            ptr, strides = plane(a, shape, k)
            planes.append([ptr + b * strides[0] + j * strides[1] for b in range(batch) for j in range(nc)])
            pitch.append(strides[2])
        return planes, pitch

    def cuda_to_jpeg(self, frames, quality: int = 95, car=None, balance: bool = False, params=None) -> list[bytes]:
        """run_cuda() followed by cv2.imencode('.jpg', canvas, [IMWRITE_JPEG_QUALITY, quality] + params) per frame-set:
        frames (and car) as run_cuda takes them; params as in ops.jpeg_encode.  The canvases stay in library scratch on
        the GPU and only the JPEG streams come back.  Runs on torch's current stream and synchronises.  Returns one
        ``bytes`` per frame-set."""
        if not self.finalized:
            self.finalize()
        ptrs = self._cuda_frames(frames)
        batch = len(ptrs) // self.n_cam
        d_car = _cuda_ptr(car, (self.BH, self.BW, 3))[0] if car is not None else None
        out, sizes = self._streams(batch, params)
        from .sharding import _torch_current_stream
        table = (C.c_void_p * len(ptrs))(*ptrs)
        with self.ctx.on_stream(_torch_current_stream(self.ctx.device)):
            L.check(self.ctx.lib.bevk_bev_frames_to_jpeg(self.ctx.h, table, batch, C.c_void_p(d_car),
                                                         L.FLAG_BALANCE if balance else 0, int(quality), L.vptr(out),
                                                         out.size, sizes))
        return _split(out, sizes)

    def _cuda_frames(self, frames):
        """Device pointers (frame-set major) of the frames run_cuda takes."""
        frame_shape = (self.FH, self.FW, 3)
        if hasattr(frames, "__cuda_array_interface__"):
            base, shape = _cuda_ptr(frames, None)
            if len(shape) != 5 or tuple(shape[1:]) != (self.n_cam,) + frame_shape:
                raise L.BevkError(f"frames must be uint8[batch][{self.n_cam}][{self.FH}][{self.FW}][3], got {tuple(shape)}")
            batch, fb = shape[0], self.FH * self.FW * 3
            ptrs = [base + i * fb for i in range(batch * self.n_cam)]
        else:
            batch, ptrs = len(frames), []
            for b, fs in enumerate(frames):
                if len(fs) != self.n_cam:
                    raise L.BevkError(f"frame-set {b} has {len(fs)} frames, expected {self.n_cam}")
                ptrs += [_cuda_ptr(f, frame_shape)[0] for f in fs]
        if batch < 1:
            raise L.BevkError("batch must be >= 1")
        return ptrs

    def run_device_cams(self, d_srcs_ptr: int, batch: int, cam_lo: int, cam_hi: int, d_out_ptr: int):
        if not self.finalized:
            self.finalize()
        L.check(self.ctx.lib.bevk_bev_run_device_cams(self.ctx.h, C.c_void_p(d_srcs_ptr), batch, cam_lo, cam_hi,
                                                      C.c_void_p(d_out_ptr)))

    def sat_sum_device(self, part_ptrs, nbytes: int, d_out_ptr: int, d_car_ptr: int = 0):
        arr = (C.c_void_p * len(part_ptrs))(*part_ptrs)
        L.check(self.ctx.lib.bevk_sat_sum_device(self.ctx.h, arr, len(part_ptrs), nbytes, C.c_void_p(d_car_ptr or None),
                                                 C.c_void_p(d_out_ptr)))

    def last_kernel_ms(self) -> float:
        ms = C.c_float()
        L.check(self.ctx.lib.bevk_last_kernel_ms(self.ctx.h, C.byref(ms)))
        return ms.value
