"""Packed YUV 4:2:2 test inputs uint8[H][W][2] (cv2's input of COLOR_YUV2BGR_YUY2 / _UYVY), shared by
tests/test_host_yuv422.py and tests/test_gpu_yuv422.py.  Each row holds pixel pairs of 4 bytes, YUYV: Y0 U0 Y1 V0,
UYVY: U0 Y0 V0 Y1; the expected BGR is what cv2.cvtColor makes of them."""
import cv2
import numpy as np

FORMATS = ("yuyv", "uyvy")
TO_BGR = {"yuyv": cv2.COLOR_YUV2BGR_YUY2, "uyvy": cv2.COLOR_YUV2BGR_UYVY}
FMT_CODE = {"yuyv": 3, "uyvy": 4}   # YUV_YUYV, YUV_UYVY of bevk_kernels.cuh


def pack(y: np.ndarray, u: np.ndarray, v: np.ndarray, fmt: str) -> np.ndarray:
    """uint8[H][W][2] from Y [H][W] and U, V [H][W/2] (one sample per pixel pair)."""
    h, w = y.shape
    out = np.empty((h, w, 2), np.uint8)
    yc, cc = (0, 1) if fmt == "yuyv" else (1, 0)
    out[..., yc] = y
    out[:, 0::2, cc] = u
    out[:, 1::2, cc] = v
    return out


def to_bgr(f: np.ndarray, fmt: str) -> np.ndarray:
    return cv2.cvtColor(f, TO_BGR[fmt])


def swap(f: np.ndarray) -> np.ndarray:
    """The same pixels in the other byte order (YUYV <-> UYVY)."""
    return np.ascontiguousarray(f[..., ::-1])


def from_bgr(img: np.ndarray, fmt: str) -> np.ndarray:
    """A camera-like 4:2:2 frame from a BGR frame: cv2's BGR -> YCrCb per pixel, chroma averaged over each pixel pair."""
    ycc = cv2.cvtColor(img, cv2.COLOR_BGR2YCrCb).astype(np.int32)
    cr = (ycc[:, 0::2, 1] + ycc[:, 1::2, 1] + 1) >> 1
    cb = (ycc[:, 0::2, 2] + ycc[:, 1::2, 2] + 1) >> 1
    return pack(ycc[..., 0].astype(np.uint8), cb.astype(np.uint8), cr.astype(np.uint8), fmt)


def random_frame(rng, w: int, h: int) -> np.ndarray:
    return rng.integers(0, 256, (h, w, 2), dtype=np.uint8)


def every_triple(fmt: str) -> np.ndarray:
    """A 4096 x 4096 frame whose pixels take every (Y, U, V) triple once: pixel pair p carries U = (p >> 7) & 255,
    V = p >> 15 and the Y values 2 (p & 127) + {0, 1}."""
    W = H = 4096
    p = np.arange(W * H // 2, dtype=np.uint32).reshape(H, W // 2)
    u, v, j = ((p >> 7) & 255).astype(np.uint8), (p >> 15).astype(np.uint8), (p & 127).astype(np.uint8)
    y = np.empty((H, W), np.uint8)
    y[:, 0::2], y[:, 1::2] = 2 * j, 2 * j + 1
    return pack(y, u, v, fmt)
