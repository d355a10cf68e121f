"""YUV 4:2:0 test inputs in cv2's single-buffer layout (uint8[H*3/2][W]), shared by tests/test_host_yuv.py and
tests/test_gpu_yuv.py: camera-like frames are BGR frames converted with cv2.cvtColor(COLOR_BGR2YUV_I420), NV12 is the
same data with the U and V planes interleaved, and the expected BGR is what cv2.cvtColor makes of either."""
import cv2
import numpy as np

FORMATS = ("nv12", "i420")
TO_BGR = {"nv12": cv2.COLOR_YUV2BGR_NV12, "i420": cv2.COLOR_YUV2BGR_I420}
FMT_CODE = {"nv12": 1, "i420": 2}


def i420_to_nv12(buf: np.ndarray) -> np.ndarray:
    h2, w = buf.shape
    h = h2 * 2 // 3
    flat = buf.reshape(-1)
    n = (w // 2) * (h // 2)
    u = flat[w * h:w * h + n]
    v = flat[w * h + n:w * h + 2 * n]
    out = np.empty_like(buf)
    out[:h] = buf[:h]
    uv = out[h:].reshape(-1)
    uv[0::2], uv[1::2] = u, v
    return out


def from_bgr(img: np.ndarray, fmt: str) -> np.ndarray:
    """A BGR frame as a YUV 4:2:0 buffer of format fmt."""
    i420 = cv2.cvtColor(img, cv2.COLOR_BGR2YUV_I420)
    return i420 if fmt == "i420" else i420_to_nv12(i420)


def to_bgr(buf: np.ndarray, fmt: str) -> np.ndarray:
    return cv2.cvtColor(buf, TO_BGR[fmt])


def random_yuv(rng, w: int, h: int) -> np.ndarray:
    return rng.integers(0, 256, (h * 3 // 2, w), dtype=np.uint8)


def every_triple(fmt: str) -> np.ndarray:
    """A 4096 x 4096 frame whose pixels take every (Y, U, V) triple once: chroma sample s carries U = s & 255,
    V = (s >> 8) & 255, and its 2 x 2 luma block the four Y values 4 (s >> 16) + {0, 1, 2, 3}."""
    W = H = 4096
    s = np.arange((W // 2) * (H // 2), dtype=np.uint32).reshape(H // 2, W // 2)
    u, v, j = (s & 255).astype(np.uint8), ((s >> 8) & 255).astype(np.uint8), (s >> 16).astype(np.uint8)
    y = np.empty((H, W), np.uint8)
    for a in range(2):
        for b in range(2):
            y[a::2, b::2] = 4 * j + 2 * a + b
    i420 = np.concatenate([y.reshape(-1), u.reshape(-1), v.reshape(-1)]).reshape(H * 3 // 2, W)
    return i420 if fmt == "i420" else i420_to_nv12(i420)
