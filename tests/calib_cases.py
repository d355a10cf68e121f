"""Seeded random calibrations for the camera-model and homography arithmetic of the kernels (undistort_point,
quantise_uv, warp_point, warp_maps_pixel), shared by tests/test_host_calib_fuzz.py (the host build of that code) and
tests/test_gpu_calib_fuzz.py (the kernels).  One seed gives one case: a camera (fisheye, or pinhole with k1 k2 p1 p2 k3),
its K, D, FOCAL_SCALE, SIZE_SCALE and principal-point offsets (P through dst_camera_matrix), the undistorted size, a
canvas size and a homography H from the undistorted frame to the canvas.

The oracle is cv2 alone: cv2.fisheye.initUndistortRectifyMap / cv2.initUndistortRectifyMap for the maps,
cv2.warpPerspective of the map planes for the BEV LUT (Camera.get_bev_maps), cv2.remap / cv2.warpPerspective for
images, oracle.cv2_path.RefBev for whole canvases.  Oracle results are cached per case."""
from __future__ import annotations

import zlib
from dataclasses import dataclass
from functools import lru_cache

import cv2
import numpy as np

from oracle import cv2_path as C

# undistorted sizes of the mild fisheye cameras at real resolutions (SIZE_SCALE 1)
_REAL_SIZES = ((3840, 2160), (2560, 2048), (1920, 1080), (1280, 1024))
# widths of the strong-distortion cameras, by W % 8: cv2.initUndistortRectifyMap's 8-column vector body (saturating
# pack) ends at W - W % 8; W % 8 == 0 has no scalar tail, 1 a one-column tail, 7 the longest
_W_MOD8 = (0, 1, 7, 0, 1, 7, 3, 5)


@dataclass(eq=False)
class CalibCase:
    name: str
    kind: str            # "mild" (real sizes, |D| <= 0.1), "scaled" (SIZE_SCALE 1.5 / 2), "strong" (wide view, large D)
    model: int           # 0 fisheye, 1 pinhole
    K: np.ndarray
    D: np.ndarray        # 4 (fisheye) or 5 (pinhole) coefficients
    FS: float
    SS: float
    FW: int              # frame size K belongs to
    FH: int
    P: np.ndarray        # dst_camera_matrix(K, FW, FH, FS, SS, off_h, off_v)
    UW: int              # undistorted size (FW * SS, FH * SS)
    UH: int
    H: np.ndarray        # homography: undistorted frame -> canvas
    BW: int
    BH: int
    horizon: str         # "none", "inside" (W <= 0 on part of the canvas) or "zero" (W == 0 exactly at some pixels)

    @property
    def fisheye(self) -> bool:
        return self.model == 0

    @property
    def d5(self) -> np.ndarray:
        d = np.zeros(5)
        d[:self.D.size] = self.D.ravel()
        return d


def _K(rng, W, H, lo, hi, dc):
    return np.array([[rng.uniform(lo, hi) * W, 0, W / 2 + rng.uniform(-dc, dc)],
                     [0, rng.uniform(lo, hi) * W, H / 2 + rng.uniform(-dc, dc)], [0, 0, 1.0]])


def _homography(rng, UW, UH, BW, BH, horizon):
    """A canvas -> undistorted-frame map with strong perspective (inverted: H takes the undistorted frame to the canvas).
    Its pre-images run past the undistorted frame; with horizon "inside" the line W = 0 crosses the canvas."""
    p = rng.normal(0, 6e-4, 2)
    if horizon == "inside":
        p[0] = -rng.uniform(1.2, 3) / BW       # W = p0 x + p1 y + 1 falls below 0 inside the canvas
    Hinv = np.array([[rng.uniform(0.5, 4), rng.normal(0, 0.5), rng.uniform(0, UW / 2)],
                     [rng.normal(0, 0.5), rng.uniform(0.5, 4), rng.uniform(0, UH / 2)],
                     [p[0], p[1], 1.0]])
    H = np.linalg.inv(Hinv)
    return H / H[2, 2]


# exact inverse (powers of two): inv(H) = [[2,0,0],[0,2,0],[2^-6, 2^-8, -1]], so W = x/64 + y/256 - 1 is exactly 0 on the
# integer points of a line through the canvas, and negative before it
_H_ZERO = np.array([[0.5, 0, 0], [0, 0.5, 0], [2.0 ** -7, 2.0 ** -9, -1.0]])


def _canvas(rng, i):
    """Canvas widths that are not multiples of 64 (warp_point's 64-pixel blocks), some below 64, one exact multiple."""
    BW = (37, 130, 200, 257, 64 * 3, 333, 96, 401)[i % 8]
    BH = int(rng.integers(30, 260))
    return BW, BH


def _case(name, kind, model, K, D, FS, SS, FW, FH, off, rng, i):
    P = C.dst_camera_matrix(K, FW, FH, FS, SS, *off)
    UW, UH = int(FW * SS), int(FH * SS)
    BW, BH = _canvas(rng, i)
    horizon = ("none", "inside", "none", "zero")[i % 4] if kind != "mild" else ("none", "inside")[i % 2]
    H = _H_ZERO.copy() if horizon == "zero" else _homography(rng, UW, UH, BW, BH, horizon)
    return CalibCase(name, kind, model, K, np.asarray(D, np.float64).ravel(), float(FS), float(SS), FW, FH, P, UW, UH, H, BW, BH,
                     horizon)


@lru_cache(maxsize=None)
def corpus() -> tuple:
    out = []
    # mild fisheye cameras at real sizes, |D| <= 0.1 (the first twelve draw exactly as the probe that found the cvRound
    # ties of the row sums: seed 0, 2560x2048 camera 5)
    rng = np.random.default_rng(0)
    for t in range(12):
        W, H = _REAL_SIZES[t % 4]
        K = _K(rng, W, H, 0.2, 0.8, 30)
        D = rng.uniform(-0.1, 0.1, (4, 1))
        FS = rng.uniform(0.3, 1.2)
        out.append(_case(f"mild{t}", "mild", 0, K, D, FS, 1, W, H, (0.0, 0.0), np.random.default_rng(100 + t), t))
    # SIZE_SCALE 2 and 1.5 with principal-point offsets: the Camera / InCalibrator geometries; both models
    rng = np.random.default_rng(1)
    for t, (FW, FH, SS, model) in enumerate(((1280, 1024, 2, 0), (1920, 1080, 1.5, 0), (1280, 1024, 2, 1), (1000, 750, 1.5, 1),
                                             (640, 512, 2, 0), (333, 250, 1.5, 1))):
        K = _K(rng, FW, FH, 0.25, 0.8, 20)
        D = rng.uniform(-0.1, 0.1, 4) if model == 0 else np.array([rng.uniform(-0.3, 0.1), rng.uniform(-0.05, 0.1),
                                                                     rng.uniform(-1e-3, 1e-3), rng.uniform(-1e-3, 1e-3),
                                                                     rng.uniform(-0.02, 0.02)])
        off = (rng.uniform(-9, 9), rng.uniform(-9, 9))
        out.append(_case(f"scaled{t}", "scaled", model, K, D, rng.uniform(0.4, 1.3), SS, FW, FH, off, rng, t))
    # strong distortion, wide field of view: map entries far outside the frame (int16 saturation in the pinhole vector
    # body, wrapping elsewhere, cvRound's INT_MIN beyond 2^31 / 32)
    rng = np.random.default_rng(5)
    for t in range(24):
        W = int(rng.integers(40, 700))
        W = W - W % 8 + _W_MOD8[t % 8]
        H = int(rng.integers(30, 500))
        K = _K(rng, W, H, 0.3, 0.9, 10)
        FS = rng.uniform(0.05, 0.4)
        if t % 2 == 0:
            D5 = np.array([rng.uniform(0.2, 3), rng.uniform(0.5, 5), rng.uniform(-0.05, 0.05), rng.uniform(-0.05, 0.05), rng.uniform(1, 30)])
        else:
            D5 = np.array([rng.uniform(-3, -0.2), rng.uniform(-5, 5), rng.uniform(-0.05, 0.05), rng.uniform(-0.05, 0.05), rng.uniform(-30, 30)])
        D4 = rng.uniform(-1, 1, 4)
        if t % 2 == 0:                         # theta_d far beyond theta: map1 wraps past 32767
            D4[3] = rng.uniform(4, 12)
        out.append(_case(f"strong_pinhole{t}", "strong", 1, K, D5, FS, 1, W, H, (0.0, 0.0), rng, t))
        out.append(_case(f"strong_fisheye{t}", "strong", 0, K, D4, FS, 1, W, H, (0.0, 0.0), rng, t + 1))
    return tuple(out)


def case_by_name(name: str) -> CalibCase:
    return next(c for c in corpus() if c.name == name)


# ------------------------------------------------------------------ the oracle (cached per case)
@lru_cache(maxsize=None)
def cv2_maps(name: str):
    """cv2's CV_16SC2 + CV_16UC1 undistortion maps of the case."""
    c = case_by_name(name)
    if c.fisheye:
        return C.undistort_maps(c.K, c.D.reshape(4, 1), c.P, c.UW, c.UH)
    return C.pinhole_maps(c.K, c.D[None, :], c.P, c.UW, c.UH)


@lru_cache(maxsize=None)
def cv2_bev_maps(name: str):
    """Camera.get_bev_maps: cv2.warpPerspective of both map planes."""
    c = case_by_name(name)
    m1, m2 = cv2_maps(name)
    return cv2.warpPerspective(m1, c.H, (c.BW, c.BH)), cv2.warpPerspective(m2, c.H, (c.BW, c.BH))


def frames(name: str, channels: int, n: int = 1, size=None):
    """n random source frames of the case (uint8[n][FH][FW][channels], or another size)."""
    c = case_by_name(name)
    w, h = size or (c.FW, c.FH)
    rng = np.random.default_rng(zlib.crc32(f"{name}/{channels}/{n}/{w}x{h}".encode()))
    return rng.integers(0, 256, (n, h, w, channels), dtype=np.uint8)


def uv32(c: CalibCase, cols=None):
    """u * 32 and v * 32 of the case, as the direct double-precision formula gives them (numpy; for locating ties and
    out-of-range entries in reports, not as an oracle)."""
    iR = np.linalg.inv(c.P)
    j = np.arange(c.UW, dtype=np.float64)[None, :] if cols is None else np.asarray(cols, np.float64)[None, :]
    i = np.arange(c.UH, dtype=np.float64)[:, None]
    _x = j * iR[0, 0] + (i * iR[0, 1] + iR[0, 2])
    _y = j * iR[1, 0] + (i * iR[1, 1] + iR[1, 2])
    _w = j * iR[2, 0] + (i * iR[2, 1] + iR[2, 2])
    with np.errstate(all="ignore"):
        x, y = _x / _w, _y / _w
        if c.fisheye:
            r = np.sqrt(x * x + y * y)
            th = np.arctan(r)
            t2 = th * th
            k = c.D
            s = np.where(r == 0, 1.0, th * (1 + k[0] * t2 + k[1] * t2 ** 2 + k[2] * t2 ** 3 + k[3] * t2 ** 4) / r)
            xd, yd = x * s, y * s
        else:
            k1, k2, p1, p2, k3 = c.d5
            r2 = x * x + y * y
            kr = 1 + ((k3 * r2 + k2) * r2 + k1) * r2
            xd = x * kr + p1 * 2 * x * y + p2 * (r2 + 2 * x * x)
            yd = y * kr + p1 * (r2 + 2 * y * y) + p2 * 2 * x * y
        return (c.K[0, 0] * xd + c.K[0, 2]) * 32, (c.K[1, 1] * yd + c.K[1, 2]) * 32


def pinhole_outside_only(c: CalibCase, got, want):
    """Where the maps differ: True when the case is pinhole, map1 equals cv2's everywhere, and every differing map2 entry
    differs only in the fraction of an axis whose map1 component puts both bilinear taps outside any frame: saturated at
    32767 (frames are at most 32767 px) or at most -2.  cv2's pinhole map is compiled in its AVX2 dispatch unit, where the
    compiler contracts products and sums into FMAs, so its last bits depend on the CPU dispatch (DESIGN.md section 7);
    there they can move a fraction, never a pixel."""
    g1, g2 = got
    w1, w2 = want
    if c.fisheye or (g1 != w1).any():
        return (g1 == w1).all() and (g2 == w2).all()
    ii, jj = np.nonzero(g2 != w2)
    dx = (g2[ii, jj] & 31) != (w2[ii, jj] & 31)
    dy = (g2[ii, jj] >> 5) != (w2[ii, jj] >> 5)
    m = w1[ii, jj].astype(np.int32)
    out = (m <= -2) | (m == 32767)
    return bool(((~dx | out[:, 0]) & (~dy | out[:, 1])).all())


def remaps_agree(c: CalibCase, got, want) -> bool:
    """cv2.remap of random frames (1 and 3 channels, the case's frame size) through both map pairs gives the same image,
    LINEAR and NEAREST."""
    for ch in (1, 3):
        f = frames(c.name, ch, 1)[0]
        f = f[..., 0] if ch == 1 else f
        for inter in (cv2.INTER_LINEAR, cv2.INTER_NEAREST):
            if not (cv2.remap(f, *got, inter) == cv2.remap(f, *want, inter)).all():
                return False
    return True


def first_diffs(c: CalibCase, got, want, n: int = 6) -> str:
    """The first differing entries: (j, i), got and want map1 / map2, and u*32, v*32 of the direct formula."""
    g1, g2 = got
    w1, w2 = want
    ii, jj = np.nonzero((g1 != w1).any(-1) | (g2 != w2))
    if ii.size == 0:
        return "no differences"
    lines = [f"{c.name}: {ii.size} entries differ"]
    for i, j in list(zip(ii, jj))[:n]:
        u, v = uv32(c, [j])
        lines.append(f"  (j,i)=({j},{i}) got {tuple(g1[i, j])} {g2[i, j]} want {tuple(w1[i, j])} {w2[i, j]} "
                     f"u*32={float(u[i, 0])!r} v*32={float(v[i, 0])!r}")
    return "\n".join(lines)
