"""Seeded calibrations of cv2's wider lens models and of rectification rotations, shared by
tests/test_host_lens_models.py (the host build of the kernels' coordinate code) and tests/test_gpu_lens_models.py (the
kernels).  One seed gives one case: a pinhole camera with 8 (rational), 12 (thin prism) or 14 (tilted) coefficients, or
with 5 and a rotation R; a fisheye camera with a rotation R; its K, D, R, P, the undistorted size, and a canvas with a
homography for the BEV LUT.

The oracle is cv2 alone: cv2.initUndistortRectifyMap / cv2.fisheye.initUndistortRectifyMap with R for the maps,
cv2.warpPerspective of the map planes for the BEV LUT, cv2.remap for images."""
from __future__ import annotations

from dataclasses import dataclass
from functools import lru_cache

import cv2
import numpy as np

from tests import calib_cases as CC

# widths of the strong pinhole cameras, by W % 8 (cv2's 8-column vector body with its saturating pack ends at W - W % 8)
_W_MOD8 = (0, 1, 7)


@dataclass(eq=False)
class LensCase:
    name: str
    kind: str            # "real" (real sizes, mild lens), "strong" (wide view, large D), "rotated" (fisheye with R)
    model: int           # 0 fisheye, 1 pinhole
    K: np.ndarray
    D: np.ndarray        # 4 (fisheye) or 5, 8, 12, 14 (pinhole) coefficients
    R: np.ndarray | None  # rectification rotation, None for eye(3)
    P: np.ndarray
    UW: int
    UH: int
    H: np.ndarray        # homography: undistorted frame -> canvas
    BW: int
    BH: int

    @property
    def fisheye(self) -> bool:
        return self.model == 0

    @property
    def n_dist(self) -> int:
        return int(self.D.size)

    @property
    def tilt(self) -> tuple:
        return (float(self.D[12]), float(self.D[13])) if self.n_dist == 14 else (0.0, 0.0)


def _rotation(rng, scale):
    return cv2.Rodrigues(rng.normal(0, scale, 3))[0]


def _pinhole_D(rng, n, strong):
    d = np.zeros(n)
    if strong:
        d[:5] = [rng.uniform(-0.8, 0.8), rng.uniform(-1, 1), rng.uniform(-0.03, 0.03), rng.uniform(-0.03, 0.03),
                 rng.uniform(-2, 2)]
    else:
        d[:5] = [rng.uniform(-0.4, 0.2), rng.uniform(-0.1, 0.1), rng.uniform(-2e-3, 2e-3), rng.uniform(-2e-3, 2e-3),
                 rng.uniform(-0.05, 0.05)]
    if n >= 8:   # rational: k4..k6 of the size calibrateCamera gives wide-angle lenses
        d[5:8] = [rng.uniform(-0.5, 0.5), rng.uniform(-0.2, 0.2), rng.uniform(-0.05, 0.05)]
        if strong:
            d[5:8] *= 3
    if n >= 12:  # thin prism, s1 s2 s3 s4 all different (a swap moves pixels)
        d[8:12] = rng.uniform(-4e-3, 4e-3, 4) * (20 if strong else 1)
    if n >= 14:  # tilt up to about 0.2 rad
        d[12:14] = rng.uniform(-0.2, 0.2, 2)
    return d


def _P(rng, K, UW, UH, fs):
    P = K.copy()
    P[0, 0] *= fs
    P[1, 1] *= fs
    P[0, 2] = UW / 2 + rng.uniform(-5, 5)
    P[1, 2] = UH / 2 + rng.uniform(-5, 5)
    return P


def _case(name, kind, model, K, D, R, P, UW, UH, rng, i):
    BW, BH = CC._canvas(rng, i)
    H = CC._homography(rng, UW, UH, BW, BH, ("none", "inside")[i % 2])
    return LensCase(name, kind, model, K, np.asarray(D, np.float64).ravel(), R, P, UW, UH, H, BW, BH)


@lru_cache(maxsize=None)
def corpus() -> tuple:
    out = []
    # pinhole cameras at real sizes: 8, 12 and 14 coefficients, the later ones rotated
    rng = np.random.default_rng(11)
    sizes = ((1280, 1024), (1920, 1080), (2560, 2048))
    for t in range(9):
        n = (8, 12, 14)[t % 3]
        W, H = sizes[t // 3]
        K = CC._K(rng, W, H, 0.4, 0.9, 20)
        R = _rotation(rng, 0.05) if t >= 5 else None
        out.append(_case(f"real{n}_{t}", "real", 1, K, _pinhole_D(rng, n, False), R, _P(rng, K, W, H, rng.uniform(0.5, 1.0)),
                         W, H, rng, t))
    # a stereo-rectified pinhole pair of 5 coefficients: R from cv2.stereoRectify
    K = CC._K(rng, 1280, 1024, 0.5, 0.8, 10)
    D5 = _pinhole_D(rng, 5, False)
    R1, R2, P1, P2, *_ = cv2.stereoRectify(K, D5, K, D5, (1280, 1024), _rotation(rng, 0.03), np.array([-0.12, 0.004, 0.002]))
    for s, (Rs, Ps) in enumerate(((R1, P1), (R2, P2))):
        out.append(_case(f"stereo5_{s}", "real", 1, K, D5, Rs, Ps[:, :3].copy(), 1280, 1024, rng, s))
    # strong distortion, wide view: W % 8 in {0, 1, 7}, every coefficient count, map entries far outside the frame
    rng = np.random.default_rng(12)
    for t in range(12):
        n = (8, 12, 14)[t % 3]
        W = int(rng.integers(60, 700))
        W = W - W % 8 + _W_MOD8[t % 3 if t < 9 else (t + 1) % 3]
        H = int(rng.integers(40, 480))
        K = CC._K(rng, W, H, 0.3, 0.9, 8)
        R = _rotation(rng, 0.08) if t % 2 else None
        out.append(_case(f"strong{n}_{t}", "strong", 1, K, _pinhole_D(rng, n, True), R, _P(rng, K, W, H, rng.uniform(0.1, 0.4)),
                         W, H, rng, t))
    # fisheye cameras with R: rotated rays that depend on the row (cv2's running row sums), at real and small sizes
    rng = np.random.default_rng(13)
    fsizes = ((1280, 1024), (2560, 2048), (1920, 1080), (640, 481), (333, 250), (1281, 720))
    for t, (W, H) in enumerate(fsizes):
        K = CC._K(rng, W, H, 0.25, 0.6, 10)
        D4 = rng.uniform(-0.05, 0.05, 4) if t < 3 else rng.uniform(-0.5, 0.5, 4)
        out.append(_case(f"rotated{t}", "rotated", 0, K, D4, _rotation(rng, 0.1), _P(rng, K, W, H, rng.uniform(0.4, 1.0)),
                         W, H, rng, t))
    return tuple(out)


def case_by_name(name: str) -> LensCase:
    return next(c for c in corpus() if c.name == name)


@lru_cache(maxsize=None)
def cv2_maps(name: str):
    """cv2's CV_16SC2 + CV_16UC1 maps of the case, with its R."""
    c = case_by_name(name)
    R = np.eye(3) if c.R is None else c.R
    if c.fisheye:
        return cv2.fisheye.initUndistortRectifyMap(c.K, c.D.reshape(4, 1), R, c.P, (c.UW, c.UH), cv2.CV_16SC2)
    return cv2.initUndistortRectifyMap(c.K, c.D, R, c.P, (c.UW, c.UH), cv2.CV_16SC2)


@lru_cache(maxsize=None)
def cv2_bev_maps(name: str):
    """Camera.get_bev_maps: cv2.warpPerspective of both map planes."""
    c = case_by_name(name)
    m1, m2 = cv2_maps(name)
    return cv2.warpPerspective(m1, c.H, (c.BW, c.BH)), cv2.warpPerspective(m2, c.H, (c.BW, c.BH))


def outside_only(c: LensCase, got, want) -> bool:
    """calib_cases.pinhole_outside_only, the one tolerated difference of pinhole maps, for a lens case."""
    return CC.pinhole_outside_only(c, got, want)


def xs_table_form(c: LensCase) -> bool:
    """Are the fisheye rays of c independent of the row (bevk_device.cuh xs_table_applies: inv(P * R) without skew and
    with last row (0, 0, *))?  Otherwise cv2's running row sums have to be walked row by row."""
    return bool(c.fisheye and _row_free(c))


def _row_free(c) -> bool:
    iR = _iR(c)
    return bool(iR[0, 1] == 0 and iR[1, 0] == 0 and iR[2, 0] == 0 and iR[2, 1] == 0)


def walks(c) -> bool:
    """Does the library walk the rays of c row by row (lens_model's walks: an R other than the identity whose inv(P * R)
    makes the rays depend on the row), for either model?"""
    return bool(c.R is not None and not (c.R == np.eye(3)).all() and not _row_free(c))


def _inv3(S):
    """OpenCV's closed-form 3x3 inverse (bevk_device.cuh inv3)."""
    M = lambda r, c: S[r, c]
    d = 1. / (M(0, 0) * (M(1, 1) * M(2, 2) - M(1, 2) * M(2, 1)) - M(0, 1) * (M(1, 0) * M(2, 2) - M(1, 2) * M(2, 0))
              + M(0, 2) * (M(1, 0) * M(2, 1) - M(1, 1) * M(2, 0)))
    return np.array([[(M(1, 1) * M(2, 2) - M(1, 2) * M(2, 1)) * d, (M(0, 2) * M(2, 1) - M(0, 1) * M(2, 2)) * d,
                      (M(0, 1) * M(1, 2) - M(0, 2) * M(1, 1)) * d],
                     [(M(1, 2) * M(2, 0) - M(1, 0) * M(2, 2)) * d, (M(0, 0) * M(2, 2) - M(0, 2) * M(2, 0)) * d,
                      (M(0, 2) * M(1, 0) - M(0, 0) * M(1, 2)) * d],
                     [(M(1, 0) * M(2, 1) - M(1, 1) * M(2, 0)) * d, (M(0, 1) * M(2, 0) - M(0, 0) * M(2, 1)) * d,
                      (M(0, 0) * M(1, 1) - M(0, 1) * M(1, 0)) * d]])


def _iR(c: LensCase):
    """inv(P * R) as lens_model forms it: cv::Matx's product order, then OpenCV's closed-form inverse."""
    if c.R is None:
        return _inv3(c.P)
    PR = np.array([[(c.P[r, 0] * c.R[0, k] + c.P[r, 1] * c.R[1, k]) + c.P[r, 2] * c.R[2, k] for k in range(3)]
                   for r in range(3)])
    return _inv3(PR)


def walked_rays(c: LensCase):
    """cv2.fisheye.initUndistortRectifyMap's rays of c: per row _x = i*iR01 + iR02, then _x += iR00 column by column (and
    the same for _y, _w), as float64[3][h][w]."""
    iR = _iR(c)
    i = np.arange(c.UH, dtype=np.float64)
    run = [i * iR[k, 1] + iR[k, 2] for k in range(3)]
    out = np.empty((3, c.UH, c.UW))
    for j in range(c.UW):
        for k in range(3):
            out[k, :, j] = run[k]
            run[k] = run[k] + iR[k, 0]
    return out


def direct_rays(c: LensCase):
    """The same rays in the direct form j*iR00 + (i*iR01 + iR02), which a map build that skipped the walk would use."""
    iR = _iR(c)
    j = np.arange(c.UW, dtype=np.float64)[None, :]
    i = np.arange(c.UH, dtype=np.float64)[:, None]
    return np.stack([j * iR[k, 0] + (i * iR[k, 1] + iR[k, 2]) for k in range(3)])


def first_diffs(c: LensCase, got, want, n: int = 6) -> str:
    """The first differing map entries of c: (j, i), got and want map1 / map2."""
    g1, g2 = got
    w1, w2 = want
    ii, jj = np.nonzero((g1 != w1).any(-1) | (g2 != w2))
    if ii.size == 0:
        return "no differences"
    lines = [f"{c.name}: {ii.size} entries differ"]
    for i, j in list(zip(ii, jj))[:n]:
        lines.append(f"  (j,i)=({j},{i}) got {tuple(g1[i, j])} {g2[i, j]} want {tuple(w1[i, j])} {w2[i, j]}")
    return "\n".join(lines)
