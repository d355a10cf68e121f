"""Seeded edge cases of cv2's wider lens models and of rectification rotations, shared by tests/test_host_lens_edges.py
(the host build of the kernels' coordinate code) and tests/test_gpu_lens_edges.py (the kernels).  Where
tests/lens_cases.py holds moderate cameras, these reach the inputs where the map arithmetic can go wrong: rays at or
behind the image plane (_w <= 0, _w == 0 exactly), rational denominators that cross zero (inf, NaN, cvRound's
INT_MIN), tilted projections whose vz changes sign, rotations up to 1.2 rad and non-orthogonal R, every W % 8 of the
pinhole vector body, degenerate map sizes, a 4K walked fisheye, and the boundaries of the LENS instance choice.

One seed gives one case, a lens_cases.LensCase: K, D, R, P, the undistorted size, and a canvas with a homography.
The oracle is cv2 alone.  cv2_rays pins how cv2 forms the rays of a map row (bevk_device.cuh row_sums), and classes()
restates the projection in NumPy to count the pixels of each edge class, so that thinning the corpus fails."""
from __future__ import annotations

from fractions import Fraction
from functools import lru_cache

import cv2
import numpy as np

from tests import calib_cases as CC
from tests import lens_cases as LC

# an exact inv(P * R): lower-triangular with power-of-two diagonal times a unit upper-triangular shift, so that
# _w = j/64 + i/256 - 13/4 is exactly 0 on the integer pixels of a line through a 320 x 240 frame, negative before it
_M_DYADIC = np.array([[2.0 ** -7, 0, -0.5], [2.0 ** -9, 2.0 ** -7, -0.625], [2.0 ** -6, 2.0 ** -8, -3.25]])
_P_DYADIC = np.array([[256.0, 0, 128], [0, 256.0, 96], [0, 0, 1]])


def _exact_inv(M):
    """inv(M) in rationals."""
    F = [[Fraction(float(v)) for v in row] for row in M]
    det = (F[0][0] * (F[1][1] * F[2][2] - F[1][2] * F[2][1]) - F[0][1] * (F[1][0] * F[2][2] - F[1][2] * F[2][0])
           + F[0][2] * (F[1][0] * F[2][1] - F[1][1] * F[2][0]))
    adj = [[F[1][1] * F[2][2] - F[1][2] * F[2][1], F[0][2] * F[2][1] - F[0][1] * F[2][2], F[0][1] * F[1][2] - F[0][2] * F[1][1]],
           [F[1][2] * F[2][0] - F[1][0] * F[2][2], F[0][0] * F[2][2] - F[0][2] * F[2][0], F[0][2] * F[1][0] - F[0][0] * F[1][2]],
           [F[1][0] * F[2][1] - F[1][1] * F[2][0], F[0][1] * F[2][0] - F[0][0] * F[2][1], F[0][0] * F[1][1] - F[0][1] * F[1][0]]]
    return [[a / det for a in row] for row in adj]


def _exact_mul(A, B):
    return [[sum(A[r][k] * B[k][c] for k in range(3)) for c in range(3)] for r in range(3)]


def dyadic_R():
    """R with inv(P_DYADIC * R) == M_DYADIC exactly: R = inv(P) * inv(M) in rationals, every entry a double."""
    R = _exact_mul(_exact_inv(_P_DYADIC), _exact_inv(_M_DYADIC))
    out = np.array([[float(v) for v in row] for row in R])
    assert all(Fraction(float(v)) == v for row in R for v in row)
    return out


def dyadic_exact(c: LC.LensCase) -> bool:
    """Are mul3(P, R) and inv3 of it exact for c, so that inv(P * R) == M_DYADIC bit for bit, as in cv2?"""
    PR = np.array([[(c.P[r, 0] * c.R[0, k] + c.P[r, 1] * c.R[1, k]) + c.P[r, 2] * c.R[2, k] for k in range(3)]
                   for r in range(3)])
    exact_PR = _exact_mul([[Fraction(float(v)) for v in row] for row in c.P], [[Fraction(float(v)) for v in row] for row in c.R])
    return (all(Fraction(float(PR[r, k])) == exact_PR[r][k] for r in range(3) for k in range(3))
            and (LC._iR(c) == _M_DYADIC).all())


def _rot(rng, angle):
    """A rotation by exactly `angle` rad about a random axis."""
    a = rng.normal(0, 1, 3)
    return cv2.Rodrigues(a / np.linalg.norm(a) * angle)[0]


def _K(W, H, f, dc=(0.0, 0.0)):
    return np.array([[f * W, 0, W / 2 + dc[0]], [0, f * W, H / 2 + dc[1]], [0, 0, 1.0]])


def _wide(K, W, H, fs):
    return LC._P(np.random.default_rng(W * 7 + H), K, W, H, fs)


def _D(n, **kw):
    names = ("k1", "k2", "p1", "p2", "k3", "k4", "k5", "k6", "s1", "s2", "s3", "s4", "tx", "ty")
    d = np.zeros(n)
    for k, v in kw.items():
        d[names.index(k)] = v
    return d


def _case(name, model, K, D, R, P, W, H, seed, horizon="none"):
    rng = np.random.default_rng(seed)
    BW, BH = CC._canvas(rng, seed)
    Hm = CC._H_ZERO.copy() if horizon == "zero" else CC._homography(rng, W, H, BW, BH, horizon)
    return LC.LensCase(name, "edge", model, K, np.asarray(D, np.float64).ravel(), R, P, W, H, Hm, BW, BH)


@lru_cache(maxsize=None)
def corpus() -> tuple:
    out = []
    rng = np.random.default_rng(41)
    # rational poles: 1 + k4 r^2 + k5 r^4 + k6 r^6 crosses zero inside the field of view, for 8, 12 and 14 coefficients
    for t, n in enumerate((8, 12, 14)):
        W, H = (200, 151, 263)[t], (150, 97, 120)[t]
        K = _K(W, H, 0.5)
        extra = dict(s1=0.01, s2=-0.004, s3=0.006, s4=0.003) if n >= 12 else {}
        if n == 14:
            extra.update(tx=0.05, ty=-0.04)
        D = _D(n, k1=-0.1, k2=0.02, p1=1e-3, k4=-0.6 - 0.1 * t, k5=0.05, k6=-0.01, **extra)
        out.append(_case(f"pole{n}", 1, K, D, None, _wide(K, W, H, 0.2), W, H, 100 + t, ("inside", "zero", "none")[t]))
    # thin-prism terms large enough to saturate map1 (the vector body) and wrap it (the scalar tail)
    for t, n in enumerate((12, 14)):
        W, H = (227, 180)[t], (140, 133)[t]
        K = _K(W, H, 0.6)
        D = _D(n, k1=-0.2, k2=0.05, k4=0.1, s1=0.4, s2=-0.35, s3=0.5, s4=0.3)
        out.append(_case(f"prism{n}", 1, K, D, None, _wide(K, W, H, 0.15), W, H, 110 + t, "inside"))
    # tilt up to about 1 rad, with vz <= 0 on part of the frame
    for t, (tx, ty) in enumerate(((1.0, -0.3), (-0.6, 0.95))):
        W, H = (240, 199)[t], (160, 150)[t]
        K = _K(W, H, 0.5)
        D = _D(14, k1=0.3, k2=0.2, k4=0.05, s1=0.02, tx=tx, ty=ty)
        out.append(_case(f"tilt{t}", 1, K, D, None, _wide(K, W, H, 0.25), W, H, 120 + t, ("zero", "inside")[t]))
    # rotations up to 1.2 rad, both models: _w <= 0 inside the frame
    for t, (model, n, ang) in enumerate(((1, 5, 1.1), (1, 8, 1.2), (1, 14, 0.9), (0, 4, 1.1), (0, 4, 1.2))):
        W, H = (216, 205, 250, 211, 170)[t], (150, 120, 133, 140, 161)[t]
        K = _K(W, H, 0.5)
        D = rng.uniform(-0.05, 0.05, 4) if model == 0 else np.concatenate([[-0.2, 0.05, 1e-3, -1e-3, 0.01], [0.05, 0.01, 0.002][:n - 5],
                                                                         np.zeros(max(0, n - 8))])
        if n == 14:
            D[12:] = [0.1, -0.05]
        out.append(_case(f"rot{'fish' if model == 0 else 'pin'}{n}_{t}", model, K, D, _rot(rng, ang), _wide(K, W, H, 0.5), W, H,
                         130 + t, "inside"))
    # a cv2.stereoRectify pair with a vertical baseline
    K = _K(320, 240, 0.8, (3.0, -2.0))
    D8 = _D(8, k1=-0.25, k2=0.08, p1=1e-3, p2=-5e-4, k3=-0.01, k4=0.1, k5=0.02, k6=-0.005)
    R1, R2, P1, P2, *_ = cv2.stereoRectify(K, D8, K, D8, (320, 240), _rot(rng, 0.04), np.array([0.003, -0.12, 0.002]))
    for s, (Rs, Ps) in enumerate(((R1, P1), (R2, P2))):
        out.append(_case(f"stereov{s}", 1, K, D8, Rs, Ps[:, :3].copy(), 320, 240, 140 + s, "inside"))
    # non-orthogonal R with a dyadic inv(P * R): _w == 0 exactly on integer pixels, both models
    K = _K(320, 240, 0.5)
    out.append(_case("dyadic_pin", 1, K, _D(8, k1=-0.2, k2=0.05, k4=0.1, k5=0.02, k6=0.001), dyadic_R(), _P_DYADIC.copy(),
                     320, 240, 150))
    out.append(_case("dyadic_fish", 0, K, np.array([0.05, -0.01, 0.002, -1e-3]), dyadic_R(), _P_DYADIC.copy(), 320, 240, 151))
    # the same inv(P * R) up to rounding, with a wide P: the line _w ~ 0 crosses the frame, and a last-bit difference in _w
    # decides between _w == 0 (NaN, INT_MIN) and a tiny _w (u near cx)
    for t, W in enumerate((320, 327, 643)):
        H = W * 3 // 4
        K = _K(W, H, 0.5)
        P = K.copy()
        P[0, 0] *= 0.15
        P[1, 1] *= 0.15
        M = np.array([[2.0 ** -7, 0, -1], [2.0 ** -9, 2.0 ** -7, -1], [2.0 ** -6, 2.0 ** -8, -2.0]])
        R = np.linalg.inv(P) @ np.linalg.inv(M)
        out.append(_case(f"neardyadic{W}", 1, K, _D(8, k1=-0.2, k2=0.05, k4=0.1, k5=0.02, k6=0.001), R, P, W, H, 160 + t))
    # every W % 8 of the pinhole vector body (rotated, rational), and rotated fisheyes at odd widths
    for r in range(8):
        W, H = 96 + 8 * r + r, 40 + 3 * r
        K = _K(W, H, 0.45)
        D = _D(8, k1=0.6, k2=-0.8, p1=0.01, k3=1.5, k4=0.4, k5=-0.2, k6=0.05)
        out.append(_case(f"wmod{r}", 1, K, D, _rot(rng, 0.15), _wide(K, W, H, 0.12), W, H, 170 + r, "inside"))
    for t, W in enumerate((97, 131, 255)):
        H = 61 + 10 * t
        K = _K(W, H, 0.4)
        out.append(_case(f"fishodd{W}", 0, K, rng.uniform(-0.3, 0.3, 4), _rot(rng, 0.3), _wide(K, W, H, 0.5), W, H, 180 + t))
    # degenerate map sizes: 1 x N and N x 1 for both models, and W from 1 to 9
    for t, (model, W, H) in enumerate(((1, 1, 37), (1, 41, 1), (0, 1, 29), (0, 33, 1))):
        K = _K(max(W, H), max(W, H), 0.5)
        D = rng.uniform(-0.1, 0.1, 4) if model == 0 else _D(12, k1=-0.2, k4=0.1, s1=0.01, s4=-0.02)
        out.append(_case(f"thin{'fish' if model == 0 else 'pin'}{W}x{H}", model, K, D, _rot(rng, 0.2), _wide(K, W, H, 0.6), W, H,
                         190 + t))
    for W in range(1, 10):
        K = _K(W, 7, 0.5)
        out.append(_case(f"narrow{W}", 1, K, _D(8, k1=-0.3, k2=0.1, k4=0.2), _rot(rng, 0.3), _wide(K, W, 7, 0.2), W, 7, 200 + W))
    # one large walked fisheye: a rotated fisheye at 3840 x 2160 (its ray scratch is about 200 MB)
    K = _K(3840, 2160, 0.3)
    out.append(_case("bigfish", 0, K, rng.uniform(-0.05, 0.05, 4), _rot(rng, 0.08), _wide(K, 3840, 2160, 0.7), 3840, 2160, 210))
    # the boundaries of the LENS instance choice: one non-zero extra coefficient, R = I given, R keeping the column table
    K = _K(160, 120, 0.6)
    P = _wide(K, 160, 120, 0.5)
    out.append(_case("only_k6", 1, K, _D(8, k1=-0.1, k6=0.01), None, P, 160, 120, 220))
    out.append(_case("only_s4", 1, K, _D(12, k1=-0.1, s4=0.002), None, P, 160, 120, 221))
    out.append(_case("only_ty", 1, K, _D(14, k1=-0.1, ty=0.02), None, P, 160, 120, 222, "zero"))
    out.append(_case("eye_pin5", 1, K, _D(5, k1=-0.1, k2=0.01), np.eye(3), P, 160, 120, 223))
    out.append(_case("eye_pin8", 1, K, _D(8, k1=-0.1, k4=0.05), np.eye(3), P, 160, 120, 224))
    out.append(_case("eye_fish", 0, K, np.array([0.05, -0.01, 0.002, -1e-3]), np.eye(3), P, 160, 120, 225))
    flip = np.diag([-1.0, -1.0, 1.0])
    out.append(_case("flip_pin", 1, K, _D(8, k1=-0.1, k4=0.05), flip, P, 160, 120, 226))
    out.append(_case("flip_fish", 0, K, np.array([0.05, -0.01, 0.002, -1e-3]), flip, P, 160, 120, 227))
    names = [c.name for c in out]
    assert len(set(names)) == len(names)
    return tuple(out)


def case_by_name(name: str) -> LC.LensCase:
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


def cv2_rays(c: LC.LensCase):
    """The rays cv2 projects, as float64[3][h][w] (_x, _y, _w).  Each row starts at i*iR01 + iR02 (the same for _y, _w).
    cv2.fisheye.initUndistortRectifyMap adds iR00 column by column (lens_cases.walked_rays).  cv2.initUndistortRectifyMap's
    8-column vector body adds 8*iR00 per block and offsets column k of a block by k*iR00, each product and sum rounded;
    its scalar tail adds iR00 column by column from where the blocks end."""
    if c.fisheye:
        return LC.walked_rays(c)
    iR = LC._iR(c)
    i = np.arange(c.UH, dtype=np.float64)
    k = np.arange(8, dtype=np.float64)
    out = np.empty((3, c.UH, c.UW))
    body = c.UW - c.UW % 8
    for p in range(3):
        run = i * iR[p, 1] + iR[p, 2]
        for j in range(0, body, 8):
            out[p, :, j:j + 8] = run[:, None] + k[None, :] * iR[p, 0]
            run = run + 8.0 * iR[p, 0]
        for j in range(body, c.UW):
            out[p, :, j] = run
            run = run + iR[p, 0]
    return out


def classes(c: LC.LensCase) -> dict:
    """Pixel counts of the edge classes of c, from a NumPy restatement of the projection on cv2's rays (not an oracle:
    it only locates the classes).  int_min: u or v NaN or beyond 2^31 / 32 (cvRound's INT_MIN); saturated / wrapped:
    a map1 component beyond int16 in the vector body (saturating pack) / elsewhere (wrapping cast); w_le0, w_eq0: _w <= 0,
    == 0; pole: the rational denominator <= 0; vz_le0: the tilted projection's vz <= 0."""
    _x, _y, _w = cv2_rays(c)
    with np.errstate(all="ignore"):
        if c.fisheye:
            x, y = _x / _w, _y / _w
            r = np.sqrt(x * x + y * y)
            th = np.arctan(r)
            t2 = th * th
            k = c.D
            s = np.where(r == 0, 1.0, th * (1 + k[0] * t2 + k[1] * t2 ** 2 + k[2] * t2 ** 3 + k[3] * t2 ** 4) / r)
            u = np.where(_w <= 0, np.where(_x > 0, -np.inf, np.inf), c.K[0, 0] * x * s + c.K[0, 2])
            v = np.where(_w <= 0, np.where(_y > 0, -np.inf, np.inf), c.K[1, 1] * y * s + c.K[1, 2])
            den = np.ones_like(_w)
            vz = np.ones_like(_w)
        else:
            d = np.zeros(14)
            d[:c.n_dist] = c.D
            k1, k2, p1, p2, k3, k4, k5, k6, s1, s2, s3, s4 = d[:12]
            w = 1 / _w
            x, y = _x * w, _y * w
            r2 = x * x + y * y
            den = 1 + ((k6 * r2 + k5) * r2 + k4) * r2
            kr = (1 + ((k3 * r2 + k2) * r2 + k1) * r2) / den
            xd = x * kr + p1 * 2 * x * y + p2 * (r2 + 2 * x * x) + s1 * r2 + s2 * r2 * r2
            yd = y * kr + p1 * (r2 + 2 * y * y) + p2 * 2 * x * y + s3 * r2 + s4 * r2 * r2
            tx, ty = (d[12], d[13]) if c.n_dist == 14 else (0.0, 0.0)
            T = _tilt(tx, ty)
            vx = T[0, 0] * xd + T[0, 1] * yd + T[0, 2]
            vy = T[1, 0] * xd + T[1, 1] * yd + T[1, 2]
            vz = T[2, 0] * xd + T[2, 1] * yd + T[2, 2]
            ip = np.where(vz != 0, 1 / vz, 1.0)
            u = c.K[0, 0] * ip * vx + c.K[0, 2]
            v = c.K[1, 1] * ip * vy + c.K[1, 2]
        iu, iv = u * 32, v * 32
        bad = ~(np.abs(iu) < 2.0 ** 31) | ~(np.abs(iv) < 2.0 ** 31)
        big = (~bad) & ((np.floor(iu / 32) > 32767) | (np.floor(iu / 32) < -32768) | (np.floor(iv / 32) > 32767)
                        | (np.floor(iv / 32) < -32768))
    body = np.zeros(_w.shape, bool)
    if not c.fisheye:
        body[:, :c.UW - c.UW % 8] = True
    rational = not c.fisheye and c.n_dist >= 8
    return {"int_min": int(bad.sum()), "saturated": int((big & body).sum()), "wrapped": int((big & ~body).sum()),
            "w_le0": int((_w <= 0).sum()), "w_eq0": int((_w == 0).sum()), "pole": int((den <= 0).sum()) if rational else 0,
            "vz_le0": int((vz <= 0).sum())}


def _tilt(tx, ty):
    """cv::detail::computeTiltProjectionMatrix(tauX, tauY)."""
    cx, sx, cy, sy = np.cos(tx), np.sin(tx), np.cos(ty), np.sin(ty)
    Rxy = np.array([[cy, 0, -sy], [0, 1, 0], [sy, 0, cy]]) @ np.array([[1, 0, 0], [0, cx, sx], [0, -sx, cx]])
    Pz = np.array([[Rxy[2, 2], 0, -Rxy[0, 2]], [0, Rxy[2, 2], -Rxy[1, 2]], [0, 0, 1]])
    return Pz @ Rxy
