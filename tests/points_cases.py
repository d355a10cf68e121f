"""Seeded corpus for cv2's point functions (bevk_points.cuh): cameras of every pinhole D length with and without tilt,
the fisheye with and without R (matrix and rvec) and P, and points at the principal point, inside the frame, far outside
(icdist < 0, theta clamped at pi/2 and flipped), NaN and +-inf.  `cv2_points` is the live cv2 call of a case."""
from __future__ import annotations

from dataclasses import dataclass, field

import cv2
import numpy as np

K = np.array([[500., 0, 320.5], [0, 510., 240.25], [0, 0, 1]])
P_NEW = np.array([[400., 0, 300], [0, 410., 250], [0, 0, 1]])
R_MAT = cv2.Rodrigues(np.array([0.05, -0.1, 0.02]))[0]
R_VEC = np.array([0.03, 0.08, -0.05])
D_FISH = np.array([0.1, 0.01, -0.01, 0.002])
H = np.array([[1.2, 0.1, -30], [0.05, 0.9, 20], [1e-4, -2e-4, 1.0]])
OPS = ("undistort", "project", "distort", "perspective")
# what the GPU tests run every op at: point counts, cv2's layouts of 2-D points, dtypes
SIZES = (0, 1, 1 << 20)
LAYOUTS = ("N12", "1N2", "N2")
DTYPES = (np.float32, np.float64)


@dataclass
class Case:
    name: str
    op: str
    model: str = "pinhole"               # "pinhole" | "fisheye"
    D: np.ndarray | None = None
    R: np.ndarray | None = None
    P: np.ndarray | None = None
    criteria: tuple = (1, 5, 0.01)
    rvec: np.ndarray = field(default_factory=lambda: np.array([0.3, -0.2, 0.1]))
    tvec: np.ndarray = field(default_factory=lambda: np.array([0.1, 0.2, 0.5]))
    alpha: float = 0.
    M: np.ndarray | None = None


def _pinhole_d(rng, n, tilt):
    d = np.concatenate([[-0.3, 0.12, 1e-3, -2e-3, -0.02], rng.normal(0, 0.03, 9)])[:n]
    if n == 14 and tilt:
        d[12:] = [0.02, -0.03]
    elif n == 14:
        d[12:] = 0
    return d


def corpus() -> list[Case]:
    rng = np.random.default_rng(20261019)
    out = []
    for n in (0, 4, 5, 8, 12, 14):
        for tilt in ((False, True) if n == 14 else (False,)):
            D = None if n == 0 else _pinhole_d(rng, n, tilt)
            t = "_tilt" if tilt else ""
            for R, P, rp in ((None, None, ""), (R_MAT, P_NEW, "_RP"), (None, P_NEW, "_P"), (R_MAT, None, "_R")):
                out.append(Case(f"und_pin{n}{t}{rp}", "undistort", D=D, R=R, P=P))
            out.append(Case(f"und_pin{n}{t}_count9", "undistort", D=D, criteria=(1, 9, 0.)))
            out.append(Case(f"proj_pin{n}{t}", "project", D=D))
    out.append(Case("und_pin5_barrel", "undistort", D=np.array([-0.9, 0.6, 0, 0, -0.2])))   # icdist < 0 far out
    for R, P, rp in ((None, None, ""), (R_MAT, P_NEW, "_RP"), (R_VEC, P_NEW, "_rvecP"), (None, P_NEW, "_P")):
        for crit, cn in (((3, 10, 1e-8), ""), ((1, 10, 0.), "_count"), ((3, 3, 1e-3), "_both3")):
            out.append(Case(f"und_fish{rp}{cn}", "undistort", "fisheye", D_FISH, R, P, crit))
    out.append(Case("und_fish_noD", "undistort", "fisheye", None, None, P_NEW, (3, 10, 1e-8)))
    out.append(Case("und_fish_strong", "undistort", "fisheye", np.array([-0.4, 0.3, -0.2, 0.1]), None, None, (3, 10, 1e-8)))
    out.append(Case("und_fish_flip", "undistort", "fisheye", np.array([-0.5, 0.1, 0, 0]), None, None, (1, 10, 0.)))
    out.append(Case("und_fish_noconv", "undistort", "fisheye", np.array([-0.4, 0.3, -0.2, 0.1]), None, None, (3, 2, 1e-14)))
    out.append(Case("proj_fish", "project", "fisheye", D_FISH))
    out.append(Case("proj_fish_alpha", "project", "fisheye", D_FISH, alpha=0.2))
    out.append(Case("proj_fish_rvec0", "project", "fisheye", D_FISH, rvec=np.zeros(3), tvec=np.zeros(3)))
    out.append(Case("dist_fish", "distort", "fisheye", D_FISH))
    out.append(Case("dist_fish_alpha", "distort", "fisheye", D_FISH, alpha=0.3))
    out.append(Case("persp", "perspective", M=H))
    out.append(Case("persp_affine", "perspective", M=np.array([[2., 0.5, 3], [-0.5, 1.5, 4], [0, 0, 1]])))
    return out


SPECIAL2 = np.array([[320.5, 240.25], [320.5 + 1e-9, 240.25], [np.nan, 1.], [5., np.nan], [np.inf, 3.], [-np.inf, np.inf],
                     [1e6, -1e6], [-3000., 5000.]])
SPECIAL3 = np.array([[0., 0., 0.], [1., 2., 0.], [1., 1., -1.], [0.5, -0.25, -3.], [np.nan, 0., 1.], [np.inf, 1., 2.],
                     [0., 0., 1e-300]])


def points(c: Case, n: int, dtype, seed: int = 0) -> np.ndarray:
    """n + the special points of case c's op, [N][1][k] of dtype (perspective: some with w == 0)."""
    rng = np.random.default_rng(seed)
    if c.op == "project":
        p = np.concatenate([rng.normal(0, 2, (n, 3)) + [0, 0, 1], SPECIAL3])
        return p.astype(dtype).reshape(-1, 1, 3)
    if c.op == "distort":
        p = np.concatenate([rng.normal(0, 1.5, (n, 2)), [[0, 0], [1e-9, 0], [np.nan, 0], [np.inf, 1], [200., -100.]]])
    elif c.op == "perspective":
        m = c.M
        # points on the line w == 0 (and within FLT_EPSILON of it)
        xs = rng.uniform(-5000, 5000, 8)
        line = np.stack([xs, -(m[2, 0] * xs + m[2, 2]) / m[2, 1]], 1) if m[2, 1] else np.zeros((0, 2))
        # near w = 0 the output is large: the rounding of w shows in its last bit (cv2's FMA against separate roundings)
        near = np.array([[-2287.7258, 3855.9158]], np.float32).astype(np.float64)
        p = np.concatenate([rng.uniform(-3000, 4000, (n, 2)), line, near, SPECIAL2])
    else:
        p = np.concatenate([rng.uniform(-2500, 3200, (n // 2, 2)), rng.uniform(0, 640, (n - n // 2, 2)), SPECIAL2])
    return p.astype(dtype).reshape(-1, 1, 2)


def cv2_points(c: Case, pts: np.ndarray) -> np.ndarray:
    if c.op == "undistort" and c.model == "pinhole":
        return cv2.undistortPointsIter(pts, K, c.D, c.R, c.P, c.criteria)
    if c.op == "undistort":
        D = np.zeros(4) if c.D is None else c.D   # cv2's fisheye reads 4 coefficients; the library's empty D is zeros
        return cv2.fisheye.undistortPoints(pts, K, D, R=c.R, P=c.P, criteria=c.criteria)
    if c.op == "project" and c.model == "pinhole":
        return cv2.projectPoints(pts, c.rvec, c.tvec, K, c.D)[0]
    if c.op == "project":
        return cv2.fisheye.projectPoints(pts, c.rvec, c.tvec, K, c.D, alpha=c.alpha)[0]
    if c.op == "distort":
        return cv2.fisheye.distortPoints(pts, K, c.D, alpha=c.alpha)
    return cv2.perspectiveTransform(pts, c.M)


def supported(c: Case, dtype) -> bool:
    """Whether the library computes case c at dtype (float64 fisheye points are refused)."""
    return np.dtype(dtype) == np.float32 or c.model == "pinhole"


def same(a, b) -> bool:
    """Equal bit for bit, NaN matching NaN."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    u = np.uint32 if a.dtype == np.float32 else np.uint64
    return bool(((a.view(u) == b.view(u)) | (np.isnan(a) & np.isnan(b))).all())


def classes() -> dict:
    """What the corpus reaches: camera classes, and point classes counted on its float64 points."""
    k = {"pinhole_n": set(), "tilt": 0, "fisheye_R": 0, "fisheye_rvec": 0, "fisheye_P": 0, "fisheye_plain": 0,
         "crit": set(), "ops": set(), "z0": 0, "z_neg": 0, "w_small": 0, "nan": 0, "inf": 0, "theta_clamped": 0,
         "theta_flipped": 0, "not_converged": 0, "icdist_neg": 0, "principal": 0}
    for c in corpus():
        k["ops"].add(c.op)
        pts = points(c, 200, np.float64, seed=len(c.name))
        flat = pts.reshape(len(pts), -1)
        k["nan"] += int(np.isnan(flat).any())
        k["inf"] += int(np.isinf(flat).any())
        if c.op == "project":
            k["z0"] += int((flat[:, 2] == 0).any())
            k["z_neg"] += int((flat[:, 2] < 0).any())
        if c.op == "perspective":
            with np.errstate(invalid="ignore"):
                w = flat[:, 0] * c.M[2, 0] + flat[:, 1] * c.M[2, 1] + c.M[2, 2]
            k["w_small"] += int((np.abs(w) <= np.finfo(np.float32).eps).any())
        if c.op != "undistort":
            continue
        pw = (flat - [K[0, 2], K[1, 2]]) / [K[0, 0], K[1, 1]]
        with np.errstate(invalid="ignore"):
            r = np.hypot(pw[:, 0], pw[:, 1])
        k["principal"] += int((r == 0).any())
        if c.model == "pinhole":
            k["pinhole_n"].add(0 if c.D is None else c.D.size)
            k["tilt"] += int(c.D is not None and c.D.size == 14 and c.D[12] != 0)
            if c.D is not None:
                d = np.zeros(14)
                d[:c.D.size] = c.D
                r2 = r * r
                with np.errstate(invalid="ignore", over="ignore"):
                    den = 1 + ((d[4] * r2 + d[1]) * r2 + d[0]) * r2
                k["icdist_neg"] += int((den < 0).any())
            continue
        k["crit"].add(c.criteria[0])
        k["fisheye_R"] += int(c.R is not None and np.size(c.R) == 9)
        k["fisheye_rvec"] += int(c.R is not None and np.size(c.R) == 3)
        k["fisheye_P"] += int(c.P is not None)
        k["fisheye_plain"] += int(c.R is None and c.P is None)
        k["theta_clamped"] += int((r > np.pi / 2).any())
        out = cv2_points(c, pts).reshape(-1, 2)
        minus = (out == -1e6).all(1).any()
        k["theta_flipped" if not c.criteria[0] & 2 else "not_converged"] += int(minus)
    return k
