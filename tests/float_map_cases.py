"""Seeded corpus of cameras and synthetic maps for cv2's float maps (CV_32FC1 / CV_32FC2).

Cameras: pinholes with 4, 5, 8, 12 and 14 coefficients, with and without a rectification rotation R, including a
cv2.stereoRectify pair at 1280x720 and one with a vertical baseline; fisheyes with and without R, one of them turned
far enough that rays fall behind the camera (+-inf map entries); widths with W % 8 of 0, 1 and 7, and a 1xN map.

Synthetic maps (synthetic_maps) hold the values where the conversion cv2.remap applies to float maps can go wrong: float
ties of x * 32 (k + 0.5) and of x itself, NaN, +-inf, +-3e9, and values just inside and outside +-32767/32 and +-32768.
classes() counts what the corpus reaches, so that thinning it fails tests/test_host_float_maps.py."""
from __future__ import annotations

import functools
from dataclasses import dataclass

import cv2
import numpy as np


@dataclass(frozen=True)
class FloatCase:
    name: str
    model: int            # 0 fisheye, 1 pinhole (BEVK_MODEL_*)
    K: np.ndarray
    D: np.ndarray
    R: np.ndarray | None
    P: np.ndarray
    W: int                # map size
    H: int
    SW: int               # size of the frames the map samples
    SH: int

    @property
    def fisheye(self) -> bool:
        return self.model == 0


def _K(f, W, H, dc=(0.0, 0.0)):
    return np.array([[f, 0, W / 2 + dc[0]], [0, f * 1.01, H / 2 + dc[1]], [0, 0, 1]], np.float64)


def _rot(rng, angle):
    v = rng.normal(size=3)
    return cv2.Rodrigues(v / np.linalg.norm(v) * angle)[0]


def _pinhole_D(rng, n):
    d = np.zeros(n)
    d[:4] = rng.normal(0, [0.15, 0.05, 0.002, 0.002])
    if n >= 5:
        d[4] = rng.normal(0, 0.01)
    if n >= 8:
        d[5:8] = rng.normal(0, [0.05, 0.01, 0.002])
    if n >= 12:
        d[8:12] = rng.normal(0, 0.002, 4)
    if n >= 14:
        d[12:14] = rng.normal(0, 0.02, 2)
    return d


def _stereo(name, W, H, T, rng):
    K1, K2 = _K(900, W, H, (3.5, -2.25)), _K(905, W, H, (-1.75, 4.5))
    D1, D2 = _pinhole_D(rng, 5), _pinhole_D(rng, 5)
    R = cv2.Rodrigues(np.array([0.01, -0.02, 0.005]))[0]
    R1, R2, P1, P2, *_ = cv2.stereoRectify(K1, D1, K2, D2, (W, H), R, np.array(T, np.float64))
    return [FloatCase(f"{name}_left", 1, K1, D1, R1, P1[:, :3].copy(), W, H, W, H),
            FloatCase(f"{name}_right", 1, K2, D2, R2, P2[:, :3].copy(), W, H, W, H)]


@functools.lru_cache(maxsize=None)
def corpus() -> tuple:
    rng = np.random.default_rng(20261018)
    cases = []
    cases += _stereo("stereo", 1280, 720, [-0.12, 0.001, 0.002], rng)
    cases += _stereo("stereo_vertical", 640, 481, [0.002, -0.1, 0.001], rng)
    for i, (n, W, H) in enumerate([(4, 640, 480), (5, 641, 360), (8, 327, 240), (12, 200, 151), (14, 263, 199)]):
        K = _K(0.8 * W, W, H, rng.normal(0, 4, 2))
        D = _pinhole_D(rng, n)
        P = _K(0.7 * W, W, H)
        cases.append(FloatCase(f"pinhole{n}", 1, K, D, None, P, W, H, W, H))
        cases.append(FloatCase(f"pinhole{n}_R", 1, K, D, _rot(rng, 0.15 + 0.05 * i), P, W, H, W, H))
    cases.append(FloatCase("pinhole5_row", 1, _K(300, 640, 480), _pinhole_D(rng, 5), _rot(rng, 0.1), _K(250, 640, 1), 640, 1,
                           640, 480))
    for name, W, H, R, fs in [("fisheye", 1280, 1024, None, 0.5), ("fisheye_R", 801, 600, _rot(rng, 0.3), 0.6),
                              ("fisheye_behind", 647, 480, _rot(rng, 1.2), 0.25)]:
        K = _K(0.3 * W, W, H, rng.normal(0, 3, 2))
        D = rng.normal(0, [0.05, 0.01, 0.005, 0.001])
        cases.append(FloatCase(name, 0, K, D, R, _K(fs * 0.3 * W, W, H), W, H, W, H))
    return tuple(cases)


def case_by_name(name: str) -> FloatCase:
    return next(c for c in corpus() if c.name == name)


@functools.lru_cache(maxsize=None)
def cv2_maps(name: str, m1type: int):
    """cv2's maps of a case: (map1, map2), map2 None for CV_32FC2."""
    c = case_by_name(name)
    R = np.eye(3) if c.R is None else c.R
    if c.fisheye:
        m1, m2 = cv2.fisheye.initUndistortRectifyMap(c.K, c.D.reshape(-1, 1), R, c.P, (c.W, c.H), m1type)
    else:
        m1, m2 = cv2.initUndistortRectifyMap(c.K, c.D, R, c.P, (c.W, c.H), m1type)
    return m1, (m2 if m2 is not None and m2.size else None)


def frames(c: FloatCase, channels: int, n: int = 1, seed: int = 5):
    """n random frames the size the case's map samples."""
    rng = np.random.default_rng(seed + c.W)
    return rng.integers(0, 256, (n, c.SH, c.SW, channels), dtype=np.uint8)


def special_values() -> np.ndarray:
    """float32 values at the conversion's edges."""
    f = np.float32
    ties32 = (np.arange(-40, 40) + 0.5) / 32            # x * 32 at k + 0.5
    ties = np.arange(-6, 6) + 0.5                        # x at k + 0.5 (NEAREST)
    big = [np.nan, np.inf, -np.inf, 3e9, -3e9, 2147483520.0, -2147483648.0, 2147483648.0]
    edges = []
    for e in (32767 / 32, -32767 / 32, 32768 / 32, -32768 / 32, 32767, -32767, 32767.5, -32768.5, 32768, -32768, 40000.5,
              -40000.5, 67108863.0, -67108864.0):
        e = f(e)
        edges += [e, np.nextafter(e, f(np.inf)), np.nextafter(e, f(-np.inf))]
    return np.concatenate([np.asarray(ties32, f), np.asarray(ties, f), np.asarray(big, f), np.asarray(edges, f)])


def synthetic_maps(W: int, H: int, SW: int, SH: int, seed: int):
    """A W x H CV_32FC1 pair (x, y) over an SW x SH frame: uniform positions around and inside the frame, ties on a
    third of the entries, and special_values() scattered through both planes."""
    rng = np.random.default_rng(seed)
    x = rng.uniform(-4, SW + 4, (H, W)).astype(np.float32)
    y = rng.uniform(-4, SH + 4, (H, W)).astype(np.float32)
    t = rng.random((H, W)) < 0.33
    x[t] = (np.round(x[t] * 32) + 0.5) / 32
    y[t] = (np.round(y[t]) + 0.5)[:]
    sv = special_values()
    for p in (x, y):
        idx = rng.choice(W * H, size=min(W * H, 3 * sv.size), replace=False)
        p.reshape(-1)[idx] = np.resize(sv, idx.size)
    return x, y


def synthetic() -> tuple:
    """(name, x, y, SW, SH) of the synthetic maps: widths with W % 8 of 0, 1 and 7 and a 1xN map."""
    return tuple((f"synthetic_{W}x{H}", *synthetic_maps(W, H, SW, SH, W * 7 + H), SW, SH)
                 for W, H, SW, SH in [(64, 48, 60, 40), (129, 33, 100, 40), (71, 40, 50, 64), (257, 1, 200, 3)])


def classes() -> dict:
    """What the corpus reaches, class by class."""
    cs = corpus()
    pin = [c for c in cs if not c.fisheye]
    fish = [c for c in cs if c.fisheye]
    sv = np.concatenate([np.concatenate([x.ravel(), y.ravel()]) for _, x, y, _, _ in synthetic()])
    fin = sv[np.isfinite(sv)].astype(np.float64)
    x32 = fin * 32
    return {
        "pinhole_n": {c.D.size for c in pin},
        "pinhole_n_with_R": {c.D.size for c in pin if c.R is not None},
        "pinhole_n_without_R": {c.D.size for c in pin if c.R is None},
        "stereo_vertical": sum(c.name.startswith("stereo_vertical") for c in pin),
        "stereo": sum(c.name.startswith("stereo_") and not c.name.startswith("stereo_vertical") for c in pin),
        "fisheye_R": sum(c.R is not None for c in fish),
        "fisheye_no_R": sum(c.R is None for c in fish),
        "fisheye_inf": sum(bool(np.isinf(cv2_maps(c.name, cv2.CV_32FC1)[0]).any()) for c in fish),
        "w_mod8": {c.W % 8 for c in cs} | {x.shape[1] % 8 for _, x, _, _, _ in synthetic()},
        "one_row": sum(c.H == 1 for c in cs) + sum(x.shape[0] == 1 for _, x, _, _, _ in synthetic()),
        "tie32": int(((x32 - np.floor(x32)) == 0.5).sum()),
        "tie1": int(((fin - np.floor(fin)) == 0.5).sum()),
        "nan": int(np.isnan(sv).sum()),
        "inf": int((sv == np.inf).sum()),
        "-inf": int((sv == -np.inf).sum()),
        "3e9": int((np.abs(fin) == np.float32(3e9)).sum()),
        "near_1024": int((np.abs(np.abs(fin) - 32767 / 32) < 1e-3).sum()),
        "near_32768": int((np.abs(np.abs(fin) - 32768) < 1e-2).sum()),
        "near_32767": int((np.abs(np.abs(fin) - 32767) < 1e-2).sum()),
    }


def same(a, b) -> bool:
    """Bit for bit, NaNs included; None only equals None."""
    if a is None or b is None:
        return a is None and b is None
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def planes(m):
    """The x and y planes of a CV_32FC1 pair or a CV_32FC2 map."""
    return (m[0], m[1]) if m[1] is not None else (m[0][..., 0], m[0][..., 1])


def far_outside_only(c: FloatCase, got, want) -> bool:
    """Where a pinhole float map differs from cv2's, both values lie at least 8 pixels outside the frame on that axis,
    where no interpolation reads a pixel.  cv2 compiles the pinhole map in its AVX2 dispatch unit with contracted FMAs
    (DESIGN.md section 7), which moves last bits; the fisheye must match exactly."""
    if c.fisheye:
        return False
    for g, w, size in zip(planes(got), planes(want), (c.SW, c.SH)):
        d = g != w
        out = lambda v: (v < -8) | (v > size + 8)
        if not (out(g[d]) & out(w[d])).all():
            return False
    return True
