"""Seeded BEV cases shared by the host fuzz (tests/test_host_math.py, tests/test_host_bev_fuzz.py) and the GPU fuzz
(tests/test_gpu_bev_fuzz.py): one seed -> one case (geometry, per-camera CV_16SC2 + CV_16UC1 maps, masks,
interpolation, frame-sets), plus the oracle every consumer compares with: cv2.remap per camera (BORDER_CONSTANT 0),
the mask weight (restate.apply_blend), the saturating compose in camera order, and -- with BALANCE -- the reference's
luminance / colour balance restated, then the car.  Maps are given to the engine through set_maps, so the host
interpreter and the device render exactly the input the oracle sees.

yuv_corpus() carries the same kind of cases with NV12 / I420 frames instead (tests/test_host_yuv.py,
tests/test_gpu_yuv_fuzz.py); its oracle is cv2.cvtColor of every frame followed by the BGR oracle."""
from __future__ import annotations

import os
import re
from dataclasses import dataclass, field, replace
from functools import lru_cache

import cv2
import numpy as np

from oracle import cv2_path as C
from oracle import restate as R
from tests import yuv_frames as Y


@dataclass
class Case:
    name: str
    kind: str                      # "local", "extreme" or "smooth"
    FW: int
    FH: int
    BW: int
    BH: int
    nearest: bool
    maps: list                     # per camera (map1 int16[BH][BW][2], map2 uint16[BH][BW])
    masks: list                    # per camera uint8[BH][BW]
    sets: list = field(default_factory=list)   # frame-sets: list (batch) of lists (camera) of uint8[FH][FW][3]
    car: np.ndarray | None = None
    yuv: list | None = None        # YUV corpus: frame-sets of YUV 4:2:0 buffers uint8[FH*3/2][FW] (sets: see yuv_bgr_case)

    @property
    def NC(self) -> int:
        return len(self.maps)

    @property
    def tma_friendly(self) -> bool:
        """Row pitch a multiple of 16 bytes: bevk_bev_finalize builds a TMA plan."""
        return (self.FW * 3) % 16 == 0


def blob(case: Case, s: int = 0, balance: bool = False, car: bool = False) -> bytes:
    """Input of tests/host/kernel_math.cu `bev` / `bevtma`: frame-set s."""
    out = [np.array([case.NC, case.FW, case.FH, case.BW, case.BH, int(case.nearest), int(balance), int(car)], np.int32).tobytes()]
    for (m1, m2), mk in zip(case.maps, case.masks):
        out += [np.ascontiguousarray(m1, np.int16).tobytes(), np.ascontiguousarray(m2, np.uint16).tobytes(),
                np.ascontiguousarray(mk, np.uint8).tobytes()]
    out += [np.ascontiguousarray(f).tobytes() for f in case.sets[s]]
    if car:
        out.append(np.ascontiguousarray(case.car).tobytes())
    return b"".join(out)


def compose(case: Case, frames, balance: bool = False):
    """The canvas before the car: remap, weight, saturating compose (+ luminance / colour balance).  None when BALANCE
    is undefined for it (a zero channel mean: the reference divides by it)."""
    if balance:
        frames = R.luminance_balance(frames)
    inter = cv2.INTER_NEAREST if case.nearest else cv2.INTER_LINEAR
    out = np.zeros((case.BH, case.BW, 3), np.uint8)
    for f, (m1, m2), mk in zip(frames, case.maps, case.masks):
        warped = cv2.remap(f, m1, m2, inter, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
        out = R.sat_add(out, R.apply_blend(warped, mk))
    if balance:
        if (out.reshape(-1, 3).sum(axis=0) == 0).any():
            return None
        out = R.color_balance(out)
    return out


def oracle(case: Case, s: int, balance: bool = False, car: bool = False):
    out = compose(case, case.sets[s], balance)
    if out is not None and car:
        out = R.sat_add(out, case.car)
    return out


# ------------------------------------------------------------------ the original host fuzz cases
def random_case(rng, case: int) -> Case:
    """Random geometry, maps (every 4th case at the int16 extremes), masks (binary, weighted, all 255) and one frame-set:
    1-3 cameras, tiny ragged canvases, every pitch alignment, both interpolations (every 3rd case nearest)."""
    NC = int(rng.integers(1, 4))
    FW, FH = int(rng.integers(8, 90)), int(rng.integers(8, 70))
    BW, BH = int(rng.integers(5, 80)), int(rng.integers(5, 75))
    nearest = bool(case % 3 == 2)
    frames, maps, masks = [], [], []
    for _ in range(NC):
        lo, hi = (-6, 6) if case % 4 else (-40000, 40000)
        m1 = np.stack([rng.integers(lo, FW + hi, (BH, BW)), rng.integers(lo, FH + hi, (BH, BW))], -1).clip(-32768, 32767).astype(np.int16)
        m2 = rng.integers(0, 1024, (BH, BW)).astype(np.uint16)
        kind = rng.integers(0, 3)
        mask = (rng.integers(0, 2, (BH, BW)) * 255 if kind == 0 else rng.integers(0, 256, (BH, BW)) if kind == 1
                else np.full((BH, BW), 255)).astype(np.uint8)
        maps.append((m1, m2)); masks.append(mask)
        frames.append(rng.integers(0, 256, (FH, FW, 3), dtype=np.uint8))
    return Case(f"random{case}", "extreme" if case % 4 == 0 else "local", FW, FH, BW, BH, nearest, maps, masks, [frames])


# ------------------------------------------------------------------ the fuzz corpus
# frame widths: TMA plan (pitch % 16 == 0), gather kernel (pitch % 4 == 0 only), per-tap path (pitch % 4 != 0); the
# widths with FW % 32 in {1, 16, 31} sample the luminance row-tail rule (OpenCV's scalar tail of 32-pixel rows)
_FW_CLASSES = ((64, 80, 112, 176, 336), (36, 44, 52, 100, 116), (33, 63, 95, 65, 97))
# canvas sizes: below 32, not a multiple of 4, a multiple of 4 but not 32, exact multiples of 32
_CANVAS = ((23, 17), (77, 45), (52, 68), (64, 96), (29, 70), (96, 64))
N_CASES = 30
# the cases every TMA configuration runs: a smooth minified one, a random-local one, an int16-extreme one (all with a
# TMA plan and 4 cameras, so that BALANCE applies)
CONFIG_CASES = ("smooth4", "local5", "extreme4")


def tma_configs():
    """BEVK_TMA_CONFIGS of bevk_api.cu: (stage bytes FS, ring slots, CTAs per SM, entry groups per slot) of every
    k_bev_tma instantiation; BEVK_TMA_CFG selects one as "FS,slots,groups"."""
    src = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "cameracalibration_b200", "csrc", "bevk_api.cu")
    line = next(ln for ln in open(src) if ln.startswith("#define BEVK_TMA_CONFIGS"))
    return [tuple(int(v) for v in m) for m in re.findall(r"X\((\d+), (\d+), (\d+), (\d+)\)", line)]


MAX_MULTS = (1, 2, 4)
DEFAULT_PLAN = (7936, 4, 4)   # (stage bytes, entry groups per slot, largest multi-pass box) of the default engine


def _masks(rng, NC, BW, BH, seed):
    """Per camera: binary wedge, weighted ramp, all 255, or random weights; some overlap above 255.  Camera NC-1 gets an
    all-zero mask and camera NC-2 a single-pixel mask when there are enough cameras; a tile-aligned hole (the car) is
    cut out of every mask on canvases that have more than one tile."""
    yy, xx = np.mgrid[0:BH, 0:BW].astype(np.float64)
    cx, cy = BW / 2, BH / 2
    out = []
    for k in range(NC):
        kind = (seed + k) % 4
        if kind == 0:                                   # binary wedge around the centre, overlapping its neighbours
            a0 = 2 * np.pi * k / NC
            ang = np.mod(np.arctan2(yy - cy, xx - cx) - a0, 2 * np.pi)
            m = np.where(ang < 2 * np.pi / NC * 1.5 + 0.3, 255, 0)
        elif kind == 1:                                 # weighted ramp along a random direction
            t = rng.uniform(0, 2 * np.pi)
            r = (xx - cx) * np.cos(t) + (yy - cy) * np.sin(t)
            m = np.clip(128 + 255 * r / max(BW, BH), 0, 255)
        elif kind == 2:                                 # all 255: FULL items where it is the first camera
            m = np.full((BH, BW), 255)
        else:                                           # random weights (sums above 255 where others overlap)
            m = rng.integers(0, 256, (BH, BW))
        out.append(m.astype(np.uint8))
    if NC >= 3:
        out[NC - 1][:] = 0
        out[NC - 2][:] = 0
        out[NC - 2][int(rng.integers(0, BH)), int(rng.integers(0, BW))] = int(rng.integers(1, 256))
    if BW > 32 and BH > 32:
        for m in out:
            m[:32, :32] = 0
    return out


def _edge_taps(rng, m1, FW, FH):
    """Taps exactly at x = FW-1, y = FH-1 and at -1 (bilinear pairs straddling the frame edges)."""
    BH, BW = m1.shape[:2]
    n = max(1, BW * BH // 8)
    for col, v in ((0, FW - 1), (1, FH - 1), (0, -1), (1, -1)):
        idx = rng.integers(0, BW * BH, n)
        m1.reshape(-1, 2)[idx, col] = v


def _smooth_maps(rng, k, FW, FH, BW, BH):
    """A random fisheye camera seen through a homography that rotates the canvas about its centre (exact 0 / 90 / 180
    degrees for the first three cameras), scales it, and tilts it so that the near field is minified 4-10x: the
    oracle's own Camera.get_bev_maps (cv2.fisheye + cv2.warpPerspective)."""
    K = np.array([[rng.uniform(0.35, 0.7) * FW, 0, FW / 2 + rng.uniform(-8, 8)],
                  [0, rng.uniform(0.35, 0.7) * FW, FH / 2 + rng.uniform(-8, 8)], [0, 0, 1.0]])
    D = rng.uniform(-0.05, 0.05, (4, 1))
    g = C.Geometry(FW=FW, FH=FH, BW=BW, BH=BH)
    theta = (0.0, np.pi / 2, np.pi)[k] if k < 3 else rng.uniform(0, 2 * np.pi)
    c, s = np.cos(theta), np.sin(theta)
    h = BH / 2
    mini = rng.uniform(4, 10)                      # minification of the near edge along canvas y (d v / d y' = sc / w^2)
    ph = rng.uniform(0.3, 0.6)                     # perspective: w = 1 + p y' runs from 1 - ph (near) to 1 + ph (far)
    sc = mini * (1 - ph) ** 2
    rot = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]]) @ np.array([[1, 0, -BW / 2], [0, 1, -BH / 2], [0, 0, 1.0]])
    persp = np.array([[sc, 0, 0], [0, sc, 0], [0, ph / h, 1.0]])
    # y' = -h is the near edge (w small: large source steps); it lands near the undistorted image's centre row
    to_und = np.array([[1, 0, FW + rng.uniform(-20, 20)], [0, 1, FH + sc * h / (1 - ph) * 0.6], [0, 0, 1.0]])
    Hinv = to_und @ persp @ rot
    H = np.linalg.inv(Hinv)
    H /= H[2, 2]
    return C.RefCamera(K, D, H, g).bev_maps


def _maps(rng, kind, NC, FW, FH, BW, BH):
    """Per camera (map1, map2) of a case of this kind: smooth fisheye + homography, random local taps within 6 px of the
    frame, or int16-extreme taps (a band of ordinary ones); local and extreme maps also get the edge taps."""
    maps = []
    for k in range(NC):
        if kind == "smooth":
            m1, m2 = _smooth_maps(rng, k, FW, FH, BW, BH)
            m1 = np.array(m1, np.int16)
        else:
            lo, hi = (-6, 6) if kind == "local" else (-40000, 40000)
            m1 = np.stack([rng.integers(lo, FW + hi, (BH, BW)), rng.integers(lo, FH + hi, (BH, BW))], -1)
            m1 = m1.clip(-32768, 32767).astype(np.int16)
            if kind == "extreme":   # a band of ordinary taps, so that extreme cases still stage some boxes
                m1[: BH // 3] = np.stack([rng.integers(0, FW, (BH // 3, BW)), rng.integers(0, FH, (BH // 3, BW))], -1)
            _edge_taps(rng, m1, FW, FH)
            m2 = rng.integers(0, 1024, (BH, BW)).astype(np.uint16)
        maps.append((m1, np.ascontiguousarray(m2, np.uint16)))
    return maps


def _frames(rng, NC, FW, FH, bright, n_sets):
    base = [rng.integers(160 if bright else 0, 256, (FH, FW, 3), dtype=np.uint8) for _ in range(NC)]
    sets = [base]
    for i in range(1, n_sets):
        sets.append([np.ascontiguousarray(np.roll(f, 31 * i + 7 * c, axis=1) ^ rng.integers(0, 32, f.shape, dtype=np.uint8))
                     for c, f in enumerate(base)])
    return sets


@lru_cache(maxsize=None)
def make_case(seed: int, n_sets: int = 9) -> Case:
    """Case `seed` of the corpus.  Kinds cycle smooth / local / extreme; frame-width classes, canvas sizes, camera counts
    (1-8; 4 -- the reference's arity, which BALANCE needs -- every other case), mask mixes, interpolation and bright
    frames (saturation) cycle with co-prime periods so that every combination class occurs."""
    rng = np.random.default_rng(1000 + seed)
    kind = ("smooth", "local", "extreme")[seed % 3]
    idx = seed // 3
    fw_class = (seed // 3 + seed) % 3 if kind != "smooth" else (0, 0, 1, 2)[idx % 4]
    FW = _FW_CLASSES[fw_class][seed % 5]
    if kind == "smooth":
        FH = int(rng.integers(120, 260))
        BW, BH = ((160, 192), (100, 90), (150, 118), (64, 77))[idx % 4]
    else:
        FH = int(rng.integers(20, 90))
        BW, BH = _CANVAS[idx % 6]
    NC = 4 if seed % 2 == 0 else int((1, 2, 3, 5, 6, 7, 8)[idx % 7])
    nearest = seed % 5 == 3
    maps = _maps(rng, kind, NC, FW, FH, BW, BH)
    masks = _masks(rng, NC, BW, BH, seed)
    bright = seed % 4 in (1, 2)
    sets = _frames(rng, NC, FW, FH, bright, n_sets)
    car = rng.integers(0, 256, (BH, BW, 3), dtype=np.uint8)
    car[rng.integers(0, 2, (BH, BW)) == 0] = 0
    return Case(f"{kind}{idx}", kind, FW, FH, BW, BH, nearest, maps, masks, sets, car)


def corpus():
    return [make_case(s) for s in range(N_CASES)]


def case_by_name(name: str) -> Case:
    return next(c for c in corpus() if c.name == name)


# ------------------------------------------------------------------ the YUV 4:2:0 corpus
# Frame-sets per YUV case: a call of up to 9 sets starts at set 0 or set 1, so that consecutive calls on one engine never
# present the same frame at the same frame index (the copy stack keeps an earlier call's conversion outside the spans).
N_YUV_SETS = 10
# The supplement: (kind, FW, FH, (BW, BH), cameras, nearest, bright).  Widths with FW % 4 == 2 (a last group of 2 pixels,
# a copy-stack pitch that is not a multiple of 4: k_bev's per-tap path), FW % 16 == 4 * k (k_bev on the copy stack, DMA
# rectangles for page-locked frames) and FW % 32 == 16 (k_bev_tma with the luminance row tail; I420 windows crossing
# the U / V halves of a buffer row); heights with FH % 4 == 2 (the I420 V plane starts mid-row); 1-8 cameras.
_YUV_SUPPLEMENT = (
    ("local", 30, 38, (52, 68), 4, False, False),
    ("extreme", 98, 54, (77, 45), 4, True, True),
    ("smooth", 118, 198, (100, 90), 4, False, False),
    ("smooth", 52, 130, (150, 118), 4, True, False),
    ("local", 112, 66, (77, 45), 4, False, True),
    ("smooth", 176, 150, (64, 77), 4, False, False),
    ("extreme", 80, 42, (96, 64), 4, False, False),
    ("extreme", 36, 42, (29, 70), 5, False, True),
    ("local", 30, 26, (23, 17), 6, True, False),
    ("extreme", 80, 34, (64, 96), 7, False, False),
    ("smooth", 64, 122, (64, 77), 8, False, True),
    ("local", 98, 30, (96, 64), 3, False, True),
    ("extreme", 118, 22, (77, 45), 2, True, False),
    ("local", 48, 20, (23, 17), 1, False, False),
)


def _yuv_sets(rng, NC, FW, FH, bright):
    """N_YUV_SETS independent frame-sets of random YUV 4:2:0 buffers (Y < 16 and chroma that saturates the conversion
    included); bright: Y in [200, 256) (saturating adds in the compose)."""
    sets = []
    for _ in range(N_YUV_SETS):
        fs = [Y.random_yuv(rng, FW, FH) for _ in range(NC)]
        if bright:
            for f in fs:
                f[:FH] = rng.integers(200, 256, (FH, FW), dtype=np.uint8)
        sets.append(fs)
    return sets


@lru_cache(maxsize=None)
def yuv_corpus() -> tuple:
    """The even-sized cases of corpus() (their maps, masks and car; bright frames where the BGR case has them) and the
    seeded supplement, each with YUV frame-sets in `yuv` and no BGR ones: yuv_bgr_case gives the frames the oracle sees."""
    out = []
    for s in range(N_CASES):
        c = make_case(s)
        if c.FW % 2 == 0 and c.FH % 2 == 0:
            rng = np.random.default_rng(2000 + s)
            out.append(replace(c, sets=[], yuv=_yuv_sets(rng, c.NC, c.FW, c.FH, s % 4 in (1, 2))))
    for i, (kind, FW, FH, (BW, BH), NC, nearest, bright) in enumerate(_YUV_SUPPLEMENT):
        rng = np.random.default_rng(3000 + i)
        maps = _maps(rng, kind, NC, FW, FH, BW, BH)
        masks = _masks(rng, NC, BW, BH, 100 + i)
        car = rng.integers(0, 256, (BH, BW, 3), dtype=np.uint8)
        car[rng.integers(0, 2, (BH, BW)) == 0] = 0
        out.append(Case(f"yuv_{kind}{i}", kind, FW, FH, BW, BH, nearest, maps, masks, [], car,
                        _yuv_sets(rng, NC, FW, FH, bright)))
    return tuple(out)


@lru_cache(maxsize=None)
def yuv_bgr_case(name: str, fmt: str) -> Case:
    """YUV corpus case `name` with sets = cv2.cvtColor(COLOR_YUV2BGR_NV12 / _I420) of its YUV frame-sets: what oracle()
    and compose() take, and what a BGR render of the same case reads."""
    c = next(c for c in yuv_corpus() if c.name == name)
    return replace(c, sets=[[Y.to_bgr(f, fmt) for f in fs] for fs in c.yuv])
