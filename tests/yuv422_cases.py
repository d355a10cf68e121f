"""The packed YUV 4:2:2 corpus (tests/test_host_yuv422.py, tests/test_gpu_yuv422.py): the even-width cases of the BEV
fuzz corpus (tests/bev_cases.py: their maps, masks and car) and a seeded 4:2:2 supplement, each with frame-sets of
YUYV frames uint8[FH][FW][2] in `yuv` (UYVY: the same pixels, tests/yuv422_frames.swap) and no BGR ones; yuv422_case
gives the frames the oracle sees: cv2.cvtColor of every frame, then the BGR oracle of tests/bev_cases.py."""
from __future__ import annotations

from dataclasses import replace
from functools import lru_cache

import numpy as np

from tests import bev_cases as B
from tests import yuv422_frames as Y2

# The 4:2:2 supplement, (kind, FW, FH, (BW, BH), cameras, nearest, bright) as bev_cases' YUV 4:2:0 one: odd heights
# (FH = 1 and 3 among them: cv2 takes any height), FW % 4 == 2 (a last group of 2 pixels) with BALANCE and with NEAREST,
# FW % 32 == 16 with BALANCE (k_bev_tma with the luminance row tail), a 2-pixel-wide frame, 1-8 cameras, int16-extreme
# and edge taps, bright frames.
_SUPPLEMENT = (
    ("local", 30, 37, (52, 68), 4, False, False),
    ("extreme", 98, 1, (77, 45), 4, True, True),
    ("smooth", 48, 131, (100, 90), 4, False, False),
    ("smooth", 118, 199, (150, 118), 4, True, False),
    ("local", 80, 3, (77, 45), 4, False, True),
    ("extreme", 112, 43, (96, 64), 4, False, False),
    ("extreme", 36, 41, (29, 70), 5, False, True),
    ("local", 30, 25, (23, 17), 6, True, False),
    ("extreme", 80, 35, (64, 96), 7, False, False),
    ("smooth", 64, 121, (64, 77), 8, False, True),
    ("local", 98, 29, (96, 64), 3, False, True),
    ("extreme", 118, 21, (77, 45), 2, True, False),
    ("local", 48, 1, (23, 17), 1, False, False),
    ("local", 2, 7, (23, 17), 2, False, True),
)
# frame-sets per case: consecutive checked calls start at set 0 or set 1, as for the YUV 4:2:0 corpus
N_SETS = B.N_YUV_SETS


def _sets(rng, NC, FW, FH, bright):
    """N_SETS independent frame-sets of random YUYV frames (Y < 16 and chroma that saturates the conversion included);
    bright: Y in [200, 256) (saturating adds in the compose)."""
    sets = []
    for _ in range(N_SETS):
        fs = [Y2.random_frame(rng, FW, FH) for _ in range(NC)]
        if bright:
            for f in fs:
                f[..., 0] = rng.integers(200, 256, (FH, FW), dtype=np.uint8)
        sets.append(fs)
    return sets


@lru_cache(maxsize=None)
def yuv422_corpus() -> tuple:
    """Every case of the 4:2:2 corpus (bev_cases.Case with YUYV frame-sets in `yuv`)."""
    out = []
    for s in range(B.N_CASES):
        c = B.make_case(s)
        if c.FW % 2 == 0:
            rng = np.random.default_rng(4000 + s)
            out.append(replace(c, name=f"p{c.name}", sets=[], yuv=_sets(rng, c.NC, c.FW, c.FH, s % 4 in (1, 2))))
    for i, (kind, FW, FH, (BW, BH), NC, nearest, bright) in enumerate(_SUPPLEMENT):
        rng = np.random.default_rng(5000 + i)
        maps = B._maps(rng, kind, NC, FW, FH, BW, BH)
        masks = B._masks(rng, NC, BW, BH, 200 + i)
        car = rng.integers(0, 256, (BH, BW, 3), dtype=np.uint8)
        car[rng.integers(0, 2, (BH, BW)) == 0] = 0
        out.append(B.Case(f"yuv422_{kind}{i}", kind, FW, FH, BW, BH, nearest, maps, masks, [], car,
                          _sets(rng, NC, FW, FH, bright)))
    return tuple(out)


@lru_cache(maxsize=None)
def yuv422_case(name: str, fmt: str) -> B.Case:
    """4:2:2 corpus case `name` with `yuv` in byte order fmt ("yuyv" / "uyvy") and sets = cv2.cvtColor of its frames
    (COLOR_YUV2BGR_YUY2 / _UYVY): what bev_cases.oracle() and compose() take, and what a BGR render of the case reads."""
    c = next(c for c in yuv422_corpus() if c.name == name)
    yuv = c.yuv if fmt == "yuyv" else [[Y2.swap(f) for f in fs] for fs in c.yuv]
    return replace(c, yuv=yuv, sets=[[Y2.to_bgr(f, fmt) for f in fs] for fs in yuv])
