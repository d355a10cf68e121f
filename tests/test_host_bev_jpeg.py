"""The encoder's BALANCE source on the CPU.  tests/host/bev_jpeg.cu encodes a raw composed canvas, its channel sums and an
optional car through GainSrc of bevk_jpeg_enc.cuh -- the gain table the device builds per CTA (gray_world_gains +
gain_entry, as k_gain) and the saturating car, applied while the blocks are loaded -- with the same __host__ __device__
functions the device runs.  Every stream must equal cv2.imencode(cv2.add(color_balance(canvas), car)) byte for byte,
color_balance being the reference's cv2 call sequence.  nvcc compiles the harness; only host code runs."""
import os
import shutil
import struct
import subprocess

import cv2
import numpy as np
import pytest

from cameracalibration_b200.build import GENCODE
from oracle import cv2_path as C
from tests.test_host_jpeg import SIZES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
QUALITIES = (1, 50, 95, 100)


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    nvcc = next((c for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc") if c and os.path.exists(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("host_bev_jpeg") / "bev_jpeg"
    build = subprocess.run([nvcc, "-O2", "-std=c++17", *GENCODE, "-o", str(out), os.path.join(ROOT, "tests", "host", "bev_jpeg.cu")],
                           capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stdout + build.stderr
    return str(out)


def _want(canvas, car, q):
    with np.errstate(divide="ignore", invalid="ignore"):      # a black channel: K / 0, as the reference divides
        img = C.color_balance(canvas.copy())
    if car is not None:
        img = cv2.add(img, car)
    return cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q])[1].tobytes()


def _check(exe, tmp_path, cases):
    """cases: [(raw canvas, car or None, quality)]: the harness's streams against cv2's."""
    blob = []
    for canvas, car, q in cases:
        h, w = canvas.shape[:2]
        csum = canvas.reshape(-1, 3).sum(axis=0, dtype=np.uint64)
        blob.append(struct.pack("<4i", w, h, q, car is not None) + csum.astype("<u8").tobytes() + np.ascontiguousarray(canvas).tobytes()
                    + (b"" if car is None else np.ascontiguousarray(car).tobytes()))
    (tmp_path / "in.bin").write_bytes(b"".join(blob))
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (r.returncode, r.stderr[-2000:])
    raw, p = (tmp_path / "out.bin").read_bytes(), 0
    for canvas, car, q in cases:
        (n,) = struct.unpack_from("<Q", raw, p)
        got = raw[p + 8:p + 8 + n]
        p += 8 + n
        want = _want(canvas, car, q)
        first = next((i for i in range(min(len(got), len(want))) if got[i] != want[i]), None)
        assert got == want, (canvas.shape, car is not None, q, len(got), len(want), first)
    assert p == len(raw)


def _canvas(rng, h, w):
    """Channel means far apart: gains above 1 (blue), near 1 (green) and below 1 (red)."""
    c = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    c[..., 0] //= 3
    c[..., 2] = 128 + c[..., 2] // 2
    return c


def test_odd_sizes_gains_and_car(exe, tmp_path):
    rng = np.random.default_rng(41)
    cases = []
    for i, (w, h) in enumerate(SIZES):
        canvas = _canvas(rng, h, w)
        car = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        car[rng.integers(0, 2, (h, w)) == 0] = 0
        for q in QUALITIES:
            cases.append((canvas, car if (i + q) % 2 else None, q))
    _check(exe, tmp_path, cases)


def test_black_channel_and_saturating_car(exe, tmp_path):
    """A channel that is 0 everywhere: its gain is K / 0 = inf, every entry saturates as on x86 (0 * inf = NaN and
    cvRound(NaN) = INT_MIN -> 0).  A bright car on a bright canvas: the cv2.add saturates."""
    rng = np.random.default_rng(42)
    black = _canvas(rng, 48, 70)
    black[..., 1] = 0
    bright = rng.integers(180, 256, (37, 50, 3), dtype=np.uint8)
    car = rng.integers(150, 256, (37, 50, 3), dtype=np.uint8)
    cases = [(black, None, q) for q in QUALITIES] + [(black, rng.integers(0, 256, black.shape, dtype=np.uint8), 95)]
    cases += [(bright, car, q) for q in QUALITIES]
    _check(exe, tmp_path, cases)


def test_bev_canvas_1000(exe, tmp_path, fx):
    """The 1000 x 1000 canvas the oracle composes from the fixture frames (before colour balance), with the car."""
    g = fx.geometry()
    raw = C.RefBev(fx.calib, g, False, False)(*fx.frames())
    _check(exe, tmp_path, [(raw, fx.car(), 95), (raw, None, 100), (raw, fx.car(), 50)])
