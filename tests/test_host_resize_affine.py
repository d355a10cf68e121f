"""cv2.resize and cv2.warpAffine on the CPU.  tests/host/resize_affine.cu runs the per-thread bodies of k_resize
(resize_frames) and of the warpAffine gathers (MODE 3 of gather_frames, gather_taps_frames and gather4_frames) over the
device's grid, from the library's own headers, and every image must equal live cv2.resize / cv2.warpAffine byte for byte
over the seeded corpus of tests/resize_affine_cases.py: 1, 3 and 4 channels, sides 1..300 and camera frame sizes, the
dsize and fx / fy forms, integer factors, fractional AREA, random and singular affine matrices, WARP_INVERSE_MAP, every
warp flag and coordinates outside int16.  nvcc compiles the harness; only host code runs."""
import os
import shutil
import struct
import subprocess

import cv2
import numpy as np
import pytest

from cameracalibration_b200.build import GENCODE
from tests import resize_affine_cases as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = {"nearest": 0, "linear": 1, "area_linear": 2, "area_fast": 3, "area": 4}


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    nvcc = next((c for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc") if c and os.path.exists(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("host_resize_affine") / "resize_affine"
    build = subprocess.run([nvcc, "-O2", "-std=c++17", "--fmad=false", "-Xcompiler", "-ffp-contract=off", *GENCODE, "-o", str(out),
                            os.path.join(ROOT, "tests", "host", "resize_affine.cu")], capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stdout + build.stderr
    return str(out)


def _stack(frames, row_pad=0, img_pad=0):
    n, h, w, ch = frames.shape
    srow = w * ch + row_pad
    simg = h * srow + img_pad
    buf = np.random.default_rng(n + h + w).integers(0, 256, (n - 1) * simg + (h - 1) * srow + w * ch, dtype=np.uint8)
    for f in range(n):
        np.lib.stride_tricks.as_strided(buf[f * simg:], (h, w, ch), (srow, ch, 1))[...] = frames[f]
    return buf, srow, simg


def _record(case, frames, word=False, row_pad=0, img_pad=0):
    n, sh, sw, ch = frames.shape
    buf, srow, simg = _stack(frames, row_pad, img_pad)
    dw, dh = case["dsize"]
    if case["op"] == "resize":
        head = struct.pack("<8i", 0, ch, sw, sh, dw, dh, n, case["interp"]) + struct.pack("<2q", srow, simg)
        extra = struct.pack("<2d", case["fx"], case["fy"]) if (dw, dh) == (0, 0) else struct.pack("<2d", 0, 0)
    else:
        head = struct.pack("<8i", 1, ch, sw, sh, dw, dh, n, 0) + struct.pack("<2q", srow, simg)
        extra = np.asarray(case["M"], "<f8").tobytes() + struct.pack("<2i", case["flags"], int(word))
    return head + extra + buf.tobytes()


def _run(exe, tmp_path, recs):
    """Runs the records; returns per record (kind, uint8[n][dh][dw][ch])."""
    (tmp_path / "in.bin").write_bytes(b"".join(r for r, _ in recs))
    r = subprocess.run([exe, "run", str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True,
                       timeout=1800)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr[-2000:])
    raw, p, res = np.fromfile(tmp_path / "out.bin", np.uint8), 0, []
    for _, (n, ch) in recs:
        dw, dh, kind = np.frombuffer(raw[p:p + 12].tobytes(), "<i4")
        p += 12
        k = n * dh * dw * ch
        res.append((int(kind), raw[p:p + k].reshape(n, dh, dw, ch)))
        p += k
    assert p == raw.size
    return res


def _check(exe, tmp_path, cases, **rec):
    recs, frames = [], []
    for c in cases:
        f = R.source(c)
        frames.append(f)
        recs.append((_record(c, f, **rec), (c["n"], c["ch"])))
    kinds = []
    for c, f, (kind, got) in zip(cases, frames, _run(exe, tmp_path, recs)):
        for i in range(c["n"]):
            w = R.want(c, f[i])
            assert got[i].shape == w.shape, (c, got.shape, w.shape)
            bad = got[i] != w
            assert not bad.any(), ({k: v for k, v in c.items() if k != "M"}, c.get("M"), i, int(bad.sum()),
                                   np.argwhere(bad)[:5].tolist())
        kinds.append(kind)
    return kinds


def test_resize_corpus(exe, tmp_path):
    kinds = _check(exe, tmp_path, R.resize_corpus(np.random.default_rng(7)))
    assert set(kinds) == set(KINDS.values())   # every body cv2 picks is exercised


def test_resize_batches_padded(exe, tmp_path):
    """Batches across GATHER_NB (grid-z groups), padded rows and images."""
    rng = np.random.default_rng(8)
    cases = []
    for i, n in enumerate((2, 8, 9, 17)):
        for interp in R.INTERS:
            c = R._resize((1, 3, 4)[i % 3], int(rng.integers(5, 60)), int(rng.integers(5, 60)), (int(rng.integers(3, 70)),
                          int(rng.integers(3, 70))), interp=interp, n=n, seed=600 + i)
            cases.append(c)
    _check(exe, tmp_path, cases, row_pad=3, img_pad=5)


def test_resize_two_forms_differ():
    """The premise of taking the scales and not only the size: fx = 0.37 and dsize = (474, 379) differ on a 1280 x 1024
    frame, and an exact 2x LINEAR downscale is cv2's INTER_AREA."""
    img = R.source(R._resize(3, 1280, 1024, seed=9))[0]
    a = cv2.resize(img, (0, 0), fx=0.37, fy=0.37)
    b = cv2.resize(img, (474, 379))
    assert a.shape == b.shape and (a != b).any()
    assert (cv2.resize(img, (640, 512)) == cv2.resize(img, (640, 512), interpolation=cv2.INTER_AREA)).all()


def test_warp_affine_corpus(exe, tmp_path):
    _check(exe, tmp_path, R.affine_corpus(np.random.default_rng(11)))


def test_warp_affine_word_path_and_batches(exe, tmp_path):
    """The 4-pixel word path (gather4_frames, 3 channels, LINEAR, dw % 4 == 0) and batches over GATHER_NB."""
    rng = np.random.default_rng(12)
    cases = []
    for i, n in enumerate((1, 3, 9)):
        M = [[1 + rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3), rng.uniform(-20, 20)],
             [rng.uniform(-0.3, 0.3), 1 + rng.uniform(-0.3, 0.3), rng.uniform(-20, 20)]]
        cases.append(R._affine(3, 64 + 4 * i, 48, M, (60 + 4 * i, 40), cv2.INTER_LINEAR, n=n, seed=700 + i))
    _check(exe, tmp_path, cases, word=True, row_pad=4, img_pad=8)
    _check(exe, tmp_path, [dict(c, flags=cv2.INTER_CUBIC) for c in cases], row_pad=1, img_pad=3)


def test_reference_scale_factor(exe, tmp_path, fx):
    """ScaleImage's factor from the corners of a board seen through a fixture calibration (the reference's calc_dist,
    run by the shim) resizes a fixture frame as cv2.resize(frame, (0, 0), fx=f, fy=f) does."""
    from cameracalibration_b200.ExtrinsicCalibration import ScaleImage
    from tests.helpers import NAMES
    frame = fx.frames(1280, 1024)[0]
    corners = R.board_corners(fx.calib[NAMES[0]][2])
    f = ScaleImage(corners).scale_factor
    assert 0.05 < f < 20, f
    case = R._resize(3, frame.shape[1], frame.shape[0], fx=f, fy=f, seed=0)
    (kind, got), = _run(exe, tmp_path, [(_record(case, frame[None]), (1, 3))])
    assert (got[0] == cv2.resize(frame, (0, 0), fx=f, fy=f)).all()
