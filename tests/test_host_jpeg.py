"""The device JPEG encoder's arithmetic on the CPU.  tests/host/jpeg_enc.cu runs the __host__ __device__ stage functions
of bevk_jpeg_enc.cuh (sampling and edge rules, islow FDCT, quantisation, dummy blocks, DC prediction, Huffman codes, the
bit writer, byte stuffing, header) serially over whole images; its streams must equal cv2.imencode's byte for byte, and
stay under bevk_jpeg_encode_bound.  nvcc compiles it; only host code runs."""
import os
import shutil
import struct
import subprocess

import cv2
import numpy as np
import pytest

from cameracalibration_b200.build import GENCODE
from oracle import cv2_path as C
from tests.helpers import NAMES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = [(1, 1), (2, 2), (16, 16), (9, 17), (37, 23), (50, 31), (50, 30), (24, 40), (42, 26), (64, 48), (200, 120),
         (18, 48), (130, 64)]                                        # (w, h)
QUALITIES = [-5, 0, 1, 10, 50, 75, 95, 100, 150, None]            # None: cv2's default


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    nvcc = next((c for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc") if c and os.path.exists(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("host_jpeg") / "jpeg_enc"
    build = subprocess.run([nvcc, "-O2", "-std=c++17", *GENCODE, "-o", str(out), os.path.join(ROOT, "tests", "host", "jpeg_enc.cu")],
                           capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stdout + build.stderr
    return str(out)


def _cv2(img, q):
    params = [] if q is None else [cv2.IMWRITE_JPEG_QUALITY, q]
    return cv2.imencode(".jpg", img, params)[1].tobytes()


def _host_encode(exe, tmp_path, cases):
    """cases: [(BGR image, quality or None)] -> [(stream, bound, entropy bits without the pad)] from the host build of
    the encoder."""
    blob = [struct.pack("<3i", img.shape[1], img.shape[0], 95 if q is None else q) + np.ascontiguousarray(img).tobytes()
            for img, q in cases]
    (tmp_path / "jpeg_in.bin").write_bytes(b"".join(blob))
    r = subprocess.run([exe, str(tmp_path / "jpeg_in.bin"), str(tmp_path / "jpeg_out.bin")], capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, (r.returncode, r.stderr[-2000:])
    raw, p, out = (tmp_path / "jpeg_out.bin").read_bytes(), 0, []
    for _ in cases:
        n, bound, bits = struct.unpack_from("<3Q", raw, p)
        out.append((raw[p + 24:p + 24 + n], bound, bits))
        p += 24 + n
    assert p == len(raw)
    return out


def _check(exe, tmp_path, cases):
    for (img, q), (got, bound, _bits) in zip(cases, _host_encode(exe, tmp_path, cases)):
        want = _cv2(img, q)
        first = next((i for i in range(min(len(got), len(want))) if got[i] != want[i]), None)
        assert got == want, (img.shape, q, len(got), len(want), first)
        assert len(got) <= bound, (img.shape, q, len(got), bound)


def test_size_content_quality_matrix(exe, tmp_path, fx):
    rng = np.random.default_rng(21)
    front = fx.img("front")
    cases = []
    for w, h in SIZES:
        for content in ("random", "fixture", "white"):
            if content == "random":
                img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            elif content == "fixture":
                img = np.ascontiguousarray(front[300:300 + h, 500:500 + w])
            else:
                img = np.full((h, w, 3), 255, np.uint8)
            cases += [(img, q) for q in QUALITIES]
    _check(exe, tmp_path, cases)


def test_every_quality_at_64x48(exe, tmp_path, fx):
    img = np.ascontiguousarray(fx.img("left")[400:448, 600:664])
    _check(exe, tmp_path, [(img, q) for q in range(0, 101)])


def test_largest_size_categories_at_q100(exe, tmp_path):
    """1-pixel checkerboards (largest AC categories) and 0/255 block steps (DC differences of category 11)."""
    yy, xx = np.mgrid[0:64, 0:96]
    checker = (((yy + xx) & 1) * 255).astype(np.uint8)
    steps = ((((yy >> 3) + (xx >> 3)) & 1) * 255).astype(np.uint8)
    colour = np.stack([checker, 255 - checker, steps], axis=-1)
    cases = [(np.repeat(checker[..., None], 3, -1), 100), (np.repeat(steps[..., None], 3, -1), 100), (colour, 100),
             (np.repeat(checker[..., None], 3, -1), 95), (colour, 1)]
    _check(exe, tmp_path, cases)


def test_bev_canvas_and_large_frames(exe, tmp_path, fx):
    """A 1000x1000 BEV canvas rendered by the oracle path, a 2560x2048 undistorted fixture frame (Camera geometry,
    SIZE_SCALE 2) and a 1920x1080 frame, at the qualities the tools use."""
    g = fx.geometry()
    canvas = C.RefBev(fx.calib, g, False, False)(*fx.frames(), fx.car())
    K, D, _ = fx.calib["front"]
    P = C.dst_camera_matrix(K, 1280, 1024, 1, 2)
    und = cv2.remap(fx.img("front"), *C.undistort_maps(K, D, P, 2560, 2048), interpolation=cv2.INTER_LINEAR)
    hd = cv2.resize(fx.img(NAMES[1]), (1920, 1080), interpolation=cv2.INTER_LINEAR)
    _check(exe, tmp_path, [(canvas, 95), (canvas, 100), (und, 100), (und, None), (hd, 90)])
