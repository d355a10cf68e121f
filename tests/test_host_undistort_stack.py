"""The batched stand-alone gathers on the CPU.  tests/host/undistort_stack.cu drives the per-thread bodies of k_gather and
k_gather4 (gather_frames / gather4_frames, from the library's headers) over the device's grid -- frame groups of
GATHER_NB in grid z -- on small batches with padded row pitches, padded image strides and unaligned bases, through a
resident map (MODE 0) or the camera model (MODE 1).  Every frame must equal cv2.remap of that frame through the
reference's maps, and the destination's padding must keep its fill.  Every tap load is audited against the frame
layout; `audit` checks that the word path's 32-bit loads never leave the taps' own rows (rounded out to whole words) at
every right-edge byte phase, which is why caller frames need no slack after them.  nvcc compiles the harness; only host
code runs."""
import os
import shutil
import struct
import subprocess

import cv2
import numpy as np
import pytest

from cameracalibration_b200.build import GENCODE
from oracle import cv2_path as C

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FILL = 0xA5


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    nvcc = next((c for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc") if c and os.path.exists(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("host_undistort_stack") / "undistort_stack"
    build = subprocess.run([nvcc, "-O2", "-std=c++17", "--fmad=false", "-Xcompiler", "-ffp-contract=off", *GENCODE, "-o", str(out),
                            os.path.join(ROOT, "tests", "host", "undistort_stack.cu")], capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stdout + build.stderr
    return str(out)


def _span(n, h, w, ch, row, img):
    return (n - 1) * img + (h - 1) * row + w * ch


def _case(rng, fx, *, mode, model, ch, linear, sw, sh, dw, dh, n, row_pad, img_pad, off, drow_pad, dimg_pad):
    """One record for the harness and what it must produce."""
    K, D, _ = fx.calib["front"]
    Ks = np.diag([sw / 1280, sh / 1024, 1.0]) @ K
    P = C.dst_camera_matrix(Ks, dw, dh, 0.5, 1)
    if model == "fisheye":
        d5 = np.r_[np.asarray(D, np.float64).ravel()[:4], 0.0]
        m1, m2 = C.undistort_maps(Ks, D, P, dw, dh)
    else:
        d5 = np.asarray(fx.D5, np.float64).ravel()
        m1, m2 = C.pinhole_maps(Ks, d5, P, dw, dh)
    srow, drow = sw * ch + row_pad, dw * ch + drow_pad
    simg, dimg = sh * srow + img_pad, dh * drow + dimg_pad
    sbytes, dbytes = _span(n, sh, sw, ch, srow, simg), _span(n, dh, dw, ch, drow, dimg)
    src = rng.integers(0, 256, sbytes, dtype=np.uint8)      # padding holds noise: a tap that reads it shows up
    frames = [np.lib.stride_tricks.as_strided(src[f * simg:], (sh, sw, ch), (srow, ch, 1)).copy() for f in range(n)]
    words = int(ch == 3 and linear and dw % 4 == 0 and off == 0 and srow % 4 == 0 and drow % 4 == 0
                and (n == 1 or (simg % 4 == 0 and dimg % 4 == 0)))
    rec = struct.pack("<10i", mode, ch, linear, words, sw, sh, dw, dh, n, off) + struct.pack("<4q", srow, simg, drow, dimg)
    if mode == 0:
        rec += np.ascontiguousarray(m1, np.int16).tobytes() + np.ascontiguousarray(m2, np.uint16).tobytes()
    else:
        model_id = 0.0 if model == "fisheye" else 1.0
        rec += np.r_[Ks.ravel(), d5, P.ravel(), model_id].astype("<f8").tobytes()
    rec += src.tobytes() + np.full(dbytes, FILL, np.uint8).tobytes()
    interp = cv2.INTER_LINEAR if linear else cv2.INTER_NEAREST
    want = [cv2.remap(f, m1, m2, interp).reshape(dh, dw, ch) for f in frames]
    return rec, dict(n=n, dh=dh, dw=dw, ch=ch, drow=drow, dimg=dimg, dbytes=dbytes, want=want, words=words)


def _run(exe, tmp_path, cases):
    (tmp_path / "in.bin").write_bytes(b"".join(r for r, _ in cases))
    r = subprocess.run([exe, "run", str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr[-2000:])
    raw, p = np.fromfile(tmp_path / "out.bin", np.uint8), 0
    for _, c in cases:
        out = raw[p:p + c["dbytes"]]
        p += c["dbytes"]
        touched = np.zeros(c["dbytes"], bool)
        for f in range(c["n"]):
            view = np.lib.stride_tricks.as_strided(out[f * c["dimg"]:], (c["dh"], c["dw"], c["ch"]), (c["drow"], c["ch"], 1))
            assert (view == c["want"][f]).all(), (f, {k: v for k, v in c.items() if k != "want"}, int((view != c["want"][f]).sum()))
            np.lib.stride_tricks.as_strided(touched[f * c["dimg"]:], view.shape, view.strides)[...] = True
        assert (out[~touched] == FILL).all(), "destination padding was written"
    assert p == raw.size
    return r.stdout


def test_word_audit_at_every_right_edge_phase(exe):
    r = subprocess.run([exe, "audit"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (r.stdout, r.stderr[-2000:])
    stats = dict(kv.split("=") for kv in r.stdout.split(":", 1)[1].split())
    assert int(stats["bad"]) == 0 and int(stats["words"]) > 0 and int(stats["bytes"]) > 0
    assert all(int(v) > 0 for v in stats["edge_phases"].split(",")), stats   # every off % 4 at the right edge


@pytest.mark.parametrize("mode", [0, 1])
def test_batched_word_path_against_cv2(exe, tmp_path, fx, mode):
    """3-channel INTER_LINEAR, dw % 4 == 0, 4-byte aligned layouts: the k_gather4 body, batches across the NB tails."""
    rng = np.random.default_rng(100 + mode)
    cases = []
    for i, n in enumerate((1, 3, 4, 5, 9)):
        for model in ("fisheye", "pinhole"):
            sw, sh = int(rng.integers(9, 48)), int(rng.integers(5, 40))
            dw, dh = 4 * int(rng.integers(2, 14)), int(rng.integers(3, 30))
            cases.append(_case(rng, fx, mode=mode, model=model, ch=3, linear=1, sw=sw, sh=sh, dw=dw, dh=dh, n=n,
                               row_pad=[0, 4, 8][i % 3] + (4 - (3 * sw) % 4) % 4, img_pad=4 * (i % 2),
                               off=0, drow_pad=4 * (i % 2), dimg_pad=8 * ((i + 1) % 2)))
    assert all(c["words"] for _, c in cases)
    out = _run(exe, tmp_path, cases)
    assert "bad=0" in out


@pytest.mark.parametrize("mode", [0, 1])
def test_batched_byte_path_against_cv2(exe, tmp_path, fx, mode):
    """The k_gather body: 1/3/4 channels, both interpolations, odd pitches and bases, dw % 4 != 0."""
    rng = np.random.default_rng(200 + mode)
    cases = []
    for i, n in enumerate((1, 3, 4, 5, 9, 2)):
        for ch in (1, 3, 4):
            for linear in (0, 1):
                model = ("fisheye", "pinhole")[(i + ch) % 2]
                sw, sh = int(rng.integers(5, 40)), int(rng.integers(5, 30))
                dw, dh = int(rng.integers(3, 37)), int(rng.integers(3, 25))
                cases.append(_case(rng, fx, mode=mode, model=model, ch=ch, linear=linear, sw=sw, sh=sh, dw=dw, dh=dh, n=n,
                                   row_pad=int(rng.integers(0, 7)), img_pad=int(rng.integers(0, 9)), off=i % 4,
                                   drow_pad=int(rng.integers(0, 5)), dimg_pad=int(rng.integers(0, 6))))
    _run(exe, tmp_path, cases)
