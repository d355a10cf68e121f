"""The YUV plane descriptor on the CPU: tests/host/yuv_planes.cu runs the host forms of k_yuv_spans' work item and
k_vsum_yuv's over frames given as separate, pitched planes (YuvFrame), from the library's headers, and this file compares
them with live cv2: cv2.cvtColorTwoPlane(y, uv, COLOR_YUV2BGR_NV12) on the pitched views, cv2.cvtColor(COLOR_YUV2BGR_I420)
of the reassembled buffer, then the oracle's luminance_balance.  cv2's single buffer must be one instance of the
descriptor, giving the chroma addresses yuv_chroma_rows gives."""
import subprocess

import numpy as np
import pytest

from oracle import cv2_path as C
from tests import bev_cases as B
from tests import yuv_frames as Y
from tests import yuv_planes as P
from tests.test_host_yuv import GEOMETRIES, _build

POISON = 0xA5


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return _build(tmp_path_factory, "yuv_planes")


def _layout(exe, fmt, FW, FH):
    r = subprocess.run([exe, "layout", str(Y.FMT_CODE[fmt]), str(FW), str(FH)], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, (fmt, FW, FH, r.stdout[-2000:], r.stderr[-2000:])
    assert "fails=0" in r.stdout


def test_dense_instance_is_cv2s_single_buffer(exe):
    """For both formats and every chroma row, the dense instance of the descriptor (offsets {0, FH*FW(, FH*FW*5/4)},
    pitches {FW, FW or FW/2(, FW/2)}) addresses the bytes yuv_chroma_rows addresses, at the fixture geometry, cfg2-cfg4
    and every size of the YUV corpus (FW % 4 == 2 and FH % 4 == 2 among them)."""
    sizes = {(FW, FH) for _, FW, FH, _, _, _ in GEOMETRIES} | {(c.FW, c.FH) for c in B.yuv_corpus()}
    assert {FW % 4 for FW, _ in sizes} == {0, 2} and {FH % 4 for _, FH in sizes} == {0, 2}
    for FW, FH in sorted(sizes):
        for fmt in Y.FORMATS:
            _layout(exe, fmt, FW, FH)


def _spans(rng, NC, FW, FH):
    """Spans that start and end anywhere, some rows empty, some whole."""
    a = rng.integers(0, FW + 1, (NC, FH, 2))
    sp = np.sort(a, axis=-1).astype(np.int32)
    sp[:, ::7] = (0, FW)
    sp[:, 3::11] = (5, 5)
    return sp


def _run(exe, tmp_path, s: P.Surfaces, arena, spans, balance):
    """The harness on the surfaces' frames read from `arena`; returns (copy stack [n][FH][FW][3], parsed stdout)."""
    n, FW, FH = s.n, s.FW, s.FH
    geo = np.zeros((n, 6), np.int64)
    geo[:, :s.off.shape[1]] = s.off
    geo[:, 3:6] = s.pitch
    if s.fmt == "nv12":
        geo[:, 2] = s.off[:, 1]
    parts = [np.array([n, FW, FH, int(balance), arena.size], np.int64).tobytes(), geo.tobytes(),
             np.ascontiguousarray(spans, np.int32).tobytes(), arena.tobytes()]
    (tmp_path / "p_in.bin").write_bytes(b"".join(parts))
    r = subprocess.run([exe, "run", str(Y.FMT_CODE[s.fmt]), str(tmp_path / "p_in.bin"), str(tmp_path / "p_out.bin")],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (s.fmt, FW, FH, r.returncode, r.stdout[-3000:], r.stderr[-2000:])
    info = {}
    for ln in r.stdout.splitlines():
        if ":" in ln:
            k, v = ln.split(":", 1)
            info[k] = v.split()
    return np.fromfile(tmp_path / "p_out.bin", np.uint8).reshape(n, FH, FW, 3), info


def _converted(spans, FW):
    NC, FH, _ = spans.shape
    x = np.arange(FW)
    lo = (spans[..., 0] >> 2) * 4
    hi = np.where(spans[..., 1] > spans[..., 0], np.minimum(FW, ((spans[..., 1] + 3) >> 2) * 4), lo)
    return (x >= lo[..., None]) & (x < hi[..., None])


def _check(exe, tmp_path, s, spans, balance, what):
    """Converted pixels equal cv2's conversion of the pitched planes (luminance-balanced with BALANCE), V sums equal
    the converted frames', nothing outside the converted groups is written, no read leaves the plane rectangles, and
    changing the padding changes nothing."""
    got, info = _run(exe, tmp_path, s, s.arena, spans, balance)
    assert int(info["audit"][1].split("=")[1]) == 0, (what, info["audit"])
    bgr = [s.bgr(i) for i in range(s.n)]
    assert [int(v) for v in info["vsum"]] == [int(b.max(-1).sum(dtype=np.int64)) for b in bgr], what
    want = C.luminance_balance(bgr) if balance else bgr
    conv = _converted(spans, s.FW)
    for k in range(s.n):
        assert (got[k][conv[k]] == want[k][conv[k]]).all(), (what, balance, k)
        assert (got[k][~conv[k]] == POISON).all(), (what, balance, k)
    rng = np.random.default_rng(s.arena.size)
    for value in (0x5A, rng.integers(0, 256, int(s.pad.sum()), dtype=np.uint8)):
        again, info2 = _run(exe, tmp_path, s, s.poisoned(value), spans, balance)
        assert (again == got).all() and info2["vsum"] == info["vsum"], (what, "padding reached the result")


@pytest.mark.parametrize("fmt", Y.FORMATS)
@pytest.mark.parametrize("FW,FH", [(64, 48), (30, 18), (98, 54)])
def test_pitched_planes_against_cv2(exe, tmp_path, fmt, FW, FH):
    """Four random frames in every layout: pitches FW, FW + 1, FW + 16 and a power of two; chroma directly after Y, after
    8 or 16 padding rows, before Y, in a separate allocation, and (I420) U and V apart; frame blocks at an odd base and
    an odd stride; with and without BALANCE.  Widths with a last group of 2 pixels, heights whose I420 V plane starts
    mid-row in the dense layout."""
    rng = np.random.default_rng(FW * FH + len(fmt))
    frames = [Y.random_yuv(rng, FW, FH) for _ in range(4)]
    spans = _spans(rng, 4, FW, FH)
    for pitch in P.PITCHES:
        for place in P.PLACES:
            for base, extra in ((0, 0), (1, 3)):
                s = P.build(frames, fmt, pitch, place, base, extra)
                for i in range(4):   # the arena holds the frames
                    assert (P.dense(s, i) == frames[i]).all()
                for balance in (False, True):
                    _check(exe, tmp_path, s, spans, balance, (fmt, pitch, place, base, extra))


@pytest.mark.parametrize("fmt", Y.FORMATS)
def test_twoplane_conversion_of_pitched_views_is_the_dense_one(fmt):
    """The oracle's premise: cv2's conversion of pitched planes equals cv2.cvtColor of the dense buffer."""
    rng = np.random.default_rng(3)
    for FW, FH in ((64, 48), (1920, 1080)):
        frames = [Y.random_yuv(rng, FW, FH)]
        s = P.build(frames, fmt, "pow2", "pad8", 1, 3)
        assert (s.bgr(0) == Y.to_bgr(frames[0], fmt)).all(), (FW, FH)


def test_decoder_surfaces_at_the_bench_geometry(exe, tmp_path, fx):
    """The bench's frames (1920 x 1080, the fixture's cameras) as 1080p decoder surfaces: pitch 2048, chroma after the
    1088-row coded height, with BALANCE, in both formats, converted over whole rows."""
    bgr_in = fx.frames(1920, 1080)
    spans = np.tile(np.array([0, 1920], np.int32), (4, 1080, 1))
    for fmt in Y.FORMATS:
        s = P.build([Y.from_bgr(f, fmt) for f in bgr_in], fmt, "pow2", "pad8")
        assert s.pitch[0] == 2048 and s.off[0, 1] - s.off[0, 0] == 1088 * 2048
        _check(exe, tmp_path, s, spans, True, (fmt, "bench"))
