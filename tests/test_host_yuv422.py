"""The packed YUV 4:2:2 source path (YUYV, UYVY) on the CPU: tests/host/yuv422.cu runs the host forms of the conversion
pre-pass (k_yuv_spans' work item), of the 4:2:2 V sum (k_vsum_yuv's) and of the ingest plan (bevk_plan.cuh) from the
library's headers, and this file compares them with live cv2: cv2.cvtColor(COLOR_YUV2BGR_YUY2 / _UYVY), then the
oracle's luminance_balance.  The copy stack the conversion leaves also goes through the host interpreters of the
render's plans (tests/host/kernel_math.cu), to show that the render reads nothing the conversion did not write."""
import subprocess
from dataclasses import replace

import numpy as np
import pytest

from oracle import cv2_path as C
from oracle import restate as R
from tests import bev_cases as B
from tests import yuv422_cases as YC
from tests import yuv422_frames as Y2
from tests.helpers import NAMES
from tests.test_host_yuv import GEOMETRIES, _build, _converted

POISON = 0xA5


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return _build(tmp_path_factory, "yuv422")


@pytest.fixture(scope="module")
def kernel_math(tmp_path_factory):
    return _build(tmp_path_factory, "kernel_math")


def _info(stdout):
    info = {}
    for ln in stdout.splitlines():
        if ":" in ln:
            k, v = ln.split(":", 1)
            info[k] = v.split()
    return info


def _run(exe, tmp_path, fmt, frames, FW, FH, balance=False, maps=None, masks=None, BW=0, BH=0, nearest=False):
    """`yuv422 plan` on NC packed frames; returns (copy stack [NC][FH][FW][3], spans [NC][FH][2], parsed stdout)."""
    NC = len(frames)
    parts = [np.array([NC, FW, FH, BW, BH, int(nearest), int(balance), int(maps is not None)], np.int32).tobytes()]
    if maps is not None:
        for (m1, m2), mk in zip(maps, masks):
            parts += [np.ascontiguousarray(m1, np.int16).tobytes(), np.ascontiguousarray(m2, np.uint16).tobytes(),
                      np.ascontiguousarray(mk, np.uint8).tobytes()]
    parts += [np.ascontiguousarray(f).tobytes() for f in frames]
    (tmp_path / "in.bin").write_bytes(b"".join(parts))
    r = subprocess.run([exe, "plan", str(Y2.FMT_CODE[fmt]), str(tmp_path / "in.bin"), str(tmp_path / "out.bin")],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (fmt, FW, FH, r.returncode, r.stdout[-3000:], r.stderr[-2000:])
    raw = np.fromfile(tmp_path / "out.bin", np.uint8)
    n = NC * FH * FW * 3
    return raw[:n].reshape(NC, FH, FW, 3), raw[n:].view(np.int32).reshape(NC, FH, 2), _info(r.stdout)


def _vsums(bgr):
    return [int(b.max(-1).sum(dtype=np.int64)) for b in bgr]


@pytest.mark.parametrize("fmt", Y2.FORMATS)
def test_yuv_bgr_every_triple_against_cv2(exe, tmp_path, fmt):
    """yuv_bgr and the packed byte positions, through the pre-pass over whole rows, for all 2^24 (Y, U, V) triples
    (both pixels of a pair take its U and V)."""
    f = Y2.every_triple(fmt)
    got, _, _ = _run(exe, tmp_path, fmt, [f], 4096, 4096)
    want = Y2.to_bgr(f, fmt)
    assert (got[0] == want).all(), int((got[0] != want).any(-1).sum())


@pytest.mark.parametrize("FW", [2, 6, 34, 38, 66, 64, 48])
def test_small_and_ragged_frames_against_cv2(exe, tmp_path, FW):
    """Widths with a last group of 2 pixels (FW % 4 == 2), widths around the 32-pixel row tail of luminance_balance,
    odd heights (1 and 3 among them, as cv2 takes them), whole-row spans, with and without BALANCE (four frames)."""
    for FH in (1, 3, 17, 24):
        rng = np.random.default_rng(FW * 100 + FH)
        for fmt in Y2.FORMATS:
            frames = [Y2.random_frame(rng, FW, FH) for _ in range(4)]
            bgr = [Y2.to_bgr(f, fmt) for f in frames]
            for balance in (False, True):
                got, _, info = _run(exe, tmp_path, fmt, frames, FW, FH, balance)
                want = C.luminance_balance(bgr) if balance else bgr
                assert [int(v) for v in info["vsum"]] == _vsums(bgr), (FW, FH, fmt)
                for k in range(4):
                    assert (got[k] == want[k]).all(), (FW, FH, fmt, balance, k)


@pytest.mark.parametrize("name,FW,FH,BW,BH,blend", GEOMETRIES)
def test_prepass_on_fixture_frames_and_ingest_covers_its_reads(exe, tmp_path, fx, name, FW, FH, BW, BH, blend):
    """The reference's cameras at each geometry, camera-like 4:2:2 frames: every pixel the pre-pass converts equals
    cv2.cvtColor (with BALANCE followed by luminance_balance); the V sums equal those of the cvtColor output; every byte
    the pre-pass reads lies inside the page-locked windows and the pageable DMA rectangles (1, 2 and 3 bands); and at the
    bench geometry the 4:2:2 ingest moves at most 0.72x the bytes of the BGR one (2 bytes per pixel against 3)."""
    g = fx.geometry(FW, FH, BW, BH)
    calib = fx.scaled_calib(g)
    maps = [C.RefCamera(*calib[n], g).bev_maps for n in NAMES]
    masks = [R.blend_mask(n, BW, BH, g.CW, g.CH) if blend else C.plain_mask(n, g) for n in NAMES]
    bgr_in = fx.frames(FW, FH)
    for fmt in Y2.FORMATS:
        frames = [Y2.from_bgr(f, fmt) for f in bgr_in]
        bgr = [Y2.to_bgr(f, fmt) for f in frames]
        for balance in (False, True):
            got, spans, info = _run(exe, tmp_path, fmt, frames, FW, FH, balance, maps, masks, BW, BH)
            assert int(info["coverage"][1].split("=")[1]) == 0, info["coverage"]
            assert [int(v) for v in info["vsum"]] == _vsums(bgr)
            want = C.luminance_balance(bgr) if balance else bgr
            conv = _converted(spans, FW)
            assert conv.any(axis=(1, 2)).all()
            for k in range(4):
                assert (got[k][conv[k]] == want[k][conv[k]]).all(), (fmt, balance, k)
                assert (got[k][~conv[k]] == POISON).all()
        b = {kv.split("=")[0]: int(kv.split("=")[1]) for kv in info["bytes"]}
        print(name, fmt, b, "fetch ratio %.3f dma ratio %.3f" % (b["fetch"] / b["bgr_fetch"], b["dma"] / b["bgr_dma"]))
        if name == "cfg4":
            assert b["fetch"] <= 0.72 * b["bgr_fetch"] and b["dma"] <= 0.72 * b["bgr_dma"], b


def _balances(case):
    """BALANCE is the reference's four-camera luminance_balance: on and off for 4-camera cases, off otherwise."""
    return (False, True) if case.NC == 4 else (False,)


def test_ingest_covers_the_prepass_on_the_422_corpus(exe, tmp_path):
    """Every case of the 4:2:2 corpus in both byte orders: the ingest windows and rectangles hold every byte the pre-pass
    reads; the converted pixels equal cv2.cvtColor, and on the 4-camera cases with BALANCE cvtColor followed by
    luminance_balance, with the V sums of the cvtColor output; nothing outside the converted groups is written."""
    cases = YC.yuv422_corpus()
    assert len(cases) >= 30
    for c0 in cases:
        for fmt in Y2.FORMATS:
            c = YC.yuv422_case(c0.name, fmt)
            frames, bgr = c.yuv[0], c.sets[0]
            for balance in _balances(c):
                got, spans, info = _run(exe, tmp_path, fmt, frames, c.FW, c.FH, balance, c.maps, c.masks, c.BW, c.BH, c.nearest)
                assert int(info["coverage"][1].split("=")[1]) == 0, (c.name, info["coverage"])
                assert [int(v) for v in info["vsum"]] == _vsums(bgr), c.name
                want = C.luminance_balance(bgr) if balance else bgr
                conv = _converted(spans, c.FW)
                for k in range(c.NC):
                    assert (got[k][conv[k]] == want[k][conv[k]]).all(), (c.name, fmt, balance, k)
                    assert (got[k][~conv[k]] == POISON).all(), (c.name, fmt, balance, k)


def _interpret(kernel_math, tmp_path, case, frames, mode):
    """kernel_math `bev` / `bevtma` (mode: argv after the mode name) on BGR frames, BALANCE and car off."""
    (tmp_path / "k_in.bin").write_bytes(B.blob(replace(case, sets=[list(frames)]), 0))
    r = subprocess.run([kernel_math, mode[0], str(tmp_path / "k_in.bin"), str(tmp_path / "k_out.bin"), *map(str, mode[1:])],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (case.name, mode, r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    return np.fromfile(tmp_path / "k_out.bin", np.uint8).reshape(case.BH, case.BW, 3)


def test_render_never_weights_an_unconverted_byte(exe, kernel_math, tmp_path):
    """The 4:2:2 pre-pass writes only the sampled spans into the shared copy stack; the rest of it holds whatever an
    earlier call left, here 0xA5.  That copy stack, rendered as BGR frames by the host interpreters of k_bev's plan and
    (16-byte friendly pitches) k_bev_tma's at the default setting, equals compose() of the cvtColor frames --
    luminance-balanced first where the pre-pass balanced -- for every case of the 4:2:2 corpus in both byte orders."""
    for c0 in YC.yuv422_corpus():
        modes = [("bev",)] + ([("bevtma", *B.DEFAULT_PLAN)] if c0.tma_friendly else [])
        for fmt in Y2.FORMATS:
            c = YC.yuv422_case(c0.name, fmt)
            bgr = c.sets[0]
            for balance in _balances(c):
                stack, _, _ = _run(exe, tmp_path, fmt, c.yuv[0], c.FW, c.FH, balance, c.maps, c.masks, c.BW, c.BH, c.nearest)
                want = B.compose(c, C.luminance_balance(bgr) if balance else bgr)
                for mode in modes:
                    got = _interpret(kernel_math, tmp_path, c, stack, mode)
                    assert (got == want).all(), (c.name, fmt, balance, mode, int((got != want).any(-1).sum()))


# ------------------------------------------------------------------ pitched single planes
def _arena(frames, pitch, base, extra, poison):
    """The packed frames in one arena: frame k's plane at base + k * (FH * pitch + extra), rows `pitch` bytes apart;
    every other byte is `poison` (a value or an array for the padding).  Returns (arena, offsets, padding mask)."""
    FH, FW = frames[0].shape[:2]
    stride = FH * pitch + extra
    arena = np.zeros(base + len(frames) * stride + 5, np.uint8)
    pad = np.ones(arena.size, bool)
    offs = []
    for k, f in enumerate(frames):
        o = base + k * stride
        offs.append(o)
        for y in range(FH):
            arena[o + y * pitch:o + y * pitch + 2 * FW] = f[y].reshape(-1)
            pad[o + y * pitch:o + y * pitch + 2 * FW] = False
    arena[pad] = poison
    return arena, offs, pad


def _pitched(exe, tmp_path, fmt, arena, offs, pitch, FW, FH, spans, balance):
    n = len(offs)
    geo = np.array([[o, pitch] for o in offs], np.int64)
    parts = [np.array([n, FW, FH, int(balance), arena.size], np.int64).tobytes(), geo.tobytes(),
             np.ascontiguousarray(spans, np.int32).tobytes(), arena.tobytes()]
    (tmp_path / "p_in.bin").write_bytes(b"".join(parts))
    r = subprocess.run([exe, "pitched", str(Y2.FMT_CODE[fmt]), str(tmp_path / "p_in.bin"), str(tmp_path / "p_out.bin")],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (fmt, FW, FH, r.returncode, r.stdout[-3000:], r.stderr[-2000:])
    return np.fromfile(tmp_path / "p_out.bin", np.uint8).reshape(n, FH, FW, 3), _info(r.stdout)


def _spans(rng, NC, FW, FH):
    """Spans that start and end anywhere, some rows empty, some whole."""
    sp = np.sort(rng.integers(0, FW + 1, (NC, FH, 2)), axis=-1).astype(np.int32)
    sp[:, ::7] = (0, FW)
    sp[:, 3::11] = (5, 5)
    return sp


@pytest.mark.parametrize("fmt", Y2.FORMATS)
@pytest.mark.parametrize("FW,FH", [(64, 47), (30, 18), (98, 1), (48, 33)])
def test_pitched_single_planes_against_cv2(exe, tmp_path, fmt, FW, FH):
    """Four random frames as one pitched plane each: pitch 2 FW, 2 FW + 4 at a 4-aligned base that is not 8-aligned,
    2 FW + 16, an odd pitch at an odd base, and a power of two; frames at a stride with extra bytes; with and without
    BALANCE.  Converted pixels equal cv2.cvtColor of the dense frames (luminance-balanced with BALANCE), the V sums are
    the converted frames', nothing outside the converted groups is written, no read leaves the plane rectangle, and
    changing the padding changes nothing."""
    rng = np.random.default_rng(FW * FH + len(fmt))
    frames = [Y2.random_frame(rng, FW, FH) for _ in range(4)]
    bgr = [Y2.to_bgr(f, fmt) for f in frames]
    spans = _spans(rng, 4, FW, FH)
    conv = _converted(spans, FW)
    row = 2 * FW
    layouts = [(row, 0, 0), (row + 4, 4, 4), (row + 16, 0, 16), (row + 3, 1, 3), (1 << int(row - 1).bit_length(), 3, 1)]
    for pitch, base, extra in layouts:
        arena, offs, pad = _arena(frames, pitch, base, extra, POISON)
        for balance in (False, True):
            got, info = _pitched(exe, tmp_path, fmt, arena, offs, pitch, FW, FH, spans, balance)
            what = (fmt, FW, FH, pitch, base, balance)
            assert int(info["audit"][1].split("=")[1]) == 0, (what, info["audit"])
            assert [int(v) for v in info["vsum"]] == _vsums(bgr), what
            want = C.luminance_balance(bgr) if balance else bgr
            for k in range(4):
                assert (got[k][conv[k]] == want[k][conv[k]]).all(), (what, k)
                assert (got[k][~conv[k]] == POISON).all(), (what, k)
            other = rng.integers(0, 256, int(pad.sum()), dtype=np.uint8)
            arena2, _, _ = _arena(frames, pitch, base, extra, other)
            again, info2 = _pitched(exe, tmp_path, fmt, arena2, offs, pitch, FW, FH, spans, balance)
            assert (again == got).all() and info2["vsum"] == info["vsum"], (what, "padding reached the result")


def test_yuv422_corpus_reaches_every_class():
    """The 4:2:2 corpus holds every class of input that selects a code path of the 4:2:2 render, so that thinning it
    fails here, without a GPU."""
    cases = YC.yuv422_corpus()
    four = [c for c in cases if c.NC == 4]
    # odd heights, FH = 1 among them, with BALANCE
    assert any(c.FH == 1 for c in cases) and any(c.FH % 2 for c in four)
    # a last group of 2 pixels with BALANCE and with NEAREST
    assert any(c.FW % 4 == 2 for c in four) and any(c.FW % 4 == 2 and c.nearest for c in cases)
    # k_bev on the copy stack (no TMA plan) and k_bev_tma with luminance_balance's row tail, with BALANCE
    assert any(not c.tma_friendly for c in four) and any(c.FW % 32 == 16 and c.tma_friendly for c in four)
    # every camera count
    assert {c.NC for c in cases} == set(range(1, 9))
    # int16-extreme and out-of-frame taps, and taps on the last column and the last row, under a non-zero mask
    taps = [(m1[mk > 0], c) for c in cases for (m1, _), mk in zip(c.maps, c.masks)]
    assert any((np.abs(t.astype(np.int32)) > 30000).any() for t, _ in taps)
    assert any(((t[:, 0] < 0) | (t[:, 0] >= c.FW) | (t[:, 1] < 0) | (t[:, 1] >= c.FH)).any() for t, c in taps)
    assert any((t[:, 0] == c.FW - 1).any() for t, c in taps) and any((t[:, 1] == c.FH - 1).any() for t, c in taps)
    # bright frames (saturating adds) among multi-camera cases
    assert any(c.NC > 1 and all(f[..., 0].min() >= 200 for f in c.yuv[0]) for c in cases)
