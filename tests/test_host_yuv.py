"""The YUV 4:2:0 source path on the CPU: tests/host/yuv.cu runs the host forms of the conversion pre-pass (k_yuv_spans'
work item), of the YUV V sum (k_vsum_yuv's) and of the ingest plan (bevk_plan.cuh) from the library's headers, and
this file compares them with live cv2: cv2.cvtColor(COLOR_YUV2BGR_NV12 / _I420), then the oracle's luminance_balance.
The copy stack the conversion leaves also goes through the host interpreters of the render's plans
(tests/host/kernel_math.cu), to show that the render reads nothing the conversion did not write."""
import os
import shutil
import subprocess
from dataclasses import replace

import numpy as np
import pytest

from cameracalibration_b200.build import GENCODE
from oracle import cv2_path as C
from oracle import restate as R
from tests import bev_cases as B
from tests import yuv_frames as Y
from tests.helpers import NAMES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POISON = 0xA5


def _build(tmp_path_factory, name):
    nvcc = next((c for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc") if c and os.path.exists(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("host_" + name) / name
    src = os.path.join(ROOT, "tests", "host", name + ".cu")
    build = subprocess.run([nvcc, "-O2", "-std=c++17", "--fmad=false", "-Xcompiler", "-ffp-contract=off", *GENCODE,
                            "-o", str(out), src], capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stdout + build.stderr
    return str(out)


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return _build(tmp_path_factory, "yuv")


@pytest.fixture(scope="module")
def kernel_math(tmp_path_factory):
    """tests/host/kernel_math.cu: the host interpreters of k_bev's and k_bev_tma's plans (`bev`, `bevtma`)."""
    return _build(tmp_path_factory, "kernel_math")


def _run(exe, tmp_path, fmt, frames, FW, FH, balance=False, maps=None, masks=None, BW=0, BH=0, nearest=False):
    """The harness on NC YUV frames; returns (copy stack [NC][FH][FW][3], spans [NC][FH][2], parsed stdout)."""
    NC = len(frames)
    parts = [np.array([NC, FW, FH, BW, BH, int(nearest), int(balance), int(maps is not None)], np.int32).tobytes()]
    if maps is not None:
        for (m1, m2), mk in zip(maps, masks):
            parts += [np.ascontiguousarray(m1, np.int16).tobytes(), np.ascontiguousarray(m2, np.uint16).tobytes(),
                      np.ascontiguousarray(mk, np.uint8).tobytes()]
    parts += [np.ascontiguousarray(f).tobytes() for f in frames]
    (tmp_path / "in.bin").write_bytes(b"".join(parts))
    r = subprocess.run([exe, "yuv", str(Y.FMT_CODE[fmt]), str(tmp_path / "in.bin"), str(tmp_path / "out.bin")],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (fmt, FW, FH, r.returncode, r.stdout[-3000:], r.stderr[-2000:])
    raw = np.fromfile(tmp_path / "out.bin", np.uint8)
    n = NC * FH * FW * 3
    info = {}
    for ln in r.stdout.splitlines():
        if ":" in ln:
            k, v = ln.split(":", 1)
            info[k] = v.split()
    return raw[:n].reshape(NC, FH, FW, 3), raw[n:].view(np.int32).reshape(NC, FH, 2), info


def _converted(spans, FW):
    """Per camera: the pixels the pre-pass converts, the spans rounded out to whole 4-pixel groups (bool[NC][FH][FW])."""
    NC, FH, _ = spans.shape
    x = np.arange(FW)
    lo = (spans[..., 0] >> 2) * 4
    hi = np.where(spans[..., 1] > spans[..., 0], np.minimum(FW, ((spans[..., 1] + 3) >> 2) * 4), lo)
    return (x >= lo[..., None]) & (x < hi[..., None])


@pytest.mark.parametrize("fmt", Y.FORMATS)
def test_yuv_bgr_every_triple_against_cv2(exe, tmp_path, fmt):
    """yuv_bgr and the chroma addressing, through the pre-pass over whole rows, for all 2^24 (Y, U, V) triples."""
    f = Y.every_triple(fmt)
    got, _, _ = _run(exe, tmp_path, fmt, [f], 4096, 4096)
    want = Y.to_bgr(f, fmt)
    assert (got[0] == want).all(), int((got[0] != want).any(-1).sum())


@pytest.mark.parametrize("FW,FH", [(64, 32), (30, 18), (98, 54)])
def test_small_and_ragged_frames_against_cv2(exe, tmp_path, FW, FH):
    """Widths that are not multiples of 4 (a last group of 2 pixels), heights with an odd chroma row count (the I420 V
    plane starts mid-row), whole-row spans, with and without BALANCE (four frames)."""
    rng = np.random.default_rng(FW * FH)
    for fmt in Y.FORMATS:
        frames = [Y.random_yuv(rng, FW, FH) for _ in range(4)]
        bgr = [Y.to_bgr(f, fmt) for f in frames]
        for balance in (False, True):
            got, _, info = _run(exe, tmp_path, fmt, frames, FW, FH, balance)
            want = C.luminance_balance(bgr) if balance else bgr
            assert [int(v) for v in info["vsum"]] == [int(b.max(-1).sum(dtype=np.int64)) for b in bgr]
            for k in range(4):
                assert (got[k] == want[k]).all(), (fmt, balance, k)


GEOMETRIES = [   # (name, FW, FH, BW, BH, blend): the fixture geometry and BASELINE's cfg2, cfg3 and cfg4 (the bench's)
    ("fixture", 1280, 1024, 1000, 1000, True),
    ("cfg2", 1280, 960, 1000, 1000, False),
    ("cfg3", 1920, 1080, 1200, 1200, True),
    ("cfg4", 1920, 1080, 1000, 1000, True),
]


@pytest.mark.parametrize("name,FW,FH,BW,BH,blend", GEOMETRIES)
def test_prepass_on_fixture_frames_and_ingest_covers_its_reads(exe, tmp_path, fx, name, FW, FH, BW, BH, blend):
    """The reference's cameras at each geometry: every pixel the pre-pass converts (the sampled spans, rounded to whole
    4-pixel groups) equals cv2.cvtColor, and with BALANCE cvtColor followed by luminance_balance; the V sums equal those
    of the cvtColor output; every byte the pre-pass reads lies inside the page-locked windows and the pageable DMA
    rectangles (1, 2 and 3 bands) -- the harness fails otherwise; and at the bench geometry the NV12 ingest moves at
    most 0.55x the bytes of the BGR one."""
    g = fx.geometry(FW, FH, BW, BH)
    calib = fx.scaled_calib(g)
    maps = [C.RefCamera(*calib[n], g).bev_maps for n in NAMES]
    masks = [R.blend_mask(n, BW, BH, g.CW, g.CH) if blend else C.plain_mask(n, g) for n in NAMES]
    bgr_in = fx.frames(FW, FH)
    for fmt in Y.FORMATS:
        frames = [Y.from_bgr(f, fmt) for f in bgr_in]
        bgr = [Y.to_bgr(f, fmt) for f in frames]
        for balance in (False, True):
            got, spans, info = _run(exe, tmp_path, fmt, frames, FW, FH, balance, maps, masks, BW, BH)
            assert int(info["coverage"][1].split("=")[1]) == 0, info["coverage"]
            assert [int(v) for v in info["vsum"]] == [int(b.max(-1).sum(dtype=np.int64)) for b in bgr]
            want = C.luminance_balance(bgr) if balance else bgr
            conv = _converted(spans, FW)
            assert conv.any(axis=(1, 2)).all()
            for k in range(4):
                assert (got[k][conv[k]] == want[k][conv[k]]).all(), (fmt, balance, k)
                assert (got[k][~conv[k]] == POISON).all()
        b = {kv.split("=")[0]: int(kv.split("=")[1]) for kv in info["bytes"]}
        print(name, fmt, b, "fetch ratio %.3f dma ratio %.3f" % (b["fetch"] / b["bgr_fetch"], b["dma"] / b["bgr_dma"]))
        if fmt == "nv12" and name == "cfg4":
            assert b["fetch"] <= 0.55 * b["bgr_fetch"] and b["dma"] <= 0.55 * b["bgr_dma"], b


def _balances(case):
    """BALANCE is the reference's four-camera luminance_balance: on and off for 4-camera cases, off otherwise."""
    return (False, True) if case.NC == 4 else (False,)


def test_ingest_covers_the_prepass_on_the_fuzz_corpus(exe, tmp_path):
    """Every case of the YUV corpus (tests/bev_cases.yuv_corpus: the even-sized fuzz corpus cases and the supplement with
    1-8 cameras, int16-extreme taps, FW % 4 == 2, FH % 4 == 2) and the even-sized original random cases (tiny frames):
    the ingest windows and rectangles hold every byte the pre-pass reads; the converted pixels equal cv2.cvtColor, and
    on the 4-camera cases with BALANCE cvtColor followed by luminance_balance, with the V sums of the cvtColor output;
    nothing outside the converted groups is written."""
    rng = np.random.default_rng(5)
    crng = np.random.default_rng(7)
    cases = [(c, c.yuv[0]) for c in B.yuv_corpus()]
    cases += [(c, [Y.random_yuv(rng, c.FW, c.FH) for _ in range(c.NC)])
              for c in [B.random_case(crng, i) for i in range(40)] if c.FW % 2 == 0 and c.FH % 2 == 0]
    assert len(cases) >= 30 and {c.FW % 4 for c, _ in cases} == {0, 2}
    for c, frames in cases:
        for fmt in Y.FORMATS:
            bgr = [Y.to_bgr(f, fmt) for f in frames]
            for balance in _balances(c):
                got, spans, info = _run(exe, tmp_path, fmt, frames, c.FW, c.FH, balance, c.maps, c.masks, c.BW, c.BH, c.nearest)
                assert int(info["coverage"][1].split("=")[1]) == 0, (c.name, info["coverage"])
                if balance:
                    assert [int(v) for v in info["vsum"]] == [int(b.max(-1).sum(dtype=np.int64)) for b in bgr], c.name
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
    """The YUV pre-pass writes only the sampled spans into the copy stack every call of a context shares; the rest of it
    holds whatever an earlier call left.  Here the rest is 0xA5: the copy stack the harness leaves, rendered as BGR frames
    by the host interpreters of k_bev's plan and (16-byte friendly pitches) k_bev_tma's at the default setting, equals
    compose() of the cvtColor frames -- luminance-balanced first where the pre-pass balanced.  A span that misses a
    sampled pixel lets 0xA5 into the canvas."""
    for c in B.yuv_corpus():
        modes = [("bev",)] + ([("bevtma", *B.DEFAULT_PLAN)] if c.tma_friendly else [])
        for fmt in Y.FORMATS:
            bgr = [Y.to_bgr(f, fmt) for f in c.yuv[0]]
            for balance in _balances(c):
                stack, _, _ = _run(exe, tmp_path, fmt, c.yuv[0], c.FW, c.FH, balance, c.maps, c.masks, c.BW, c.BH, c.nearest)
                want = B.compose(c, C.luminance_balance(bgr) if balance else bgr)
                for mode in modes:
                    got = _interpret(kernel_math, tmp_path, c, stack, mode)
                    assert (got == want).all(), (c.name, fmt, balance, mode, int((got != want).any(-1).sum()))


def test_yuv_corpus_reaches_every_class():
    """The YUV corpus holds every class of input that selects a code path of the YUV render, so that thinning it fails
    here, without a GPU."""
    cases = B.yuv_corpus()
    four = [c for c in cases if c.NC == 4]
    # a last group of 2 pixels (byte stores; a copy-stack pitch that is no multiple of 4: k_bev's per-tap path), with
    # BALANCE and with NEAREST
    assert any(c.FW % 4 == 2 for c in four) and any(c.FW % 4 == 2 and c.nearest for c in cases)
    # k_bev on the copy stack, page-locked frames ingested by DMA rectangles
    assert any(c.FW % 16 and c.FW % 4 == 0 for c in cases)
    # k_bev_tma with luminance_balance's row tail; I420 windows that cross the halves of a buffer row
    assert any(c.FW % 32 == 16 for c in four)
    # the I420 V plane starting mid-row, with BALANCE, on both kernel paths
    assert {c.tma_friendly for c in four if c.FH % 4 == 2} == {True, False}
    # every camera count: frame indexing, empty (camera NC-1) and single-pixel (NC-2) masks from three cameras on
    assert {c.NC for c in cases} == set(range(1, 9))
    # int16-extreme and out-of-frame taps, and taps on the last column and the last row, under a non-zero mask
    taps = [(m1[mk > 0], c) for c in cases for (m1, _), mk in zip(c.maps, c.masks)]
    assert any((np.abs(t.astype(np.int32)) > 30000).any() for t, _ in taps)
    assert any(((t[:, 0] < 0) | (t[:, 0] >= c.FW) | (t[:, 1] < 0) | (t[:, 1] >= c.FH)).any() for t, c in taps)
    assert any((t[:, 0] == c.FW - 1).any() for t, c in taps) and any((t[:, 1] == c.FH - 1).any() for t, c in taps)
    # bright frames (saturating adds) among multi-camera cases
    assert any(c.NC > 1 and all(f[:c.FH].min() >= 200 for f in c.yuv[0]) for c in cases)
