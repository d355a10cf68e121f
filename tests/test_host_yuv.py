"""The YUV 4:2:0 source path on the CPU: tests/host/yuv.cu runs the host forms of the conversion pre-pass (k_yuv_spans'
work item), of the YUV V sum (k_vsum_yuv's) and of the ingest plan (bevk_plan.cuh) from the library's headers, and
this file compares them with live cv2: cv2.cvtColor(COLOR_YUV2BGR_NV12 / _I420), then the oracle's luminance_balance."""
import os
import shutil
import subprocess

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


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    nvcc = next((c for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc") if c and os.path.exists(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("host_yuv") / "yuv"
    src = os.path.join(ROOT, "tests", "host", "yuv.cu")
    build = subprocess.run([nvcc, "-O2", "-std=c++17", "--fmad=false", "-Xcompiler", "-ffp-contract=off", *GENCODE,
                            "-o", str(out), src], capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stdout + build.stderr
    return str(out)


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


def test_ingest_covers_the_prepass_on_the_fuzz_corpus(exe, tmp_path):
    """Every even-sized case of tests/bev_cases.py -- the fuzz corpus (1-8 cameras, int16-extreme taps) and the original
    random cases (tiny frames, widths that are not multiples of 4): the ingest windows and rectangles hold every byte the
    pre-pass reads, and the converted pixels equal cv2.cvtColor."""
    rng = np.random.default_rng(5)
    crng = np.random.default_rng(7)
    cases = [c for c in B.corpus() + [B.random_case(crng, i) for i in range(40)] if c.FW % 2 == 0 and c.FH % 2 == 0]
    assert len(cases) >= 16 and {c.FW % 4 for c in cases} == {0, 2}
    for c in cases:
        frames = [Y.random_yuv(rng, c.FW, c.FH) for _ in range(c.NC)]
        for fmt in Y.FORMATS:
            got, spans, info = _run(exe, tmp_path, fmt, frames, c.FW, c.FH, False, c.maps, c.masks, c.BW, c.BH, c.nearest)
            assert int(info["coverage"][1].split("=")[1]) == 0, (c.name, info["coverage"])
            conv = _converted(spans, c.FW)
            for k, f in enumerate(frames):
                want = Y.to_bgr(f, fmt)
                assert (got[k][conv[k]] == want[conv[k]]).all(), (c.name, fmt, k)
