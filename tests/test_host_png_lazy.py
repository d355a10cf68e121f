"""The device PNG encoder's hash-chain path on the CPU.  tests/host/png_lazy.cu runs png::normalise(..., hash_chain)
and the __host__ __device__ stage functions of bevk_png_enc.cuh (filters, lazy_match per position, lazy_chain between
canonical positions, zlib's trees and block choice with real distances, symbol codes, zlib header with FLEVEL, Adler-32,
IDAT framing) serially over whole images; every stream of the tests/png_lazy_cases.py corpus must equal
cv2.imencode(".png", img, params) byte for byte and stay within the bound, the corpus must reach every class, the
normaliser must refuse exactly the lists cv2 writes with levels 0..3 under a hash-chain strategy, BILEVEL or
ZLIBBUFFER_SIZE, and no block zlib could not have stored (its start slid out of the window) comes out stored."""
import os
import shutil
import subprocess
import zlib

import cv2
import numpy as np
import pytest

from cameracalibration_b200.build import GENCODE
from tests import png_lazy_cases as PL
from tests.test_host_png import chunks, cv2_png, host_run

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C, S, F, B, Z = (cv2.IMWRITE_PNG_COMPRESSION, cv2.IMWRITE_PNG_STRATEGY, cv2.IMWRITE_PNG_FILTER, cv2.IMWRITE_PNG_BILEVEL,
                 cv2.IMWRITE_PNG_ZLIBBUFFER_SIZE)


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    nvcc = next((c for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc") if c and os.path.exists(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("host_png_lazy") / "png_lazy"
    build = subprocess.run([nvcc, "-O2", "-std=c++17", *GENCODE, "-o", str(out), os.path.join(ROOT, "tests", "host", "png_lazy.cu")],
                           capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stdout + build.stderr
    return str(out)


@pytest.fixture(scope="module")
def corpus_run(exe, tmp_path_factory):
    cases = PL.cases()
    return cases, host_run(exe, tmp_path_factory.mktemp("png_lazy_corpus"), [(img, p) for _, img, p in cases])


def test_png_lazy_corpus_matches_cv2(corpus_run):
    """Every case byte-equal to live cv2 and within the bound; the host program itself exits non-zero if a block whose
    raw span exceeds the window's MAX_DIST comes out stored (DESIGN.md section 2)."""
    cases, got = corpus_run
    bad = []
    for (name, img, params), (ok, _, stream, bound) in zip(cases, got):
        assert ok == 0, name
        assert len(stream) <= bound, name
        if stream != cv2_png(img, params):
            bad.append(name)
    assert not bad, bad


def test_png_lazy_corpus_reaches_every_class(corpus_run):
    cases, got = corpus_run
    seen = 0
    for _, cls, _, _ in got:
        seen |= cls
    missing = [v for k, v in PL.CLASSES.items() if not (seen >> k) & 1]
    assert not missing, missing
    forms = {tuple(p) for _, _, p in cases}
    assert {(C, lv, S, st) for lv in range(4, 10) for st in (0, 1, 4)} <= forms
    assert {tuple(p) for p in PL.FILTER_LISTS.values()} <= forms


def test_png_lazy_header_flevel(corpus_run):
    """FLEVEL of cv2's zlib header: 1 at levels 4..5, 2 at 6, 3 at 7..9, 0 under Z_FIXED."""
    cases, got = corpus_run
    for (name, _, params), (_, _, stream, _) in zip(cases, got):
        if not name.startswith("blocks_301x237_l") or len(params) != 4 or params[2] != S:
            continue
        level, st = params[1], params[3]
        flg = chunks(stream)[1][1][1]
        want = 0 if st == PL.FIXED else 1 if level < 6 else 2 if level == 6 else 3
        assert flg >> 6 == want, name


# Lists for the normaliser's hash-chain reading: levels, strategies, orders, clamping and refusals
NORMALISE_LISTS = [
    [C, 4], [C, 9], [C, 12], [C, 3], [C, 1], [C, 0], [C, -2], [S, 0], [S, 1], [S, 4], [C, 6, S, 1], [C, 6, S, 4],
    [C, 3, S, 4], [C, 5, S, 3], [C, 5, S, 2], [S, 0, C, 5], [C, 9, F, 8], [F, 32, C, 4], [C, 7, S, 9], [C, 2, S, 0],
    [C, 9, B, 1], [C, 9, B, 0], [C, 9, Z, 8192], [C, 4, S, 0, C, 3], [C, 3, S, 3, C, 8], [],
]


def test_png_lazy_normaliser_agrees_with_cv2(exe, tmp_path):
    """Accepted lists (result 0 or 3 for the Z_RLE / Z_HUFFMAN_ONLY ones) are written as cv2 writes them; refused ones
    (2) are level 0 (stored blocks), deflate_fast's levels 1..3 (its header says so: FLEVEL 0 at level 1, and the
    stream differs from deflate_slow's at level 4), BILEVEL != 0 or ZLIBBUFFER_SIZE."""
    rng = np.random.default_rng(8)
    img = PL.P._stripes(rng, 50, 64)
    got = host_run(exe, tmp_path, [(img, p) for p in NORMALISE_LISTS])
    for params, (ok, _, stream, _) in zip(NORMALISE_LISTS, got):
        want = cv2_png(img, params)
        if ok == 0:
            assert stream == want, params
            continue
        assert stream == b"", params
        if ok == 3:   # a Z_RLE / Z_HUFFMAN_ONLY list: tests/test_host_png.py covers those
            continue
        assert ok == 2, params
        if want is None or B in params[::2] and params[params.index(B) + 1] != 0 or Z in params[::2]:
            continue
        z = b"".join(d for t, d in chunks(want) if t == b"IDAT")
        raw, rb = zlib.decompress(z), 3 * img.shape[1] + 1
        co = zlib.compressobj(4, zlib.DEFLATED, 13, 8, zlib.Z_DEFAULT_STRATEGY)
        body = b"".join(co.compress(raw[y * rb:(y + 1) * rb]) for y in range(img.shape[0])) + co.flush()
        assert z[2:] != body[2:], params
        assert (z[1] >> 6) in (0, 1), params   # level 0..1: FLEVEL 0; 2..3: FLEVEL 1


def test_png_lazy_bound_holds_for_noise(exe, tmp_path):
    rng = np.random.default_rng(12)
    recs = [(rng.integers(0, 256, (h, w, 3), dtype=np.uint8), p) for w, h in ((1, 1), (5, 3), (700, 200), (3, 6000))
            for p in ([C, 9], [C, 4, S, 4], [C, 6, S, 1])]
    for (img, p), (ok, _, stream, bound) in zip(recs, host_run(exe, tmp_path, recs)):
        assert ok == 0 and stream == cv2_png(img, p) and len(stream) <= bound
