"""The device PNG encoder on the CPU.  tests/host/png_enc.cu runs png::normalise and the __host__ __device__ stage
functions of bevk_png_enc.cuh (filters, the Z_RLE / Z_HUFFMAN_ONLY parse, zlib's trees and block choice, symbol codes,
zlib header, Adler-32, IDAT framing, CRC-32) serially over whole images; every stream of the tests/png_cases.py corpus
must equal cv2.imencode(".png", img, params) byte for byte and stay within the bound, the corpus must reach every stream
class, and the normaliser must agree with cv2 on which lists it takes and how it reads them."""
import os
import shutil
import struct
import subprocess
import zlib

import cv2
import numpy as np
import pytest

from cameracalibration_b200.build import GENCODE
from tests import png_cases as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C, S, F, B, Z = (cv2.IMWRITE_PNG_COMPRESSION, cv2.IMWRITE_PNG_STRATEGY, cv2.IMWRITE_PNG_FILTER, cv2.IMWRITE_PNG_BILEVEL,
                 cv2.IMWRITE_PNG_ZLIBBUFFER_SIZE)


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    nvcc = next((c for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc") if c and os.path.exists(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("host_png") / "png_enc"
    build = subprocess.run([nvcc, "-O2", "-std=c++17", *GENCODE, "-o", str(out), os.path.join(ROOT, "tests", "host", "png_enc.cu")],
                           capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stdout + build.stderr
    return str(out)


def host_run(exe, tmp_path, records):
    """records: [(BGR image, params)] -> [(normalise result, class bits, stream, bound)] from the host build."""
    blob = [struct.pack(f"<3i{len(p)}i", img.shape[1], img.shape[0], len(p), *p) + np.ascontiguousarray(img).tobytes()
            for img, p in records]
    (tmp_path / "in.bin").write_bytes(b"".join(blob))
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, (r.returncode, r.stderr[-2000:])
    raw, p, out = (tmp_path / "out.bin").read_bytes(), 0, []
    for _ in records:
        ok, cls = struct.unpack_from("<2i", raw, p)
        n, bound = struct.unpack_from("<2Q", raw, p + 8)
        out.append((ok, cls, raw[p + 24:p + 24 + n], bound))
        p += 24 + n
    assert p == len(raw)
    return out


def cv2_png(img, params):
    ok, buf = cv2.imencode(".png", img, list(params))
    return buf.tobytes() if ok else None


def chunks(stream):
    p, out = 8, []
    while p < len(stream):
        n = struct.unpack_from(">I", stream, p)[0]
        out.append((stream[p + 4:p + 8], stream[p + 8:p + 8 + n]))
        p += 12 + n
    return out


@pytest.fixture(scope="module")
def corpus_run(exe, tmp_path_factory):
    cases = P.cases()
    return cases, host_run(exe, tmp_path_factory.mktemp("png_corpus"), [(img, p) for _, img, p in cases])


def test_png_corpus_matches_cv2(corpus_run):
    cases, got = corpus_run
    bad = []
    for (name, img, params), (ok, _, stream, bound) in zip(cases, got):
        assert ok == 0, name
        want = cv2_png(img, params)
        assert len(stream) <= bound, name
        if stream != want:
            bad.append((name, len(stream), len(want)))
    assert not bad, bad


def test_png_corpus_reaches_every_class(corpus_run):
    cases, got = corpus_run
    seen = 0
    for _, cls, _, _ in got:
        seen |= cls
    missing = [v for k, v in P.CLASSES.items() if not (seen >> k) & 1]
    assert not missing, missing
    sizes = {(img.shape[1], img.shape[0]) for _, img, _ in cases}
    assert {(1, 1), (65500, 1), (1, 65500)} <= sizes
    assert any(w == 1 and h > 1 for w, h in sizes) and any(h == 1 and w > 1 for w, h in sizes)
    forms = {tuple(p) for _, _, p in cases}
    assert {tuple(p) for p in P.PARAMS.values()} <= forms


def test_png_window_thresholds(corpus_run):
    """libpng's window rule at its thresholds: 16383 filtered bytes gets a reduced window in the header, 16426 does not;
    a 1x1 image gets CINFO 0."""
    cases, got = corpus_run
    head = {name: chunks(stream)[1][1][:2].hex() for (name, _, _), (_, _, stream, _) in zip(cases, got)}
    assert head["noise_14x381_default"] == "6805" and head["noise_14x382_default"] == "7801"
    assert head["smooth_64x50_default"] == "6805" and head["1x1_default"] == "081d"


def test_png_empty_final_block(corpus_run):
    """14 x 381 under HUFFMAN_ONLY is exactly 16383 literals: zlib flushes them as one full block and Z_FINISH adds an
    empty final static block (3 + 7 bits), so the stream ends in the bytes of that block."""
    cases, got = corpus_run
    (_, cls, stream, _), = [g for (n, _, _), g in zip(cases, got) if n == "noise_14x381_huff"]
    assert (cls >> 3) & 1
    z = b"".join(d for t, d in chunks(stream) if t == b"IDAT")
    assert zlib.decompress(z) is not None
    assert stream == cv2_png(next(img for n, img, _ in cases if n == "noise_14x381_huff"), [S, cv2.IMWRITE_PNG_STRATEGY_HUFFMAN_ONLY])


# Parameter lists for the normaliser: both orders, clamping, fallbacks, refusals
NORMALISE_LISTS = [
    [], [S, 3], [S, 2], [C, 1, S, 3], [C, 5, S, 3], [C, 9, S, 2], [C, 12, S, 3], [C, -1, S, 3], [C, 0, S, 3],
    [S, 3, C, 5], [S, 2, C, 1], [C, 5], [C, 1], [S, 0], [S, 1], [S, 4], [S, 7], [S, -3], [C, 3, S, 7],
    [F, 8], [F, 16], [F, 32], [F, 64], [F, 128], [F, 56], [F, 248], [F, 0], [F, 24], [F, 255], [F, -1],
    [F, 32, C, 3, S, 3], [C, 3, S, 3, F, 8], [C, 3, F, 64, S, 2], [F, 8, S, 3],
    [B, 0], [B, 0, S, 2], [B, 1], [Z, 8192], [Z, 1024, S, 3], [C, 4, S, 3, C, 6, S, 2], [S, 2, S, 3],
    [C, 2, S, 3, S, 0], [S, 3, B, 1],
]


def test_png_normaliser_agrees_with_cv2(exe, tmp_path):
    """Every list: the host build accepts it exactly when it is one the encoder reproduces, and then writes cv2's
    bytes; cv2's own reading of the list (strategy, level, filters) is pinned by the streams themselves.  Lists the
    encoder refuses are ones where cv2 uses zlib's hash-chain parse or stored blocks (checked on cv2's zlib header and
    by recompressing), or fails / is not 3-channel."""
    assert len(NORMALISE_LISTS) >= 40
    rng = np.random.default_rng(7)
    img = P._stripes(rng, 50, 64)
    got = host_run(exe, tmp_path, [(img, p) for p in NORMALISE_LISTS])
    for params, (ok, _, stream, _) in zip(NORMALISE_LISTS, got):
        want = cv2_png(img, params)
        if ok == 0:
            assert stream == want, params
            continue
        assert stream == b"", params
        if want is None or B in params[::2] and params[params.index(B) + 1] != 0:
            continue
        if Z in params[::2]:
            assert ok == 2, params
            continue
        assert ok == 2, params
        # cv2 parsed this list with something other than Z_RLE / Z_HUFFMAN_ONLY: its deflate data is neither
        z = b"".join(d for t, d in chunks(want) if t == b"IDAT")
        raw, rb = zlib.decompress(z), 3 * img.shape[1] + 1
        for strategy in (zlib.Z_RLE, zlib.Z_HUFFMAN_ONLY):
            co = zlib.compressobj(1, zlib.DEFLATED, 15, 8, strategy)
            body = b"".join(co.compress(raw[y * rb:(y + 1) * rb]) for y in range(img.shape[0])) + co.flush()
            assert z[2:] != body[2:], (params, strategy)


def test_png_normaliser_rejects_other_keys(exe, tmp_path):
    img = np.zeros((4, 4, 3), np.uint8)
    got = host_run(exe, tmp_path, [(img, [cv2.IMWRITE_JPEG_QUALITY, 90]), (img, [15, 1]), (img, [21, 0])])
    assert [g[0] for g in got] == [1, 1, 1]


def test_png_bound_holds_for_noise(exe, tmp_path):
    rng = np.random.default_rng(11)
    recs = [(rng.integers(0, 256, (h, w, 3), dtype=np.uint8), p) for w, h in ((1, 1), (5, 3), (700, 200), (3, 6000))
            for p in ([], [S, 2], [C, 9, S, 3])]
    for (img, p), (ok, _, stream, bound) in zip(recs, host_run(exe, tmp_path, recs)):
        assert ok == 0 and stream == cv2_png(img, p) and len(stream) <= bound
