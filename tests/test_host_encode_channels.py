"""The grey and BGRA encoder stages on the CPU.  tests/host/encode_channels.cu runs the __host__ __device__ stage
functions of bevk_jpeg_enc.cuh and bevk_png_enc.cuh serially over the tests/encode_channels_cases.py corpus: every
baseline JPEG stream must equal cv2.imencode byte for byte and stay within its bound, every PNG's filtered bytes must
equal what cv2's IDAT data inflates to, under the IHDR colour type cv2 writes, and under the hash-chain lists (levels 4..9)
the whole zlib stream must equal cv2's IDAT data, window slides included.  The header constants, the grey
progressive scan script and the bounds are pinned against cv2's streams too."""
import os
import shutil
import struct
import subprocess
import zlib

import cv2
import numpy as np
import pytest

from cameracalibration_b200.build import GENCODE
from tests import encode_channels_cases as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    nvcc = next((c for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc") if c and os.path.exists(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("host_encode_channels") / "encode_channels"
    build = subprocess.run([nvcc, "-O2", "-std=c++17", *GENCODE, "-o", str(out),
                            os.path.join(ROOT, "tests", "host", "encode_channels.cu")], capture_output=True, text=True,
                           timeout=600)
    assert build.returncode == 0, build.stdout + build.stderr
    return str(out)


def split_quality(params):
    q, rest = 95, []
    for k, v in zip(params[::2], params[1::2]):
        if k == cv2.IMWRITE_JPEG_QUALITY:
            q = v
        else:
            rest += [k, v]
    return q, rest


def host_run(exe, tmp_path, records):
    """records: [(ext, image [H][W][C], params)] -> [(status, info, bound, bytes, zlib bytes, class bits)]"""
    blob = []
    for ext, img, params in records:
        h, w, c = img.shape
        q, p = split_quality(params) if ext == ".jpg" else (0, list(params))
        blob.append(struct.pack(f"<6i{len(p)}i", int(ext == ".png"), w, h, c, q, len(p), *p) +
                    np.ascontiguousarray(img).tobytes())
    (tmp_path / "in.bin").write_bytes(b"".join(blob))
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True,
                       timeout=1200)
    assert r.returncode == 0, (r.returncode, r.stderr[-2000:])
    raw, p, out = (tmp_path / "out.bin").read_bytes(), 0, []
    for _ in records:
        status, info, cls = struct.unpack_from("<3i", raw, p)
        bound, n, nz = struct.unpack_from("<3Q", raw, p + 12)
        out.append((status, info, bound, raw[p + 36:p + 36 + n], raw[p + 36 + n:p + 36 + n + nz], cls))
        p += 36 + n + nz
    assert p == len(raw)
    return out


def png_chunks(stream):
    p, out = 8, []
    while p < len(stream):
        n = struct.unpack_from(">I", stream, p)[0]
        out.append((stream[p + 4:p + 8], stream[p + 8:p + 8 + n]))
        p += 12 + n
    return out


def cv2_one(ext, img, params):
    return cv2.imencode(ext, img[..., 0] if img.shape[-1] == 1 else img, list(params))[1].tobytes()


@pytest.fixture(scope="module")
def corpus_run(exe, tmp_path_factory):
    recs = [(ext, im, p) for _, ext, imgs, p in E.cases() for im in imgs]
    return recs, host_run(exe, tmp_path_factory.mktemp("enc_channels"), recs)


def test_corpus_jpeg_baseline_matches_cv2(corpus_run):
    recs, got = corpus_run
    bad, seen = [], 0
    for (ext, img, params), (status, _, bound, s, _, _) in zip(recs, got):
        if ext != ".jpg":
            continue
        want = cv2_one(ext, img, params)
        assert len(want) <= bound, (img.shape, params)
        if status == 2:   # progressive: the scan structure is checked below, the bytes on the GPU
            continue
        assert status == 0, params
        seen += 1
        if s != want:
            bad.append((img.shape, params))
    assert seen > 100 and not bad, bad[:10]


def test_corpus_png_filter_stage_matches_cv2(corpus_run):
    recs, got = corpus_run
    bad, seen = [], 0
    for (ext, img, params), (status, colour, bound, f, z, _) in zip(recs, got):
        if ext != ".png":
            continue
        assert status == 0, params
        want = cv2_one(ext, img, params)
        assert len(want) <= bound
        ch = png_chunks(want)
        assert ch[0][0] == b"IHDR" and ch[0][1][9] == colour
        idat = b"".join(d for t, d in ch if t == b"IDAT")
        seen += 1
        if zlib.decompress(idat) != f or (z and z != idat):
            bad.append((img.shape, params))
    assert seen > 100 and not bad, bad[:10]


def test_hash_chain_window_slides(exe, tmp_path):
    """The window cases: every zlib stream equals cv2's, and for grey and BGRA rows alike they reach both outcomes of a
    head at w_size exactly MAX_DIST back that the row length decides: searched (class 19) and NIL because a row ends at
    2 w_size - 1 (class 20).  With rows taken as 3W + 1 bytes long instead of C*W + 1, 14 of these streams differ from
    cv2's."""
    cases = E.window_cases()
    got = host_run(exe, tmp_path, [(ext, imgs[0], p) for _, ext, imgs, p in cases])
    seen = {1: 0, 4: 0}
    for (name, ext, imgs, params), (status, _, _, _, z, cls) in zip(cases, got):
        assert status == 0 and z, name
        idat = b"".join(d for t, d in png_chunks(cv2_one(ext, imgs[0], params)) if t == b"IDAT")
        assert z == idat, name
        seen[imgs.shape[-1]] |= cls
    for c, cls in seen.items():
        assert all((cls >> k) & 1 for k in (19, 20)), (c, hex(cls))


def segments(stream):
    segs, p = [], 2
    while p < len(stream) - 2:
        m, ln = stream[p + 1], struct.unpack_from(">H", stream, p + 2)[0]
        segs.append((m, stream[p + 4:p + 2 + ln]))
        p += 2 + ln
        if m == 0xDA:   # skip the entropy-coded data to the next marker that is not a stuffed byte or RSTn
            while not (stream[p] == 0xFF and stream[p + 1] not in (0x00, *range(0xD0, 0xD8))):
                p += 1
    return segs


def test_grey_header_constants():
    from cameracalibration_b200 import _lib as L  # noqa: F401  (the package imports without a GPU)
    rng = np.random.default_rng(1)
    g = E.image(rng, 19, 23, 1)[..., 0]
    s = cv2.imencode(".jpg", g)[1].tobytes()
    assert s.index(b"\xff\xda") + 10 == 328                     # kGreyHeaderBytes
    assert s.index(b"\xff\xc4") == 102                              # kGreyHeaderPrefix
    r = cv2.imencode(".jpg", g, [cv2.IMWRITE_JPEG_RST_INTERVAL, 2])[1].tobytes()
    assert r.index(b"\xff\xda") + 10 == 328 + 6 and r[r.index(b"\xff\xda") - 6:r.index(b"\xff\xda") - 4] == b"\xff\xdd"
    for sf in (0x111111, 0x211111, 0x121111, 0x221111, 0x411111):   # SAMPLING_FACTOR does not reach a grey stream
        assert cv2.imencode(".jpg", g, [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, sf])[1].tobytes() == s


def test_grey_progressive_script():
    """cv2's grey progressive stream: six SOS segments with the script's bands and approximations, one component each,
    five DHT segments (DC0 before the first scan, AC0 before every AC scan)."""
    rng = np.random.default_rng(2)
    g = E.image(rng, 40, 50, 1)[..., 0]
    segs = segments(cv2.imencode(".jpg", g, [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes())
    sos = [s for m, s in segs if m == 0xDA]
    assert [(s[0], s[1], s[2], s[3], s[4], s[5]) for s in sos] == [
        (1, 1, 0x00, 0, 0, 0x01), (1, 1, 0x00, 1, 5, 0x02), (1, 1, 0x00, 6, 63, 0x02), (1, 1, 0x00, 1, 63, 0x21),
        (1, 1, 0x00, 0, 0, 0x10), (1, 1, 0x00, 1, 63, 0x10)]
    dht = [s[0] for m, s in segs if m == 0xC4]
    assert dht == [0x00, 0x10, 0x10, 0x10, 0x10]
    assert [m for m, _ in segs].index(0xC2) < [m for m, _ in segs].index(0xDA)


def test_bounds_hold_for_noise(exe, tmp_path):
    rng = np.random.default_rng(4)
    recs = [(ext, rng.integers(0, 256, (h, w, c), dtype=np.uint8), p) for w, h in ((1, 1), (9, 17), (130, 70))
            for c in (1, 4) for ext, p in ((".jpg", [cv2.IMWRITE_JPEG_QUALITY, 100]), (".jpg", [cv2.IMWRITE_JPEG_QUALITY, 100,
                                                                                             cv2.IMWRITE_JPEG_PROGRESSIVE, 1]),
                                           (".png", []), (".png", [cv2.IMWRITE_PNG_STRATEGY, 2]))]
    for (ext, img, p), (status, _, bound, s, _, _) in zip(recs, host_run(exe, tmp_path, recs)):
        want = cv2_one(ext, img, p)
        assert len(want) <= bound, (ext, img.shape, p)
        if ext == ".jpg" and status == 0:
            assert s == want


def test_refused_png_lists(exe, tmp_path):
    img = np.zeros((4, 4, 1), np.uint8)
    lists = [[cv2.IMWRITE_PNG_COMPRESSION, 0], [cv2.IMWRITE_PNG_COMPRESSION, 2], [cv2.IMWRITE_PNG_STRATEGY, 0],
             [cv2.IMWRITE_PNG_BILEVEL, 1], [cv2.IMWRITE_PNG_ZLIBBUFFER_SIZE, 4096]]
    got = host_run(exe, tmp_path, [(".png", img, p) for p in lists])
    assert [g[0] for g in got] == [2] * len(lists)
