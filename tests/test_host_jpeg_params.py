"""The device JPEG encoder under cv2.imwrite's JPEG parameters, on the CPU.  tests/host/jpeg_params.cu runs jpeg::normalise
and the __host__ __device__ stage functions of bevk_jpeg_enc.cuh in the general MCU layout serially over whole images;
every stream of the tests/jpeg_params_cases.py corpus must equal cv2.imencode(".jpg", img, [IMWRITE_JPEG_QUALITY, q] +
params) byte for byte (the DHT segments compared first, so the optimal-table builder is pinned apart from the entropy
data) and stay within the params bound, and the normaliser must agree with cv2 on every rule."""
import os
import shutil
import struct
import subprocess

import cv2
import numpy as np
import pytest

from cameracalibration_b200.build import GENCODE
from tests import jpeg_params_cases as J

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    nvcc = next((c for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc") if c and os.path.exists(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("host_jpeg_params") / "jpeg_params"
    build = subprocess.run([nvcc, "-O2", "-std=c++17", *GENCODE, "-o", str(out), os.path.join(ROOT, "tests", "host", "jpeg_params.cu")],
                           capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stdout + build.stderr
    return str(out)


def cv2_stream(img, q, params):
    return cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q] + list(params))[1].tobytes()


def host_run(exe, tmp_path, records):
    """records: [(BGR image, quality, params)] -> [(opts dict, stream, bound, bits)] from the host build."""
    blob = [struct.pack(f"<4i{len(p)}i", img.shape[1], img.shape[0], q, len(p), *p) + np.ascontiguousarray(img).tobytes()
            for img, q, p in records]
    (tmp_path / "in.bin").write_bytes(b"".join(blob))
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, (r.returncode, r.stderr[-2000:])
    raw, p, out = (tmp_path / "out.bin").read_bytes(), 0, []
    for _ in records:
        ok, hy, vy, qy, qc, rst, opt, prog = struct.unpack_from("<8i", raw, p)
        n, bound, bits, padmask, ffend = struct.unpack_from("<5Q", raw, p + 32)
        out.append((dict(ok=ok, hy=hy, vy=vy, qy=qy, qc=qc, rst=rst, optimize=opt, progressive=prog, padmask=padmask,
                         ffend=ffend), raw[p + 72:p + 72 + n], bound, bits))
        p += 72 + n
    assert p == len(raw)
    return out


def segments(stream):
    """[(marker, payload)] of the header up to SOS, then ("ECS", rest)."""
    segs, p = [], 2
    while True:
        m, ln = stream[p + 1], struct.unpack_from(">H", stream, p + 2)[0]
        segs.append((m, stream[p + 4:p + 2 + ln]))
        p += 2 + ln
        if m == 0xDA:
            segs.append(("ECS", stream[p:]))
            return segs


def header_opts(stream):
    """(hy, vy, luma table, chroma table, DRI present) read off a stream."""
    segs = segments(stream)
    sof = next(s for m, s in segs if m == 0xC0)
    dqt = {s[0]: s[1:65] for m, s in segs if m == 0xDB}
    return sof[7] >> 4, sof[7] & 15, dqt[0], dqt[1], any(m == 0xDD for m, _ in segs)


def assert_same(got, want, what):
    if got == want:
        return
    gs, ws = segments(got), segments(want)
    # DHT segments apart: a table difference is reported before any entropy-data difference
    assert [s for s in gs if s[0] == 0xC4] == [s for s in ws if s[0] == 0xC4], (what, "DHT")
    first = next((i for i in range(min(len(got), len(want))) if got[i] != want[i]), None)
    raise AssertionError((what, len(got), len(want), first))


def test_corpus_reaches_every_class():
    have = set().union(*(c.classes for c in J.cases()))
    missing = J.required_classes() - have
    assert not missing, sorted(missing)


def test_corpus_byte_equal_to_cv2(exe, tmp_path):
    records, whats = [], []
    for c in J.cases():
        for k, img in enumerate(c.images):
            records.append((img, c.quality, c.params))
            whats.append((c.name, k, img.shape))
    padmask = ffend = 0
    n_opt_dht = 0
    for (img, q, params), what, (opts, got, bound, bits) in zip(records, whats, host_run(exe, tmp_path, records)):
        assert opts["ok"] == 1, what
        want = cv2_stream(img, q, params)
        assert_same(got, want, what)
        assert len(got) <= bound, (what, len(got), bound)
        # the params bound is what bevk_jpeg_encode_bound_params reports: header (+ DRI), blocks at 1660 bits (1665
        # with optimised tables) plus 7 pad bits per interval, doubled for stuffing, 2 bytes per RSTn, EOI
        hy, vy, rst = opts["hy"], opts["vy"], opts["rst"]
        mcus = -(-img.shape[1] // (8 * hy)) * -(-img.shape[0] // (8 * vy))
        nint = -(-mcus // rst) if rst else 1
        blocks = J.blocks_per_image(img.shape[1], img.shape[0], hy, vy)
        maxbits = 1665 if opts["optimize"] else 1660
        assert bound == 623 + (6 if rst else 0) + 2 * ((blocks * maxbits + 7 * nint) // 8) + 2 * (nint - 1) + 2, what
        padmask |= opts["padmask"]
        ffend |= opts["ffend"] and rst > 0
        if opts["optimize"]:
            dht = [s for s in segments(want) if s[0] == 0xC4]
            assert all(len(s) <= (16 + 1 + 162 if s[0] >> 4 else 16 + 1 + 12) for _, s in dht), what
            n_opt_dht += 1
    assert padmask == 0xFF, bin(padmask)                    # every pad length 0-7 occurs at an interval's end
    assert ffend, "no restart interval whose data ends in 0xFF"
    assert n_opt_dht > 20


def test_dht_segments_and_largest_streams(exe, tmp_path):
    """DHT segments equal cv2's (Annex K, and the optimal tables of flat, noise and checkerboard images, pinned apart
    from the entropy data), and 4:4:4 noise at q100 with one MCU per interval and optimised tables stays within the
    params bound."""
    rng = np.random.default_rng(5)
    img = rng.integers(0, 256, (96, 80, 3), dtype=np.uint8)
    flat = np.full((40, 48, 3), 77, np.uint8)
    yy, xx = np.mgrid[0:40, 0:48]
    checker = np.repeat((((yy + xx) & 1) * 255).astype(np.uint8)[..., None], 3, -1)
    recs = [(img, 100, [J.SAMPLING, sf]) for sf in J.SAMPLINGS] + [(img, 100, [J.LUMA, 100, J.CHROMA, 99])]
    recs += [(im, 100, [J.SAMPLING, 0x111111, J.OPTIMIZE, 1, J.RST, r]) for im in (img, flat, checker) for r in (0, 1)]
    for (im, q, p), (_, got, bound, _) in zip(recs, host_run(exe, tmp_path, recs)):
        want = cv2_stream(im, q, p)
        assert [s for s in segments(got) if s[0] == 0xC4] == [s for s in segments(want) if s[0] == 0xC4]
        assert got == want and len(got) <= bound


NORMALISER_LISTS = [
    [], [5, 80], [5, 150], [5, -1], [5, 0], [5, 100], [6, 80], [6, 80, 5, 80], [5, 80, 6, 80], [5, 90, 6, 70],
    [6, 70, 5, 90], [5, 90, 6, -4], [5, 90, 6, 300], [5, 100, 6, 101], [5, 0, 6, 1], [5, 1, 6, 0], [5, 60, 1, 10],
    [1, 10, 5, 60], [1, 10, 6, 60], [1, -7], [1, 0], [1, 200], [5, -20, 6, 40],
    [7, 0x111111], [7, 0x211111], [7, 0x121111], [7, 0x221111], [7, 0x411111], [7, 0x141111], [7, 0x222222],
    [7, 0x112111], [7, 0], [7, -1], [7, 0x111111, 7, 0x3], [7, 0x411111, 5, 50, 6, 60], [7, 0x411111, 5, 50, 6, 50],
    [7, 0x211111, 6, 20], [2, 0], [3, 0], [4, 0], [4, -3], [3, 0, 2, 0, 4, -65536],
]


def test_normaliser_agrees_with_cv2(exe, tmp_path):
    """jpeg::normalise against the header cv2 writes: Y sampling byte, both quantisation tables, no DRI.  QUALITY
    pairs inside the list are accepted by the normaliser (bevk_jpeg_set_params refuses them; the call's quality is
    normalise's first argument)."""
    img = np.random.default_rng(9).integers(0, 256, (20, 36, 3), dtype=np.uint8)
    recs = [(img, q, p) for p in NORMALISER_LISTS for q in (-5, 0, 40, 95, 101)]
    for (im, q, p), (opts, got, _, _) in zip(recs, host_run(exe, tmp_path, recs)):
        want = cv2_stream(im, q, p)
        hy, vy, lq, cq, dri = header_opts(want)
        assert (opts["ok"], opts["hy"], opts["vy"], dri) == (1, hy, vy, False), (q, p, opts)
        got_h = header_opts(got)
        assert got_h[2] == lq and got_h[3] == cq, (q, p, opts)
        assert got == want, (q, p)


def test_normaliser_flags_and_refusals(exe, tmp_path):
    """Odd lists and unknown keys are refused; RST_INTERVAL is clamped to [0, 65535].  OPTIMIZE and PROGRESSIVE are read
    as cv2 reads them, on above 0 only: a PROGRESSIVE list is progressive exactly when cv2 writes SOF2 for it, and every
    other list's stream equals cv2's (PROGRESSIVE streams are not written here: no stream)."""
    img = np.random.default_rng(3).integers(0, 256, (24, 40, 3), dtype=np.uint8)
    recs = [(img, 95, p) for p in ([5], [8, 1], [0, 1], [4, 1], [4, 65536], [4, -1], [4, 70000])]
    res = [o for o, *_ in host_run(exe, tmp_path, recs)]
    assert [r["ok"] for r in res] == [0, 0, 0] + [1] * 4
    assert [r["rst"] for r in res[3:7]] == [1, 65535, 0, 65535]
    # cv2 writes a DRI for a positive interval
    assert header_opts(cv2_stream(img, 95, [4, 1]))[4]
    flags = [[3, -1], [3, 5], [2, -2], [2, 1]]
    for p, (opts, got, _, _) in zip(flags, host_run(exe, tmp_path, [(img, 95, p) for p in flags])):
        want = cv2_stream(img, 95, p)
        assert opts["ok"] == 1, p
        assert opts["progressive"] == any(m == 0xC2 for m, _ in segments(want)), (p, opts)
        if not opts["progressive"]:
            assert_same(got, want, p)
