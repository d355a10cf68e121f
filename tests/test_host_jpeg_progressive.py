"""The progressive JPEG coder on the CPU.  tests/host/jpeg_progressive.cu runs the __host__ __device__ stage functions of
bevk_jpeg_prog.cuh serially over whole images; every stream of the tests/jpeg_progressive_cases.py corpus must equal
cv2.imencode(".jpg", img, [IMWRITE_JPEG_QUALITY, q] + params) byte for byte (each scan's DHT and SOS compared before the
data) and stay within the bound, the kernels' parallel run resolution must place every flush where the serial state
machine does, and the corpus must reach every flush cause.  Mutating the rules must break the comparison."""
import os
import shutil
import struct
import subprocess

import cv2
import numpy as np
import pytest

from cameracalibration_b200.build import GENCODE
from tests import jpeg_progressive_cases as J

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAUSES = ("symbol", "eob-0x7fff", "correction-bits", "restart", "end-of-scan")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    nvcc = next((c for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc") if c and os.path.exists(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("host_jpeg_progressive") / "jpeg_progressive"
    build = subprocess.run([nvcc, "-O2", "-std=c++17", *GENCODE, "-o", str(out),
                            os.path.join(ROOT, "tests", "host", "jpeg_progressive.cu")], capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stdout + build.stderr
    return str(out)


def cv2_stream(img, q, params):
    return cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q] + list(params))[1].tobytes()


def host_run(exe, tmp_path, records, mutation=0):
    """records: [(BGR image, quality, params)] -> [(meta dict, stream)] from the host build."""
    blob = [struct.pack(f"<4i{len(p)}i", img.shape[1], img.shape[0], q, len(p), *p) + np.ascontiguousarray(img).tobytes()
            for img, q, p in records]
    (tmp_path / "in.bin").write_bytes(b"".join(blob))
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin"), str(mutation)], capture_output=True, text=True,
                       timeout=1800)
    assert r.returncode == 0, (r.returncode, r.stderr[-2000:])
    raw, p, out = (tmp_path / "out.bin").read_bytes(), 0, []
    for _ in records:
        ok, prog, par_ok = struct.unpack_from("<3i", raw, p)
        *causes, bound, n = struct.unpack_from("<7Q", raw, p + 12)
        out.append((dict(ok=ok, progressive=prog, parallel_ok=par_ok, causes=dict(zip(CAUSES, causes)), bound=bound),
                    raw[p + 68:p + 68 + n]))
        p += 68 + n
    assert p == len(raw)
    return out


def scans(stream):
    """[(header segments before the SOS, SOS payload, entropy data with RSTn)] of each scan."""
    out, p, segs = [], 2, []
    while True:
        m = stream[p + 1]
        if m == 0xD9:
            return out
        ln = struct.unpack_from(">H", stream, p + 2)[0]
        payload = stream[p + 4:p + 2 + ln]
        p += 2 + ln
        if m != 0xDA:
            segs.append((m, payload))
            continue
        q = p
        while not (stream[q] == 0xFF and stream[q + 1] not in (0x00,) and not 0xD0 <= stream[q + 1] <= 0xD7):
            q += 1
        out.append((segs, payload, stream[p:q]))
        segs, p = [], q


def frame_marker(stream):
    """The SOFn marker of a stream (0xC0 baseline, 0xC2 progressive)."""
    p = 2
    while not 0xC0 <= stream[p + 1] <= 0xC2:
        p += 2 + struct.unpack_from(">H", stream, p + 2)[0]
    return stream[p + 1]


def assert_same(got, want, what):
    if got == want:
        return
    gs, ws = scans(got), scans(want)
    assert len(gs) == len(ws), (what, len(gs), len(ws))
    for k, (g, w) in enumerate(zip(gs, ws)):
        assert g[0] == w[0], (what, "scan", k, "DHT / DRI")
        assert g[1] == w[1], (what, "scan", k, "SOS")
        assert g[2] == w[2], (what, "scan", k, "data", len(g[2]), len(w[2]))
    raise AssertionError((what, len(got), len(want)))


def corpus_records(small=False):
    records, whats = [], []
    for c in J.cases(small):
        for k, img in enumerate(c.images):
            records.append((img, c.quality, c.params))
            whats.append((c.name, k, img.shape))
    return records, whats


def test_corpus_reaches_every_class():
    have = set().union(*(c.classes for c in J.cases()))
    missing = J.required_classes() - have
    assert not missing, sorted(missing)


def test_corpus_byte_equal_to_cv2(exe, tmp_path):
    records, whats = corpus_records()
    causes = dict.fromkeys(CAUSES, 0)
    for (img, q, params), what, (meta, got) in zip(records, whats, host_run(exe, tmp_path, records)):
        assert meta["ok"] == 1, what
        want = cv2_stream(img, q, params)
        assert meta["progressive"] == J.params_progressive(params) == (frame_marker(want) == 0xC2), what
        if not meta["progressive"]:
            continue
        assert meta["parallel_ok"] == 1, what
        assert_same(got, want, what)
        assert len(got) <= meta["bound"], (what, len(got), meta["bound"])
        for k, v in meta["causes"].items():
            causes[k] += v
    # every flush cause is reached by the corpus
    assert all(causes.values()), causes


def test_script_and_headers(exe, tmp_path):
    """Ten scans in cv2's order, SOF2, the DHTs before each SOS and one DRI after scan 1's DHTs."""
    img = J.smooth(np.random.default_rng(3), 40, 24)
    want = cv2_stream(img, 90, J.P + [J.RST, 2])
    ss = scans(want)
    assert b"\xff\xc2" in want and len(ss) == 10
    sos = [(s[1][0], tuple(s[1][1:1 + 2 * s[1][0]:2]), s[1][-3], s[1][-2], s[1][-1]) for s in ss]
    assert sos == [(3, (1, 2, 3), 0, 0, 1), (1, (1,), 1, 5, 2), (1, (3,), 1, 63, 1), (1, (2,), 1, 63, 1), (1, (1,), 6, 63, 2),
                   (1, (1,), 1, 63, 0x21), (3, (1, 2, 3), 0, 0, 0x10), (1, (3,), 1, 63, 0x10), (1, (2,), 1, 63, 0x10),
                   (1, (1,), 1, 63, 0x10)]
    assert [m for m, _ in ss[0][0] if m != 0xDB and m != 0xC2 and m != 0xE0] == [0xC4, 0xC4, 0xDD]
    assert [len(s[0]) for s in ss[1:]] == [1, 1, 1, 1, 1, 0, 1, 1, 1]
    # 40 x 24 at 4:2:0 with RST_INTERVAL 2: DC scans 2 markers, luma scans 7, chroma scans 2
    assert [s[2].count(b"\xff\xd0") + sum(s[2].count(bytes([0xFF, 0xD0 + k])) for k in range(1, 8)) for s in ss] == \
        [2, 7, 2, 2, 7, 7, 2, 2, 2, 7]
    (meta, got), = host_run(exe, tmp_path, [(img, 90, J.P + [J.RST, 2])])
    assert got == want


def test_progressive_implies_optimize():
    img = J.smooth(np.random.default_rng(4), 48, 32)
    assert cv2_stream(img, 90, [2, 1]) == cv2_stream(img, 90, [2, 1, 3, 1]) == cv2_stream(img, 90, [2, 7, 3, 0])


@pytest.mark.parametrize("mutation", [1, 2, 3], ids=["corr-limit-1000", "scans-3-4-swapped", "dc-logical-shift"])
def test_mutations_are_caught(exe, tmp_path, mutation):
    """Each mutation of a rule must make some corpus stream differ from cv2."""
    records, whats = corpus_records(small=True)
    records += [(c.images[0], c.quality, c.params) for c in J.cases() if c.name == "corr"]   # crosses the 937-bit flush
    differs = 0
    for (img, q, params), (meta, got) in zip(records, host_run(exe, tmp_path, records, mutation)):
        if meta["progressive"]:
            differs += got != cv2_stream(img, q, params)
    assert differs > 0
