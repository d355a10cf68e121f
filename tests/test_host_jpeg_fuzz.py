"""The encoder corpus of tests/jpeg_cases.py on the CPU: every class it promises is present, and every image of it goes
through tests/host/jpeg_enc.cu (the __host__ __device__ stages of bevk_jpeg_enc.cuh run serially) with streams equal
to cv2.imencode's, within bevk_jpeg_encode_bound, and entropy bit counts that agree with cv2's stream."""
from tests import jpeg_cases as J
from tests.test_host_jpeg import _host_encode, exe  # noqa: F401  (exe: the module fixture that builds the harness)

BATCH_CLASSES = ("cta_starts_mid_image", "cta_starts_mid_mcu", "mixed_batch", "n_over_100", "q_clamped")


def test_jpeg_corpus_reaches_every_class():
    got = set()
    for c in J.corpus():
        got |= J.case_classes(c)
        for s in J.streams(c.name):
            got |= J.stream_classes(s)
    want = ({f"w16_{r}" for r in range(16)} | {f"h16_{r}" for r in range(16)}
            | {f"{a}_{d}" for a in "wh" for d in J.SMALL_DIMS + (J.MAX_DIM,)}
            | {f"layout_{x}" for x in J.LAYOUTS} | {f"content_{x}" for x in list(J.CONTENTS) + ["mixed"]}
            | {f"nblk_{b}" for b in J.BATCH_SIZES} | set(BATCH_CLASSES) | set(J.STREAM_CLASSES))
    assert not want - got, f"classes the corpus misses: {sorted(want - got)}"
    qualities = {c.quality for c in J.corpus()}
    assert {-5, 0, 100, 150} <= qualities and len(qualities & set(range(1, 100))) >= 10, sorted(qualities)
    assert {(J.MAX_DIM, 1), (J.MAX_DIM, 17), (1, J.MAX_DIM), (17, J.MAX_DIM)} <= {(c.W, c.H) for c in J.corpus()}


def test_host_harness_over_corpus(exe, tmp_path):  # noqa: F811
    cases = [(img, c.quality, c.name, want) for c in J.corpus() for img, want in zip(c.images, J.streams(c.name))]
    mods = set()
    for k in range(0, len(cases), 400):
        part = cases[k:k + 400]
        for (img, q, name, want), (got, bound, bits) in zip(part, _host_encode(exe, tmp_path, [(i, q) for i, q, _, _ in part])):
            first = next((i for i in range(min(len(got), len(want))) if got[i] != want[i]), None)
            assert got == want, (name, img.shape, q, len(got), len(want), first)
            assert len(got) <= bound, (name, len(got), bound)
            e = J.entropy_segment(want)
            assert (bits + 7) // 8 == len(e), (name, bits, len(e))
            if e[-1] & 1 == 0:                      # no pad: the stream ends on a whole byte
                assert bits == 8 * len(e), (name, bits, len(e))
            mods |= {m for m in (8, 32) if bits % m == 0}
    assert mods == {8, 32}, mods
