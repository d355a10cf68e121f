"""The fuzz corpus of tests/test_gpu_bev_fuzz.py on the CPU: every case through the plan compilers and their host
interpreters (tests/host/kernel_math.cu `bev` and `bevtma`) at every (stage bytes, entry groups per slot, largest
multi-pass box) setting the GPU test builds engines with, each against the cv2 oracle of tests/bev_cases.py.

tma_plan_info does not report item kinds, so the GPU run alone cannot show that it met multi-pass items, GATHER items
with out-of-frame taps, saturating adds, FULL items, both orientations, empty or edge tiles.  The plan compiler is
deterministic: the per-kind counts the interpreter prints here are what the device ran on the same input.  Summed over
the cases a setting renders, every kind the setting can produce must occur -- so an edit that thins the corpus fails
here, without a GPU."""
import subprocess

import numpy as np

from tests import bev_cases as B
from tests.test_host_math import exe  # noqa: F401  (module fixture: builds kernel_math)


def _kinds(stdout):
    line = next(ln for ln in stdout.splitlines() if ln.startswith("tma kinds:"))
    return {k: int(v) for k, v in (t.split("=") for t in line.split(":", 1)[1].split())}


def _run(exe_path, tmp_path, case, mode_args, balance, car):
    (tmp_path / "in.bin").write_bytes(B.blob(case, 0, balance, car))
    r = subprocess.run([exe_path, mode_args[0], str(tmp_path / "in.bin"), str(tmp_path / "out.bin"), *map(str, mode_args[1:])],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (case.name, mode_args, r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    return np.fromfile(tmp_path / "out.bin", np.uint8).reshape(case.BH, case.BW, 3), r.stdout


def _settings():
    """(stage bytes, groups, max mult) -> names of the corpus cases the GPU test renders at that plan setting."""
    out = {B.DEFAULT_PLAN: [c.name for c in B.corpus() if c.tma_friendly]}
    for fs, _slots, _ctas, eg in B.tma_configs():
        for mm in B.MAX_MULTS:
            out.setdefault((fs, eg, mm), [])
            out[(fs, eg, mm)] += [n for n in B.CONFIG_CASES if n not in out[(fs, eg, mm)]]
    return out


def test_fuzz_corpus_on_the_host_reaches_every_plan_feature(exe, tmp_path):  # noqa: F811
    cases = {c.name: c for c in B.corpus()}
    # BALANCE runs on the 4-camera cases: between them they sample OpenCV's luminance row tails of 1, 16 and 31 px and
    # every kernel path (TMA plan, gather, per-tap)
    four = [c for c in cases.values() if c.NC == 4]
    assert {1, 16, 31} <= {c.FW % 32 for c in four}, sorted((c.name, c.FW) for c in four)
    assert {(c.FW * 3) % 16 == 0 for c in four} == {True, False} and any((c.FW * 3) % 4 for c in four), sorted((c.name, c.FW) for c in four)
    # every case through the round-1 plan (k_bev's), frame-set 0; BALANCE with the car on the 4-camera cases
    for c in cases.values():
        balance = c.NC == 4 and B.oracle(c, 0, True, True) is not None
        got, _ = _run(exe, tmp_path, c, ("bev",), balance, balance)
        want = B.oracle(c, 0, balance, balance)
        assert (got == want).all(), (c.name, balance, int((got != want).sum()))
    for (fs, eg, mm), names in _settings().items():
        total = {}
        for n in names:
            c = cases[n]
            balance = c.NC == 4 and B.oracle(c, 0, True, True) is not None
            got, out = _run(exe, tmp_path, c, ("bevtma", fs, eg, mm), balance, balance)
            want = B.oracle(c, 0, balance, balance)
            assert (got == want).all(), (n, (fs, eg, mm), balance, int((got != want).sum()))
            for k, v in _kinds(out).items():
                total[k] = total.get(k, 0) + v
        # items of 2 FS exist only when the plan may make them, and 4 FS ones likewise
        need = [k for k in total if not (k == "fs2" and mm < 2) and not (k == "fs4" and mm < 4)]
        assert all(total[k] > 0 for k in need), ((fs, eg, mm), names, total)
        assert (mm >= 2 or total["fs2"] == 0) and (mm >= 4 or total["fs4"] == 0), ((fs, eg, mm), total)
