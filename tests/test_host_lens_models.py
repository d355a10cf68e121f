"""cv2's rational, thin-prism and tilted pinhole models and rectification rotations (both models) on the CPU:
tests/host/lens_models.cu runs the kernels' camera set-up and coordinate code (lens_model, walk_rays,
undistort_point<LENS>, warp_maps_pixel<1, LENS>; host forms, no FMA contraction) over the seeded cases of
tests/lens_cases.py, compared with live cv2 byte for byte."""
import os
import shutil
import subprocess

import cv2
import numpy as np
import pytest

from cameracalibration_b200.build import GENCODE
from tests import calib_cases as CC
from tests import lens_cases as LC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    nvcc = next((c for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc") if c and os.path.exists(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("lens_models") / "lens_models"
    build = subprocess.run([nvcc, "-O2", "-std=c++17", "--fmad=false", "-Xcompiler", "-ffp-contract=off", *GENCODE, "-o", str(out),
                            os.path.join(ROOT, "tests", "host", "lens_models.cu")], capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stdout + build.stderr
    return str(out)


def _run(exe, args, values, code=0):
    r = subprocess.run([exe] + [str(a) for a in args], input=" ".join(float(v).hex() for v in values), capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == code, (r.returncode, r.stdout, r.stderr)
    return r.stdout


def _planes(path, w, h):
    raw = np.fromfile(path, np.uint8)
    return raw[:w * h * 4].view(np.int16).reshape(h, w, 2), raw[w * h * 4:].view(np.uint16).reshape(h, w)


def _maps(exe, tmp_path, model, K, D, R, P, w, h, instance=-1):
    out = tmp_path / "maps.bin"
    values = list(np.ravel(K)) + list(np.ravel(D)) + ([] if R is None else list(np.ravel(R))) + list(np.ravel(P))
    text = _run(exe, ["maps", model, w, h, np.size(D), int(R is not None), instance, out], values)
    return _planes(out, w, h), text.split()[:2] == ["lens", "1"]


def _remaps_agree(c, got, want):
    """cv2.remap of a random 3-channel frame through both map pairs gives the same image, LINEAR and NEAREST."""
    f = np.random.default_rng(7).integers(0, 256, (c.UH, c.UW, 3), dtype=np.uint8)
    return all((cv2.remap(f, *got, i) == cv2.remap(f, *want, i)).all() for i in (cv2.INTER_LINEAR, cv2.INTER_NEAREST))


def test_lens_corpus_reaches_every_class():
    """The corpus holds every class of input the wider models and R bring, so that thinning it fails here."""
    cases = LC.corpus()
    pin = [c for c in cases if not c.fisheye]
    fish = [c for c in cases if c.fisheye]
    # every coefficient count cv2 adds, at real sizes and strongly distorted; tilt up to about 0.2 rad
    for n in (8, 12, 14):
        assert {c.kind for c in pin if c.n_dist == n} == {"real", "strong"}, n
    assert {(c.UW, c.UH) for c in pin if c.kind == "real"} >= {(1280, 1024), (1920, 1080), (2560, 2048)}
    tilts = np.abs([t for c in pin for t in c.tilt])
    assert 0.15 < tilts.max() <= 0.2
    assert all(len(set(c.D[8:12])) == 4 for c in pin if c.n_dist >= 12)   # s1..s4 distinct: a swap moves the map
    # rotations for both models, rational ones too; a cv2.stereoRectify pair
    assert any(c.R is not None for c in pin if c.n_dist == 5) and any(c.R is not None for c in pin if c.n_dist >= 8)
    assert all(c.R is not None for c in fish) and any(not LC.xs_table_form(c) for c in fish)
    assert any(c.name.startswith("stereo") for c in pin)
    # the vector body's saturating pack: widths with W % 8 in {0, 1, 7}, saturated map1 entries among them
    strong = [c for c in pin if c.kind == "strong"]
    assert {c.UW % 8 for c in strong} >= {0, 1, 7}
    for r in (1, 7):
        assert any(((LC.cv2_maps(c.name)[0] == 32767) | (LC.cv2_maps(c.name)[0] == -32768)).any() for c in strong if c.UW % 8 == r)
    # fisheye at real sizes, and odd widths
    assert {(c.UW, c.UH) for c in fish} >= {(1280, 1024), (2560, 2048)} and any(c.UW % 2 for c in fish)


def test_lens_maps_vs_cv2(exe, tmp_path):
    """The map of every case, as k_undistort_map builds it (the instance the library picks), == cv2's maps with R: no
    tolerance for the fisheye, calib_cases.pinhole_outside_only for the pinhole (whose cv2 build contracts FMAs), with
    identical remapped images."""
    n = n_tolerated = 0
    for c in LC.corpus():
        got, lens = _maps(exe, tmp_path, c.model, c.K, c.D, c.R, c.P, c.UW, c.UH)
        want = LC.cv2_maps(c.name)
        # the LENS = 1 instance exactly when the camera needs it: extra pinhole terms, or rays walked row by row
        needs = (not c.fisheye and (np.any(c.D[5:] != 0))) or LC.walks(c)
        assert lens == needs, c.name
        n += c.UW * c.UH
        if not ((got[0] == want[0]).all() and (got[1] == want[1]).all()):
            assert not c.fisheye and LC.outside_only(c, got, want), LC.first_diffs(c, got, want)
            assert _remaps_agree(c, got, want), c.name
            n_tolerated += int((got[1] != want[1]).sum())
    assert n > 35_000_000 and n_tolerated < 1000   # about 100 of 40 M entries, all in the strong cases


def test_rotated_fisheye_rays_are_walked(exe, tmp_path):
    """The rays the map code of every rotated fisheye projects (camera_ray in the instance the library picks) are
    cv2's running row sums bit for bit, and they are not the direct form: a map build that skipped the row walk, or a
    walk in another order, fails here even where no cvRound tie shows it in the maps."""
    cases = [c for c in LC.corpus() if c.fisheye and not LC.xs_table_form(c)]
    assert cases
    for c in cases:
        out = tmp_path / "rays.bin"
        _run(exe, ["rays", 0, c.UW, c.UH, 4, 1, out], list(c.K.ravel()) + list(c.D) + list(c.R.ravel()) + list(c.P.ravel()))
        got = np.fromfile(out, np.float64).reshape(3, c.UH, c.UW)
        want = LC.walked_rays(c)
        bad = got != want
        assert not bad.any(), (c.name, int(bad.sum()), np.argwhere(bad)[:3])
        assert (want != LC.direct_rays(c)).any(), c.name


def test_full_instance_equals_todays_on_calib_cases(exe, tmp_path):
    """On every camera of calib_cases (4-coefficient fisheye, 5-coefficient pinhole, R = I), the LENS = 1 instance
    computes exactly the bytes of the LENS = 0 instance, so choosing between them can never change a map."""
    for c in CC.corpus():
        D = c.D if c.fisheye else c.d5
        base, lens = _maps(exe, tmp_path, c.model, c.K, D, None, c.P, c.UW, c.UH, instance=0)
        assert not lens, c.name
        full, _ = _maps(exe, tmp_path, c.model, c.K, D, None, c.P, c.UW, c.UH, instance=1)
        assert (base[0] == full[0]).all() and (base[1] == full[1]).all(), c.name
        # R = I given explicitly is R = NULL
        withI, _ = _maps(exe, tmp_path, c.model, c.K, D, np.eye(3), c.P, c.UW, c.UH)
        assert (base[0] == withI[0]).all() and (base[1] == withI[1]).all(), c.name


def test_bev_lut_vs_cv2_pinhole(exe, tmp_path):
    """k_warp_maps<1, LENS> of every unrotated pinhole case (and the 5-coefficient strong cases of calib_cases) ==
    cv2.warpPerspective of cv2's map planes."""
    cases = [c for c in LC.corpus() if not c.fisheye and c.R is None]
    assert {c.n_dist for c in cases} == {8, 12, 14}
    for c in cases:
        out = tmp_path / "bev.bin"
        _run(exe, ["bevmaps", 1, c.UW, c.UH, c.n_dist, c.BW, c.BH, out],
             list(c.K.ravel()) + list(c.D) + list(c.P.ravel()) + list(c.H.ravel()))
        got, want = _planes(out, c.BW, c.BH), LC.cv2_bev_maps(c.name)
        assert (got[0] == want[0]).all() and (got[1] == want[1]).all(), (c.name, LC.first_diffs(c, got, want))


@pytest.mark.parametrize("model,n", [(1, 1), (1, 2), (1, 3), (1, 6), (1, 7), (1, 9), (1, 13), (1, 15),
                                     (0, 1), (0, 3), (0, 5), (0, 8)])
def test_refuses_d_lengths_cv2_refuses(exe, tmp_path, model, n):
    """A pinhole D of other than 0, 4, 5, 8, 12 or 14 coefficients, a fisheye D of other than 0 or 4: refused as cv2
    refuses them."""
    c = CC.corpus()[0]
    _run(exe, ["maps", model, 64, 48, n, 0, -1, tmp_path / "x.bin"], list(c.K.ravel()) + [0.01] * n + list(c.P.ravel()), code=5)
    K, D = c.K, np.full(n, 0.01)
    fn = cv2.fisheye.initUndistortRectifyMap if model == 0 else cv2.initUndistortRectifyMap
    with pytest.raises(cv2.error):
        fn(K, D.reshape(-1, 1) if model == 0 else D, np.eye(3), c.P, (64, 48), cv2.CV_16SC2)
