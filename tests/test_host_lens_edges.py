"""The edge cases of tests/lens_edge_cases.py on the CPU: tests/host/lens_models.cu runs the kernels' camera set-up and
coordinate code (lens_model, row_sums / walk_rays, undistort_point<LENS>, warp_maps_pixel<1, LENS>; host forms, no FMA
contraction) on every case, compared with live cv2 under the rules of tests/test_host_lens_models.py: no tolerance for
the fisheye, calib_cases.pinhole_outside_only plus identical cv2.remap images for the pinhole."""
import numpy as np

from tests import lens_cases as LC
from tests import lens_edge_cases as E
from tests.test_host_lens_models import _maps, _planes, _remaps_agree, _run, exe  # noqa: F401  (exe: the module fixture)


def test_lens_edge_corpus_reaches_every_class():
    """The corpus holds every edge class, counted from the NumPy restatement, so that thinning it fails here."""
    cases = E.corpus()
    total = {}
    for c in cases:
        for k, v in E.classes(c).items():
            total[k] = total.get(k, 0) + v
    missing = [k for k in ("int_min", "saturated", "wrapped", "w_le0", "w_eq0", "pole", "vz_le0") if total.get(k, 0) == 0]
    assert not missing, (missing, total)
    pin = [c for c in cases if not c.fisheye]
    fish = [c for c in cases if c.fisheye]
    # pixels of every W % 8 class of the pinhole vector body, in rotated (walked) cameras
    assert {c.UW % 8 for c in pin if LC.walks(c)} == set(range(8))
    # rational poles for 8, 12 and 14 coefficients; vz <= 0 under a tilt of about 1 rad
    assert {c.n_dist for c in pin if E.classes(c)["pole"]} >= {8, 12, 14}
    assert max(abs(t) for c in pin for t in c.tilt) >= 0.95
    # rotations up to 1.2 rad with _w <= 0 in the frame, for both models
    ang = lambda c: np.linalg.norm(__import__("cv2").Rodrigues(c.R)[0]) if c.R is not None else 0.0
    for group in (pin, fish):
        assert any(ang(c) > 1.15 and E.classes(c)["w_le0"] for c in group)
    # _w == 0 exactly on integer pixels through an exact (dyadic) inv(P * R), for both models
    dy = [c for c in cases if c.name.startswith("dyadic")]
    assert {c.model for c in dy} == {0, 1} and all(E.dyadic_exact(c) and E.classes(c)["w_eq0"] for c in dy)
    # a stereoRectify pair with a vertical baseline; odd-width rotated fisheyes; 1 x N and N x 1 maps; W = 1..9
    assert sum(c.name.startswith("stereov") for c in pin) == 2
    assert any(c.UW % 2 and LC.walks(c) for c in fish)
    assert {(c.model, c.UW == 1, c.UH == 1) for c in cases if 1 in (c.UW, c.UH)} >= {(0, True, False), (0, False, True),
                                                                                  (1, True, False), (1, False, True)}
    assert {c.UW for c in pin} >= set(range(1, 10))
    # one walked fisheye at 3840 x 2160
    assert any(c.fisheye and LC.walks(c) and (c.UW, c.UH) == (3840, 2160) for c in cases)
    # the LENS choice boundaries: one extra coefficient alone (k6, s4, tauY), R = I given, R keeping the column table
    extra = lambda c, i: c.n_dist > i and c.D[i] != 0 and np.count_nonzero(c.D[5:]) == 1
    assert all(any(extra(c, i) for c in pin) for i in (7, 11, 13))
    assert {c.model for c in cases if c.R is not None and (c.R == np.eye(3)).all()} == {0, 1}
    assert {c.model for c in cases if c.R is not None and not (c.R == np.eye(3)).all() and not LC.walks(c)} == {0, 1}


def _args(c):
    return list(c.K.ravel()) + list(c.D) + ([] if c.R is None else list(c.R.ravel())) + list(c.P.ravel())


def test_lens_edge_maps_vs_cv2(exe, tmp_path):
    """The map of every edge case, as k_undistort_map builds it in the instance the library picks, == cv2's: no tolerance
    for the fisheye, pinhole_outside_only with identical remapped images for the pinhole; and the instance is LENS = 1
    exactly when the camera has extra pinhole terms or walks its rays."""
    for c in E.corpus():
        got, lens = _maps(exe, tmp_path, c.model, c.K, c.D, c.R, c.P, c.UW, c.UH)
        assert lens == ((not c.fisheye and bool(np.any(c.D[5:] != 0))) or LC.walks(c)), c.name
        want = E.cv2_maps(c.name)
        if not ((got[0] == want[0]).all() and (got[1] == want[1]).all()):
            assert not c.fisheye and LC.outside_only(c, got, want), LC.first_diffs(c, got, want)
            assert _remaps_agree(c, got, want), c.name


def test_lens_edge_rays_are_cv2s(exe, tmp_path):
    """The rays every edge case projects (camera_ray in the instance the library picks: walked, column table or direct)
    are cv2's running sums bit for bit: per column for the fisheye, per 8-column block with in-block offsets and a
    running scalar tail for the pinhole."""
    for c in E.corpus():
        out = tmp_path / "rays.bin"
        _run(exe, ["rays", c.model, c.UW, c.UH, c.n_dist, int(c.R is not None), out], _args(c))
        got = np.fromfile(out, np.float64).reshape(3, c.UH, c.UW)
        bad = got != E.cv2_rays(c)
        assert not bad.any(), (c.name, int(bad.sum()), np.argwhere(bad)[:3])


def test_lens_edge_bev_lut_vs_cv2(exe, tmp_path):
    """k_warp_maps<1, LENS> of every unrotated pinhole edge case (poles, large thin prism, tilt, LENS boundaries) under
    its homography, horizons crossing the canvas among them, == cv2.warpPerspective of cv2's map planes."""
    cases = [c for c in E.corpus() if not c.fisheye and (c.R is None or (c.R == np.eye(3)).all())]
    assert {c.n_dist for c in cases} >= {5, 8, 12, 14}
    for c in cases:
        out = tmp_path / "bev.bin"
        _run(exe, ["bevmaps", 1, c.UW, c.UH, c.n_dist, c.BW, c.BH, out], list(c.K.ravel()) + list(c.D) + list(c.P.ravel())
             + list(c.H.ravel()))
        got, want = _planes(out, c.BW, c.BH), E.cv2_bev_maps(c.name)
        assert (got[0] == want[0]).all() and (got[1] == want[1]).all(), (c.name, LC.first_diffs(c, got, want))
