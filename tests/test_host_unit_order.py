"""k_bev_tma's work units on the CPU: the plan compiler's tile order (bevk_plan_tma.cuh tile_order: a Hilbert curve over
the tile grid, the cheapest tiles last) decoded as the producer decodes a unit (tile u / groups, frame-set group
u % groups) hands out every (tile, group) exactly once, for batches that are and are not multiples of the four
frame-sets of a unit, tile grids that are not powers of two, and the output-window skip of camera-sharded slabs.  nvcc
compiles the harness; only host code runs."""
import os
import shutil
import subprocess

import pytest

from cameracalibration_b200.build import GENCODE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    nvcc = next((c for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc") if c and os.path.exists(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("unit_order") / "unit_order"
    build = subprocess.run([nvcc, "-O2", "-std=c++17", *GENCODE, "-o", str(out), os.path.join(ROOT, "tests", "host", "unit_order.cu")],
                           capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stdout + build.stderr
    return str(out)


TAILS = [10, 0, 100, 37]   # the plan's default share of cheapest tiles kept for the end, none, all, an odd one
GEOMETRIES = [(32, 32), (38, 38), (31, 17), (1, 1), (3, 40), (63, 63)]   # tiles x, y: bench 1000², cfg3 1200², odd shapes


@pytest.mark.parametrize("tail", TAILS)
@pytest.mark.parametrize("batch", [1, 3, 4, 7, 9, 32])
def test_units_cover_every_tile_and_group_once(exe, tail, batch):
    for i, (tx, ty) in enumerate(GEOMETRIES):
        r = subprocess.run([exe, str(tx), str(ty), str(batch), str(tail), str(i + 7 * batch)], capture_output=True, text=True,
                           timeout=120)
        assert r.returncode == 0 and r.stdout.startswith("ok"), (tx, ty, r.stdout, r.stderr)


@pytest.mark.parametrize("tail", TAILS)
def test_window_skip_keeps_the_slab_tiles(exe, tail):
    # camera-sharded slab of a 1000x1000 canvas (tile-aligned bounding box of some cameras' masks) and an unaligned window
    for win in ((0, 0, 1024, 384), (320, 96, 700, 1000), (33, 65, 34, 66)):
        for batch in (1, 7, 32):
            r = subprocess.run([exe, "32", "32", str(batch), str(tail), "5", *map(str, win)], capture_output=True, text=True,
                               timeout=120)
            assert r.returncode == 0 and r.stdout.startswith("ok"), (win, batch, r.stdout, r.stderr)
