"""Python argument rules of ops.resize and ops.warp_affine that hold without a device: cv2's output size from dsize or
fx / fy, and the refusals made before any library call."""
import cv2
import numpy as np
import pytest

from cameracalibration_b200 import _lib as L
from cameracalibration_b200 import ops


def test_resize_size_follows_cv2():
    rng = np.random.default_rng(3)
    for sw, sh in [(9, 7), (5, 3), (1280, 1024), (1, 1)]:
        img = np.zeros((sh, sw), np.uint8)
        for fx, fy in [(0.5, 0.5), (1.5, 2.5), (0.37, 0.37), *rng.uniform(0.1, 3, (20, 2)).tolist()]:
            if round(sw * fx) < 1 or round(sh * fy) < 1:
                continue
            want = cv2.resize(img, (0, 0), fx=fx, fy=fy).shape
            assert ops.resize_size((sw, sh), (0, 0), fx, fy) == (want[1], want[0])
            assert ops.resize_size((sw, sh), None, fx, fy) == (want[1], want[0])
        assert ops.resize_size((sw, sh), (4, 6), 9.0, 9.0) == (4, 6)   # a dsize wins over fx, fy, as in cv2
    for fx, fy in [(0, 0), (0.5, 0), (-1, 1)]:
        with pytest.raises(L.BevkError, match="fx > 0"):
            ops.resize_size((10, 10), (0, 0), fx, fy)
    with pytest.raises(L.BevkError, match="empty"):
        ops.resize_size((10, 10), (0, 0), 0.01, 0.5)


def test_refused_before_the_library():
    img = np.zeros((8, 8, 3), np.uint8)
    with pytest.raises(L.BevkError, match="BORDER_CONSTANT"):
        ops.warp_affine(img, np.eye(2, 3), (8, 8), borderMode=cv2.BORDER_REFLECT)
    with pytest.raises(L.BevkError, match="BORDER_CONSTANT"):
        ops.warp_affine(img, np.eye(2, 3), (8, 8), borderValue=(1, 0, 0))
    assert (ops.INTER_LINEAR_EXACT, ops.INTER_NEAREST_EXACT, ops.WARP_INVERSE_MAP) == (
        cv2.INTER_LINEAR_EXACT, cv2.INTER_NEAREST_EXACT, cv2.WARP_INVERSE_MAP)
