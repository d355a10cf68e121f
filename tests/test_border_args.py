"""Python argument rules of the gathers' borderMode / borderValue that hold without a device: the refusals made before
any library call, and the constants, which are cv2's."""
import cv2
import numpy as np
import pytest

from cameracalibration_b200 import _lib as L
from cameracalibration_b200 import ops


def test_border_refusals_before_the_library():
    """BORDER_TRANSPARENT without out= and a borderValue of more than four values raise BevkError from every gather
    before the library is called.  The constants are cv2's."""
    img = np.zeros((8, 8, 3), np.uint8)
    m1, m2 = np.zeros((4, 4, 2), np.int16), np.zeros((4, 4), np.uint16)
    fx = np.zeros((4, 4), np.float32)
    calls = [lambda **k: ops.warp_affine_border(img, np.eye(2, 3), (8, 8), **k),
             lambda **k: ops.warp_perspective(img, np.eye(3), (8, 8), **k),
             lambda **k: ops.remap(img, m1, m2, cv2.INTER_LINEAR, **k),
             lambda **k: ops.remap(img, fx, fx, cv2.INTER_LINEAR, **k)]
    for call in calls:
        with pytest.raises(L.BevkError, match="needs out="):
            call(borderMode=cv2.BORDER_TRANSPARENT)
        with pytest.raises(L.BevkError, match="up to 4 values"):
            call(borderValue=(1, 2, 3, 4, 5))
    assert (ops.INTER_LINEAR_EXACT, ops.INTER_NEAREST_EXACT, ops.WARP_INVERSE_MAP) == (
        cv2.INTER_LINEAR_EXACT, cv2.INTER_NEAREST_EXACT, cv2.WARP_INVERSE_MAP)
    assert (ops.BORDER_CONSTANT, ops.BORDER_REPLICATE, ops.BORDER_REFLECT, ops.BORDER_WRAP, ops.BORDER_REFLECT_101,
            ops.BORDER_TRANSPARENT) == (cv2.BORDER_CONSTANT, cv2.BORDER_REPLICATE, cv2.BORDER_REFLECT, cv2.BORDER_WRAP,
                                        cv2.BORDER_REFLECT_101, cv2.BORDER_TRANSPARENT)
