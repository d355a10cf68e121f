"""Drop-in for the hot-path part of the reference's IntrinsicCalibration/intrinsicCalib.py:
``InCalibrator(camera_type).undistort(img)`` with the undistortion map cached on the GPU
(reference: intrinsicCalib.py:90-103 fisheye, :150-163 pinhole, :193-195 undistort).

Chessboard detection and cv2.fisheye.calibrate / cv2.calibrateCamera (the offline
estimation of K and D, reference :44-88, :105-148, :179-208) are outside the hot path
(SURVEY 2 row 6): here K and D are *given* -- ``set_calibration(K, D)`` or by assigning
``camera.data.camera_mat`` / ``camera.data.dist_coeff`` and calling
``camera._get_undistort_maps()``, which is exactly the hand-off the reference's own
``update()`` performs after calibrating.
"""
from __future__ import annotations

import argparse

import numpy as np

from .. import ops

parser = argparse.ArgumentParser(description="Camera Intrinsic Calibration (H100 undistortion path)")
parser.add_argument("-type", "--CAMERA_TYPE", default="fisheye", type=str)
parser.add_argument("-fw", "--FRAME_WIDTH", default=1280, type=int)
parser.add_argument("-fh", "--FRAME_HEIGHT", default=1024, type=int)
parser.add_argument("-fs", "--FOCAL_SCALE", default=0.5, type=float)
parser.add_argument("-ss", "--SIZE_SCALE", default=1, type=float)
args = parser.parse_known_args([])[0]


class CalibData:
    def __init__(self):
        self.type = None
        self.camera_mat = None
        self.dist_coeff = None
        self.rvecs = None
        self.tvecs = None
        self.reproj_err = None
        self.ok = False
        self._und = None
        self._maps = None

    # the maps stay on the device; numpy copies are fetched on first access
    @property
    def map1(self):
        return self._fetch()[0]

    @property
    def map2(self):
        return self._fetch()[1]

    def _fetch(self):
        if self._und is None:
            return (None, None)
        if self._maps is None:
            self._maps = self._und.maps()
        return self._maps


class _Model:
    kind = "fisheye"

    def __init__(self):
        self.data = CalibData()
        self.data.type = self.kind.upper()
        self.inited = False

    def _get_camera_mat_dst(self, camera_mat):
        P = np.array(camera_mat, np.float64)
        P[0, 0] *= args.FOCAL_SCALE
        P[1, 1] *= args.FOCAL_SCALE
        P[0, 2] = args.FRAME_WIDTH / 2 * args.SIZE_SCALE
        P[1, 2] = args.FRAME_HEIGHT / 2 * args.SIZE_SCALE
        return P

    def _get_undistort_maps(self):
        d = self.data
        size = (int(args.FRAME_WIDTH * args.SIZE_SCALE), int(args.FRAME_HEIGHT * args.SIZE_SCALE))
        d._und = ops.Undistorter(d.camera_mat, d.dist_coeff, self._get_camera_mat_dst(d.camera_mat), size,
                                 model=self.kind)
        d._maps = None

    def update(self, corners, frame_size):
        raise Exception("calibration (cv2.fisheye.calibrate / cv2.calibrateCamera) is outside the GPU hot path; "
                        "estimate K, D with the reference and pass them to set_calibration()")


class Fisheye(_Model):
    kind = "fisheye"


class Normal(_Model):
    kind = "pinhole"

    def __init__(self):
        super().__init__()
        self.data.type = "NORMAL"


class InCalibrator:
    def __init__(self, camera):
        if camera == "fisheye":
            self.camera = Fisheye()
        elif camera == "normal":
            self.camera = Normal()
        else:
            raise Exception("camera should be fisheye/normal")
        self.corners = []

    @staticmethod
    def get_args():
        return args

    def set_calibration(self, camera_mat, dist_coeff):
        """K and D as cv2 calibrated them: a fisheye D of 4 coefficients, a "normal" (pinhole) D of 4, 5, 8, 12 or 14."""
        d = self.camera.data
        d.camera_mat = np.asarray(camera_mat, np.float64)
        d.dist_coeff = np.asarray(dist_coeff, np.float64)
        d.ok = True
        self.camera._get_undistort_maps()
        return d

    def undistort(self, img):
        d = self.camera.data
        if d._und is None:
            if d.camera_mat is None:
                raise Exception("no calibration: call set_calibration(K, D) first")
            self.camera._get_undistort_maps()
        return d._und(img)

    def undistort_points(self, pts):
        """Raw-frame pixels -> pixels of undistort(img)'s image: cv2.fisheye.undistortPoints(pts, K, D, P=P) (a "normal"
        camera: cv2.undistortPoints) with the P that undistort uses, bit for bit; NumPy or CUDA points."""
        d = self.camera.data
        if d.camera_mat is None:
            raise Exception("no calibration: call set_calibration(K, D) first")
        P = self.camera._get_camera_mat_dst(d.camera_mat)
        if self.camera.kind == "fisheye":
            return ops.fisheye_undistort_points(pts, d.camera_mat, d.dist_coeff, P=P)
        return ops.undistort_points(pts, d.camera_mat, d.dist_coeff, P=P)

    def calibrate(self, img):
        return self.camera.data

    def __call__(self, raw_frame):
        raise Exception("chessboard detection / calibration is outside the GPU hot path (see module docstring)")
