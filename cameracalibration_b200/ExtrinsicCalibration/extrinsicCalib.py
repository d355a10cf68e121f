"""Drop-in for the hot-path part of the reference's ExtrinsicCalibration/extrinsicCalib.py:
``ExCalibrator.warp()`` = cv2.warpPerspective(src_img, homography, dst size) on the GPU
(reference extrinsicCalib.py:166-169), ``ScaleImage`` with its cv2.resize on the GPU (:90-132) and
``CenterImage.translate`` = cv2.warpAffine on the GPU (:53-58).  Picking the centre with the mouse
(``CenterImage.__call__``) is interactive and raises here: set ``x`` and ``y`` directly.

Estimating the homography (chessboard corners in two views + cv2.findHomography(RANSAC),
reference :155-183) is offline, irregular work outside the hot path (SURVEY 2 row 8): set
``src_img``, ``dst_img`` (only its shape is used) and ``homography`` directly, or use
``set_views(src_img, dst_img, homography)``.
"""
from __future__ import annotations

import argparse

import numpy as np

from .. import ops

parser = argparse.ArgumentParser(description="Homography from Source to Destination Image (H100 warp path)")
parser.add_argument("-id", "--CAMERA_ID", default=1, type=int)
parser.add_argument("-bw", "--BORAD_WIDTH", default=7, type=int, help="Chess Board Width (corners number)")
parser.add_argument("-bh", "--BORAD_HEIGHT", default=6, type=int, help="Chess Board Height (corners number)")
parser.add_argument("-size", "--SCALED_SIZE", default=10, type=int, help="Scaled Chess Board Square Size (image pixel)")
args = parser.parse_known_args([])[0]


class CenterImage:
    def __init__(self):
        self.x = 0
        self.y = 0

    def translate(self, img):
        """cv2.warpAffine(img, [[1, 0, W // 2 - x], [0, 1, H // 2 - y]], (W, H)) on the GPU; img a NumPy image or a
        CUDA array [H][W][C]."""
        H, W = int(img.shape[0]), int(img.shape[1])
        M = np.float32([[1, 0, W // 2 - self.x], [0, 1, H // 2 - self.y]])
        return ops.warp_affine(img, M, (W, H))

    def __call__(self, raw_frame):
        raise Exception("picking the image centre with the mouse is interactive: set x and y, then call translate()")


class ScaleImage:
    def __init__(self, corners):
        self.calc_dist(corners)
        print("scale image from {} to {}".format(self.dist_square, args.SCALED_SIZE))
        self.scale_factor = args.SCALED_SIZE / self.dist_square

    def calc_dist(self, corners):
        import cv2   # host-side arithmetic on the corner list only
        dist_total = 0
        for i in range(args.BORAD_HEIGHT):
            dist = cv2.norm(corners[i * args.BORAD_WIDTH, :], corners[(i + 1) * args.BORAD_WIDTH - 1, :], cv2.NORM_L2)
            dist_total += dist / (args.BORAD_WIDTH - 1)
        self.dist_square = dist_total / args.BORAD_HEIGHT

    def padding(self, img, width, height):
        H, W = img.shape[0], img.shape[1]
        top = bottom = (height - H) // 2
        if top + bottom + H < height:
            bottom += 1
        left = right = (width - W) // 2
        if left + right + W < width:
            right += 1
        out = np.zeros((top + H + bottom, left + W + right) + img.shape[2:], img.dtype)   # cv2.copyMakeBorder, zeros
        out[top:top + H, left:left + W] = img
        return out

    def center_crop(self, img, width, height):
        H, W = img.shape[0], img.shape[1]
        top = (H - height) // 2
        left = (W - width) // 2
        return img[top:top + height, left:left + width]

    def __call__(self, raw_frame):
        width, height = raw_frame.shape[1], raw_frame.shape[0]
        raw_frame = ops.resize(raw_frame, (0, 0), fx=self.scale_factor, fy=self.scale_factor)
        if self.scale_factor < 1:
            return self.padding(raw_frame, width, height)
        return self.center_crop(raw_frame, width, height)


class ExCalibrator:
    def __init__(self):
        self.src_corners_total = np.empty([0, 1, 2])
        self.dst_corners_total = np.empty([0, 1, 2])
        self.src_img = None
        self.dst_img = None
        self.homography = None

    @staticmethod
    def get_args():
        return args

    def set_views(self, src_img, dst_img, homography):
        self.src_img, self.dst_img = src_img, dst_img
        self.homography = np.asarray(homography, np.float64)
        return self.homography

    def warp(self):
        if self.src_img is None or self.dst_img is None or self.homography is None:
            raise Exception("src_img, dst_img and homography must be set before warp()")
        return ops.warp_perspective(self.src_img, self.homography, (self.dst_img.shape[1], self.dst_img.shape[0]))

    def __call__(self, src_img, dst_img):
        raise Exception("corner detection / cv2.findHomography is outside the GPU hot path (see module docstring)")
