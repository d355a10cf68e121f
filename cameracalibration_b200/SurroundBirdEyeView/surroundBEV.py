"""Drop-in for the reference's SurroundBirdEyeView/surroundBEV.py on libbevk.so.

Same public surface -- ``BevGenerator(blend, balance)(front, back, left, right, car)``,
``BevGenerator.get_args()``, ``Camera``, ``Mask``, ``BlendMask``, ``padding``,
``luminance_balance``, ``color_balance`` -- with every per-pixel operation executed by
the sm_90a kernels behind the C ABI (include/bevk.h).  Host-side work kept here is
what the reference also does once at construction: loading K/D/H, building the
destination camera matrix, and rasterising the 4 mask polygons with cv2.fillPoly
(SURVEY K11, out of GPU scope).

Differences from the reference that are deliberate:
  * argparse does not consume sys.argv at import (the reference's import-time
    ``parse_args()`` kills any host program with foreign flags, surroundBEV.py:17);
    ``get_args()`` returns the same mutable namespace with the same attribute names.
  * K/D/H are read from ``args.DATA_DIR`` (default ``<this dir>/data``, the reference's
    layout ``{name}/camera_{name}_{K,D,H}.npy``) or passed as ``calib={name: (K, D, H)}``.
    ``calib={name: (K, D, H, "pinhole")}`` takes a pinhole camera instead of a fisheye, with D of
    4, 5, 8, 12 or 14 coefficients as cv2.initUndistortRectifyMap takes it.
  * ``BevGenerator.run_batch`` renders many frame-sets per call (the reference has no
    batch API); ``BevGenerator(..., interpolation=cv2.INTER_NEAREST)`` selects nearest-neighbour
    sampling with cv2.remap's exact fixed-point-map semantics (the reference always uses bilinear).
"""
from __future__ import annotations

import argparse
import os

import numpy as np

from .. import _lib as L
from .. import ops

_DEFAULTS = [  # flag, dest, default, type  (reference: surroundBEV.py:6-16)
    ("-fw", "FRAME_WIDTH", 1280, int), ("-fh", "FRAME_HEIGHT", 1024, int),
    ("-bw", "BEV_WIDTH", 1000, int), ("-bh", "BEV_HEIGHT", 1000, int),
    ("-cw", "CAR_WIDTH", 250, int), ("-ch", "CAR_HEIGHT", 400, int),
    ("-fs", "FOCAL_SCALE", 1, float), ("-ss", "SIZE_SCALE", 2, float),
    ("-blend", "BLEND_FLAG", False, bool), ("-balance", "BALANCE_FLAG", False, bool),
]
parser = argparse.ArgumentParser(description="Generate Surrounding Camera Bird Eye View (H100 engine)")
for _flag, _dest, _default, _type in _DEFAULTS:
    parser.add_argument(_flag, "--" + _dest, default=_default, type=_type)
parser.add_argument("--DATA_DIR", default=os.path.join(os.path.dirname(os.path.abspath(__file__)), "data"), type=str)
args = parser.parse_known_args([])[0]   # defaults only; main() re-parses the real command line

NAMES = ("front", "back", "left", "right")


def _cv2():
    import cv2   # host-side image plumbing only (fillPoly, copyMakeBorder, imread)
    return cv2


# ----------------------------------------------------------------------------------------
# geometry snapshot (the reference copies args into module globals in init_args, :300-310)
# ----------------------------------------------------------------------------------------
class _Geo:
    __slots__ = ("FW", "FH", "BW", "BH", "CW", "CH", "FS", "SS")

    def __init__(self, a=None):
        a = a or args
        self.FW, self.FH, self.BW, self.BH = a.FRAME_WIDTH, a.FRAME_HEIGHT, a.BEV_WIDTH, a.BEV_HEIGHT
        self.CW, self.CH, self.FS, self.SS = a.CAR_WIDTH, a.CAR_HEIGHT, a.FOCAL_SCALE, a.SIZE_SCALE

    @property
    def und_size(self):
        return int(self.FW * self.SS), int(self.FH * self.SS)

    def key(self):
        return tuple(getattr(self, s) for s in self.__slots__)


_geo = _Geo()


def padding(img, width, height):
    """Centre ``img`` on a zero canvas of width x height (extra pixel goes right / bottom)."""
    h, w = img.shape[:2]
    top, left = (height - h) // 2, (width - w) // 2
    return _cv2().copyMakeBorder(img, top, height - h - top, left, width - w - left,
                                 _cv2().BORDER_CONSTANT, value=(0, 0, 0))


def color_balance(image):
    """Grey-world channel gains (reference surroundBEV.py:43-55), on the GPU."""
    return ops.color_balance(image)


def luminance_balance(images):
    """Equalise mean V=max(B,G,R) across the frames through OpenCV's 8-bit HSV round trip
    (reference surroundBEV.py:57-79), on the GPU."""
    return ops.luminance_balance(list(images))


# ----------------------------------------------------------------------------------------
class Camera:
    """One camera: K, D, H, destination matrix, undistort maps, BEV maps.  A fisheye, or a pinhole when calib has a
    fourth element "pinhole"."""

    def __init__(self, name, calib=None, geo: _Geo | None = None):
        self.name = name
        self._g = geo or _geo
        if calib is None:
            base = os.path.join(args.DATA_DIR, name, "camera_" + name + "_")
            calib = tuple(np.load(base + s + ".npy") for s in "KDH")
        self.model = calib[3] if len(calib) > 3 else "fisheye"
        if self.model not in ("fisheye", "pinhole"):
            raise L.BevkError(f'camera {name}: model must be "fisheye" or "pinhole", got {self.model!r}')
        self.camera_mat, self.dist_coeff, self.homography = (np.asarray(m, np.float64) for m in calib[:3])
        self.camera_mat_dst = self.get_camera_mat_dst()
        self._und = None
        self._und_maps = None
        self._bev_maps = None
        self._bev1 = None

    def get_camera_mat_dst(self):
        g = self._g
        P = self.camera_mat.copy()
        P[0, 0] *= g.FS
        P[1, 1] *= g.FS
        P[0, 2] = g.FW / 2 * g.SS
        P[1, 2] = g.FH / 2 * g.SS
        return P

    # maps live on the device; the numpy views are materialised only if somebody asks
    def _undistorter(self):
        if self._und is None:
            self._und = ops.Undistorter(self.camera_mat, self.dist_coeff, self.camera_mat_dst, self._g.und_size,
                                        model=self.model)
        return self._und

    def get_undistort_maps(self):
        return self._undistorter().maps()

    @property
    def undistort_maps(self):
        if self._und_maps is None:
            self._und_maps = self.get_undistort_maps()
        return self._und_maps

    def get_bev_maps(self):
        return self._single().get_maps(0)

    @property
    def bev_maps(self):
        if self._bev_maps is None:
            self._bev_maps = self.get_bev_maps()
        return self._bev_maps

    def _single(self):
        """1-camera engine with an all-pass mask: raw2bev through the fused kernel."""
        if self._bev1 is None:
            g = self._g
            e = ops.BevEngine(1, (g.FW, g.FH), (g.BW, g.BH))
            e.set_camera(0, self.camera_mat, self.dist_coeff, self.camera_mat_dst, g.und_size, self.homography, self.model)
            e.set_mask(0, np.full((g.BH, g.BW), 255, np.uint8))
            e.finalize()
            self._bev1 = e
        return self._bev1

    def undistort(self, img):
        return self._undistorter()(img)

    def warp_homography(self, img):
        g = self._g
        if img.dtype == np.uint8:
            return ops.warp_perspective(img, self.homography, (g.BW, g.BH))
        # the reference also pushes the undistortion map planes through this method (get_bev_maps)
        if img.dtype == np.int16 and img.ndim == 3 and img.shape[2] == 2:
            return ops.warp_perspective_maps(img, np.zeros(img.shape[:2], np.uint16), self.homography, (g.BW, g.BH))[0]
        if img.dtype == np.uint16 and img.ndim == 2:
            return ops.warp_perspective_maps(np.zeros(img.shape + (2,), np.int16), img, self.homography, (g.BW, g.BH))[1]
        raise L.BevkError("warp_homography: uint8 images or CV_16SC2 / CV_16UC1 map planes only")

    def raw2bev(self, img):
        return self._single().run([[img]])[0]


# ----------------------------------------------------------------------------------------
def _plain_points(name, g: _Geo):
    BW, BH, CW, CH = g.BW, g.BH, g.CW, g.CH
    inner = {"tl": ((BW - CW) / 2, (BH - CH) / 2), "tr": ((BW + CW) / 2, (BH - CH) / 2),
             "bl": ((BW - CW) / 2, (BH + CH) / 2), "br": ((BW + CW) / 2, (BH + CH) / 2)}
    table = {"front": [(0, 0), (BW, 0), inner["tr"], inner["tl"]],
             "back": [(0, BH), (BW, BH), inner["br"], inner["bl"]],
             "left": [(0, 0), (0, BH), inner["bl"], inner["tl"]],
             "right": [(BW, 0), (BW, BH), inner["br"], inner["tr"]]}
    if name not in table:
        raise Exception("name should be front/back/left/right")
    return np.array(table[name]).astype(np.int32)


def _blend_points(name, g: _Geo):
    BW, BH, CW, CH = g.BW, g.BH, g.CW, g.CH
    tl, tr = ((BW - CW) / 2, (BH - CH) / 2), ((BW + CW) / 2, (BH - CH) / 2)
    bl, br = ((BW - CW) / 2, (BH + CH) / 2), ((BW + CW) / 2, (BH + CH) / 2)
    table = {"front": [(0, 0), (BW, 0), (BW, BH / 5), tr, tl, (0, BH / 5)],
             "back": [(0, BH), (BW, BH), (BW, BH - BH / 5), br, bl, (0, BH - BH / 5)],
             "left": [(0, 0), (0, BH), (BW / 5, BH), bl, tl, (BW / 5, 0)],
             "right": [(BW, 0), (BW, BH), (BW - BW / 5, BH), br, tr, (BW - BW / 5, 0)]}
    if name not in table:
        raise Exception("name should be front/back/left/right")
    return np.array(table[name]).astype(np.int32)


def _seam_lines(g: _Geo):
    """FL, FR, BL, BR, LF, LB, RF, RB as int32[8][2][2] (BlendMask.get_lines)."""
    BW, BH, CW, CH = g.BW, g.BH, g.CW, g.CH
    tl, tr = ((BW - CW) / 2, (BH - CH) / 2), ((BW + CW) / 2, (BH - CH) / 2)
    bl, br = ((BW - CW) / 2, (BH + CH) / 2), ((BW + CW) / 2, (BH + CH) / 2)
    segs = [[(0, BH / 5), tl], [(BW, BH / 5), tr], [(0, BH - BH / 5), bl], [(BW, BH - BH / 5), br],
            [(BW / 5, 0), tl], [(BW / 5, BH), bl], [(BW - BW / 5, 0), tr], [(BW - BW / 5, BH), br]]
    return np.array(segs).astype(np.int32)


def _fill(points, g: _Geo):
    return _cv2().fillPoly(np.zeros((g.BH, g.BW), np.uint8), [points], 255)


class Mask:
    """Binary 4-gon mask of one camera's canvas sector."""

    def __init__(self, name, geo: _Geo | None = None):
        self._g = geo or _geo
        self.mask = self.get_mask(name)

    def get_points(self, name):
        return _plain_points(name, self._g)

    def get_mask(self, name):
        return _fill(self.get_points(name), self._g)

    def __call__(self, img):
        return ops.apply_mask(img, self.mask, blend=False)


_blend_cache: dict = {}


class BlendMask:
    """6-gon mask with distance-ratio weights in the overlap wedges (computed on the GPU)."""

    def __init__(self, name, geo: _Geo | None = None):
        self._g = g = geo or _geo
        if name not in NAMES:
            raise Exception("name should be front/back/left/right")
        self.get_lines()
        key = g.key()
        if key not in _blend_cache:
            polys = np.stack([self.get_mask(n) for n in NAMES])
            eng = ops.BevEngine(1, (g.FW, g.FH), (g.BW, g.BH))
            _blend_cache.clear()
            _blend_cache[key] = eng.blend_masks(polys, _seam_lines(g))
        self.mask = _blend_cache[key][NAMES.index(name)].copy()
        self._weight = None

    @property
    def weight(self):
        if self._weight is None:
            self._weight = (np.repeat(self.mask[:, :, np.newaxis], 3, axis=2) / 255.0).astype(np.float32)
        return self._weight

    def get_points(self, name):
        return _blend_points(name, self._g)

    def get_mask(self, name):
        return _fill(self.get_points(name), self._g)

    def get_lines(self):
        ln = _seam_lines(self._g)
        (self.lineFL, self.lineFR, self.lineBL, self.lineBR,
         self.lineLF, self.lineLB, self.lineRF, self.lineRB) = (ln[i] for i in range(8))

    def __call__(self, img):
        return ops.apply_mask(img, self.mask, blend=True)


# ----------------------------------------------------------------------------------------
class BevGenerator:
    def __init__(self, blend=None, balance=None, calib=None, interpolation=None):
        self.init_args()
        g = self._g = _Geo()
        self.blend = args.BLEND_FLAG if blend is None else blend
        self.balance = args.BALANCE_FLAG if balance is None else balance
        self.cameras = [Camera(n, None if calib is None else calib[n], g) for n in NAMES]
        self.masks = [(BlendMask if self.blend else Mask)(n, g) for n in NAMES]
        self.engine = ops.BevEngine(len(NAMES), (g.FW, g.FH), (g.BW, g.BH))
        if interpolation is not None:   # extension: cv2.INTER_NEAREST (0) / cv2.INTER_LINEAR (1, the reference)
            self.engine.set_interpolation(interpolation)
        for i, (cam, mk) in enumerate(zip(self.cameras, self.masks)):
            self.engine.set_camera(i, cam.camera_mat, cam.dist_coeff, cam.camera_mat_dst, g.und_size, cam.homography,
                                   cam.model)
            self.engine.set_mask(i, mk.mask)
        self.engine.finalize()

    @staticmethod
    def get_args():
        return args

    def init_args(self):
        global _geo, FRAME_WIDTH, FRAME_HEIGHT, BEV_WIDTH, BEV_HEIGHT, CAR_WIDTH, CAR_HEIGHT, FOCAL_SCALE, SIZE_SCALE
        _geo = _Geo()
        FRAME_WIDTH, FRAME_HEIGHT, BEV_WIDTH, BEV_HEIGHT = _geo.FW, _geo.FH, _geo.BW, _geo.BH
        CAR_WIDTH, CAR_HEIGHT, FOCAL_SCALE, SIZE_SCALE = _geo.CW, _geo.CH, _geo.FS, _geo.SS

    def __call__(self, front, back, left, right, car=None):
        return self.engine.run([[front, back, left, right]], car, self.balance)[0]

    def points_to_bev(self, name, pts):
        """Pixels of camera `name`'s raw frame -> BEV canvas pixels (BevEngine.camera_to_canvas)."""
        return self.engine.camera_to_canvas(NAMES.index(name), pts)

    def points_from_bev(self, name, pts):
        """BEV canvas pixels -> pixels of camera `name`'s raw frame (BevEngine.canvas_to_camera)."""
        return self.engine.canvas_to_camera(NAMES.index(name), pts)

    def run_batch(self, frame_sets, car=None, out=None, pixel_format="bgr", out_format="bgr"):
        """frame_sets: iterable of (front, back, left, right) tuples -> uint8[n][BH][BW][3].  pixel_format "nv12" /
        "i420": the frames are YUV 4:2:0 buffers uint8[FH*3//2][FW] (cv2's layout), converted to BGR on the GPU exactly
        as cv2.cvtColor does.  pixel_format "yuyv" / "uyvy": packed YUV 4:2:2 camera frames uint8[FH][FW][2], as
        cv2.cvtColor(frame, COLOR_YUV2BGR_YUY2 / _UYVY) makes them BGR.  out_format "nv12" / "i420": the canvases come
        back as uint8[n][BH*3//2][BW], each
        cv2.cvtColor(canvas, COLOR_BGR2YUV_I420) (NV12: U and V interleaved), converted on the GPU."""
        return self.engine.run([list(fs) for fs in frame_sets], car, self.balance, out, pixel_format=pixel_format,
                               out_format=out_format)

    def run_cuda(self, frames, car=None, out=None, stream=None, pixel_format="bgr", out_format="bgr"):
        """Frame-sets that are already on the GPU (uint8 CUDA array [n][4][FH][FW][3] in front/back/left/right
        order, or nested lists of per-frame CUDA arrays) -> CUDA array [n][BH][BW][3]; nothing crosses PCIe.
        pixel_format "nv12" / "i420": one uint8 CUDA array [n][4][FH*3//2][FW] of YUV 4:2:0 frames; "yuyv" / "uyvy":
        one uint8 CUDA array [n][4][FH][FW][2] of packed 4:2:2 frames.  out_format
        "nv12" / "i420": the result is uint8[n][BH*3//2][BW] YUV 4:2:0 canvases (see run_batch)."""
        return self.engine.run_cuda(frames, car, self.balance, out, stream, pixel_format=pixel_format, out_format=out_format)

    def run_cuda_planes(self, y, c=None, v=None, pixel_format="nv12", car=None, out=None, stream=None, out_format="bgr"):
        """run_cuda on YUV 4:2:0 frame-sets given plane by plane, as a video decoder leaves them on the GPU (pitched
        rows, each plane at its own address): y uint8 CUDA array [n][4][FH][FW], c [n][4][FH/2][FW] interleaved U,V
        ("nv12") or [n][4][FH/2][FW/2] U ("i420"), v the V plane ("i420"); or nested lists of per-frame plane tuples.
        "yuyv" / "uyvy": y alone, the packed frames [n][4][FH][FW][2] with padded rows.  See BevEngine.run_cuda_planes."""
        return self.engine.run_cuda_planes(y, c, v, pixel_format, car, self.balance, out, stream, out_format=out_format)

    def jpeg(self, front, back, left, right, car=None, quality=95, params=None):
        """cv2.imencode('.jpg', self(front, back, left, right, car), [IMWRITE_JPEG_QUALITY, quality] + params) -- the
        bytes main()'s cv2.imwrite('./surround.jpg', surround) writes (reference surroundBEV.py:340) -- encoded on the
        GPU: only the JPEG stream crosses PCIe.  params: cv2.imwrite's other JPEG pairs (see ops.jpeg_encode)."""
        return self.engine.run_to_jpeg([[front, back, left, right]], quality, car, self.balance, params)[0]

    def jpeg_batch(self, frame_sets, car=None, quality=95, params=None):
        """frame_sets: iterable of (front, back, left, right) host tuples -> one JPEG ``bytes`` per frame-set."""
        return self.engine.run_to_jpeg([list(fs) for fs in frame_sets], quality, car, self.balance, params)

    def jpeg_cuda(self, frames, car=None, quality=95, params=None):
        """Frame-sets already on the GPU (as run_cuda takes them) -> one JPEG ``bytes`` per frame-set."""
        return self.engine.cuda_to_jpeg(frames, quality, car, self.balance, params)


FRAME_WIDTH, FRAME_HEIGHT, BEV_WIDTH, BEV_HEIGHT = _geo.FW, _geo.FH, _geo.BW, _geo.BH
CAR_WIDTH, CAR_HEIGHT, FOCAL_SCALE, SIZE_SCALE = _geo.CW, _geo.CH, _geo.FS, _geo.SS


def main(argv=None):
    global args
    cv2 = _cv2()
    parser.parse_args(argv, namespace=args)
    d = args.DATA_DIR
    frames = [cv2.imread(os.path.join(d, n, n + ".jpg")) for n in NAMES]
    car = padding(cv2.imread(os.path.join(d, "car.jpg")), args.BEV_WIDTH, args.BEV_HEIGHT)
    surround = BevGenerator()(*frames, car)
    cv2.imwrite("./surround.jpg", surround)
    return surround


if __name__ == "__main__":
    main()
