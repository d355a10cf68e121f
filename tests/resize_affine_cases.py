"""Seeded corpus of cv2.resize and cv2.warpAffine cases, shared by the CPU harness test (test_host_resize_affine.py) and
the GPU test (test_gpu_resize_affine.py).  Each case is a dict: op "resize" (dsize, fx, fy, interp) or "affine" (M, dsize,
flags), with channels, source size and a frame count; `source(case)` makes its frames and `want(case, frame)` runs cv2."""
import cv2
import numpy as np

INTERS = (cv2.INTER_NEAREST, cv2.INTER_LINEAR, cv2.INTER_AREA)
WARP_FLAGS = (cv2.INTER_NEAREST, cv2.INTER_LINEAR, cv2.INTER_CUBIC, cv2.INTER_AREA, cv2.INTER_LANCZOS4)


def _resize(ch, sw, sh, dsize=(0, 0), fx=0.0, fy=0.0, interp=cv2.INTER_LINEAR, n=1, seed=0):
    return dict(op="resize", ch=ch, sw=sw, sh=sh, dsize=tuple(int(v) for v in dsize), fx=float(fx), fy=float(fy),
                interp=interp, n=n, seed=seed)


def _affine(ch, sw, sh, M, dsize, flags=cv2.INTER_LINEAR, n=1, seed=0):
    return dict(op="affine", ch=ch, sw=sw, sh=sh, M=np.asarray(M, np.float64).reshape(2, 3), dsize=tuple(int(v) for v in dsize),
                flags=int(flags), n=n, seed=seed)


def resize_corpus(rng):
    cases = []
    # sides 1..300: dsize and fx / fy forms, up, down and mixed, every flag and channel count
    for i in range(150):
        ch = (1, 3, 4)[i % 3]
        interp = INTERS[i % 3]
        sw, sh = int(rng.integers(1, 301)), int(rng.integers(1, 301))
        if i % 2:
            dw, dh = int(rng.integers(1, 301)), int(rng.integers(1, 301))
            cases.append(_resize(ch, sw, sh, (dw, dh), interp=interp, seed=i))
        else:
            fx, fy = float(rng.uniform(0.05, 3.5)), float(rng.uniform(0.05, 3.5))
            if round(sw * fx) < 1 or round(sh * fy) < 1:
                fx, fy = 1.5, 0.7
            cases.append(_resize(ch, sw, sh, fx=fx, fy=fy, interp=interp, seed=i))
    # integer factors 2, 3 and 4 (AREA's whole-cell body, LINEAR's 2x redirect), with and without a partial edge cell
    for k, (f, sw, sh) in enumerate([(2, 64, 48), (2, 67, 45), (3, 90, 63), (3, 91, 65), (4, 128, 96), (4, 130, 99)]):
        for interp in INTERS:
            cases.append(_resize((1, 3, 4)[k % 3], sw, sh, fx=1 / f, fy=1 / f, interp=interp, seed=100 + k))
            cases.append(_resize((3, 4, 1)[k % 3], sw, sh, (sw // f, sh // f), interp=interp, seed=200 + k))
    # fractional AREA downscales and upscales whose first and last rows use the unclamped row weights
    for k, (sw, sh, dw, dh) in enumerate([(100, 80, 37, 29), (255, 3, 99, 2), (17, 300, 5, 111), (40, 30, 97, 71),
                                           (3, 2, 300, 7), (1, 1, 5, 9), (200, 150, 333, 40)]):
        for interp in INTERS:
            cases.append(_resize((1, 3, 4)[k % 3], sw, sh, (dw, dh), interp=interp, seed=300 + k))
    # the two forms give different pixels for the same output size
    cases.append(_resize(3, 1280, 1024, fx=0.37, fy=0.37, seed=400))
    cases.append(_resize(3, 1280, 1024, (474, 379), seed=401))
    # frame sizes of the pipeline
    for k, (sw, sh, dsize, fx, interp) in enumerate([(1280, 1024, (640, 480), 0, cv2.INTER_LINEAR),
                                                     (1280, 1024, (640, 512), 0, cv2.INTER_AREA),
                                                     (1280, 1024, (427, 341), 0, cv2.INTER_AREA),
                                                     (1920, 1080, (0, 0), 0.5, cv2.INTER_LINEAR),
                                                     (1920, 1080, (0, 0), 0.6, cv2.INTER_AREA),
                                                     (1920, 1080, (2880, 1620), 0, cv2.INTER_LINEAR)]):
        cases.append(_resize(3, sw, sh, dsize, fx=fx, fy=fx, interp=interp, seed=500 + k))
    return cases


def affine_corpus(rng):
    cases = []
    for i in range(40):
        ch = (1, 3, 4)[i % 3]
        flags = WARP_FLAGS[i % 5] | (cv2.WARP_INVERSE_MAP if i % 4 == 3 else 0)
        sw, sh = int(rng.integers(1, 200)), int(rng.integers(1, 200))
        dw, dh = int(rng.integers(1, 200)), int(rng.integers(1, 200))
        a = rng.uniform(-0.5, 0.5, 4) + [1, 0, 0, 1] if i % 2 else rng.uniform(-2, 2, 4)
        t = rng.uniform(-60, 60, 2)
        cases.append(_affine(ch, sw, sh, [[a[0], a[1], t[0]], [a[2], a[3], t[1]]], (dw, dh), flags, seed=i))
    # singular matrices: the inverse is the zero matrix
    for k, M in enumerate([[[1, 2, 3], [2, 4, 5]], [[0, 0, 7], [0, 0, 9]], [[0.5, 0, 0], [0, 0, 0]]]):
        for flags in (cv2.INTER_LINEAR, cv2.INTER_NEAREST, cv2.INTER_CUBIC):
            cases.append(_affine(3, 50, 40, M, (30, 20), flags, seed=60 + k))
    # fixed-point coordinates outside int16, and beyond int32 (cv2's saturate_cast gives INT_MIN)
    for k, M in enumerate([[[1, 0, 40000], [0, 1, -40000]], [[300, 0, 0], [0, -250, 0]], [[1, 0, 3e6], [0, 1, 0]],
                           [[1e7, 0, 0], [0, 1, 0]], [[1, 0.1, -33000], [0.2, 1, 32800]]]):
        for flags in WARP_FLAGS:
            cases.append(_affine((1, 3, 4)[k % 3], 90, 70, M, (80, 60), flags | cv2.WARP_INVERSE_MAP * (k % 2), seed=70 + k))
    # CenterImage.translate's matrix (float32, as the reference builds it) at a camera frame's size
    for k, (x, y) in enumerate([(600, 500), (700, 530), (1, 1023)]):
        M = np.float32([[1, 0, 640 - x], [0, 1, 512 - y]])
        cases.append(_affine(3, 1280, 1024, M, (1280, 1024), cv2.INTER_LINEAR, seed=80 + k))
    return cases


def board_corners(H, bw=7, bh=6, square=10.0, origin=(400.0, 150.0)):
    """Chessboard corners as cv2.findChessboardCorners lists them (float32 [bw * bh][1][2], row by row) for a board lying
    flat in front of a camera: a square grid in the bird's-eye canvas, mapped into the camera image through inv(H) of a
    fixture calibration."""
    g = np.array([[origin[0] + i * square, origin[1] + j * square] for j in range(bh) for i in range(bw)], np.float64)
    return cv2.perspectiveTransform(g[:, None, :], np.linalg.inv(H)).astype(np.float32)


def source(case):
    """uint8[n][sh][sw][ch] frames of the case."""
    r = np.random.default_rng(1000 + case["seed"])
    n, sh, sw, ch = case["n"], case["sh"], case["sw"], case["ch"]
    img = r.integers(0, 256, (n, sh, sw, ch), dtype=np.uint8)
    if sh > 8 and sw > 8:   # smooth regions as well as noise: rounding ties of the weights show up on both
        yy, xx = np.mgrid[0:sh, 0:sw]
        img[:, : sh // 2] = ((xx[: sh // 2, :, None] * 7 + yy[: sh // 2, :, None] * 3 + np.arange(ch)) % 256).astype(np.uint8)
    return img


def want(case, frame):
    """cv2's output for one uint8[sh][sw][ch] frame of the case, as uint8[dh][dw][ch]."""
    f = frame[..., 0] if case["ch"] == 1 else frame
    if case["op"] == "resize":
        out = cv2.resize(f, case["dsize"], fx=case["fx"], fy=case["fy"], interpolation=case["interp"])
    else:
        out = cv2.warpAffine(f, case["M"], case["dsize"], flags=case["flags"])
    return out.reshape(out.shape[0], out.shape[1], case["ch"])
