"""The YUV 4:2:0 canvas output on the CPU: tests/host/yuv_out.cu runs the host form of k_canvas_yuv's work item
(canvas_yuv_item, with bgr_yuv) from the library's header over whole canvases, and this file compares it with live cv2:
cv2.cvtColor(COLOR_BGR2YUV_I420) of the BGR canvas (NV12: tests/yuv_frames.i420_to_nv12 of it); with GAIN, of the
oracle's color_balance of the raw canvas followed by the saturating add of the car."""
import subprocess

import cv2
import numpy as np
import pytest

from oracle import cv2_path as C
from oracle import restate as R
from tests import yuv_frames as Y
from tests.test_host_yuv import _build


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return _build(tmp_path_factory, "yuv_out")


def _run(exe, tmp_path, fmt, canvases, gain=False, car=None, out_off=0):
    """The harness on BGR canvases [batch][BH][BW][3]; returns (YUV canvases [batch][BH*3/2][BW], word path taken)."""
    batch, BH, BW, _ = canvases.shape
    parts = [np.array([BW, BH, batch, int(car is not None), out_off], np.int32).tobytes()]
    if gain:
        parts.append(canvases.reshape(batch, -1, 3).sum(axis=1, dtype=np.uint64).tobytes())
    if car is not None:
        parts.append(np.ascontiguousarray(car).tobytes())
    parts.append(np.ascontiguousarray(canvases).tobytes())
    (tmp_path / "in.bin").write_bytes(b"".join(parts))
    r = subprocess.run([exe, "yuv_out", str(Y.FMT_CODE[fmt]), str(int(gain)), str(tmp_path / "in.bin"), str(tmp_path / "out.bin")],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (fmt, BW, BH, r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    words = int(r.stdout.split("words:")[1].split()[0])
    return np.fromfile(tmp_path / "out.bin", np.uint8).reshape(batch, BH * 3 // 2, BW), words


def _want(canvas, fmt, gain=False, car=None):
    """cvtColor(BGR2YUV_I420) of the canvas (GAIN: of color_balance(canvas), then the car added with saturation)."""
    if gain:
        with np.errstate(divide="ignore", invalid="ignore"):   # a black channel: K / 0, as the reference divides
            canvas = C.color_balance(canvas)
        if car is not None:
            canvas = R.sat_add(canvas, car)
    return Y.from_bgr(canvas, fmt)


def every_colour_image():
    """An 8192 x 8192 BGR image whose even/even pixels (the top-left pixels of the 2 x 2 chroma blocks) take each of the
    2^24 colours once, and whose other three pixels of each block take other colours: a chroma rule that averages or
    that reads another pixel of the block fails on it."""
    s = np.arange(1 << 24, dtype=np.uint32).reshape(4096, 4096)
    img = np.empty((8192, 8192, 3), np.uint8)
    for a in range(2):
        for b in range(2):
            v = s ^ np.uint32([0, 0x5A3C96, 0xC3A50F, 0x3FC0F0][2 * a + b])
            img[a::2, b::2] = np.stack([v & 255, (v >> 8) & 255, (v >> 16) & 255], -1).astype(np.uint8)
    return img


def test_bgr_yuv_every_colour_against_cv2(exe, tmp_path):
    """bgr_yuv and the top-left chroma rule through the work item over an 8192^2 canvas: Y of every colour, and U and
    V of every colour taken from its block's top-left pixel, equal cv2.cvtColor(COLOR_BGR2YUV_I420); no Y, U or V leaves
    [16, 235] / [16, 240]."""
    img = every_colour_image()
    want = cv2.cvtColor(img, cv2.COLOR_BGR2YUV_I420)
    got, words = _run(exe, tmp_path, "i420", img[None])
    assert words == 1
    assert (got[0] == want).all(), int((got[0] != want).sum())
    assert 16 <= want[:8192].min() and want[:8192].max() <= 235
    assert 16 <= want[8192:].min() and want[8192:].max() <= 240
    # the chroma depends on the top-left pixel alone: a copy with the other three pixels changed has the same U and V
    img[0::2, 1::2] ^= 0x11
    img[1::2] ^= 0x22
    assert (cv2.cvtColor(img, cv2.COLOR_BGR2YUV_I420)[8192:] == want[8192:]).all()


SIZES = [(64, 32), (30, 18), (40, 6), (98, 54), (200, 100), (1000, 10)]   # BW % 4 in {0, 2}, BW % 16 != 0, BH % 4 == 2


@pytest.mark.parametrize("BW,BH", SIZES)
def test_canvases_against_cv2(exe, tmp_path, BW, BH):
    """Whole canvases in both layouts, plain and with GAIN (colour balance), with and without the car, at output base
    offsets 0..3: the word path (BW % 4 == 0 and an aligned output) and the byte path.  The third canvas has a channel
    that is 0 everywhere: its gain is K / 0 = inf, and 0 * inf = NaN rounds as on x86 (cvRound(NaN) = INT_MIN -> 0)."""
    rng = np.random.default_rng(BW * 1000 + BH)
    canvases = rng.integers(0, 256, (3, BH, BW, 3), dtype=np.uint8)
    canvases[1] //= 3                            # darker canvases: gains far from 1
    canvases[2][..., 1] = 0                      # a black channel
    car = rng.integers(0, 256, (BH, BW, 3), dtype=np.uint8)
    car[rng.random((BH, BW)) < 0.7] = 0          # the car overlay is mostly black
    paths = set()
    for fmt in Y.FORMATS:
        for gain, c in ((False, None), (True, None), (True, car)):
            for off in range(4):
                got, words = _run(exe, tmp_path, fmt, canvases, gain, c, off)
                paths.add(words)
                for b in range(3):
                    want = _want(canvases[b], fmt, gain, c)
                    assert (got[b] == want).all(), (fmt, gain, c is not None, off, b, int((got[b] != want).sum()))
    assert paths == ({0, 1} if BW % 4 == 0 else {0})


def test_layouts_are_cv2s_round_trip(exe, tmp_path):
    """The I420 and NV12 canvases decode with cv2.cvtColor(COLOR_YUV2BGR_I420 / _NV12) to the same image."""
    rng = np.random.default_rng(3)
    canvas = rng.integers(0, 256, (1, 50, 98, 3), dtype=np.uint8)
    back = [Y.to_bgr(_run(exe, tmp_path, fmt, canvas)[0][0], fmt) for fmt in Y.FORMATS]
    assert (back[0] == back[1]).all()
