"""cv2.resize and cv2.warpAffine on the H100, byte for byte against live cv2, through all four entry points: the host
calls (bevk_resize / bevk_warp_affine) and the device-batch calls (bevk_resize_stack / bevk_warp_affine_stack) over the
corpus of tests/resize_affine_cases.py, padded rows and images, batches across GATHER_NB, the word and byte paths of the
warpAffine gather, a CUDA-graph capture and replay, the shim's ScaleImage and CenterImage.translate, and the refusals."""
import ctypes as C

import cv2
import numpy as np
import pytest

from tests import resize_affine_cases as R

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def ctx():
    from cameracalibration_b200 import _lib as L
    return L.default_context()


def _call(case, src, ctx, out=None):
    from cameracalibration_b200 import ops
    if case["op"] == "resize":
        return ops.resize(src, case["dsize"], fx=case["fx"], fy=case["fy"], interpolation=case["interp"], ctx=ctx, out=out)
    return ops.warp_affine(src, case["M"], case["dsize"], flags=case["flags"], ctx=ctx, out=out)


def _corpus():
    return R.resize_corpus(np.random.default_rng(7)) + R.affine_corpus(np.random.default_rng(11))


def test_host_entry_points(ctx):
    for c in _corpus():
        f = R.source(c)[0]
        got = _call(c, f[..., 0] if c["ch"] == 1 else f, ctx)
        w = R.want(c, f)
        assert (got.reshape(w.shape) == w).all(), ({k: v for k, v in c.items() if k != "M"}, int((got.reshape(w.shape) != w).sum()))


def _padded(frames, row_pad, img_pad, dev):
    """frames [n][h][w][c] copied into a device pool with padded rows and images; returns the strided view."""
    n, h, w, ch = frames.shape
    row, img = w * ch + row_pad, h * (w * ch + row_pad) + img_pad
    pool = torch.randint(0, 256, (n * img,), dtype=torch.uint8, device=dev)
    view = pool.as_strided((n, h, w, ch), (img, row, ch, 1))
    view.copy_(torch.from_numpy(frames).to(dev))
    return view


def test_device_batches_padded(ctx):
    """The corpus as device batches (n = 1, 3, 9 and 17: across GATHER_NB), with padded source and output rows and images."""
    from cameracalibration_b200 import ops
    dev = torch.device("cuda", ctx.device)
    for i, c in enumerate(_corpus()[::3]):
        c = dict(c, n=(1, 3, 9, 17)[i % 4])
        frames = R.source(c)
        src = _padded(frames, i % 5, (i * 3) % 7, dev)
        dw, dh = ops.resize_size((c["sw"], c["sh"]), c["dsize"], c["fx"], c["fy"]) if c["op"] == "resize" else c["dsize"]
        out = _padded(np.zeros((c["n"], dh, dw, c["ch"]), np.uint8), (i * 7) % 5, i % 3, dev)
        _call(c, src, ctx, out=out)
        torch.cuda.synchronize()
        got = out.cpu().numpy()
        for f in range(c["n"]):
            w = R.want(c, frames[f])
            assert (got[f] == w).all(), ({k: v for k, v in c.items() if k != "M"}, f, int((got[f] != w).sum()))


def test_word_and_byte_paths(ctx):
    """An aligned 3-channel batch takes the word path (k_gather4), the same frames at an odd base address the byte path
    (k_gather); resize reports k_resize."""
    from cameracalibration_b200 import ops
    dev = torch.device("cuda", ctx.device)
    c = R._affine(3, 640, 480, [[0.9, 0.1, 12.5], [-0.05, 1.1, -7.25]], (640, 480), cv2.INTER_LINEAR, n=5, seed=3)
    frames = R.source(c)
    want = [R.want(c, f) for f in frames]
    aligned = torch.from_numpy(frames).to(dev)
    got = ops.warp_affine(aligned, c["M"], c["dsize"], ctx=ctx)
    assert ops.last_path(ctx) == "word"
    assert all((g == w).all() for g, w in zip(got.cpu().numpy(), want))
    pool = torch.zeros(frames.size + 1, dtype=torch.uint8, device=dev)
    odd = pool[1:].view(frames.shape)
    odd.copy_(aligned)
    got = ops.warp_affine(odd, c["M"], c["dsize"], ctx=ctx)
    assert ops.last_path(ctx) == "byte"
    assert all((g == w).all() for g, w in zip(got.cpu().numpy(), want))
    ops.resize(odd, (320, 240), ctx=ctx)
    assert ops.last_path(ctx) == "resize"


def test_graph_capture_and_replay(ctx):
    """Both stack calls captured into one CUDA graph on the ctx stream and replayed on new frames written into the captured
    buffers."""
    from cameracalibration_b200 import _lib as L
    dev = torch.device("cuda", ctx.device)
    cr = R._resize(3, 320, 256, (160, 128), interp=cv2.INTER_AREA, n=9, seed=21)
    ca = R._affine(3, 320, 256, [[1, 0, 17], [0, 1, -9]], (320, 256), cv2.INTER_CUBIC, n=9, seed=22)
    src = torch.from_numpy(R.source(cr)).to(dev)
    o1 = torch.empty((9, 128, 160, 3), dtype=torch.uint8, device=dev)
    o2 = torch.empty((9, 256, 320, 3), dtype=torch.uint8, device=dev)
    sp, M = C.c_void_p(src.data_ptr()), L.dptr(ca["M"])

    def calls():
        assert ctx.lib.bevk_resize_stack(ctx.h, sp, 320 * 256 * 3, 320, 256, 320 * 3, 3, 9, C.c_void_p(o1.data_ptr()),
                                         160 * 128 * 3, 160, 128, 160 * 3, 0.0, 0.0, cv2.INTER_AREA) == 0
        assert ctx.lib.bevk_warp_affine_stack(ctx.h, sp, 320 * 256 * 3, 320, 256, 320 * 3, 3, 9, M, C.c_void_p(o2.data_ptr()),
                                              320 * 256 * 3, 320, 256, 320 * 3, cv2.INTER_CUBIC) == 0
    ctx.set_stream(None)
    torch.cuda.synchronize()
    calls()
    ctx.sync()
    with ctx.graph_capture() as g:
        calls()
    new = R.source(dict(cr, seed=23))
    src.copy_(torch.from_numpy(new).to(dev))
    o1.zero_()
    o2.zero_()
    torch.cuda.synchronize()
    g.launch(2)
    ctx.sync()
    g.destroy()
    for f in range(9):
        assert (o1[f].cpu().numpy() == R.want(cr, new[f])).all()
        assert (o2[f].cpu().numpy() == R.want(ca, new[f])).all()


def test_reference_scale_and_translate(ctx, fx):
    """The shim's ScaleImage and CenterImage.translate against the reference's code run with cv2 (restated here: its
    module parses sys.argv at import)."""
    from cameracalibration_b200.ExtrinsicCalibration import CenterImage, ScaleImage
    from tests.helpers import NAMES
    frame = fx.frames(1280, 1024)[0]
    for i, name in enumerate(NAMES[:2]):
        s = ScaleImage(R.board_corners(fx.calib[name][2], origin=(400.0 + 150 * i, 150.0)))
        f = s.scale_factor
        want = cv2.resize(frame, (0, 0), fx=f, fy=f)
        W, H = frame.shape[1], frame.shape[0]
        if f < 1:
            t, l = (H - want.shape[0]) // 2, (W - want.shape[1]) // 2
            want = cv2.copyMakeBorder(want, t, H - want.shape[0] - t, l, W - want.shape[1] - l, cv2.BORDER_CONSTANT,
                                      value=(0, 0, 0))
        else:
            t, l = (want.shape[0] - H) // 2, (want.shape[1] - W) // 2
            want = want[t:t + H, l:l + W]
        assert (s(frame) == want).all(), (name, f)
    c = CenterImage()
    for x, y in [(600, 500), (700, 530), (3, 1020)]:
        c.x, c.y = x, y
        M = np.float32([[1, 0, frame.shape[1] // 2 - x], [0, 1, frame.shape[0] // 2 - y]])
        assert (c.translate(frame) == cv2.warpAffine(frame, M, frame.shape[1::-1])).all()
    with pytest.raises(Exception, match="interactive"):
        c(frame)


def test_refusals_write_nothing(ctx):
    """Refused flags return BEVK_ERR_UNSUPPORTED (-4) and leave the destination as it was; an overlapping destination and
    an image stride smaller than an image are BEVK_ERR_ARG (-1)."""
    from cameracalibration_b200 import _lib as L
    dev = torch.device("cuda", ctx.device)
    src = torch.from_numpy(R.source(R._resize(3, 64, 48, n=2, seed=31))).to(dev)
    out = torch.full((2, 24, 32, 3), 77, dtype=torch.uint8, device=dev)
    sp, op = C.c_void_p(src.data_ptr()), C.c_void_p(out.data_ptr())
    M = L.dptr(np.array([[1, 0, 2], [0, 1, 3]], np.float64))
    for interp in (cv2.INTER_CUBIC, cv2.INTER_LANCZOS4, cv2.INTER_LINEAR_EXACT, cv2.INTER_NEAREST_EXACT):
        assert ctx.lib.bevk_resize_stack(ctx.h, sp, 64 * 48 * 3, 64, 48, 64 * 3, 3, 2, op, 32 * 24 * 3, 32, 24, 32 * 3, 0.0, 0.0,
                                         interp) == -4
    for flags in (cv2.INTER_LINEAR_EXACT, cv2.INTER_NEAREST_EXACT, 7, cv2.INTER_LINEAR | 32):
        assert ctx.lib.bevk_warp_affine_stack(ctx.h, sp, 64 * 48 * 3, 64, 48, 64 * 3, 3, 2, M, op, 32 * 24 * 3, 32, 24, 32 * 3,
                                              flags) == -4
    # the fx form with a size that is not cv2's for it, strides smaller than an image, an overlapping destination
    assert ctx.lib.bevk_resize_stack(ctx.h, sp, 64 * 48 * 3, 64, 48, 64 * 3, 3, 2, op, 32 * 24 * 3, 32, 24, 32 * 3, 0.4, 0.5,
                                     cv2.INTER_LINEAR) == -1
    assert ctx.lib.bevk_resize_stack(ctx.h, sp, 64 * 48 * 3 - 1, 64, 48, 64 * 3, 3, 2, op, 32 * 24 * 3, 32, 24, 32 * 3, 0.0, 0.0,
                                     cv2.INTER_LINEAR) == -1
    assert ctx.lib.bevk_warp_affine_stack(ctx.h, sp, 64 * 48 * 3, 64, 48, 64 * 3, 3, 2, M, op, 32 * 24 * 3 - 5, 32, 24, 32 * 3,
                                          cv2.INTER_LINEAR) == -1
    inside = C.c_void_p(src.data_ptr() + 100)
    assert ctx.lib.bevk_resize_stack(ctx.h, sp, 64 * 48 * 3, 64, 48, 64 * 3, 3, 2, inside, 32 * 24 * 3, 32, 24, 32 * 3, 0.0, 0.0,
                                     cv2.INTER_LINEAR) == -1
    assert ctx.lib.bevk_warp_affine_stack(ctx.h, sp, 64 * 48 * 3, 64, 48, 64 * 3, 3, 2, M, inside, 32 * 24 * 3, 32, 24, 32 * 3,
                                          cv2.INTER_LINEAR) == -1
    torch.cuda.synchronize()
    assert (out == 77).all()
