"""BEV canvases from NV12 and I420 frames on the GPU.  Inputs are fixture frames converted with
cv2.cvtColor(COLOR_BGR2YUV_I420) (NV12: the same planes interleaved); every canvas must equal, byte for byte,
cv2.cvtColor(frame, COLOR_YUV2BGR_NV12 / _I420) followed by the cv2 call sequence of the reference, and the engine's own
BGR render of the cvtColor output.  Both formats in every case."""
import ctypes

import cv2
import numpy as np
import pytest

from oracle import cv2_path as C
from oracle import restate as R
from tests import yuv_frames as Y
from tests.helpers import NAMES
from tests.test_gpu_graph_frames import _replay_after_other_stack
from tests.test_gpu_tma import _engine

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from cameracalibration_b200 import ops as o
    return o


def _oracle(calib, g, masks, blend, balance, bgr, car=None, nearest=False):
    """The reference's call sequence on BGR frames (RefBev; with nearest its cv2.remap is INTER_NEAREST)."""
    if not nearest:
        ref = C.RefBev(calib, g, blend, balance, masks=masks)
        return ref(*bgr, car)
    assert not balance
    out = np.zeros((g.BH, g.BW, 3), np.uint8)
    for n, f, mk in zip(NAMES, bgr, masks):
        m1, m2 = C.RefCamera(*calib[n], g).bev_maps
        w = cv2.remap(f, m1, m2, cv2.INTER_NEAREST, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
        out = R.sat_add(out, R.apply_blend(w, mk) if blend else R.apply_plain(w, mk))
    return out if car is None else R.sat_add(out, car)


def _sets(fx, g, n, fmt):
    """n frame-sets: (YUV frames, their cvtColor BGR) -- fixture frames, then fixture frames blended with noise."""
    bgr_in = [fx.frames(g.FW, g.FH)] + [fx.perturbed_frames(g.FW, g.FH, i) for i in range(1, n)]
    yuv = [[Y.from_bgr(f, fmt) for f in s] for s in bgr_in]
    return yuv, [[Y.to_bgr(f, fmt) for f in s] for s in yuv]


@pytest.mark.parametrize("blend", [False, True])
def test_fixture_geometry_host_frames(ops, fx, blend):
    """1280x1024 -> 1000^2 with the reference's calibration: plain and blend, BALANCE on and off, with and without the
    car, pageable host frames; a 2-set batch."""
    g = fx.geometry()
    e, masks = _engine(ops, fx, g, blend, calib=fx.calib)
    car = fx.car()
    for fmt in Y.FORMATS:
        yuv, bgr = _sets(fx, g, 2, fmt)
        for balance in (False, True):
            for c in (None, car):
                got = e.run(yuv, c, balance, pixel_format=fmt)
                assert e.last_path() == "tma"
                assert (got == e.run(bgr, c, balance)).all(), (fmt, balance, c is not None)
                for b in range(2):
                    want = _oracle(fx.calib, g, masks, blend, balance, bgr[b], c)
                    assert (got[b] == want).all(), (fmt, balance, c is not None, b, int((got[b] != want).sum()))


def test_nearest(ops, fx):
    from cameracalibration_b200 import _lib as L
    g = fx.geometry()
    masks = [R.blend_mask(n, g.BW, g.BH, g.CW, g.CH) for n in NAMES]
    e = ops.BevEngine(4, (g.FW, g.FH), (g.BW, g.BH))
    for i, n in enumerate(NAMES):
        K, D, H = fx.calib[n]
        e.set_camera(i, K, D, C.dst_camera_matrix(K, g.FW, g.FH, g.FS, g.SS), (int(g.FW * g.SS), int(g.FH * g.SS)), H)
        e.set_mask(i, masks[i])
    e.set_interpolation(L.INTER_NEAREST)
    e.finalize()
    car = fx.car()
    for fmt in Y.FORMATS:
        yuv, bgr = _sets(fx, g, 1, fmt)
        got = e.run(yuv, car, pixel_format=fmt)[0]
        assert (got == e.run(bgr, car)[0]).all(), fmt
        assert (got == _oracle(fx.calib, g, masks, True, False, bgr[0], car, nearest=True)).all(), fmt


def test_cfg3_blend_balance_car_host_and_device(ops, fx):
    """cfg3 (1920x1080 -> 1200^2, blend + BALANCE + car): pageable and page-locked host frames and a device stack."""
    import torch
    from cameracalibration_b200 import _lib as L
    g = fx.geometry(1920, 1080, 1200, 1200)
    e, masks = _engine(ops, fx, g, True)
    calib = fx.scaled_calib(g)
    car = fx.car(1200, 1200)
    dev = torch.device("cuda", e.ctx.device)
    for fmt in Y.FORMATS:
        yuv, bgr = _sets(fx, g, 2, fmt)
        want = [_oracle(calib, g, masks, True, True, s, car) for s in bgr]
        got = e.run(yuv, car, True, pixel_format=fmt)
        pinned = []
        for s in yuv:
            pinned.append([])
            for f in s:
                p = L.pinned_empty(f.shape)
                p[:] = f
                pinned[-1].append(p)
        got_p = e.run(pinned, car, True, pixel_format=fmt)
        d = torch.from_numpy(np.stack([np.stack(s) for s in yuv])).to(dev)
        got_d = e.run_cuda(d, torch.from_numpy(car).to(dev), True, pixel_format=fmt)
        torch.cuda.synchronize()
        got_d = got_d.cpu().numpy()
        for b in range(2):
            for name, x in (("pageable", got[b]), ("pinned", got_p[b]), ("device", got_d[b])):
                assert (x == want[b]).all(), (fmt, name, b, int((x != want[b]).sum()))


def test_cfg4_batch_of_32_device(ops, fx):
    """cfg4 (1920x1080 -> 1000^2, blend), a batch of 32 frame-sets as one device array [32][4][1620][1920]."""
    import torch
    g = fx.geometry(1920, 1080, 1000, 1000)
    e, masks = _engine(ops, fx, g, True)
    calib = fx.scaled_calib(g)
    dev = torch.device("cuda", e.ctx.device)
    for fmt in Y.FORMATS:
        yuv, bgr = _sets(fx, g, 32, fmt)
        d = torch.from_numpy(np.stack([np.stack(s) for s in yuv])).to(dev)
        got = e.run_cuda(d, pixel_format=fmt)
        assert e.last_path() == "tma"
        ref = e.run_cuda(torch.from_numpy(np.stack([np.stack(s) for s in bgr])).to(dev))
        torch.cuda.synchronize()
        got, ref = got.cpu().numpy(), ref.cpu().numpy()
        assert (got == ref).all(), (fmt, int((got != ref).sum()))
        for b in (0, 13, 31):
            want = _oracle(calib, g, masks, True, False, bgr[b])
            assert (got[b] == want).all(), (fmt, b)


def test_page_locked_ingest_moves_the_yuv_windows(ops, fx):
    """Page-locked host frames are fetched by the SMs (zero-copy windows), pageable ones by DMA rectangles: same
    canvases; the NV12 bytes are about half the BGR ones, and the pageable count is what host_copy_bytes reports."""
    from cameracalibration_b200 import _lib as L
    g = fx.geometry()
    e, masks = _engine(ops, fx, g, True, calib=fx.calib)
    bgr_in = fx.frames()
    pin_bgr = []
    for f in bgr_in:
        p = L.pinned_empty(f.shape)
        p[:] = f
        pin_bgr.append(p)
    e.run([pin_bgr])
    bgr_zero_copy = e.last_h2d_bytes()
    for fmt in Y.FORMATS:
        yuv = [Y.from_bgr(f, fmt) for f in bgr_in]
        pinned = []
        for f in yuv:
            p = L.pinned_empty(f.shape)
            p[:] = f
            pinned.append(p)
        a = e.run([pinned], pixel_format=fmt)[0].copy()
        zc = e.last_h2d_bytes()
        b = e.run([yuv], pixel_format=fmt)[0]
        dma = e.last_h2d_bytes()
        assert (a == b).all(), fmt
        assert dma == e.host_copy_bytes(pixel_format=fmt)[0]
        assert 0 < zc <= 0.55 * bgr_zero_copy, (fmt, zc, bgr_zero_copy)
        assert dma <= 0.55 * e.host_copy_bytes()[0]
        assert e.host_copy_bytes(True, fmt)[0] == 4 * g.FW * g.FH * 3 // 2


def test_device_stack_unaligned_base_and_stride(ops, fx):
    """run_stack on YUV frames at an odd base address and an odd frame stride."""
    import torch
    g = fx.geometry()
    e, masks = _engine(ops, fx, g, True, calib=fx.calib)
    dev = torch.device("cuda", e.ctx.device)
    car = torch.from_numpy(fx.car()).to(dev)
    fb = g.FW * g.FH * 3 // 2
    stride, n = fb + 3, 3
    for fmt in Y.FORMATS:
        yuv, bgr = _sets(fx, g, n, fmt)
        host = np.full(1 + n * 4 * stride, 0xEE, np.uint8)
        for i, f in enumerate(f for s in yuv for f in s):
            host[1 + i * stride:1 + i * stride + fb] = f.reshape(-1)
        d = torch.from_numpy(host).to(dev)
        for balance in (False, True):
            out = torch.empty((n, g.BH, g.BW, 3), dtype=torch.uint8, device=dev)
            e.run_stack(d.data_ptr() + 1, stride, n, out.data_ptr(), car.data_ptr(), balance, pixel_format=fmt)
            e.ctx.sync()
            assert e.last_path() == "tma"
            got = out.cpu().numpy()
            want = e.run(bgr, fx.car(), balance)
            assert (got == want).all(), (fmt, balance, int((got != want).sum()))


@pytest.mark.parametrize("balance", [False, True])
def test_graph_replay_reads_the_captured_yuv_stack(ops, fx, balance):
    """Capture run_stack on YUV stack A, make an eager call on stack B, replay: A's canvases."""
    import torch
    g = fx.geometry()
    e, _ = _engine(ops, fx, g, True, calib=fx.calib)
    dev = torch.device("cuda", e.ctx.device)
    n, fb = 3, g.FW * g.FH * 3 // 2
    car = torch.from_numpy(fx.car()).to(dev)
    for fmt in Y.FORMATS:
        yuv, bgr = _sets(fx, g, n, fmt)
        a = np.stack([np.stack(s) for s in yuv])
        d_a, d_b = torch.from_numpy(a).to(dev), torch.from_numpy(np.ascontiguousarray(a[::-1]) ^ 0x21).to(dev)

        def call(d, out):
            e.run_stack(d.data_ptr(), fb, n, out.data_ptr(), car.data_ptr(), balance, pixel_format=fmt)

        want_a, want_b, got = _replay_after_other_stack(torch, e, call, d_a, d_b, (n, g.BH, g.BW, 3))
        assert e.last_path() == "tma"
        assert (want_a == e.run(bgr, fx.car(), balance)).all()
        assert (got == want_a).all(), (fmt, int((got != want_a).sum()), bool((got == want_b).all()))


def test_refusals(ops, fx):
    import torch
    from cameracalibration_b200 import _lib as L
    g = fx.geometry(640, 512, 500, 500)
    e, _ = _engine(ops, fx, g, False)
    dev = torch.device("cuda", e.ctx.device)
    yuv = [Y.from_bgr(f, "nv12") for f in fx.frames(640, 512)]
    # wrong shapes, dtypes and names
    with pytest.raises(L.BevkError, match="uint8"):
        e.run([fx.frames(640, 512)], pixel_format="nv12")
    with pytest.raises(L.BevkError, match="uint8"):
        e.run([[f.astype(np.int16) for f in yuv]], pixel_format="i420")
    with pytest.raises(L.BevkError, match="pixel_format"):
        e.run([yuv], pixel_format="yuyv")
    with pytest.raises(L.BevkError, match="frames must be uint8"):
        e.run_cuda(torch.zeros((1, 4, 512, 640), dtype=torch.uint8, device=dev), pixel_format="nv12")
    with pytest.raises(L.BevkError, match="one uint8 CUDA array"):
        e.run_cuda([[torch.zeros((768, 640), dtype=torch.uint8, device=dev)] * 4], pixel_format="nv12")
    lib, h, V = e.ctx.lib, e.ctx.h, ctypes.c_void_p
    d = torch.zeros((4, 768, 640), dtype=torch.uint8, device=dev)
    out = torch.zeros((1, 500, 500, 3), dtype=torch.uint8, device=dev)
    assert lib.bevk_bev_run_stack(h, V(d.data_ptr()), 768 * 640, 1, None, L.FLAG_NV12 | L.FLAG_I420, V(out.data_ptr())) == -1
    assert lib.bevk_bev_run_stack(h, V(d.data_ptr()), 768 * 640 - 1, 1, None, L.FLAG_NV12, V(out.data_ptr())) == -1
    # every entry point with flags other than bevk_bev_run / _run_stack / _host_copy_bytes refuses the YUV bits
    table = (V * 4)(*[d.data_ptr()] * 4)
    hp = (V * 4)(*[f.ctypes.data for f in yuv])
    sizes = (ctypes.c_uint64 * 4)(1, 1, 1, 1)
    streams = np.zeros(1 << 16, np.uint8)
    ssz = (ctypes.c_uint64 * 1)()
    n_own = ctypes.c_int()
    for flag in (L.FLAG_NV12, L.FLAG_I420, L.FLAG_NV12 | L.FLAG_BALANCE):
        rcs = {
            "run_device": lib.bevk_bev_run_device(h, V(d.data_ptr()), 1, None, flag, V(out.data_ptr())),
            "run_frames": lib.bevk_bev_run_frames(h, table, 1, None, flag, V(out.data_ptr())),
            "run_jpeg": lib.bevk_bev_run_jpeg(h, hp, sizes, 1, None, flag, L.vptr(streams)),
            "run_to_jpeg": lib.bevk_bev_run_to_jpeg(h, hp, 640, 1, None, flag, 95, L.vptr(streams), streams.size, ssz),
            "frames_to_jpeg": lib.bevk_bev_frames_to_jpeg(h, table, 1, None, flag, 95, L.vptr(streams), streams.size, ssz),
            "run_sharded": lib.bevk_bev_run_sharded(h, V(d.data_ptr()), 768 * 640, 1, None, flag, V(out.data_ptr())),
            "run_scattered": lib.bevk_bev_run_scattered(h, V(d.data_ptr()), 768 * 640, 1, None, flag, V(out.data_ptr()),
                                                        ctypes.byref(n_own)),
        }
        assert all(rc == -4 for rc in rcs.values()), (flag, rcs)
        assert "BGR frames only" in lib.bevk_last_error().decode()
    e.ctx.sync()
    # odd frame sizes: cv2 refuses them, and so do the Python layer and the C ABI
    go = fx.geometry(641, 512, 500, 500)
    eo, _ = _engine(ops, fx, go, False)
    with pytest.raises(L.BevkError, match="even"):
        eo.run([[np.zeros((768, 641), np.uint8)] * 4], pixel_format="nv12")
    for flag in (L.FLAG_NV12, L.FLAG_I420):
        assert lib.bevk_bev_run_stack(eo.ctx.h, V(d.data_ptr()), 768 * 642, 1, None, flag, V(out.data_ptr())) == -4
        a, b = ctypes.c_int64(), ctypes.c_int64()
        assert lib.bevk_bev_host_copy_bytes(eo.ctx.h, flag, ctypes.byref(a), ctypes.byref(b)) == -4
        p = (V * 4)(*[np.zeros(1, np.uint8).ctypes.data] * 4)
        assert lib.bevk_bev_run(eo.ctx.h, p, 641, 1, None, flag, L.vptr(np.zeros((500, 500, 3), np.uint8))) == -4
