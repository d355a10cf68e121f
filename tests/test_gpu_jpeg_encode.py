"""GPU test of the device JPEG encoder (bevk_jpeg_encode / bevk_undistort_jpeg, ops.jpeg_encode, Undistorter.jpeg and
Tools/undistort.py -dstformat jpg): every stream must equal cv2.imencode's / the file cv2.imwrite writes, byte for byte."""
import ctypes

import cv2
import numpy as np
import pytest

from oracle import cv2_path as C
from oracle import restate as R
from tests.helpers import NAMES

pytestmark = pytest.mark.gpu


def _cv2(img, q=95):
    return cv2.imencode(".jpg", np.ascontiguousarray(img), [cv2.IMWRITE_JPEG_QUALITY, q])[1].tobytes()


def test_device_canvases_batch_of_32(fx):
    """32 canvases rendered on the device by the engine (the bench workload's output), encoded in place at q95 and q100."""
    import torch
    from cameracalibration_b200 import ops
    g = fx.geometry()
    e = ops.BevEngine(4, (g.FW, g.FH), (g.BW, g.BH))
    masks = [R.blend_mask(n, g.BW, g.BH, g.CW, g.CH) for n in NAMES]
    for i, n in enumerate(NAMES):
        K, D, H = fx.calib[n]
        e.set_camera(i, K, D, C.dst_camera_matrix(K, g.FW, g.FH, g.FS, g.SS), (int(g.FW * g.SS), int(g.FH * g.SS)), H)
        e.set_mask(i, masks[i])
    e.finalize()
    frames = np.stack([np.stack(fx.perturbed_frames(g.FW, g.FH, b)) for b in range(32)])
    canvases = e.run_cuda(torch.from_numpy(frames).cuda())
    host = canvases.cpu().numpy()
    assert len({host[b].tobytes() for b in range(32)}) == 32
    for q in (95, 100):
        streams = ops.jpeg_encode(canvases, q, ctx=e.ctx)
        assert len(streams) == 32
        for b in range(32):
            assert streams[b] == _cv2(host[b], q), (q, b)


def test_padded_rows_and_images():
    """Row pitch > 3W and image stride > H * pitch, read in place."""
    import torch
    from cameracalibration_b200 import ops
    rng = np.random.default_rng(31)
    N, H, W = 3, 45, 70
    base = torch.from_numpy(rng.integers(0, 256, (N, H + 5, 3 * W + 29), dtype=np.uint8)).cuda()
    view = base[:, :H, :3 * W].unflatten(2, (W, 3))
    iface = view.__cuda_array_interface__
    assert iface["strides"] is not None and iface["strides"][1] > 3 * W and iface["strides"][0] > H * iface["strides"][1]
    host = view.cpu().numpy()
    for q in (75, 100):
        assert ops.jpeg_encode(view, q) == [_cv2(host[i], q) for i in range(N)]
    assert ops.jpeg_encode(view[1]) == [_cv2(host[1])]          # one image [H][W][3] with a padded pitch


def test_odd_sizes_and_quality_sweep():
    from cameracalibration_b200 import ops
    rng = np.random.default_rng(32)
    for w, h in ((1, 1), (9, 17), (37, 23), (1001, 999)):
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        if w > 500:                                              # a smooth image too: long zero runs, ZRL, EOB
            yy, xx = np.mgrid[0:h, 0:w]
            img[: h // 2] = np.stack([(xx * 255 // w), (yy * 255 // h), ((xx + yy) & 255)], -1)[: h // 2].astype(np.uint8)
        for q in (1, 50, 95, 100):
            assert ops.jpeg_encode(img, q) == [_cv2(img, q)], (w, h, q)
    img = rng.integers(0, 256, (48, 64, 3), dtype=np.uint8)
    batch = np.stack([img, 255 - img])
    for q in list(range(-5, 106, 7)) + [150]:
        assert ops.jpeg_encode(batch, q) == [_cv2(batch[0], q), _cv2(batch[1], q)], q
    assert ops.jpeg_encode(img) == [cv2.imencode(".jpg", img)[1].tobytes()]      # cv2's default quality is 95


@pytest.mark.parametrize("fused", [False, True])
def test_undistorter_jpeg_2560x2048(fx, fused):
    from cameracalibration_b200 import ops
    K, D, _ = fx.calib["front"]
    P = C.dst_camera_matrix(K, 1280, 1024, 1, 2)
    u = ops.Undistorter(K, D, P, (2560, 2048), fused=fused)
    src = fx.img("front")
    want_img = cv2.remap(src, *C.undistort_maps(K, D, P, 2560, 2048), interpolation=cv2.INTER_LINEAR)
    assert (u(src) == want_img).all()
    for q in (100, 95):
        assert u.jpeg(src, q) == _cv2(want_img, q), q
    near = cv2.remap(src, *C.undistort_maps(K, D, P, 2560, 2048), interpolation=cv2.INTER_NEAREST)
    assert u.jpeg(src, 90, ops.INTER_NEAREST) == _cv2(near, 90)
    with pytest.raises(Exception, match="uint8\\[h\\]\\[w\\]\\[3\\]"):
        u.jpeg(cv2.cvtColor(src, cv2.COLOR_BGR2GRAY))
    u.close()


def test_tools_undistort_cli_jpg_files_identical(fx, tmp_path):
    """Tools/undistort.py -dstformat jpg -quality 100: the files equal the reference loop's cv2.remap + cv2.imwrite."""
    from cameracalibration_b200.Tools import undistort as T
    (tmp_path / "in").mkdir()
    (tmp_path / "out").mkdir()
    (tmp_path / "ref").mkdir()
    K, D, _ = fx.calib["front"]
    np.save(tmp_path / "K.npy", K)
    np.save(tmp_path / "D.npy", D)
    for n in NAMES:
        cv2.imwrite(str(tmp_path / "in" / f"{n}.png"), fx.img(n))
    m1, m2 = C.undistort_maps(K, D, C.dst_camera_matrix(K, 1280, 1024, 1, 1), 1280, 1024)
    for fused in ("0", "1"):
        written = T.main(["-path_read", str(tmp_path / "in") + "/", "-path_save", str(tmp_path / "out") + "/", "-path_k",
                          str(tmp_path / "K.npy"), "-path_d", str(tmp_path / "D.npy"), "-srcformat", "png", "-dstformat", "jpg",
                          "-quality", "100", "-fused", fused, "-workers", "2"])
        assert sorted(written) == sorted(f"{n}.png" for n in NAMES)
        for entry in written:
            img = cv2.imread(str(tmp_path / "in" / entry))
            ref = str(tmp_path / "ref" / (entry[:-4] + ".jpg"))
            cv2.imwrite(ref, cv2.remap(img, m1, m2, interpolation=cv2.INTER_LINEAR), [cv2.IMWRITE_JPEG_QUALITY, 100])
            got = (tmp_path / "out" / (entry[:-4] + ".jpg")).read_bytes()
            assert got == open(ref, "rb").read(), (fused, entry)


def test_capacity_and_channel_errors():
    import torch
    from cameracalibration_b200 import _lib as L
    from cameracalibration_b200 import ops
    ctx = L.default_context()
    rng = np.random.default_rng(33)
    img = rng.integers(0, 256, (2, 40, 56, 3), dtype=np.uint8)
    d = torch.from_numpy(img).cuda()
    want = [_cv2(img[0], 90), _cv2(img[1], 90)]
    total = sum(len(s) for s in want)
    sizes = (ctypes.c_uint64 * 2)()
    buf = np.full(total + 64, 0xA5, np.uint8)
    rc = ctx.lib.bevk_jpeg_encode(ctx.h, ctypes.c_void_p(d.data_ptr()), 40 * 56 * 3, 56 * 3, 2, 56, 40, 90, L.vptr(buf), total - 1,
                                  sizes)
    assert rc == -1                                             # BEVK_ERR_ARG
    assert "capacity" in ctx.lib.bevk_last_error().decode()
    assert list(sizes) == [len(s) for s in want]
    assert (buf == 0xA5).all()                                  # nothing written, in particular nothing past capacity
    rc = ctx.lib.bevk_jpeg_encode(ctx.h, ctypes.c_void_p(d.data_ptr()), 40 * 56 * 3, 56 * 3, 2, 56, 40, 90, L.vptr(buf), total, sizes)
    assert rc == 0
    assert buf[:total].tobytes() == b"".join(want) and (buf[total:] == 0xA5).all()
    for bad in (np.zeros((8, 8, 4), np.uint8), np.zeros((8, 8), np.uint8), np.zeros((2, 8, 8, 1), np.uint8),
                np.zeros((8, 8, 3), np.float32)):
        with pytest.raises(L.BevkError, match="uint8"):
            ops.jpeg_encode(bad)
    with pytest.raises(L.BevkError, match="uint8"):
        ops.jpeg_encode(torch.zeros((8, 8, 4), dtype=torch.uint8, device="cuda"))
    with pytest.raises(L.BevkError, match="size"):
        ops.jpeg_encode_bound(0, 8)
