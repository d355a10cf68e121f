"""Every image entry point (remap, undistort, warpPerspective, warpAffine, resize; host, device-batch and JPEG forms) under
every channel count and interpolation or flag it accepts, and the refusals of one bad argument each.

Each accepted call must equal cv2 byte for byte (cv2.remap through cv2's own undistortion maps, cv2.warpPerspective,
cv2.warpAffine, cv2.resize, and cv2.imencode of those images for the JPEG forms), enqueue the expected number of kernels
(bevk_launch_count) and report the expected kernel in bevk_undistort_last_path.  Host sources and destinations are dense
and row-padded; device batches have n = 1 and n = 3, padded rows and images, and a base off a 4-byte boundary.  The host
form and the n = 1 device form of an operation give the same bytes.  Each refusal returns its status code and message,
enqueues nothing and leaves the destination as it was."""
import ctypes as C

import cv2
import numpy as np
import pytest

from oracle import cv2_path as CV

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

V = C.c_void_p
ARG, UNSUP = -1, -4
NEAREST, LINEAR, CUBIC, AREA, LANCZOS4 = 0, 1, 2, 3, 4
GATHER_INTERPS = (NEAREST, LINEAR, CUBIC, AREA, LANCZOS4)
INVERSE = 16                                     # WARP_INVERSE_MAP
SW, SH, DW, DH = 72, 50, 96, 40                  # 4-byte rows at 3 channels on both sides: the word path is reachable
FILL = 0xA5
H = np.array([[1.05, 0.03, -3.0], [0.02, 0.97, 2.0], [1e-4, 2e-4, 1.0]])
M = np.array([[0.9, 0.1, 3.5], [-0.05, 1.1, -2.25]])
PATH_WORD, PATH_BYTE, PATH_TAPS, PATH_RESIZE = 4, 1, 2, 3


class Rig:
    """A context of its own with four undistorter slots: fisheye and pinhole, map-resident and fused (slot 7 unset)."""

    def __init__(self, fx):
        from cameracalibration_b200 import _lib as L
        self.L = L
        self.ctx = L.Context(0)
        self.lib, self.h = self.ctx.lib, self.ctx.h
        self.dev = torch.device("cuda", self.ctx.device)
        K, D, _ = fx.calib["front"]
        K = np.diag([SW / 1280, SH / 1024, 1.0]) @ K
        P = CV.dst_camera_matrix(K, DW, DH, 0.6, 1)
        eye = np.eye(3)
        self.model = {"fisheye": (0, K, np.asarray(D, np.float64).reshape(-1), P),
                      "pinhole": (1, K, np.asarray(fx.D5, np.float64).reshape(-1), P)}
        self.maps = {"fisheye": cv2.fisheye.initUndistortRectifyMap(K, D, eye, P, (DW, DH), cv2.CV_16SC2),
                     "pinhole": cv2.initUndistortRectifyMap(K, fx.D5, eye, P, (DW, DH), cv2.CV_16SC2)}
        self.slots = {}
        for slot, (model, fused) in enumerate((("fisheye", 0), ("fisheye", 1), ("pinhole", 0), ("pinhole", 1))):
            m, K_, D_, P_ = self.model[model]
            L.check(self.lib.bevk_undistorter_set(self.h, slot, m, L.dptr(K_), L.dptr(D_), D_.size, L.dptr(P_), DW, DH, fused))
            self.slots[(model, fused)] = slot
        self.rng = np.random.default_rng(20261018)

    def launches(self):
        return int(self.lib.bevk_launch_count(self.h))

    def path(self):
        return int(self.lib.bevk_undistort_last_path(self.h))

    def error(self):
        return self.lib.bevk_last_error().decode()

    def image(self, w, h, ch):
        return self.rng.integers(0, 256, (h, w) if ch == 1 else (h, w, ch), dtype=np.uint8)


@pytest.fixture(scope="module")
def rig(fx):
    return Rig(fx)


# ------------------------------------------------------------------ the operations
# An operation: name, channels, its argument (interp / flags), the C calls and cv2's result.
def _dsize(op):
    return (36, 25) if op.get("fxy") else (DW, DH)


def _ops(rig):
    out = []
    for ch in (1, 3, 4):
        for interp in GATHER_INTERPS:
            out.append(dict(kind="remap", ch=ch, arg=interp, map2=True))
            out.append(dict(kind="perspective", ch=ch, arg=interp))
            for flags in (interp, interp | INVERSE):
                out.append(dict(kind="affine", ch=ch, arg=flags))
            for (model, fused) in rig.slots:
                out.append(dict(kind="undistort", ch=ch, arg=interp, model=model, fused=fused))
        out.append(dict(kind="remap", ch=ch, arg=NEAREST, map2=False))
        for interp in (NEAREST, LINEAR, AREA):
            out.append(dict(kind="resize", ch=ch, arg=interp))
            out.append(dict(kind="resize", ch=ch, arg=interp, fxy=True))
    return out


def _name(op):
    return "-".join(str(v) for v in op.values())


def _want(rig, op, src):
    dsize = _dsize(op)
    if op["kind"] == "remap":
        m1, m2 = rig.maps["fisheye"]
        return cv2.remap(src, m1, m2 if op["map2"] else None, op["arg"])
    if op["kind"] == "undistort":
        return cv2.remap(src, *rig.maps[op["model"]], op["arg"])
    if op["kind"] == "perspective":
        return cv2.warpPerspective(src, H, dsize, flags=op["arg"])
    if op["kind"] == "affine":
        return cv2.warpAffine(src, M, dsize, flags=op["arg"])
    if op.get("fxy"):
        return cv2.resize(src, None, fx=0.5, fy=0.5, interpolation=op["arg"])
    return cv2.resize(src, dsize, interpolation=op["arg"])


def _host_call(rig, op, sp, sstride, dp, dstride, ch=None, sw=SW, sh=SH, dw=None, dh=None, arg=None, slot=None, m1=True,
               m2=True, mat=True):
    """The host form of op; every argument can be overridden (refusals)."""
    L, lib, h = rig.L, rig.lib, rig.h
    ch = op["ch"] if ch is None else ch
    dw = _dsize(op)[0] if dw is None else dw
    dh = _dsize(op)[1] if dh is None else dh
    arg = op["arg"] if arg is None else arg
    k = op["kind"]
    if k == "remap":
        maps = rig.maps["fisheye"]
        return lib.bevk_remap(h, sp, sw, sh, sstride, ch, L.vptr(maps[0]) if m1 else None,
                              L.vptr(maps[1]) if m2 and op["map2"] else None, dw, dh, dp, dstride, arg)
    if k == "undistort":
        slot = rig.slots[(op["model"], op["fused"])] if slot is None else slot
        return lib.bevk_undistort(h, slot, sp, sw, sh, sstride, ch, dp, dw, dh, dstride, arg)
    if k == "perspective":
        return lib.bevk_warp_perspective(h, sp, sw, sh, sstride, ch, L.dptr(H) if mat else None, dp, dw, dh, dstride, arg)
    if k == "affine":
        return lib.bevk_warp_affine(h, sp, sw, sh, sstride, ch, L.dptr(M) if mat else None, dp, dw, dh, dstride, arg)
    fxy = (0.5, 0.5) if op.get("fxy") else (0.0, 0.0)
    return lib.bevk_resize(h, sp, sw, sh, sstride, ch, dp, dw, dh, dstride, *fxy, arg)


def _device_call(rig, op, sp, sis, srs, n, dp, dis, drs, ch=None, sw=SW, sh=SH, dw=None, dh=None, arg=None, slot=None,
                 mat=True, entry=None):
    """The device form of op (undistort: bevk_undistort_stack_interp, or `entry`)."""
    L, lib, h = rig.L, rig.lib, rig.h
    ch = op["ch"] if ch is None else ch
    dw = _dsize(op)[0] if dw is None else dw
    dh = _dsize(op)[1] if dh is None else dh
    arg = op["arg"] if arg is None else arg
    k = op["kind"]
    if k == "undistort":
        slot = rig.slots[(op["model"], op["fused"])] if slot is None else slot
        f = entry or lib.bevk_undistort_stack_interp
        return f(h, slot, sp, sis, sw, sh, srs, ch, n, dp, dis, dw, dh, drs, arg)
    if k == "affine":
        return lib.bevk_warp_affine_stack(h, sp, sis, sw, sh, srs, ch, n, L.dptr(M) if mat else None, dp, dis, dw, dh, drs, arg)
    fxy = (0.5, 0.5) if op.get("fxy") else (0.0, 0.0)
    return lib.bevk_resize_stack(h, sp, sis, sw, sh, srs, ch, n, dp, dis, dw, dh, drs, *fxy, arg)


def _path(op, ch, dw, sh, spitch, dpitch, sbase, dbase, n=1, sis=0, dis=0):
    """bevk_undistort_last_path after op: k_resize, k_gather_taps, or k_gather4's word path when its rule holds."""
    if op["kind"] == "resize":
        return PATH_RESIZE
    interp = op["arg"] & 7
    interp = LINEAR if interp == AREA else interp
    if interp in (CUBIC, LANCZOS4):
        return PATH_TAPS
    al = sbase | dbase | spitch | dpitch | ((sis | dis) if n > 1 else 0)
    maps_ok = op["kind"] != "remap" or op["map2"]
    word = ch == 3 and interp == LINEAR and dw % 4 == 0 and al % 4 == 0 and spitch < (1 << 31) // sh and maps_ok
    return PATH_WORD if word else PATH_BYTE


def _padded_host(img, pad):
    """img inside a FILL-padded buffer whose rows are `pad` bytes longer: (buffer, pointer, row stride)."""
    h, w = img.shape[:2]
    row = img[0].size
    buf = np.full((h, row + pad), FILL, np.uint8)
    buf[:, :row] = img.reshape(h, row)
    return buf, V(buf.ctypes.data), row + pad


def _padded_device(rig, frames, row_pad, img_pad, offset):
    """frames [n][h][w][c] in a FILL device pool at byte `offset`, rows and images padded: (pool, pointer, image stride,
    row stride)."""
    n, h, w, ch = frames.shape
    row = w * ch + row_pad
    img = h * row + img_pad
    pool = torch.full((offset + n * img + 64,), FILL, dtype=torch.uint8, device=rig.dev)
    view = pool[offset:offset + n * img].as_strided((n, h, w, ch), (img, row, ch, 1))
    view.copy_(torch.from_numpy(np.ascontiguousarray(frames)).to(rig.dev))
    torch.cuda.synchronize(rig.dev)              # the library's stream does not wait for torch's
    return pool, pool.data_ptr() + offset, img, row


def _read_device(rig, pool, ptr, n, h, w, ch, img, row):
    """n frames [h][w][ch] at ptr (inside pool) with the given strides, as NumPy, once the ctx stream has written them."""
    rig.ctx.sync()
    off = ptr - pool.data_ptr()
    return pool[off:off + n * img].as_strided((n, h, w, ch), (img, row, ch, 1)).cpu().numpy()


@pytest.mark.parametrize("kind", ["remap", "undistort", "perspective", "affine", "resize"])
def test_every_operation_host_and_device(rig, kind):
    L = rig.L
    for op in (o for o in _ops(rig) if o["kind"] == kind):
        ch = op["ch"]
        dw, dh = _dsize(op)
        src = rig.image(SW, SH, ch)
        want = _want(rig, op, src).reshape(dh, dw, ch)
        # host forms: dense, and row-padded on both sides
        for spad, dpad in ((0, 0), (5, 3)):
            sbuf, sp, ss = _padded_host(src, spad)
            dbuf = np.full((dh, dw * ch + dpad), FILL, np.uint8)
            n0 = rig.launches()
            L.check(_host_call(rig, op, sp, ss, V(dbuf.ctypes.data), dw * ch + dpad))
            assert rig.launches() - n0 == 1, _name(op)
            assert rig.path() == _path(op, ch, dw, SH, SW * ch, dw * ch, 0, 0), (_name(op), spad)
            assert (dbuf[:, :dw * ch].reshape(dh, dw, ch) == want).all(), (_name(op), spad, dpad)
            assert (dbuf[:, dw * ch:] == FILL).all()
        if kind in ("remap", "perspective"):
            continue
        # device forms: n = 1 dense; n = 3 padded; n = 3 padded at an odd base
        frames = np.stack([src] + [rig.image(SW, SH, ch) for _ in range(2)]).reshape(3, SH, SW, ch)
        wants = [want] + [_want(rig, op, f.reshape(src.shape)).reshape(dh, dw, ch) for f in frames[1:]]
        for n, rpad, ipad, off in ((1, 0, 0, 0), (3, 4, 12, 0), (3, 3, 7, 1)):
            spool, sp, sis, srs = _padded_device(rig, frames[:n], rpad, ipad, off)
            dpool, dp, dis, drs = _padded_device(rig, np.zeros((n, dh, dw, ch), np.uint8), rpad, ipad, off)
            n0 = rig.launches()
            L.check(_device_call(rig, op, V(sp), sis, srs, n, V(dp), dis, drs))
            assert rig.launches() - n0 == 1, _name(op)
            assert rig.path() == _path(op, ch, dw, SH, srs, drs, sp, dp, n, sis, dis), (_name(op), n, off)
            got = _read_device(rig, dpool, dp, n, dh, dw, ch, dis, drs)
            for i in range(n):
                assert (got[i] == wants[i]).all(), (_name(op), n, rpad, off, i)
            if n == 1:
                assert (got[0] == dbuf[:, :dw * ch].reshape(dh, dw, ch)).all(), _name(op)   # host form == device form


def test_undistort_stack_nearest_linear(rig):
    """bevk_undistort_stack: the NEAREST / LINEAR entry point gives bevk_undistort_stack_interp's bytes."""
    for (model, fused) in rig.slots:
        for ch in (1, 3, 4):
            for interp in (NEAREST, LINEAR):
                op = dict(kind="undistort", ch=ch, arg=interp, model=model, fused=fused)
                frames = np.stack([rig.image(SW, SH, ch) for _ in range(3)]).reshape(3, SH, SW, ch)
                spool, sp, sis, srs = _padded_device(rig, frames, 4, 12, 0)
                dpool, dp, dis, drs = _padded_device(rig, np.zeros((3, DH, DW, ch), np.uint8), 4, 12, 0)
                n0 = rig.launches()
                rig.L.check(_device_call(rig, op, V(sp), sis, srs, 3, V(dp), dis, drs, entry=rig.lib.bevk_undistort_stack))
                assert rig.launches() - n0 == 1
                assert rig.path() == _path(op, ch, DW, SH, srs, drs, sp, dp, 3, sis, dis)
                got = _read_device(rig, dpool, dp, 3, DH, DW, ch, dis, drs)
                for i in range(3):
                    want = _want(rig, op, frames[i].reshape((SH, SW) if ch == 1 else (SH, SW, ch)))
                    assert (got[i] == want.reshape(DH, DW, ch)).all(), (model, fused, ch, interp, i)


def _encode_launches(rig, images):
    """Kernels bevk_jpeg_encode enqueues for n device images (the encoder part of a JPEG form's launches)."""
    n = len(images)
    d = torch.from_numpy(np.ascontiguousarray(np.stack(images))).to(rig.dev)
    torch.cuda.synchronize(rig.dev)
    out, sizes = np.zeros(n * (1 << 16), np.uint8), (C.c_uint64 * n)()
    n0 = rig.launches()
    rig.L.check(rig.lib.bevk_jpeg_encode(rig.h, V(d.data_ptr()), DW * DH * 3, DW * 3, n, DW, DH, 90, V(out.ctypes.data),
                                         out.size, sizes))
    return rig.launches() - n0


def _streams(out, sizes):
    res, off = [], 0
    for s in sizes:
        res.append(out[off:off + s].tobytes())
        off += s
    return res


def test_jpeg_forms(rig):
    """bevk_undistort_jpeg (host frame) and bevk_undistort_stack_jpeg (device frames) == cv2.imencode of cv2.remap."""
    L = rig.L
    L.check(rig.lib.bevk_jpeg_set_params(rig.h, None, 0))
    for (model, fused), slot in rig.slots.items():
        for interp in GATHER_INTERPS:
            op = dict(kind="undistort", ch=3, arg=interp, model=model, fused=fused)
            frames = np.stack([rig.image(SW, SH, 3) for _ in range(3)])
            wants = [_want(rig, op, f) for f in frames]
            jpgs = [cv2.imencode(".jpg", w, [cv2.IMWRITE_JPEG_QUALITY, 90])[1].tobytes() for w in wants]
            enc1 = _encode_launches(rig, wants[:1])
            for spad in (0, 5):
                sbuf, sp, ss = _padded_host(frames[0], spad)
                out, size = np.zeros(1 << 16, np.uint8), C.c_uint64()
                n0 = rig.launches()
                L.check(rig.lib.bevk_undistort_jpeg(rig.h, slot, sp, SW, SH, ss, interp, 90, V(out.ctypes.data), out.size,
                                                    C.byref(size)))
                assert rig.launches() - n0 == 1 + enc1, (model, fused, interp)
                assert rig.path() == _path(op, 3, DW, SH, SW * 3, DW * 3, 0, 0)
                assert out[:size.value].tobytes() == jpgs[0], (model, fused, interp, spad)
            for n, rpad, ipad, off in ((1, 0, 0, 0), (3, 4, 12, 0), (3, 3, 7, 1)):
                spool, sp, sis, srs = _padded_device(rig, frames[:n], rpad, ipad, off)
                out, sizes = np.zeros(n << 16, np.uint8), (C.c_uint64 * n)()
                enc = _encode_launches(rig, wants[:n])
                n0 = rig.launches()
                L.check(rig.lib.bevk_undistort_stack_jpeg(rig.h, slot, V(sp), sis, SW, SH, srs, n, interp, 90,
                                                          V(out.ctypes.data), out.size, sizes))
                assert rig.launches() - n0 == 1 + enc, (model, fused, interp, n)
                assert rig.path() == _path(op, 3, DW, SH, srs, DW * 3, sp, 0, n, sis, DW * DH * 3), (model, fused, interp, n, off)
                assert _streams(out, list(sizes)) == jpgs[:n], (model, fused, interp, n, off)


def test_map_builders(rig):
    """bevk_undistort_map, bevk_undistorter_maps (resident and fused slots) and bevk_warp_maps == cv2's maps."""
    L, lib, h = rig.L, rig.lib, rig.h
    for model, (m, K, D, P) in rig.model.items():
        want = rig.maps[model]
        m1, m2 = np.zeros((DH, DW, 2), np.int16), np.zeros((DH, DW), np.uint16)
        n0 = rig.launches()
        L.check(lib.bevk_undistort_map(h, m, L.dptr(K), L.dptr(D), D.size, L.dptr(P), DW, DH, L.vptr(m1), L.vptr(m2)))
        assert rig.launches() - n0 == 1
        assert (m1 == want[0]).all() and (m2 == want[1]).all(), model
        for fused in (0, 1):
            m1, m2 = np.zeros((DH, DW, 2), np.int16), np.zeros((DH, DW), np.uint16)
            n0 = rig.launches()
            L.check(lib.bevk_undistorter_maps(h, rig.slots[(model, fused)], L.vptr(m1), L.vptr(m2)))
            assert rig.launches() - n0 == fused, (model, fused)           # a fused slot evaluates its model
            assert (m1 == want[0]).all() and (m2 == want[1]).all(), (model, fused)
        o1, o2 = np.zeros((30, 50, 2), np.int16), np.zeros((30, 50), np.uint16)
        n0 = rig.launches()
        L.check(lib.bevk_warp_maps(h, L.vptr(want[0]), L.vptr(want[1]), DW, DH, L.dptr(H), 50, 30, L.vptr(o1), L.vptr(o2)))
        assert rig.launches() - n0 == 1
        assert (o1 == cv2.warpPerspective(want[0], H, (50, 30))).all(), model
        assert (o2 == cv2.warpPerspective(want[1], H, (50, 30))).all(), model


# ------------------------------------------------------------------ refusals
def _host_refusals(kind):
    """(overrides of _host_call, status, message fragment): one bad argument each."""
    rows = [(dict(sp=None), ARG, "null src"), (dict(dp=None), ARG, "null dst"), (dict(sw=0), ARG, "size"),
            (dict(dw=0), ARG, "holds a" if kind == "undistort" else "size"), (dict(ch=2), UNSUP, "channels"),
            (dict(sstride=-1), ARG, "src stride"),
            (dict(dstride=-1), ARG, "dst stride")]
    if kind == "remap":
        rows += [(dict(arg=5), UNSUP, "interp 5"), (dict(m1=False), ARG, "null map1"), (dict(m2=False), ARG, "needs map2")]
    if kind == "undistort":
        rows += [(dict(arg=5), UNSUP, "interp 5"), (dict(slot=7), ARG, "not set"), (dict(slot=8), ARG, "not set"),
                 (dict(dw=DW - 1), ARG, "holds a"), (dict(dh=DH + 1), ARG, "holds a")]
    if kind == "perspective":
        rows += [(dict(arg=5), UNSUP, "interp 5"), (dict(mat=False), ARG, "null H")]
    if kind == "affine":
        rows += [(dict(arg=5), UNSUP, "interp 5"), (dict(arg=32), UNSUP, "warpAffine flags"), (dict(mat=False), ARG, "null M")]
    if kind == "resize":
        rows += [(dict(arg=CUBIC), UNSUP, "resize interp"), (dict(dw=DW + 1, fxy=True), ARG, "images")]
    return rows


@pytest.mark.parametrize("kind", ["remap", "undistort", "perspective", "affine", "resize"])
def test_host_refusals(rig, kind):
    op = dict(kind=kind, ch=3, arg=LINEAR, map2=True, model="fisheye", fused=0)
    src = rig.image(SW, SH, 3)
    for kw, code, msg in _host_refusals(kind):
        o = dict(op, fxy=kw.pop("fxy", False))
        dw, dh = _dsize(o)
        dbuf = np.full((DH + 1, (DW + 1) * 3), FILL, np.uint8)
        args = dict(sp=V(src.ctypes.data), sstride=SW * 3, dp=V(dbuf.ctypes.data), dstride=dbuf.shape[1])
        if kw.get("sstride") == -1:
            kw["sstride"] = SW * 3 - 1
        if kw.get("dstride") == -1:
            kw["dstride"] = dw * 3 - 1
        args.update(kw)
        n0 = rig.launches()
        rc = _host_call(rig, o, **args)
        assert rc == code and msg in rig.error(), (kind, kw, rc, rig.error())
        assert rig.launches() == n0, (kind, kw)
        assert (dbuf == FILL).all(), (kind, kw)


def _device_refusals(kind, img, row, dimg, drow):
    rows = [(dict(sp=None), ARG, "null src"), (dict(dp=None), ARG, "null dst"), (dict(sw=0), ARG, "size"),
            (dict(dw=0), ARG, "holds a" if kind.startswith("undistort") else "size"), (dict(ch=2), UNSUP, "channels"),
            (dict(n=0), ARG, "n must"),
            (dict(srs=row - 1), ARG, "src stride"), (dict(drs=drow - 1), ARG, "dst stride"),
            (dict(sis=img - 1), ARG, "src image stride"), (dict(dis=dimg - 1), ARG, "dst image stride"),
            (dict(dp="src+1"), ARG, "overlaps"), (dict(dp="src"), ARG, "overlaps")]
    if kind == "undistort":
        rows += [(dict(arg=5), UNSUP, "interp 5"), (dict(slot=7), ARG, "not set"), (dict(dw=DW - 4), ARG, "holds a"),
                 (dict(dh=DH - 1), ARG, "holds a")]
    if kind == "undistort_stack":
        rows += [(dict(arg=CUBIC), UNSUP, "bevk_undistort_stack takes"), (dict(arg=5), UNSUP, "bevk_undistort_stack takes"),
                 (dict(slot=7), ARG, "not set"), (dict(dw=DW - 4), ARG, "holds a")]
    if kind == "affine":
        rows += [(dict(arg=5), UNSUP, "interp 5"), (dict(arg=32), UNSUP, "warpAffine flags"), (dict(mat=False), ARG, "null M")]
    if kind == "resize":
        rows += [(dict(arg=CUBIC), UNSUP, "resize interp"), (dict(dw=DW + 1, fxy=True), ARG, "images")]
    return rows


@pytest.mark.parametrize("kind", ["undistort", "undistort_stack", "affine", "resize"])
def test_device_refusals(rig, kind):
    op = dict(kind="undistort" if kind == "undistort_stack" else kind, ch=3, arg=LINEAR, model="fisheye", fused=0)
    entry = rig.lib.bevk_undistort_stack if kind == "undistort_stack" else None
    row, img = SW * 3, SH * SW * 3
    drow, dimg = DW * 3, DH * DW * 3
    src = torch.zeros((3 * img,), dtype=torch.uint8, device=rig.dev)
    torch.cuda.synchronize(rig.dev)
    for kw, code, msg in _device_refusals(kind, img, row, dimg, drow):
        o = dict(op, fxy=kw.pop("fxy", False))
        dst = torch.full((3 * dimg + 4 * drow,), FILL, dtype=torch.uint8, device=rig.dev)
        torch.cuda.synchronize(rig.dev)
        args = dict(sp=V(src.data_ptr()), sis=img, srs=row, n=3, dp=V(dst.data_ptr()), dis=dimg, drs=drow)
        if kw.get("dp") == "src":
            kw["dp"] = V(src.data_ptr())
        elif kw.get("dp") == "src+1":
            kw["dp"] = V(src.data_ptr() + img)
        args.update(kw)
        if kind == "resize" and o["fxy"]:
            args["dis"] = max(args["dis"], 25 * 36 * 3)
        n0 = rig.launches()
        rc = _device_call(rig, o, entry=entry, **args)
        assert rc == code and msg in rig.error(), (kind, kw, rc, rig.error())
        assert rig.launches() == n0, (kind, kw)
        assert (dst == FILL).all(), (kind, kw)
        assert (src == 0).all(), (kind, kw)


def test_jpeg_refusals(rig):
    L, lib, h = rig.L, rig.lib, rig.h
    L.check(lib.bevk_jpeg_set_params(h, None, 0))
    slot = rig.slots[("fisheye", 0)]
    src = rig.image(SW, SH, 3)
    for kw, code, msg in [(dict(slot=7), ARG, "not set"), (dict(sp=None), ARG, "null src"), (dict(arg=5), UNSUP, "interp 5"),
                          (dict(sw=0), ARG, "size"), (dict(ss=SW * 3 - 1), ARG, "src stride")]:
        a = dict(slot=slot, sp=V(src.ctypes.data), sw=SW, ss=SW * 3, arg=LINEAR)
        a.update(kw)
        out, size = np.full(1 << 16, FILL, np.uint8), C.c_uint64(7)
        n0 = rig.launches()
        rc = lib.bevk_undistort_jpeg(h, a["slot"], a["sp"], a["sw"], SH, a["ss"], a["arg"], 90, V(out.ctypes.data), out.size,
                                     C.byref(size))
        assert rc == code and msg in rig.error(), (kw, rc, rig.error())
        assert rig.launches() == n0 and (out == FILL).all() and size.value == 7, kw
    row, img = SW * 3, SH * SW * 3
    d = torch.zeros((3 * img,), dtype=torch.uint8, device=rig.dev)
    torch.cuda.synchronize(rig.dev)
    for kw, code, msg in [(dict(slot=7), ARG, "not set"), (dict(sp=None), ARG, "null src"), (dict(arg=5), UNSUP, "interp 5"),
                          (dict(n=0), ARG, "n must"), (dict(srs=row - 1), ARG, "src stride"),
                          (dict(sis=img - 1), ARG, "src image stride")]:
        a = dict(slot=slot, sp=V(d.data_ptr()), sis=img, srs=row, n=3, arg=LINEAR)
        a.update(kw)
        out, sizes = np.full(3 << 16, FILL, np.uint8), (C.c_uint64 * 3)(7, 7, 7)
        n0 = rig.launches()
        rc = lib.bevk_undistort_stack_jpeg(h, a["slot"], a["sp"], a["sis"], SW, SH, a["srs"], a["n"], a["arg"], 90,
                                           V(out.ctypes.data), out.size, sizes)
        assert rc == code and msg in rig.error(), (kw, rc, rig.error())
        assert rig.launches() == n0 and (out == FILL).all() and list(sizes) == [7, 7, 7], kw
