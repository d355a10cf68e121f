"""cv2's border modes on the CPU.  tests/host/remap_border.cu runs the per-thread bodies of k_gather_border,
k_gather_taps_border and k_gather4_border (gather_frames_border, and gather_taps_frames / gather4_frames with BD = true)
with a border built by make_border, over the device's grid,
from the library's own headers; every image must equal live cv2.remap / cv2.warpPerspective / cv2.warpAffine with the
same borderMode and borderValue bit for bit (float32: the same bit pattern, or NaN where cv2 gives NaN):

- every border mode (CONSTANT, REPLICATE, REFLECT, WRAP, REFLECT_101, TRANSPARENT) x depth (8U, 16U, 16S, 32F) x channel
  count (1, 3, 4) x interpolation x MODE 0-5, and the 3-channel LINEAR word path;
- border values negative, over the depth's range, at .5 ties, NaN and +-inf (cv2's scalarToRawData conversion);
- 1- and 2-pixel sources, windows across every edge, int16-extreme maps, warps that fall wholly outside;
- BORDER_TRANSPARENT over a destination filled beforehand;
- border_index against a NumPy restatement of cv2.borderInterpolate for every int16 position (widened by the Lanczos4
  window) and lengths 1-64 and a few large ones, the restatement itself pinned against cv2.borderInterpolate;
- the warps cv2 computes with other arithmetic than remap's, pinned in both directions (cv2_warp_differs).

nvcc compiles the harness; only host code runs."""
import os
import shutil
import struct
import subprocess

import cv2
import numpy as np
import pytest

from cameracalibration_b200.build import GENCODE
from tests import bev_cases as B
from tests.test_host_remap_depth import _mild_camera, cv2_warp_differs, same, ndiff

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INTERS = (cv2.INTER_NEAREST, cv2.INTER_LINEAR, cv2.INTER_CUBIC, cv2.INTER_LANCZOS4)
DEPTHS = {0: np.uint8, 2: np.uint16, 3: np.int16, 5: np.float32}
DEPTH_IDS = ["8u", "16u", "16s", "32f"]
MODES = (cv2.BORDER_CONSTANT, cv2.BORDER_REPLICATE, cv2.BORDER_REFLECT, cv2.BORDER_WRAP, cv2.BORDER_REFLECT_101,
         cv2.BORDER_TRANSPARENT)
VALUES = [(0, 0, 0, 0), (300, -2, 7.5, 8.5), (-40000.5, 70000.4, 2.5, -0.5), (np.nan, np.inf, -np.inf, 1e10),
          (65535, 32767, -32768, 1.5), (17.25, 0, 0, 0)]


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    nvcc = next((c for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc") if c and os.path.exists(c)), None)
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("host_remap_border") / "remap_border"
    build = subprocess.run([nvcc, "-O2", "-std=c++17", "--fmad=false", "-Xcompiler", "-ffp-contract=off", *GENCODE, "-o", str(out),
                            os.path.join(ROOT, "tests", "host", "remap_border.cu")], capture_output=True, text=True, timeout=900)
    assert build.returncode == 0, build.stdout + build.stderr
    return str(out)


def values(rng, depth, shape, special=0.0):
    """Random elements over the depth's range; a fraction `special` of them the depth's extremes."""
    dt = DEPTHS[depth]
    if depth == 5:
        v = (rng.standard_normal(shape) * 10.0 ** rng.uniform(-3, 4, shape)).astype(np.float32)
        ext = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1e-45, 3.4028235e38, 65535.0], np.float32)
    else:
        info = np.iinfo(dt)
        v = rng.integers(info.min, int(info.max) + 1, shape).astype(dt)
        ext = np.array([info.min, info.max, 0], dt)
    if special:
        m = rng.random(shape) < special
        v[m] = rng.choice(ext, int(m.sum()))
    return v


def _stack(frames, row_pad=0, img_pad=0):
    n, h, w, ch = frames.shape
    es = frames.itemsize
    srow = (w * ch + row_pad) * es
    simg = h * srow + img_pad * es
    size = (n - 1) * simg + (h - 1) * srow + w * ch * es
    buf = np.random.default_rng(n * 7 + h * 3 + w).integers(0, 256, size, dtype=np.uint8)
    typed = buf.view(frames.dtype)
    for f in range(n):
        np.lib.stride_tricks.as_strided(typed[f * simg // es:], (h, w, ch), (srow, ch * es, es))[...] = frames[f]
    return buf, srow, simg


class Case:
    """One harness record and the cv2 call it must equal."""

    def __init__(self, mode, inter, frames, dw, dh, extra, border, bval, arg=0, words=False, row_pad=0, img_pad=0,
                 call=None, fill=None):
        n, sh, sw, ch = frames.shape
        depth = {np.dtype(v): k for k, v in DEPTHS.items()}[frames.dtype]
        if words:   # k_gather4 runs on 4-byte aligned rows and images only (gather4_ok)
            row_pad += -(sw * ch + row_pad) % 4
            img_pad -= img_pad % 4
        buf, srow, simg = _stack(frames, row_pad, img_pad)
        if fill is None:
            fill = values(np.random.default_rng(dw * 31 + dh), depth, (n, dh, dw, ch))
        self.fill = np.ascontiguousarray(fill.astype(frames.dtype))
        bv = (tuple(bval) + (0, 0, 0, 0))[:4]
        self.rec = (struct.pack("<12i", mode, ch, inter, depth, sw, sh, dw, dh, n, arg, border, int(words)) +
                    struct.pack("<4d", *[float(v) for v in bv]) + struct.pack("<2q", srow, simg) + extra + buf.tobytes() +
                    self.fill.tobytes())
        self.mode, self.inter, self.frames, self.dw, self.dh = mode, inter, frames, dw, dh
        self.border, self.bval, self.call, self.ch, self.dtype, self.n = border, bval, call, ch, frames.dtype, n

    def want(self, f, maps=None):
        frame = self.frames[f]
        src = frame[..., 0] if self.ch == 1 else frame
        dst = self.fill[f][..., 0].copy() if self.ch == 1 else self.fill[f].copy()
        kw = dict(borderMode=self.border, borderValue=self.bval, dst=dst)
        out = self.call(src, kw) if maps is None else cv2.remap(src, maps[0], maps[1], self.inter, **kw)
        return out.reshape(out.shape[:2] + (self.ch,))


def maps_case(inter, frames, m1, m2, border, bval, **kw):
    dh, dw = m1.shape[:2]
    extra = np.ascontiguousarray(m1, np.int16).tobytes() + (b"" if m2 is None else np.ascontiguousarray(m2, np.uint16).tobytes())
    return Case(0, inter, frames, dw, dh, extra, border, bval, int(m2 is not None),
                call=lambda s, k: cv2.remap(s, m1, m2, inter, **k), **kw)


def fmaps_case(inter, frames, x, y, border, bval, **kw):
    dh, dw = x.shape[:2]
    extra = np.ascontiguousarray(x, np.float32).tobytes() + (b"" if y is None else np.ascontiguousarray(y, np.float32).tobytes())
    return Case(4, inter, frames, dw, dh, extra, border, bval, cv2.CV_32FC2 if y is None else cv2.CV_32FC1,
                call=lambda s, k: cv2.remap(s, x, y, inter, **k), **kw)


def model_case(mode, inter, frames, K, d5, P, model, dw, dh, border, bval):
    extra = np.r_[np.ravel(K), d5, np.ravel(P), float(model)].astype("<f8").tobytes()
    return Case(mode, inter, frames, dw, dh, extra, border, bval)


def persp_case(inter, frames, H, dw, dh, border, bval, **kw):
    return Case(2, inter, frames, dw, dh, np.asarray(H, "<f8").tobytes(), border, bval,
                call=lambda s, k: cv2.warpPerspective(s, H, (dw, dh), flags=inter, **k), **kw)


def affine_case(inter, frames, M, inv, dw, dh, border, bval, **kw):
    fl = inter | (cv2.WARP_INVERSE_MAP if inv else 0)
    return Case(3, inter, frames, dw, dh, np.asarray(M, "<f8").tobytes(), border, bval, int(inv),
                call=lambda s, k: cv2.warpAffine(s, M, (dw, dh), flags=fl, **k), **kw)


def cv2_border_differs(mode, depth, inter, border):
    """The border cases bevk refuses (BEVK_ERR_UNSUPPORTED) because cv2 4.13 leaves remap's arithmetic there: LINEAR
    under BORDER_TRANSPARENT at 32F (the windows across the edge), in every MODE; warpPerspective (MODE 2) NEAREST and
    LINEAR at 16S under BORDER_REPLICATE and BORDER_TRANSPARENT.  test_every_combination pins it in both directions."""
    linear = inter in (cv2.INTER_LINEAR, cv2.INTER_AREA)
    if depth == 5 and linear and border == cv2.BORDER_TRANSPARENT:
        return True
    return mode == 2 and depth == 3 and (linear or inter == cv2.INTER_NEAREST) and border in (
        cv2.BORDER_REPLICATE, cv2.BORDER_TRANSPARENT)


def run(exe, tmp_path, cases, differ=False):
    """Runs the cases; each must equal cv2 (differ=False) or each must differ from it somewhere (differ=True)."""
    (tmp_path / "in.bin").write_bytes(b"".join(c.rec for c in cases))
    r = subprocess.run([exe, "run", str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True,
                       timeout=1800)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr[-2000:])
    raw, p, bad = np.fromfile(tmp_path / "out.bin", np.uint8), 0, []
    for c in cases:
        npx = c.dh * c.dw
        k = c.n * npx * c.ch * c.dtype.itemsize
        imgs = raw[p:p + k].view(c.dtype).reshape(c.n, c.dh, c.dw, c.ch)
        p += k
        maps = None
        if c.mode == 1:
            maps = (raw[p:p + 4 * npx].view(np.int16).reshape(c.dh, c.dw, 2),
                    raw[p + 4 * npx:p + 6 * npx].view(np.uint16).reshape(c.dh, c.dw))
            p += 6 * npx
        elif c.mode == 5:
            maps = (raw[p:p + 4 * npx].view(np.float32).reshape(c.dh, c.dw),
                    raw[p + 4 * npx:p + 8 * npx].view(np.float32).reshape(c.dh, c.dw))
            p += 8 * npx
        for f in range(c.n):
            want = c.want(f, maps)
            if not same(imgs[f], want, c.inter):
                bad.append((c.mode, c.dtype.name, c.ch, c.inter, c.border, c.bval, f, ndiff(imgs[f], want)))
    assert p == raw.size
    keys = {(c.mode, c.dtype.name, c.ch, c.inter, c.border) for c in cases}
    if differ:
        assert {b[:5] for b in bad} == keys, sorted(keys - {b[:5] for b in bad})
    else:
        assert not bad, "\n".join(map(str, sorted({b[:5] for b in bad})))


@pytest.mark.parametrize("depth", DEPTHS, ids=DEPTH_IDS)
def test_every_combination(exe, tmp_path, depth):
    """Every border mode x channel count x interpolation x MODE 0-5 at this depth, with windows inside, across the edges
    and wholly outside, a border value per case from VALUES, and the word path for 3-channel 8-bit LINEAR."""
    rng = np.random.default_rng(1000 + depth)
    cases, refused = [], []
    sw, sh, dw, dh = 13, 11, 48, 36
    i = 0
    for border in MODES:
        for mode in range(6):
            for ch in (1, 3, 4):
                for inter in INTERS:
                    if mode in (2, 3) and cv2_warp_differs(mode, depth, inter, ch):
                        continue
                    i += 1
                    bval = VALUES[i % len(VALUES)]
                    words = depth == 0 and ch == 3 and inter == cv2.INTER_LINEAR and border != cv2.BORDER_TRANSPARENT
                    frames = values(rng, depth, (2, sh, sw, ch), 0.05)
                    n0 = len(cases)
                    if mode == 0:
                        m1 = np.stack([rng.integers(-20, sw + 20, (dh, dw)), rng.integers(-20, sh + 20, (dh, dw))],
                                      -1).astype(np.int16)
                        m2 = None if inter == cv2.INTER_NEAREST and ch == 3 else rng.integers(0, 1024, (dh, dw)).astype(np.uint16)
                        words &= m2 is not None
                        cases.append(maps_case(inter, frames, m1, m2, border, bval, words=words))
                    elif mode in (1, 5):
                        K, d5, P, model = _mild_camera(sw, sh, fisheye=(ch != 3))
                        P = P.copy()
                        P[0, 0] *= 0.4
                        P[1, 1] *= 0.4   # zoomed out: the undistorted frame sits inside a border
                        cases.append(model_case(mode, inter, frames, K, d5, P, model, dw, dh, border, bval))
                    elif mode == 2:
                        H = np.array([[0.3, 0.05, 1.3], [-0.04, 0.35, -2.2], [1e-3, -2e-3, 1.0]])
                        cases.append(persp_case(inter, frames, H, dw, dh, border, bval, words=words))
                    elif mode == 3:
                        M = cv2.getRotationMatrix2D((sw / 2, sh / 2), 17.0 + ch, 2.5)
                        cases.append(affine_case(inter, frames, M, ch == 4, dw, dh, border, bval, words=words))
                    else:
                        x = rng.uniform(-20, sw + 20, (dh, dw)).astype(np.float32)
                        y = rng.uniform(-20, sh + 20, (dh, dw)).astype(np.float32)
                        if ch == 3:
                            cases.append(fmaps_case(inter, frames, np.stack([x, y], -1), None, border, bval, words=words))
                        else:
                            cases.append(fmaps_case(inter, frames, x, y, border, bval))
                    if cv2_border_differs(mode, depth, inter, border):
                        refused.append(cases.pop(n0))
    run(exe, tmp_path, cases)
    if refused:
        run(exe, tmp_path, refused, differ=True)


@pytest.mark.parametrize("depth", DEPTHS, ids=DEPTH_IDS)
def test_border_values(exe, tmp_path, depth):
    """Each border value of VALUES and a few scalars under every mode, through maps whose windows cross every edge."""
    rng = np.random.default_rng(1100 + depth)
    cases = []
    sw, sh, dw, dh = 9, 7, 40, 32
    vals = VALUES + [(np.nan,), (-np.inf, np.nan), (255.5, 254.5, -0.5, 0.5), (-1e-30, 1e-30, 3.4e38, -3.5e38)]
    for j, bval in enumerate(vals):
        for border in MODES:
            ch, inter = (1, 3, 4)[j % 3], INTERS[(j + border) % 4]
            frames = values(rng, depth, (1, sh, sw, ch), 0.05)
            m1 = np.stack([rng.integers(-6, sw + 6, (dh, dw)), rng.integers(-6, sh + 6, (dh, dw))], -1).astype(np.int16)
            m2 = rng.integers(0, 1024, (dh, dw)).astype(np.uint16)
            m2[rng.random((dh, dw)) < 0.2] = 0
            if not cv2_border_differs(0, depth, inter, border):
                cases.append(maps_case(inter, frames, m1, m2, border, bval))
    run(exe, tmp_path, cases)


@pytest.mark.parametrize("depth", DEPTHS, ids=DEPTH_IDS)
def test_small_sources_and_extreme_maps(exe, tmp_path, depth):
    """1- and 2-pixel sources and every small size up to 5 around the frame; the int16-extreme and near-edge map recipes
    of the BEV fuzz corpus; batches across GATHER_NB with padded rows and images."""
    rng = np.random.default_rng(1200 + depth)
    cases = []
    i = 0
    for sw in (1, 2, 3, 5):
        for sh in (1, 2, 4):
            for border in MODES:
                i += 1
                ch, inter, n = (1, 3, 4)[i % 3], INTERS[i % 4], (1, 3, 9)[i % 3]
                frames = values(rng, depth, (n, sh, sw, ch), 0.05)
                xs, ys = np.meshgrid(np.arange(-11, sw + 11), np.arange(-11, sh + 11))
                m1 = np.stack([xs, ys], -1).astype(np.int16)
                m2 = rng.integers(0, 1024, xs.shape).astype(np.uint16)
                if not cv2_border_differs(0, depth, inter, border):
                    cases.append(maps_case(inter, frames, m1, m2, border, VALUES[i % len(VALUES)], row_pad=i % 3,
                                           img_pad=i % 4))
    for i, kind in enumerate(("extreme", "local", "extreme", "local")):
        FW, FH = (2, 33, 1, 64)[i], (2, 21, 3, 40)[i]
        for j, (m1, m2) in enumerate(B._maps(rng, kind, 2, FW, FH, 77, 45)):
            for border in MODES:
                ch, inter = (1, 3, 4)[(i + j + border) % 3], INTERS[(2 * i + j + border) % 4]
                frames = values(rng, depth, (2, FH, FW, ch), 0.05)
                if not cv2_border_differs(0, depth, inter, border):
                    cases.append(maps_case(inter, frames, m1, m2, border, VALUES[(i + border) % len(VALUES)], row_pad=i))
    run(exe, tmp_path, cases)


@pytest.mark.parametrize("depth", DEPTHS, ids=DEPTH_IDS)
def test_warps_outside_and_transparent(exe, tmp_path, depth):
    """Warps that fall wholly or mostly outside the source (zoomed out, shifted away), and BORDER_TRANSPARENT over a
    destination filled beforehand, through warpPerspective and warpAffine with and without WARP_INVERSE_MAP."""
    rng = np.random.default_rng(1300 + depth)
    cases = []
    for i in range(24):
        border = MODES[i % 6]
        ch, inter = (1, 3, 4)[i % 3], INTERS[(i // 3) % 4]
        sw, sh, dw, dh = int(rng.integers(3, 40)), int(rng.integers(3, 30)), 4 * int(rng.integers(2, 16)), int(rng.integers(4, 40))
        frames = values(rng, depth, (1 + i % 2, sh, sw, ch), 0.02)
        bval = VALUES[i % len(VALUES)]
        far = 1e4 if i % 4 == 0 else 0.0
        if not cv2_warp_differs(2, depth, inter, ch) and not cv2_border_differs(2, depth, inter, border):
            H = np.array([[rng.uniform(2, 6), rng.uniform(-.5, .5), rng.uniform(-20, 20) + far],
                          [rng.uniform(-.5, .5), rng.uniform(2, 6), rng.uniform(-20, 20)], [rng.uniform(-1e-3, 1e-3), 0, 1]])
            cases.append(persp_case(inter, frames, H, dw, dh, border, bval))
        if not cv2_warp_differs(3, depth, inter, ch) and not cv2_border_differs(3, depth, inter, border):
            M = np.array([[rng.uniform(-4, 4), rng.uniform(-1, 1), rng.uniform(-20, 40) - far],
                          [rng.uniform(-1, 1), rng.uniform(-4, 4), rng.uniform(-20, 40)]])
            words = depth == 0 and ch == 3 and inter == cv2.INTER_LINEAR and border != cv2.BORDER_TRANSPARENT
            cases.append(affine_case(inter, frames, M, bool(i & 8), dw, dh, border, bval, words=words, row_pad=4 * (i % 2)))
    run(exe, tmp_path, cases)


def border_interpolate(p, n, mode):
    """cv2.borderInterpolate restated in NumPy, loop for loop, over an array of positions."""
    p = np.array(p, np.int64)
    out = p.copy()
    inside = (p >= 0) & (p < n)
    if mode == cv2.BORDER_REPLICATE:
        out = np.where(p < 0, 0, n - 1)
    elif mode in (cv2.BORDER_REFLECT, cv2.BORDER_REFLECT_101):
        d = int(mode == cv2.BORDER_REFLECT_101)
        if n == 1:
            out = np.zeros_like(p)
        else:
            q = p.copy()
            while True:
                o = (q < 0) | (q >= n)
                if not o.any():
                    break
                q = np.where(o & (q < 0), -q - 1 + d, np.where(o, n - 1 - (q - n) - d, q))
            out = q
    elif mode == cv2.BORDER_WRAP:
        q = p.copy()
        neg = q < 0
        q[neg] -= np.fix((q[neg] - n + 1) / n).astype(np.int64) * n
        q = np.where(q >= n, q % n, q)
        out = q
    else:
        out = np.full_like(p, -1)
    return np.where(inside, p, out)


def test_border_interpolate_restatement():
    """The NumPy restatement equals cv2.borderInterpolate itself on a sample of positions, lengths and modes."""
    rng = np.random.default_rng(7)
    for mode in (cv2.BORDER_CONSTANT, cv2.BORDER_REPLICATE, cv2.BORDER_REFLECT, cv2.BORDER_WRAP, cv2.BORDER_REFLECT_101):
        for n in list(range(1, 20)) + [63, 64, 1000, 32767, 65536]:
            ps = np.r_[np.arange(-40, 40), rng.integers(-32776, 32776, 60), -32776, 32775]
            got = border_interpolate(ps, n, mode)
            want = [cv2.borderInterpolate(int(p), n, mode) for p in ps]
            assert list(got) == want, (mode, n)


def test_border_index_every_position(exe, tmp_path):
    """border_index (the device rule) against the restatement for every position in [-32776, 32775], lengths 1-64 and a
    few large ones, in every mode that indexes the source."""
    pairs = [(n, m) for m in (cv2.BORDER_CONSTANT, cv2.BORDER_REPLICATE, cv2.BORDER_REFLECT, cv2.BORDER_WRAP,
                              cv2.BORDER_REFLECT_101) for n in list(range(1, 65)) + [97, 1080, 1920, 32767, 32768, 70000]]
    (tmp_path / "idx.bin").write_bytes(struct.pack("<i", len(pairs)) + b"".join(struct.pack("<2i", n, m) for n, m in pairs))
    r = subprocess.run([exe, "index", str(tmp_path / "idx.bin"), str(tmp_path / "idx.out")], capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr
    got = np.fromfile(tmp_path / "idx.out", np.int32).reshape(len(pairs), -1)
    ps = np.arange(-32776, 32776)
    for k, (n, m) in enumerate(pairs):
        assert np.array_equal(got[k], border_interpolate(ps, n, m)), (n, m)


def test_cv2_border_premises():
    """What the library refuses and converts, read off cv2: borderMode 0-5 accepted, 6, 7 and REFLECT | BORDER_ISOLATED
    refused; a scalar borderValue is (v, 0, 0, 0); values converted with cvRound half to even and saturation (NaN, inf and
    values beyond int give INT_MIN before saturation), float32 keeps NaN and inf."""
    src = np.zeros((4, 4), np.uint8)
    m1, m2 = np.full((1, 1, 2), -100, np.int16), np.zeros((1, 1), np.uint16)
    for mode in MODES:
        cv2.remap(src, m1, m2, cv2.INTER_LINEAR, borderMode=mode)
    for mode in (6, 7, cv2.BORDER_REFLECT | cv2.BORDER_ISOLATED):
        with pytest.raises(cv2.error):
            cv2.remap(src, m1, m2, cv2.INTER_LINEAR, borderMode=mode)
    px = lambda dt, bv: cv2.remap(np.zeros((4, 4, 4), dt), m1, m2, cv2.INTER_LINEAR, borderValue=bv).ravel().tolist()
    assert px(np.uint8, (300, -2, 7.5, 8.5)) == [255, 0, 8, 8]
    assert px(np.uint8, (np.nan, np.inf, -np.inf, 1e10)) == [0, 0, 0, 0]
    assert px(np.uint16, (70000.4, -1, 2.5, 3.5)) == [65535, 0, 2, 4]
    assert px(np.int16, (np.nan, 1e10, -40000, 32767.5)) == [-32768, -32768, -32768, 32767]
    assert px(np.uint8, 5) == [5, 0, 0, 0]
    f = px(np.float32, (np.nan, np.inf, -np.inf, 1e10))
    assert np.isnan(f[0]) and f[1:] == [np.inf, -np.inf, np.float32(1e10)]
