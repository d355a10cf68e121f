"""Seeded corpus for the grey and BGRA device encoders (bevk_jpeg_encode_channels, bevk_png_encode_channels,
ops.imencode): image sizes over every MCU edge class, batches with padded pitches, and the cv2 parameter lists each
format takes.  Every case is (name, ext, images uint8[N][H][W][C], params) with params cv2's whole list."""
import cv2
import numpy as np

Q, P, O, R, LQ, CQ, SF = (cv2.IMWRITE_JPEG_QUALITY, cv2.IMWRITE_JPEG_PROGRESSIVE, cv2.IMWRITE_JPEG_OPTIMIZE,
                          cv2.IMWRITE_JPEG_RST_INTERVAL, cv2.IMWRITE_JPEG_LUMA_QUALITY, cv2.IMWRITE_JPEG_CHROMA_QUALITY,
                          cv2.IMWRITE_JPEG_SAMPLING_FACTOR)
PC, PS, PF = cv2.IMWRITE_PNG_COMPRESSION, cv2.IMWRITE_PNG_STRATEGY, cv2.IMWRITE_PNG_FILTER

JPEG_LISTS = {
    "q1": [Q, 1], "q50": [Q, 50], "q95": [], "q100": [Q, 100],
    "luma30": [LQ, 30], "luma30_chroma80": [LQ, 30, CQ, 80], "chroma80": [CQ, 80],
    "sf111": [SF, 0x111111], "sf211": [SF, 0x211111], "sf121": [SF, 0x121111], "sf221": [SF, 0x221111],
    "sf411": [SF, 0x411111],
    "opt": [O, 1], "rst1": [R, 1], "rst3": [R, 3], "rst65535": [R, 65535], "opt_rst3": [O, 1, R, 3],
    "prog": [P, 1], "prog_rst3": [P, 1, R, 3], "prog_opt": [P, 1, O, 1], "prog_rst1_q50": [P, 1, R, 1, Q, 50],
}
PNG_LISTS = {
    "default": [], "rle": [PS, cv2.IMWRITE_PNG_STRATEGY_RLE], "huff": [PS, cv2.IMWRITE_PNG_STRATEGY_HUFFMAN_ONLY],
    "f_none": [PF, 8], "f_sub": [PF, 16], "f_up": [PF, 32], "f_avg": [PF, 64], "f_paeth": [PF, 128],
    "f_fast": [PF, 56], "f_all": [PF, 248], "f_all_rle_l5": [PC, 5, PS, 3, PF, 248],
    "l4": [PC, 4], "l6": [PC, 6], "l9": [PC, 9],
    "l4_filtered": [PC, 4, PS, cv2.IMWRITE_PNG_STRATEGY_FILTERED], "l6_filtered": [PC, 6, PS, 1],
    "l9_filtered": [PC, 9, PS, 1], "l4_fixed": [PC, 4, PS, cv2.IMWRITE_PNG_STRATEGY_FIXED], "l6_fixed": [PC, 6, PS, 4],
    "l9_fixed": [PC, 9, PS, 4],
}


def image(rng, h, w, c, kind="smooth"):
    """A uint8[h][w][c] image: smooth gradients with noise (compressible) or uniform noise."""
    if kind == "noise":
        return rng.integers(0, 256, (h, w, c), dtype=np.uint8)
    y, x = np.mgrid[0:h, 0:w]
    base = np.stack([(x * (3 + k) + y * (5 - k) + 40 * k) % 256 for k in range(c)], -1).astype(np.int32)
    return np.clip(base + rng.integers(-6, 7, (h, w, c)), 0, 255).astype(np.uint8)


def grey_sizes():
    """Every W % 8 and H % 8 class, 1-pixel sides and one 65500-pixel side."""
    s = [(8 + a, 8 + b) for a in range(8) for b in range(8)]
    return s + [(1, 1), (1, 9), (13, 1), (65500, 2), (3, 65500)]


def bgra_sizes():
    """Every W % 16 and H % 16 class (the MCU edges of 4:2:0 and 4:1:1), and 1-pixel sides."""
    return [(16 + a, 16 + (a * 7 + 3) % 16) for a in range(16)] + [(16 + (b * 5) % 16, 16 + b) for b in range(16)] + \
        [(1, 1), (1, 17), (33, 1)]


def plant(img, offsets, pattern):
    """Write pattern at these offsets of img's filtered stream under FILTER NONE (rows of C*W + 1 bytes, each led by its
    filter byte; BGRA stored as RGBA)."""
    h, w, c = img.shape
    rb = c * w + 1
    flat = img.reshape(h, w * c)
    for off in offsets:
        y, col = divmod(off, rb)
        assert 1 <= col and col + len(pattern) <= rb, (off, rb)
        for k, v in enumerate(pattern):
            i = col - 1 + k
            flat[y, i if c != 4 or i & 1 else i ^ 2] = v
    return img


def window_cases(seed=77):
    """Hash-chain PNGs past one 32 KiB window: noise with one 4-byte string at filtered offsets 32768 and 65274, so the
    search at 65274 meets the head at w_size exactly MAX_DIST (32506) back.  Whether zlib searches it depends on the row
    length (C*W + 1) through the window slide, so grey and BGRA images whose rows are not 3W + 1 long pin it: with rows
    of 301 bytes (grey 300 wide, BGRA 75 wide) the head is searched, with rows of 257 a row ends at 2 w_size - 1 and the
    head is NIL."""
    rng = np.random.default_rng(seed)
    out = []
    for c, w, h in ((1, 300, 250), (4, 75, 250), (1, 256, 300), (4, 64, 300)):
        for k in range(4):
            # background bytes below 16 and a string led by a byte with bit 4 set: zlib's 15-bit hash of the string's
            # first 3 bytes then occurs only at the two planted offsets, so the chain at 65274 leads to 32768
            pattern = [0x90 | int(rng.integers(0, 16)), *rng.integers(16, 256, 3)]
            img = plant(rng.integers(0, 16 if k < 3 else 256, (h, w, c), dtype=np.uint8), (32768, 65274), pattern)
            for name, p in (("l9_none", [PC, 9, PF, 8]), ("l6_none", [PC, 6, PF, 8]), ("l9_filtered_none", [PC, 9, PS, 1, PF, 8])):
                out.append((f"window_{'grey' if c == 1 else 'bgra'}_{w}x{h}_{k}_{name}", ".png", img[None], p))
    return out


def cases(seed=2026):
    rng = np.random.default_rng(seed)
    out = []
    # every size class, one list each in rotation (cheap sizes get the full sweep below)
    jl, pl = list(JPEG_LISTS.items()), list(PNG_LISTS.items())
    for k, (w, h) in enumerate(grey_sizes()):
        big = max(w, h) > 1000
        img = image(rng, h, w, 1, "noise" if k % 3 == 0 else "smooth")[None]
        name, p = jl[k % len(jl)] if not big else ("q95", [])
        out.append((f"grey_{w}x{h}_{name}", ".jpg", img, p))
        name, p = pl[k % len(pl)] if not big else ("default", [])
        out.append((f"grey_{w}x{h}_{name}", ".png", img, p))
    for k, (w, h) in enumerate(bgra_sizes()):
        img = image(rng, h, w, 4, "noise" if k % 3 == 0 else "smooth")[None]
        name, p = jl[(k * 5) % len(jl)]
        out.append((f"bgra_{w}x{h}_{name}", ".jpg", img, p))
        name, p = pl[(k * 3) % len(pl)]
        out.append((f"bgra_{w}x{h}_{name}", ".png", img, p))
    # every list on one grey and one BGRA image of awkward size
    for c, (w, h) in ((1, (61, 45)), (4, (53, 38))):
        img = image(rng, h, w, c)[None]
        for name, p in JPEG_LISTS.items():
            out.append((f"{'grey' if c == 1 else 'bgra'}_{w}x{h}_{name}", ".jpg", img, p))
        for name, p in PNG_LISTS.items():
            out.append((f"{'grey' if c == 1 else 'bgra'}_{w}x{h}_{name}", ".png", img, p))
    # batches
    for c in (1, 4):
        imgs = np.stack([image(rng, 29, 70, c, kind) for kind in ("smooth", "noise", "smooth")])
        who = "grey" if c == 1 else "bgra"
        for name in ("q95", "opt_rst3", "prog", "prog_rst3"):
            out.append((f"batch3_{who}_{name}", ".jpg", imgs, JPEG_LISTS[name]))
        for name in ("default", "huff", "l6"):
            out.append((f"batch3_{who}_{name}", ".png", imgs, PNG_LISTS[name]))
    return out + window_cases()


def padded(images, row_pad, image_pad):
    """A view of images [N][H][W][C] whose rows are row_pad bytes and images image_pad bytes longer than dense."""
    n, h, w, c = images.shape
    row = w * c + row_pad
    img = h * row + image_pad
    buf = np.full(n * img + 64, 0xA5, np.uint8)
    view = np.lib.stride_tricks.as_strided(buf, (n, h, w, c), (img, row, c, 1))
    view[...] = images
    return buf, view


def cv2_streams(ext, images, params):
    """cv2.imencode of every image of [N][H][W][C] (grey as [H][W])."""
    res = []
    for im in images:
        ok, buf = cv2.imencode(ext, im[..., 0] if im.shape[-1] == 1 else im, list(params))
        assert ok
        res.append(buf.tobytes())
    return res
