"""Seeded corpus for the device PNG encoder (bevk_png_enc.cuh): images and cv2.imwrite PNG parameter lists chosen so
that together they reach every stream class the encoder has to get right (tests/test_host_png.py checks that they do).

Each case is (name, BGR image uint8[H][W][3], params list).  The oracle is cv2.imencode('.png', img, params) alone."""
import cv2
import numpy as np

C, S, F = cv2.IMWRITE_PNG_COMPRESSION, cv2.IMWRITE_PNG_STRATEGY, cv2.IMWRITE_PNG_FILTER
RLE, HUFF = cv2.IMWRITE_PNG_STRATEGY_RLE, cv2.IMWRITE_PNG_STRATEGY_HUFFMAN_ONLY

# Every accepted form of a parameter list (the normaliser test covers the refused ones)
PARAMS = {
    "default": [],
    "rle": [S, RLE],
    "huff": [S, HUFF],
    "rle_l5": [C, 5, S, RLE],
    "huff_l9": [C, 9, S, HUFF],
    "rle_l1": [C, 1, S, RLE],
    "rle_clamp": [C, 12, S, RLE],
    "filter_none": [F, cv2.IMWRITE_PNG_FILTER_NONE],
    "filter_up": [F, cv2.IMWRITE_PNG_FILTER_UP],
    "filter_avg_huff": [S, HUFF, F, cv2.IMWRITE_PNG_FILTER_AVG],
    "filter_paeth": [F, cv2.IMWRITE_PNG_FILTER_PAETH],
    "filter_fast_l3": [C, 3, S, RLE, F, cv2.IMWRITE_PNG_FAST_FILTERS],
    "filter_all": [F, cv2.IMWRITE_PNG_ALL_FILTERS],
    "filter_bad": [F, 24],
    "bilevel0": [cv2.IMWRITE_PNG_BILEVEL, 0],
    "strategy_bad": [S, 7],
}


def _smooth(rng, h, w):
    y, x = np.mgrid[0:h, 0:w]
    a = rng.uniform(0.5, 3.0, 3)
    img = np.stack([(x * a[0] + y * a[1]) / 4, (x * a[2] + 40) / 3, (y * a[0] + x) / 5], -1)
    return (img % 256).astype(np.uint8)


def _noise(rng, h, w):
    return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)


def _flat(rng, h, w):
    return np.full((h, w, 3), rng.integers(0, 256, 3), np.uint8)


def _blocks(rng, h, w):
    """Flat tiles with noisy borders: runs of every length, matches of 3, rows that favour each filter."""
    img = np.zeros((h, w, 3), np.uint8)
    for y0 in range(0, h, 7):
        for x0 in range(0, w, 5):
            img[y0:y0 + 7, x0:x0 + 5] = rng.integers(0, 256, 3)
    mask = rng.random((h, w)) < 0.05
    img[mask] = rng.integers(0, 256, (int(mask.sum()), 3))
    return img


def _stripes(rng, h, w):
    """Rows alternating between horizontal gradients, vertical copies and noise: each adaptive filter wins some row."""
    img = _smooth(rng, h, w)
    for y in range(h):
        k = y % 5
        if k == 1 and y:
            img[y] = img[y - 1]
        elif k == 2:
            img[y] = rng.integers(0, 256, (w, 3))
        elif k == 3 and y:
            img[y] = ((img[y - 1].astype(int) + np.arange(w)[:, None]) % 256).astype(np.uint8)
    return img


def _runs3(rng, h, w):
    """Triples of equal bytes in the SUB-filtered row: runs of exactly 3 and matches of exactly 3."""
    img = np.zeros((h, w, 3), np.uint8)
    img[:, :, :] = (np.arange(w)[None, :, None] // 2 * 37 % 256)
    return img


def cases():
    rng = np.random.default_rng(20261017)
    out = []

    def add(name, img, params):
        out.append((name, np.ascontiguousarray(img), list(params)))

    for pname, params in PARAMS.items():
        add(f"smooth_64x50_{pname}", _smooth(rng, 50, 64), params)
        add(f"stripes_83x61_{pname}", _stripes(rng, 61, 83), params)
    for pname in ("default", "huff", "rle_l5", "filter_all"):
        params = PARAMS[pname]
        add(f"noise_400x300_{pname}", _noise(rng, 300, 400), params)
        add(f"blocks_301x237_{pname}", _blocks(rng, 237, 301), params)
        add(f"flat_640x480_{pname}", _flat(rng, 480, 640), params)
        add(f"smooth_1000x300_{pname}", _smooth(rng, 300, 1000), params)
    # edges of the geometry
    for pname in ("default", "rle_l5", "filter_paeth", "huff"):
        params = PARAMS[pname]
        add(f"1x1_{pname}", _noise(rng, 1, 1), params)
        add(f"w1_{pname}", _noise(rng, 37, 1), params)
        add(f"h1_{pname}", _noise(rng, 1, 53), params)
        add(f"65500x1_{pname}", _smooth(rng, 1, 65500), params)
        add(f"1x65500_{pname}", _smooth(rng, 65500, 1), params)
    add("runs3_90x20", _runs3(rng, 20, 90), [])
    add("runs3_90x20_l5", _runs3(rng, 20, 90), PARAMS["rle_l5"])
    # window-bits thresholds: 14 x 381 is 16383 filtered bytes (reduced window; and exactly one full block of literals
    # under HUFFMAN_ONLY, so an empty final block), 14 x 382 is past the threshold
    for h in (381, 382):
        for pname in ("default", "huff"):
            add(f"noise_14x{h}_{pname}", _noise(rng, h, 14), PARAMS[pname])
    add("noise_13x5_default", _noise(rng, 5, 13), [])
    add("noise_100x100_huff", _noise(rng, 100, 100), PARAMS["huff"])
    # found by a seeded search: an 8195-byte zlib stream, so the Adler-32 trailer starts in one IDAT and ends in the next
    add("adler_split_3x850", np.random.default_rng(3850).integers(0, 256, (850, 3, 3), dtype=np.uint8), [])
    return out


# Stream classes the corpus must reach (bit numbers of tests/host/png_enc.cu)
CLASSES = {0: "stored block", 1: "static block", 2: "dynamic block", 3: "empty final block", 4: "match of 258",
           5: "match of 3", 6: "run of exactly 3", 7: "match across a row boundary", 8: "adaptive NONE",
           9: "adaptive SUB", 10: "adaptive UP", 11: "adaptive AVG", 12: "adaptive PAETH",
           13: "window-reduced zlib header", 14: "more than one IDAT", 15: "Adler-32 split across two IDATs"}
