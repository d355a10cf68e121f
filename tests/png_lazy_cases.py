"""Seeded corpus for the device PNG encoder's hash-chain path (zlib's deflate_slow, levels 4..9 under the DEFAULT,
FILTERED and FIXED strategies; bevk_png_enc.cuh lazy_match / lazy_chain).  Images and cv2.imwrite PNG parameter lists
chosen so that together they reach every class of tests/host/png_lazy.cu (tests/test_host_png_lazy.py checks that they
do).

Each case is (name, BGR image uint8[H][W][3], params list).  The oracle is cv2.imencode('.png', img, params) alone."""
import cv2
import numpy as np

from tests import png_cases as P

C, S, F = cv2.IMWRITE_PNG_COMPRESSION, cv2.IMWRITE_PNG_STRATEGY, cv2.IMWRITE_PNG_FILTER
DEFAULT, FILTERED, FIXED = cv2.IMWRITE_PNG_STRATEGY_DEFAULT, cv2.IMWRITE_PNG_STRATEGY_FILTERED, cv2.IMWRITE_PNG_STRATEGY_FIXED
NONE = cv2.IMWRITE_PNG_FILTER_NONE
MAX_DIST = 32768 - 262   # zlib's MAX_DIST for the full window (images above 16384 filtered bytes)

# Accepted list forms beyond [COMPRESSION, level, STRATEGY, s]
FILTER_LISTS = {
    "l6_none": [C, 6, F, NONE],
    "l9_paeth": [C, 9, F, cv2.IMWRITE_PNG_FILTER_PAETH],
    "l5_filtered_fast": [C, 5, S, FILTERED, F, cv2.IMWRITE_PNG_FAST_FILTERS],
    "sub_then_l7": [F, cv2.IMWRITE_PNG_FILTER_SUB, C, 7],
    "l8_up_fixed": [C, 8, S, FIXED, F, cv2.IMWRITE_PNG_FILTER_UP],
    "l12_clamped": [C, 12],
}


def _planted(rng, h, w, copies):
    """Noise image whose NONE-filtered stream (a 0 filter byte, then the row in RGB order) holds copies of stream bytes:
    copies = [(dst, src, length)] in stream positions; the copies stay inside rows."""
    rb = 3 * w + 1
    f = rng.integers(0, 256, h * rb, dtype=np.uint8)
    f[::rb] = 0
    for dst, src, n in copies:
        assert dst // rb == (dst + n - 1) // rb and dst % rb and src % rb and src // rb == (src + n - 1) // rb
        f[dst:dst + n] = f[src:src + n]
    rgb = f.reshape(h, rb)[:, 1:].reshape(h, w, 3)
    return np.ascontiguousarray(rgb[:, :, ::-1])


def _tail_repeat(rng, h, w):
    """Noise whose last 150 bytes repeat twice earlier (at 1000 and 2000 bytes back): tail matches that reach the end."""
    rb = 3 * w + 1
    n = h * rb
    return _planted(rng, h, w, [(n - 150, n - 150 - 1000, 150), (n - 150 - 1000, n - 150 - 2000, 150)]), n


def _slid_head(w, match_len):
    """The head exactly MAX_DIST back at the window's first slide: a 12-byte copy from 32768 to T = 32768 + MAX_DIST
    (seed 3 leaves no other position of T's hash in between), with a copy of match_len bytes ending at T (none: 0).
    Whether zlib's window slides before T's search depends on the last parse step before T and the last row end below
    65536: with the match, widths 642 (row end 65518) make the head NIL; 1456 (a row ends at 65535) makes it NIL
    whatever the parse; 1000 (row end 63021) leaves the window full and the head searched."""
    rb, t = 3 * w + 1, 32768 + MAX_DIST
    copies = [(t, 32768, 12)] + ([(t - match_len, t - match_len - 2 * rb, match_len)] if match_len else [])
    return _planted(np.random.default_rng(3), 66500 // rb + 2, w, copies)


def cases():
    rng = np.random.default_rng(20261018)
    out = []

    def add(name, img, params):
        out.append((name, np.ascontiguousarray(img), list(params)))

    smooth, stripes, blocks = P._smooth(rng, 50, 64), P._stripes(rng, 61, 83), P._blocks(rng, 237, 301)
    for level in range(4, 10):
        for sname, st in (("default", DEFAULT), ("filtered", FILTERED), ("fixed", FIXED)):
            params = [C, level, S, st]
            add(f"smooth_64x50_l{level}_{sname}", smooth, params)
            add(f"stripes_83x61_l{level}_{sname}", stripes, params)
            add(f"blocks_301x237_l{level}_{sname}", blocks, params)
    for fname, params in FILTER_LISTS.items():
        add(f"stripes_83x61_{fname}", stripes, params)
        add(f"blocks_301x237_{fname}", blocks, params)
    # stored blocks and the 16383-symbol split
    add("noise_100x100_l6", P._noise(rng, 100, 100), [C, 6])
    add("noise_300x200_l9", P._noise(rng, 200, 300), [C, 9])
    # 258-byte matches, long chains of equal bytes
    add("flat_640x480_l9", P._flat(rng, 480, 640), [C, 9])
    add("smooth_1000x300_l6", P._smooth(rng, 300, 1000), [C, 6])
    add("smooth_1000x300_l9", P._smooth(rng, 300, 1000), [C, 9])
    # MAX_DIST: a 10-byte copy exactly MAX_DIST back (the head); a copy 100 back whose chain successor is MAX_DIST back
    # (cut); a 3-byte copy 5000 back (TOO_FAR) and a 4-byte one (Z_FILTERED drops it)
    rb = 3 * 400 + 1
    a0, b0, c0, d0 = 50 * rb + 20, 60 * rb + 30, 70 * rb + 40, 75 * rb + 40
    limits = _planted(rng, 120, 400, [(a0 + MAX_DIST, a0, 10), (b0 + MAX_DIST - 100, b0, 10), (b0 + MAX_DIST, b0, 10),
                                      (c0 + 5000, c0, 3), (d0 + 5000, d0, 4)])
    for level in (4, 6, 9):
        add(f"limits_400x120_l{level}", limits, [C, level, F, NONE])
        add(f"limits_400x120_l{level}_filtered", limits, [C, level, S, FILTERED, F, NONE])
    tail, _ = _tail_repeat(rng, 40, 200)
    for level in (5, 9):
        add(f"tail_200x40_l{level}", tail, [C, level, F, NONE])
    # exactly 16383 symbols ending in a match: 16382 literals (Z_FILTERED keeps noise free of matches) and one 102-byte
    # tail copy, so zlib flushes a full block and Z_FINISH adds an empty final one
    n = 26 * 634
    add("empty_final_211x26_l4", _planted(rng, 26, 211, [(n - 102, n - 102 - 10 * 634, 102)]), [C, 4, S, FILTERED, F, NONE])
    # a final block of exactly 16383 symbols ending in the literal of the last byte, tallied at Z_FINISH without the
    # block-full check: no empty block after it (Z_FILTERED keeps 14 x 381 noise all literals)
    for level in (4, 9):
        add(f"noise_14x381_l{level}_filtered", P._noise(np.random.default_rng(381), 381, 14), [C, level, S, FILTERED])
    # the head at the window slide (k w_size, exactly MAX_DIST back)
    add("slid_head_nil_642_l4", _slid_head(642, 20), [C, 4, F, NONE])
    add("slid_head_nil_642_l9", _slid_head(642, 20), [C, 9, F, NONE])
    add("slid_head_full_1000_l6", _slid_head(1000, 20), [C, 6, F, NONE])
    add("slid_head_full_642_l9", _slid_head(642, 0), [C, 9, F, NONE])
    add("slid_head_rowend_1456_l9", _slid_head(1456, 20), [C, 9, F, NONE])
    # reduced windows, geometry edges
    for level in (4, 9):
        add(f"1x1_l{level}", P._noise(rng, 1, 1), [C, level])
        add(f"w1_l{level}", P._noise(rng, 37, 1), [C, level])
        add(f"h1_l{level}", P._smooth(rng, 1, 53), [C, level])
        add(f"noise_14x381_l{level}", P._noise(rng, 381, 14), [C, level])
    add("runs3_90x20_l7", P._runs3(rng, 20, 90), [C, 7])
    return out


# Stream classes the corpus must reach (bit numbers of tests/host/png_lazy.cu)
CLASSES = {0: "window slide", 1: "reduced window", 2: "more than one block", 3: "empty final block", 4: "stored block",
           5: "match of 258", 6: "nice_match exit", 7: "chain cut at max_chain", 8: "good_match quartering",
           9: "TOO_FAR drop", 10: "Z_FILTERED drop", 11: "head at exactly MAX_DIST",
           12: "chain successor at exactly MAX_DIST", 13: "hash collision", 14: "tail match reaching the end",
           15: "dynamic block with real distance codes", 16: "final 16383-symbol block ending in the last literal",
           17: "static block under Z_FIXED", 18: "slid-window head made NIL by the parse",
           19: "slid-window head searched (window full)", 20: "slid-window head NIL whatever the parse"}
