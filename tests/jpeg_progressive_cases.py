"""Seeded corpus of the progressive JPEG coder (bevk_jpeg_encode_params with IMWRITE_JPEG_PROGRESSIVE), shared by
tests/test_host_jpeg_progressive.py (the host build of the stage functions) and tests/test_gpu_jpeg_progressive.py (the
device pipeline).  The oracle is cv2.imencode(".jpg", img, [IMWRITE_JPEG_QUALITY, q] + params) alone.  It covers:

- all five sampling factors, with every W and H residue modulo the MCU, and 1- and 65500-px sides;
- q1 to q100, noise at q100 (the largest categories), LUMA / CHROMA quality forcing 4:4:4;
- flat images with at least 32,767 blocks in one scan and no restarts (the 0x7FFF flush), and content whose refinement
  scans buffer more than 937 correction bits (the correction-bit flush);
- restart intervals 1, 2, mcux - 1, mcux, mcux + 1, the block-count edges of the single-component scans, more than 8
  intervals per scan, and 65535;
- batches whose 128-block CTAs start mid-image;
- cv2's reading of the flag values: [P, -1], [P, 2], [O, -1, P, 0] and [P, 1, O, 0].
"""
from collections import namedtuple

import numpy as np

from tests.jpeg_params_cases import CTA_BLOCKS, SAMPLINGS, blocks_per_image, image

PROGRESSIVE, OPTIMIZE, RST, LUMA, CHROMA, SAMPLING = 2, 3, 4, 5, 6, 7       # cv2.IMWRITE_JPEG_*
P = [PROGRESSIVE, 1]

Case = namedtuple("Case", "name images quality params classes")


def smooth(rng, w, h):
    """Low-amplitude texture: most blocks have a few small AC coefficients, so refinement scans carry long runs of
    correction bits."""
    yy, xx = np.mgrid[0:h, 0:w]
    base = 128 + 40 * np.sin(xx / 3.0) * np.cos(yy / 4.0)
    img = base[..., None] + rng.normal(0, 6, (h, w, 3))
    return np.clip(img, 0, 255).astype(np.uint8)


def cases(small=False):
    """small: a cut of the corpus for the mutation runs."""
    rng = np.random.default_rng(20261018)
    out = []
    for sf, (hy, vy) in SAMPLINGS.items():
        p = P + [SAMPLING, sf]
        for w in range(1, 8 * hy + 2):
            out.append(Case(f"w{w}-{sf:x}", [image(rng, w, 11, "gradient" if w % 2 else "noise")], 90, p,
                            {f"wres-{sf:x}-{w % (8 * hy)}"}))
        for h in range(1, 8 * vy + 2):
            out.append(Case(f"h{h}-{sf:x}", [image(rng, 13, h, "noise" if h % 2 else "gradient")], 75, p,
                            {f"hres-{sf:x}-{h % (8 * vy)}"}))
        out.append(Case(f"noise100-{sf:x}", [image(rng, 48, 40, "noise")], 100, p, {"q100-noise"}))
        out.append(Case(f"checker-{sf:x}", [image(rng, 40, 24, "checker")], 100, p, {"q100-checker"}))
        # batches: 128-block CTAs start mid-image
        w, h = 40, 24
        nblk = blocks_per_image(w, h, hy, vy)
        n = CTA_BLOCKS // nblk + 5
        out.append(Case(f"batch-{sf:x}", [image(rng, w, h, ("noise", "flat", "gradient")[i % 3]) for i in range(n)], 85, p,
                        {"batch-midimage"}))
        out.append(Case(f"lc-{sf:x}", [image(rng, 37, 29, "gradient")], 95, p + [LUMA, 90, CHROMA, 70], {"forced444"}))
        if small:
            break
    for w, h in ((65500, 1), (1, 65500), (65500, 9)):
        out.append(Case(f"{w}x{h}", [image(rng, w, h, "gradient")], 95, P, {"65500"}))
    out.append(Case("1x1", [image(rng, 1, 1, "noise")], 95, P, {"1px"}))
    for q in (1, 5, 25, 50, 75, 95, 100):
        out.append(Case(f"q{q}", [smooth(rng, 64, 48)], q, P, {f"q{q}"}))
    # 0x7FFF flush: a flat 4:4:4 image with 33,024 blocks per component and no restarts (2048 x 1032 px)
    out.append(Case("flat-eob", [image(rng, 2048, 1032, "flat")], 95, P + [SAMPLING, 0x111111], {"eob-flush"}))
    # correction-bit flush: 1-px checkerboard blocks each leave one correction bit and no symbol in the last luma
    # refinement, so runs pass 937 bits after 938 blocks
    out.append(Case("corr", [image(rng, 256, 256, "checker")], 100, P + [SAMPLING, 0x111111], {"corr-flush"}))
    out.append(Case("smooth", [smooth(rng, 256, 192)], 98, P, {"smooth"}))
    # restart intervals: 4:2:0 image 40 x 24 (mcux 3, 6 MCUs; luma 5 x 3 = 15 blocks, chroma 6 blocks)
    rimg = [image(rng, 40, 24, "noise"), smooth(rng, 40, 24)]
    for r in (1, 2, 3, 4, 5, 6, 7, 14, 15, 16, 65535):
        out.append(Case(f"rst{r}", rimg, 90, P + [RST, r], {f"rst-{r}"}))
    out.append(Case("rst-many", [smooth(rng, 96, 64)], 95, P + [RST, 3], {"rst-wrap"}))
    out.append(Case("rst-444", [image(rng, 45, 37, "noise")], 92, P + [SAMPLING, 0x111111, RST, 7], {"rst-444"}))
    # cv2's value reading
    vimg = [image(rng, 33, 17, "gradient")]
    for name, params in (("p-neg", [PROGRESSIVE, -1]), ("p-2", [PROGRESSIVE, 2]), ("o-neg-p0", [OPTIMIZE, -1, PROGRESSIVE, 0]),
                         ("p1-o0", [PROGRESSIVE, 1, OPTIMIZE, 0]), ("p-opt", [PROGRESSIVE, 1, OPTIMIZE, 1])):
        out.append(Case(name, vimg, 90, params, {f"flags-{name}"}))
    return out


def required_classes():
    req = {"q100-noise", "q100-checker", "batch-midimage", "forced444", "65500", "1px", "eob-flush", "corr-flush", "smooth", "rst-wrap",
           "rst-444"}
    req |= {f"q{q}" for q in (1, 5, 25, 50, 75, 95, 100)} | {f"rst-{r}" for r in (1, 2, 3, 4, 5, 6, 7, 14, 15, 16, 65535)}
    req |= {f"flags-{n}" for n in ("p-neg", "p-2", "o-neg-p0", "p1-o0", "p-opt")}
    for sf, (hy, vy) in SAMPLINGS.items():
        req |= {f"wres-{sf:x}-{r}" for r in range(8 * hy)} | {f"hres-{sf:x}-{r}" for r in range(8 * vy)}
    return req


def params_progressive(params):
    """Whether cv2 4.13 writes a progressive stream for params (its last PROGRESSIVE value > 0)."""
    v = 0
    for k in range(0, len(params), 2):
        if params[k] == PROGRESSIVE:
            v = params[k + 1]
    return v > 0
