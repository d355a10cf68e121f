"""Seeded corpus of the device JPEG encoder under cv2.imwrite's JPEG parameters (bevk_jpeg_set_params), shared by
tests/test_host_jpeg_params.py (the host build of the stage functions) and tests/test_gpu_jpeg_params.py (the device
pipeline).  The oracle is cv2.imencode(".jpg", img, [IMWRITE_JPEG_QUALITY, q] + params) alone.  It covers:

- every sampling factor cv2 writes (4:4:4, 4:2:2, 4:4:0, 4:2:0, 4:1:1): every W and H residue modulo the MCU size
  (sides 1-17 and 33, and 18-32 for 4:1:1's 32-px MCU), and 65500-px sides;
- the quality rules: LUMA_QUALITY replacing QUALITY, CHROMA_QUALITY with and without LUMA_QUALITY, in either order,
  out-of-range values, luma != chroma forcing 4:4:4 under every SAMPLING_FACTOR, unknown sampling values, and the
  default-valued keys (PROGRESSIVE 0, OPTIMIZE 0, RST_INTERVAL 0 / -1);
- noise, gradients, flat images and 1-px checkerboards at q100 (largest categories);
- batches of 3-, 4- and 6-block-per-MCU images whose 128-block CTAs start mid-image (and mid-MCU for 3 and 6 blocks);
- restart intervals 0, 1, 2, 3, mcux - 1, mcux, mcux + 1, total MCUs - 1 / + 0 / + 1, 65535, -1 and 65536 (clamped),
  more than 8 intervals (marker wrap); across the corpus every pad length 0-7 and an interval whose data ends in 0xFF
  (tests/test_host_jpeg_params.py reads both off the streams);
- optimised tables on flat images (one or two symbols per table), noise (every AC symbol), checkerboards (largest
  categories) and batches whose images each get their own tables; optimise x restart x every sampling factor.
"""
from collections import namedtuple

import numpy as np

PROGRESSIVE, OPTIMIZE, RST, LUMA, CHROMA, SAMPLING = 2, 3, 4, 5, 6, 7       # cv2.IMWRITE_JPEG_*
SAMPLINGS = {0x111111: (1, 1), 0x211111: (2, 1), 0x121111: (1, 2), 0x221111: (2, 2), 0x411111: (4, 1)}
CTA_BLOCKS = 128                                                              # jpeg::kBlockThreads

Case = namedtuple("Case", "name images quality params classes")


def image(rng, w, h, kind):
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == "flat":
        return np.full((h, w, 3), rng.integers(0, 256, 3, dtype=np.uint8), np.uint8)
    if kind == "checker":
        yy, xx = np.mgrid[0:h, 0:w]
        c = (((yy + xx) & 1) * 255).astype(np.uint8)
        return np.ascontiguousarray(np.stack([c, 255 - c, (((yy >> 3) + (xx >> 3)) & 1) * 255], -1).astype(np.uint8))
    yy, xx = np.mgrid[0:h, 0:w]                                              # gradient with colour edges
    g = np.stack([(xx * 7 + yy * 3) & 255, (xx * 2 + 5 * yy) & 255, ((xx // 5 + yy // 3) & 1) * 200 + 20], -1)
    return g.astype(np.uint8)


def blocks_per_image(w, h, hy, vy):
    return -(-w // (8 * hy)) * -(-h // (8 * vy)) * (hy * vy + 2)


def cases():
    rng = np.random.default_rng(20261017)
    out = []
    for sf, (hy, vy) in SAMPLINGS.items():
        p = [SAMPLING, sf]
        sides = list(range(1, 18)) + [33] + (list(range(18, 33)) if hy == 4 else [])
        for w in sides:
            out.append(Case(f"w{w}-{sf:x}", [image(rng, w, 13, "gradient" if w % 2 else "noise")], 90, p,
                            {f"wres-{sf:x}-{w % (8 * hy)}", f"hres-{sf:x}-{13 % (8 * vy)}"}))
        for h in range(1, 18):
            out.append(Case(f"h{h}-{sf:x}", [image(rng, 11, h, "noise" if h % 2 else "gradient")], 75, p,
                            {f"hres-{sf:x}-{h % (8 * vy)}", f"wres-{sf:x}-{11 % (8 * hy)}"}))
        for w, h in ((65500, 1), (1, 65500), (65500, 9), (9, 65500)):
            out.append(Case(f"{w}x{h}-{sf:x}", [image(rng, w, h, "gradient")], 95, p, {f"65500-{sf:x}"}))
        for kind in ("flat", "checker"):
            out.append(Case(f"{kind}-{sf:x}", [image(rng, 48, 40, kind)], 100, p, {f"{kind}-{sf:x}"}))
        # luma != chroma forces 4:4:4 under every sampling factor, in either order of the pairs
        img = image(rng, 37, 29, "gradient")
        out.append(Case(f"lc-{sf:x}", [img], 95, p + [LUMA, 90, CHROMA, 70], {f"forced444-{sf:x}"}))
        out.append(Case(f"cl-{sf:x}", [img], 95, [CHROMA, 70] + p + [LUMA, 90], {f"forced444-{sf:x}"}))
        out.append(Case(f"ll-{sf:x}", [img], 95, [LUMA, 85, CHROMA, 85] + p, {f"equal-lc-{sf:x}"}))
        # batches: 128-block CTAs start mid-image (and mid-MCU unless 128 % blocks-per-MCU == 0)
        w, h = {1: (24, 24), 2: (40, 8)}.get(hy * vy, (40, 24))
        if hy * vy == 2 and vy == 2:
            w, h = (8, 48)
        nblk = blocks_per_image(w, h, hy, vy)
        n = CTA_BLOCKS // nblk + 7
        imgs = [image(rng, w, h, ("noise", "flat", "gradient")[i % 3]) for i in range(n)]
        starts = {(c * CTA_BLOCKS) % nblk for c in range(1, n * nblk // CTA_BLOCKS + 1)}
        bpm = hy * vy + 2
        cls = {f"batch-bpm{bpm}"} | ({f"batch-midmcu-bpm{bpm}"} if any(s % bpm for s in starts) else set())
        out.append(Case(f"batch-{sf:x}", imgs, 85, p, cls | ({"batch-midimage"} if any(starts) else set())))
    img = image(rng, 53, 41, "gradient")
    rules = [
        ("default", 95, [], "default"),
        ("luma-replaces", 50, [LUMA, 80], "luma-replaces"),
        ("luma-over", 50, [LUMA, 150], "luma-out-of-range"),
        ("luma-neg", 50, [LUMA, -3], "luma-ignored"),
        ("luma-zero", 50, [LUMA, 0], "luma-zero"),
        ("chroma-alone", 50, [CHROMA, 80], "chroma-ignored"),
        ("chroma-neg", 50, [LUMA, 60, CHROMA, -1], "chroma-ignored"),
        ("chroma-over", 50, [LUMA, 70, CHROMA, 150], "chroma-out-of-range"),
        ("both-100", 50, [LUMA, 100, CHROMA, 120], "equal-after-clamp"),
        ("luma0-chroma1", 50, [LUMA, 0, CHROMA, 1], "differ-same-table"),
        ("luma-replaces-low", 30, [LUMA, 60], "luma-replaces"),
        ("q-neg", -5, [SAMPLING, 0x111111], "quality-out-of-range"),
        ("q-zero", 0, [SAMPLING, 0x211111], "quality-out-of-range"),
        ("q-over", 150, [SAMPLING, 0x121111], "quality-out-of-range"),
        ("sf-bad", 90, [SAMPLING, 0x222222], "sampling-fallback"),
        ("sf-zero", 90, [SAMPLING, 0], "sampling-fallback"),
        ("sf-neg", 90, [SAMPLING, -1], "sampling-fallback"),
        ("sf-twice", 90, [SAMPLING, 0x111111, SAMPLING, 0x411111], "sampling-last-wins"),
        ("defaults", 90, [PROGRESSIVE, 0, OPTIMIZE, 0, RST, 0, RST, -1], "default-valued-keys"),
    ]
    for name, q, params, cls in rules:
        out.append(Case(name, [img], q, params, {cls}))
    for sf in SAMPLINGS:                                                     # noise at q100 under the largest bound
        out.append(Case(f"noise100-{sf:x}", [image(rng, 64, 48, "noise")], 100, [SAMPLING, sf], {f"noise100-{sf:x}"}))
    # restart intervals on a 4:2:0 image of 4 x 3 MCUs
    rimg = [image(rng, 53, 41, "noise"), image(rng, 53, 41, "gradient")]
    mcux, total = 4, 12
    for r in (0, 1, 2, 3, mcux - 1, mcux, mcux + 1, total - 1, total, total + 1, 65535, -1, 65536):
        out.append(Case(f"rst{r}", rimg, 90, [RST, r], {f"rst-{r}"} | ({"marker-wrap"} if 0 < r and -(-total // r) > 8 else set())))
    for k in range(6):                                                       # many intervals: pad lengths, 0xFF ends
        out.append(Case(f"rst-noise{k}", [image(rng, 96, 64, "noise")], (100, 95, 90, 80, 60, 30)[k], [RST, 1 + k % 2],
                        {"rst-many"}))
    # optimised tables
    for kind in ("flat", "noise", "checker", "gradient"):
        out.append(Case(f"opt-{kind}", [image(rng, 48, 40, kind)], 100 if kind != "gradient" else 75, [OPTIMIZE, 1],
                        {f"opt-{kind}"}))
    out.append(Case("opt-flat-tiny", [image(rng, 8, 8, "flat")], 50, [OPTIMIZE, 7], {"opt-flat"}))
    w, h = 40, 24                                                            # 36 blocks: CTAs start mid-image
    out.append(Case("opt-batch", [image(rng, w, h, ("noise", "flat", "checker", "gradient")[i % 4]) for i in range(13)], 90,
                    [OPTIMIZE, 1], {"opt-batch"}))
    for sf in SAMPLINGS:                                                     # optimise x restart x sampling
        imgs = [image(rng, 45, 37, "noise"), image(rng, 45, 37, "gradient"), image(rng, 45, 37, "flat")]
        for r in (0, 1, 3):
            out.append(Case(f"opt-rst{r}-{sf:x}", imgs, 92, [SAMPLING, sf, OPTIMIZE, 1, RST, r], {f"opt-rst{r}-{sf:x}"}))
    out.append(Case("opt-rst1-444-q100", [image(rng, 64, 48, "noise")], 100, [SAMPLING, 0x111111, OPTIMIZE, 1, RST, 1],
                    {"opt-rst-bound"}))
    out.append(Case("opt-lc", [image(rng, 37, 29, "gradient")], 95, [LUMA, 90, CHROMA, 60, OPTIMIZE, 1, RST, 2],
                    {"opt-lc"}))
    return out


def required_classes():
    req = {"default", "luma-replaces", "luma-out-of-range", "luma-ignored", "luma-zero", "chroma-ignored",
           "chroma-out-of-range", "equal-after-clamp", "differ-same-table", "quality-out-of-range", "sampling-fallback",
           "sampling-last-wins", "default-valued-keys", "batch-midimage", "batch-midmcu-bpm3", "batch-midmcu-bpm6",
           "batch-bpm4", "marker-wrap", "rst-many", "opt-flat", "opt-noise", "opt-checker", "opt-gradient", "opt-batch",
           "opt-rst-bound", "opt-lc"}
    req |= {f"rst-{r}" for r in (0, 1, 2, 3, 4, 5, 11, 12, 13, 65535, -1, 65536)}
    for sf, (hy, vy) in SAMPLINGS.items():
        req |= {f"wres-{sf:x}-{r}" for r in range(8 * hy)} | {f"hres-{sf:x}-{r}" for r in range(8 * vy)}
        req |= {f"65500-{sf:x}", f"flat-{sf:x}", f"checker-{sf:x}", f"forced444-{sf:x}", f"equal-lc-{sf:x}",
                f"noise100-{sf:x}"} | {f"opt-rst{r}-{sf:x}" for r in (0, 1, 3)}
    return req
