"""Seeded corpus of the device JPEG encoder (bevk_jpeg_enc.cuh), shared by tests/test_host_jpeg_fuzz.py (the host build
of the per-block stages) and tests/test_gpu_jpeg_fuzz.py (the device pipeline).  One case is a batch of equal-sized BGR
images, a quality and a memory layout; its oracle is cv2.imencode(".jpg", img, [IMWRITE_JPEG_QUALITY, q]) and nothing
else.

The corpus covers:
- geometry: every W % 16 and H % 16 residue (right-edge, bottom-edge and corner dummy blocks, or none), W and H of
  1, 2, 7, 8, 9, 15, 16, 17, and 65500 x 1, 65500 x 17, 1 x 65500, 17 x 65500 (JPEG_MAX_DIMENSION);
- content: noise (long codes, 0xFF-dense streams), smooth gradients (ZRL and EOB runs), flat images (EOB-only blocks),
  1-px checkerboards and 8-px 0/255 steps at q100 (AC category 10, DC category 11);
- quality: spread over 0-100 plus the clamped -5 and 150;
- batches of images of 6, 12, 18, 120, 126 and 132 blocks, n up to 130: the 128-block CTAs of k_jpeg_blocks /
  k_jpeg_dc / k_jpeg_pack start mid-image and mid-MCU; mixed batches of flat and noise images (short streams next to
  long ones);
- layouts: dense, padded rows, padded image stride, a base at byte offset 1-3, a crop of a larger tensor, NumPy input.

Stream classes are read off cv2's own stream (entropy-coded segment between SOS and EOI, unstuffed): last byte 0xFF (a
stuffed pad), a 0xFF at offset 127 mod 128 (the last byte of a stuffing chunk), length 0 mod 128 (whole chunks), one
chunk, more than 1000 chunks, and -- when the last bit is 0, which a 1-bit pad never leaves -- bit counts 0 mod 8 and
0 mod 32 (no partial last word).  The rare ones are found by a seeded search below, so the corpus is fixed."""
from __future__ import annotations

from dataclasses import dataclass
from functools import lru_cache

import cv2
import numpy as np

CHUNK = 128                      # bytes per stuffing chunk (jpeg::kChunk)
CTA_BLOCKS = 128                 # blocks per CTA of the per-block kernels (jpeg::kBlockThreads)
LAYOUTS = ("dense", "pitch", "stride", "offset1", "offset2", "offset3", "view", "numpy")
SMALL_DIMS = (1, 2, 7, 8, 9, 15, 16, 17)
MAX_DIM = 65500
# (W, H) per block count of an image (blocks = 6 * MCUs): 1, 2, 3, 20, 21 and 22 MCUs, two shapes each
BATCH_SIZES = {6: ((16, 16), (13, 11)), 12: ((17, 16), (32, 9)), 18: ((48, 16), (40, 13)), 120: ((80, 64), (65, 50)),
               126: ((112, 48), (100, 33)), 132: ((176, 32), (170, 20))}
BATCH_NS = (1, 2, 7, 11, 22, 23, 43, 64, 127, 130)


@dataclass(eq=False)
class JpegCase:
    name: str
    images: np.ndarray           # uint8[n][H][W][3]
    quality: int
    layout: str
    content: str

    @property
    def n(self) -> int:
        return self.images.shape[0]

    @property
    def W(self) -> int:
        return self.images.shape[2]

    @property
    def H(self) -> int:
        return self.images.shape[1]

    @property
    def nblk(self) -> int:
        return 6 * ((self.W + 15) // 16) * ((self.H + 15) // 16)


# ------------------------------------------------------------------ contents
def noise(rng, h, w):
    return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)


def gradient(rng, h, w):
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    a, b = rng.uniform(0.2, 3, 2)
    return np.stack([xx * a * 255 / max(w, 1), yy * b * 255 / max(h, 1), (xx + yy) * 127 / max(w + h, 1)], -1).clip(0, 255).astype(np.uint8)


def flat(rng, h, w):
    return np.full((h, w, 3), rng.integers(0, 256, 3), np.uint8)


def checker(rng, h, w):
    yy, xx = np.mgrid[0:h, 0:w]
    c = ((yy + xx) & 1).astype(np.uint8) * 255
    return np.stack([c, 255 - c, c], -1)


def steps(rng, h, w):
    yy, xx = np.mgrid[0:h, 0:w]
    c = (((yy >> 3) + (xx >> 3)) & 1).astype(np.uint8) * 255
    return np.stack([c, c, 255 - c], -1)


CONTENTS = {"noise": noise, "gradient": gradient, "flat": flat, "checker": checker, "steps": steps}


# ------------------------------------------------------------------ the oracle and the stream classes
def encode(img, q) -> bytes:
    ok, s = cv2.imencode(".jpg", np.ascontiguousarray(img), [cv2.IMWRITE_JPEG_QUALITY, int(q)])
    assert ok
    return s.tobytes()


def entropy_segment(stream: bytes) -> bytes:
    """The entropy-coded segment of a baseline stream (after the SOS segment, before EOI), unstuffed."""
    p = 2
    while True:
        assert stream[p] == 0xFF, p
        marker, length = stream[p + 1], int.from_bytes(stream[p + 2:p + 4], "big")
        p += 2 + length
        if marker == 0xDA:
            break
    assert stream[-2:] == b"\xff\xd9"
    return stream[p:-2].replace(b"\xff\x00", b"\xff")


def stream_classes(stream: bytes) -> set:
    e = entropy_segment(stream)
    out = set()
    if e[-1] == 0xFF:
        out.add("pad_ff")
    if any(e[i] == 0xFF for i in range(CHUNK - 1, len(e), CHUNK)):
        out.add("ff_at_chunk_end")
    if len(e) % CHUNK == 0:
        out.add("len_0_mod_128")
    if len(e) <= CHUNK:
        out.add("one_chunk")
    if len(e) > 1000 * CHUNK:
        out.add("over_1000_chunks")
    if e[-1] & 1 == 0:                          # the pad is 1 bits: a last bit 0 means no pad
        out.add("bits_0_mod_8")
        if len(e) % 4 == 0:
            out.add("bits_0_mod_32")
    return out


STREAM_CLASSES = ("pad_ff", "ff_at_chunk_end", "len_0_mod_128", "one_chunk", "over_1000_chunks", "bits_0_mod_8",
                  "bits_0_mod_32")


def case_classes(c: JpegCase) -> set:
    """Geometry, batch, quality and layout classes of a case (stream classes: stream_classes of its cv2 streams)."""
    out = {f"w16_{c.W % 16}", f"h16_{c.H % 16}", f"layout_{c.layout}", f"content_{c.content}"}
    for d in SMALL_DIMS + (MAX_DIM,):
        if c.W == d:
            out.add(f"w_{d}")
        if c.H == d:
            out.add(f"h_{d}")
    if c.quality < 0 or c.quality > 100:
        out.add("q_clamped")
    if c.nblk in BATCH_SIZES:
        out.add(f"nblk_{c.nblk}")
    total = c.nblk * c.n
    for k in range(1, (total - 1) // CTA_BLOCKS + 1):
        r = (k * CTA_BLOCKS) % c.nblk
        if r:
            out.add("cta_starts_mid_image")
            if r % 6:
                out.add("cta_starts_mid_mcu")
    if c.n > 1 and c.content == "mixed":
        out.add("mixed_batch")
    if c.n >= 100:
        out.add("n_over_100")
    return out


# ------------------------------------------------------------------ the corpus
def _case(name, rng, W, H, q, layout, content, n=1):
    if content == "mixed":                      # flat and noise images alternate
        imgs = [flat(rng, H, W) if i % 2 else noise(rng, H, W) for i in range(n)]
    else:
        imgs = [CONTENTS[content](rng, H, W) for _ in range(n)]
        if content in ("checker", "steps") and n > 1:
            imgs = [np.roll(im, i, axis=1) for i, im in enumerate(imgs)]
    return JpegCase(name, np.ascontiguousarray(np.stack(imgs)), int(q), layout, content)


def _search(rng, want: str, sizes, qualities, tries: int = 4000) -> JpegCase:
    """The first seeded noise image whose cv2 stream has class `want`."""
    for t in range(tries):
        W, H = sizes[t % len(sizes)]
        q = qualities[t % len(qualities)]
        img = noise(rng, H, W)
        if want in stream_classes(encode(img, q)):
            return JpegCase(f"search_{want}", img[None], int(q), LAYOUTS[t % len(LAYOUTS)], "noise")
    raise AssertionError(f"no seeded image reaches {want}")


@lru_cache(maxsize=None)
def corpus() -> tuple:
    out = []
    rng = np.random.default_rng(4242)
    names = tuple(CONTENTS)
    # every W % 16 and H % 16 residue, on sizes with several MCUs
    for r in range(16):
        W, H = 32 + r, 48 + (7 * r) % 16
        q = int(rng.integers(0, 101))
        out.append(_case(f"res{r}_{W}x{H}", rng, W, H, q, LAYOUTS[r % len(LAYOUTS)], names[r % len(names)], n=1 + r % 3))
    # small dimensions: every pair of W, H in 1, 2, 7, 8, 9, 15, 16, 17
    for i, W in enumerate(SMALL_DIMS):
        for j, H in enumerate(SMALL_DIMS):
            k = i * len(SMALL_DIMS) + j
            q = (-5, 150, 0, 100, 1, 50, 95, 75, 30)[(k // 3) % 9] if k % 3 else int(rng.integers(0, 101))
            out.append(_case(f"small_{W}x{H}", rng, W, H, q, LAYOUTS[k % len(LAYOUTS)], names[k % len(names)], n=1 + k % 4))
    # JPEG_MAX_DIMENSION
    for W, H, content, q in ((MAX_DIM, 1, "noise", 100), (MAX_DIM, 17, "gradient", 90), (1, MAX_DIM, "checker", 100),
                             (17, MAX_DIM, "noise", 60)):
        out.append(_case(f"max_{W}x{H}", rng, W, H, q, "dense", content))
    # largest size categories at q100, and a long noise stream (more than 1000 stuffing chunks)
    for content in ("checker", "steps"):
        out.append(_case(f"{content}_q100", rng, 96, 64, 100, "pitch", content, n=2))
    out.append(_case("noise_320x240_q100", rng, 320, 240, 100, "stride", "noise", n=2))
    out.append(_case("gradient_640x480", rng, 640, 480, 97, "view", "gradient"))
    # batches across 128-block CTA boundaries: images of 6, 12, 18, 120, 126, 132 blocks
    k = 0
    for nblk, shapes in BATCH_SIZES.items():
        for s, (W, H) in enumerate(shapes):
            for n in BATCH_NS[s::2]:
                if nblk >= 120 and n > 64 and s == 0:
                    continue
                content = ("mixed", "noise", "gradient", "flat", "mixed")[k % 5]
                q = (100, 90, 5, 75, 150, 60, 0, 99)[k % 8]
                out.append(_case(f"batch{nblk}_{W}x{H}_n{n}", rng, W, H, q, LAYOUTS[k % len(LAYOUTS)], content, n=n))
                k += 1
    # rare stream classes, by seeded search
    rng = np.random.default_rng(77)
    small = ((16, 16), (24, 16), (17, 9), (33, 31), (40, 24))
    for want, sizes, qualities in (("pad_ff", small, (100, 98, 92)), ("ff_at_chunk_end", ((64, 64),), (100,)),
                                   ("len_0_mod_128", ((48, 40), (56, 48), (64, 32)), (100, 97, 93, 88)),
                                   ("bits_0_mod_32", small, (100, 95, 80)), ("bits_0_mod_8", small, (90, 70))):
        out.append(_search(rng, want, sizes, qualities))
    out.append(_case("flat_8x8", rng, 8, 8, 95, "dense", "flat"))
    return tuple(out)


@lru_cache(maxsize=None)
def streams(name: str) -> tuple:
    """cv2's streams of the case's images."""
    c = case_by_name(name)
    return tuple(encode(img, c.quality) for img in c.images)


def case_by_name(name: str) -> JpegCase:
    return next(c for c in corpus() if c.name == name)
