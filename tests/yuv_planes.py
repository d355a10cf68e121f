"""YUV 4:2:0 frames as a video decoder leaves them: each plane at its own address, rows padded to a pitch, shared by
tests/test_host_yuv_planes.py and tests/test_gpu_yuv_planes.py.  Frames come in cv2's single-buffer layout
(tests/yuv_frames.py) and are laid out in one byte arena; the bytes outside every plane rectangle (row padding, gaps,
whatever lies between planes) hold a poison value that a test can change to show that nothing reads them."""
from dataclasses import dataclass

import cv2
import numpy as np

PITCHES = ("dense", "odd", "pad16", "pow2")   # FW, FW + 1, FW + 16, the next power of two (2048 for 1920 or 1280)
# chroma directly after Y, after 8 / 16 padding rows (1080 + 8 = 1088: a 1080p surface's coded height), before Y in
# memory, in a separate allocation (its own region of the arena), and (I420) U and V in separate allocations
PLACES = ("after", "pad8", "pad16", "before", "separate", "apart")


def pitch_of(kind: str, FW: int) -> int:
    return {"dense": FW, "odd": FW + 1, "pad16": FW + 16, "pow2": max(256, 1 << (FW - 1).bit_length())}[kind]


def chroma_pitch(fmt: str, FW: int, py: int) -> int:
    """The chroma pitch that goes with a Y pitch: the same for NV12; for I420 half of it, rounded up (FFmpeg's linesize)."""
    return py if fmt == "nv12" else FW // 2 + (py - FW + 1) // 2


def split(f: np.ndarray, fmt: str):
    """The planes (Y, UV) or (Y, U, V) of a frame in cv2's single-buffer layout, as 2-D arrays."""
    FH, FW = f.shape[0] * 2 // 3, f.shape[1]
    if fmt == "nv12":
        return [f[:FH], f[FH:]]
    flat, n = f.reshape(-1), (FW // 2) * (FH // 2)
    return [f[:FH], flat[FW * FH:FW * FH + n].reshape(FH // 2, FW // 2), flat[FW * FH + n:].reshape(FH // 2, FW // 2)]


def plane_shapes(fmt: str, FW: int, FH: int):
    return [(FH, FW), (FH // 2, FW)] if fmt == "nv12" else [(FH, FW), (FH // 2, FW // 2), (FH // 2, FW // 2)]


@dataclass
class Surfaces:
    fmt: str
    FW: int
    FH: int
    arena: np.ndarray       # uint8 bytes
    off: np.ndarray         # int64[n][nplanes]: byte offset of plane p of frame i in the arena
    pitch: tuple            # row pitch of each plane
    pad: np.ndarray         # bool[arena]: bytes outside every plane rectangle
    stride: int | None      # common frame stride of every plane (a surface pool), or None (scattered)

    @property
    def n(self):
        return self.off.shape[0]

    def view(self, arena, i, p):
        """Plane p of frame i as a pitched 2-D view of `arena`."""
        h, w = plane_shapes(self.fmt, self.FW, self.FH)[p]
        return np.lib.stride_tricks.as_strided(arena[self.off[i, p]:], (h, w), (self.pitch[p], 1), writeable=False)

    def poisoned(self, value) -> np.ndarray:
        """A copy of the arena whose padding holds `value` (a byte, or an array of the padding's size)."""
        a = self.arena.copy()
        a[self.pad] = value
        return a

    def bgr(self, i, arena=None):
        """cv2's conversion of frame i read from its pitched planes: cvtColorTwoPlane for NV12, cvtColor of the
        reassembled single buffer for I420."""
        a = self.arena if arena is None else arena
        if self.fmt == "nv12":   # the UV plane as cv2 takes it: FW/2 x FH/2 pixels of two channels
            uv = np.lib.stride_tricks.as_strided(a[self.off[i, 1]:], (self.FH // 2, self.FW // 2, 2), (self.pitch[1], 2, 1),
                                                 writeable=False)
            return cv2.cvtColorTwoPlane(self.view(a, i, 0), uv, cv2.COLOR_YUV2BGR_NV12)
        dense = np.concatenate([self.view(a, i, p).reshape(-1) for p in range(3)]).reshape(self.FH * 3 // 2, self.FW)
        return cv2.cvtColor(dense, cv2.COLOR_YUV2BGR_I420)

    def pool(self):
        """(byte offset of frame 0's Y plane, frame stride, plane offsets relative to it) of a surface pool."""
        assert self.stride is not None
        y0 = int(self.off[0, 0])
        return y0, self.stride, [int(o) - y0 for o in self.off[0]] + [0] * (3 - self.off.shape[1])


def build(frames, fmt: str, pitch: str = "dense", place: str = "after", base: int = 0, extra: int = 0,
          scatter: bool = False, fill: int = 0xA5) -> Surfaces:
    """Frames (cv2 layout, uint8[FH*3/2][FW]) laid out as surfaces in one arena starting at byte `base`.  A frame block
    holds the frame's Y plane (and, unless place is "separate" / "apart", its chroma planes); blocks are the block size
    + `extra` bytes apart, in the same order as the frames, or (scatter) shuffled and unevenly spaced, so that
    the frames form no pool.  Chroma in its own region (or regions) sits at the same frame stride as the Y blocks."""
    FH, FW = frames[0].shape[0] * 2 // 3, frames[0].shape[1]
    n, npl = len(frames), (2 if fmt == "nv12" else 3)
    py = pitch_of(pitch, FW)
    pc = chroma_pitch(fmt, FW, py)
    ys, cs = FH * py, (FH // 2) * pc
    chroma = [cs] * (npl - 1)
    if place in ("after", "pad8", "pad16"):
        pad = {"after": 0, "pad8": 8, "pad16": 16}[place] * py
        rel = [0, ys + pad] + ([ys + pad + cs] if npl == 3 else [])
        region, block = [0] * npl, ys + pad + sum(chroma)
    elif place == "before":
        rel = [sum(chroma), 0] + ([cs] if npl == 3 else [])
        region, block = [0] * npl, ys + sum(chroma)
    elif place == "separate":
        rel = [0, 0] + ([cs] if npl == 3 else [])
        region, block = [0, 1, 1][:npl], max(ys, sum(chroma))
    else:   # apart
        rel = [0] * npl
        region, block = [0, 1, 2][:npl], ys
    S = block + extra
    slots = np.arange(n)
    if scatter:
        slots = np.random.default_rng(n * 7 + FW).permutation(n)
        S += 48
    gap = 37
    starts = [base + r * (n * S + gap) for r in range(3)]
    off = np.zeros((n, npl), np.int64)
    for i in range(n):
        step = slots[i] * S + (16 * (slots[i] % 3) if scatter else 0)
        for p in range(npl):
            off[i, p] = starts[region[p]] + step + rel[p]
    pitches = (py, pc, pc)[:npl]
    shapes = plane_shapes(fmt, FW, FH)
    size = int(max(off[i, p] + (shapes[p][0] - 1) * pitches[p] + shapes[p][1] for i in range(n) for p in range(npl))) + 19
    arena = np.full(size, fill, np.uint8)
    pad = np.ones(size, bool)
    for i, f in enumerate(frames):
        for p, pl in enumerate(split(f, fmt)):
            for r in range(pl.shape[0]):
                o = int(off[i, p]) + r * pitches[p]
                arena[o:o + pl.shape[1]] = pl[r]
                assert pad[o:o + pl.shape[1]].all(), "planes overlap"
                pad[o:o + pl.shape[1]] = False
    return Surfaces(fmt, FW, FH, arena, off, pitches + (0,) * (3 - npl), pad, None if scatter else S)


def dense(s: Surfaces, i: int, arena=None) -> np.ndarray:
    """Frame i back in cv2's single-buffer layout."""
    a = s.arena if arena is None else arena
    return np.concatenate([s.view(a, i, p).reshape(-1) for p in range(s.off.shape[1])]).reshape(s.FH * 3 // 2, s.FW)
