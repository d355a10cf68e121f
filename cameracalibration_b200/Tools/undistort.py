"""Batch fisheye undistortion on the GPU -- counterpart of the reference's Tools/undistort.py:25-77.

The undistortion map is built once on the device and never leaves it.  With ``-dstformat jpg`` (the
default) each image costs one upload, one gather kernel and the device JPEG encoder, and only the
compressed stream comes back -- the same bytes cv2.imwrite writes; so does ``-dstformat png`` at
``-quality`` 4 and above (zlib levels 4..9; the default 100 is level 9) through the device PNG encoder.
Other formats, and PNG at levels 0..3, download the image and encode it with cv2 as the reference does.  Decoding the source files stays on the host with cv2.  The
command line accepts the reference's flags with the same defaults; boolean flags additionally understand
0/1/true/false (the reference's ``type=bool`` turns every non-empty string into True), and ``-fused 1``
evaluates the camera model inside the gather kernel instead of keeping a map in HBM; ``-workers N`` sizes
the thread pool that decodes source files and writes finished ones while the GPU calls run.
"""
from __future__ import annotations

import argparse
import os

import numpy as np

from .. import ops

# intrinsics of the reference's sample camera (Tools/undistort.py:28-32), used when -load is off
_SAMPLE_K = (350.4931893001142, 0.0, 647.6297467576265,
             0.0, 352.43072872484805, 513.5196785119657,
             0.0, 0.0, 1.0)
_SAMPLE_D = (-0.03367245449576437, 0.015380779195912842, -0.018654590946883556, 0.0058128945633924185)

_FLAGS = (  # name, default, converter
    ("width", 1280, int), ("height", 1024, int), ("load", True, "flag"),
    ("path_read", "./data/", str), ("path_save", "./", str),
    ("path_k", "./data/camera_0_K.npy", str), ("path_d", "./data/camera_0_D.npy", str),
    ("focalscale", 1, float), ("sizescale", 1, float), ("offset_h", 0, float), ("offset_v", 0, float),
    ("srcformat", "jpg", str), ("dstformat", "jpg", str), ("quality", 100, int), ("name", None, str),
    ("fused", False, "flag"), ("workers", min(8, os.cpu_count() or 1), int),
)


def _as_flag(text) -> bool:
    return str(text).strip().lower() not in ("", "0", "false", "no", "off")


def make_parser() -> argparse.ArgumentParser:
    parser = argparse.ArgumentParser(description="Fisheye camera undistortion of a directory of images (H100)")
    for name, default, conv in _FLAGS:
        parser.add_argument("-" + name, default=default, type=_as_flag if conv == "flag" else conv)
    return parser


def _intrinsics(opts):
    if not opts.load:
        return np.array(_SAMPLE_K).reshape(3, 3), np.array(_SAMPLE_D).reshape(4, 1)
    for path, what in ((opts.path_k, "K"), (opts.path_d, "D")):
        if not os.path.exists(path):
            raise Exception(f"Camera {what} File Path not exist")
    return np.load(opts.path_k), np.load(opts.path_d)


def build_undistorter(opts) -> ops.Undistorter:
    """Destination intrinsics as the reference forms them (:42-46): scaled focal length, optical axis
    centred on the scaled frame plus the optional offsets."""
    K, D = _intrinsics(opts)
    P = np.array(K, np.float64)
    P[0, 0] *= opts.focalscale
    P[1, 1] *= opts.focalscale
    P[0, 2] = opts.width / 2 * opts.sizescale + opts.offset_h
    P[1, 2] = opts.height / 2 * opts.sizescale + opts.offset_v
    size = (int(opts.width * opts.sizescale), int(opts.height * opts.sizescale))
    return ops.Undistorter(K, D, P, size, fused=opts.fused)


def _write_bytes(path, data):
    with open(path, "wb") as f:
        f.write(data)


def _save(cv2, opts, stem_in_save_dir, bare_stem, img):
    if opts.dstformat == "png":
        cv2.imwrite(stem_in_save_dir + ".png", img, [cv2.IMWRITE_PNG_COMPRESSION, opts.quality])
    else:   # the reference writes other formats next to the working directory
        cv2.imwrite(bare_stem + "." + opts.dstformat, img)


def run_directory(opts, undistorter, cv2):
    """Decode -> undistort -> encode over a directory, overlapped: a thread pool decodes the next files
    and writes finished ones (cv2 releases the GIL in imread/imwrite) while the GPU call for the current
    image runs on the calling thread.  For ``-dstformat jpg`` that call is ``undistorter.jpeg`` -- undistort
    and encode on the device, the pool only writes the bytes (likewise ``undistorter.png`` for PNG at levels 4..9);
    other formats are encoded by cv2 in the pool.
    Files are processed and numbered in ``os.listdir`` order exactly as the reference's serial loop does
    (:59-77); at most ``2 * workers`` decoded images are held at a time."""
    from collections import deque
    from concurrent.futures import ThreadPoolExecutor

    suffix = "." + opts.srcformat
    entries = [e for e in os.listdir(opts.path_read) if e[-4:] == suffix]
    workers = max(1, int(opts.workers))
    written, encodes = [], deque()
    device_jpeg = opts.dstformat == "jpg"
    device_png = opts.dstformat == "png" and opts.quality >= 4   # cv2 clamps the level to 9
    with ThreadPoolExecutor(max_workers=workers) as pool:
        decodes, upcoming = deque(), iter(entries)

        def top_up():
            while len(decodes) < 2 * workers:
                entry = next(upcoming, None)
                if entry is None:
                    return
                decodes.append((entry, pool.submit(cv2.imread, os.path.join(opts.path_read, entry))))

        top_up()
        counter = 1
        while decodes:
            entry, pending = decodes.popleft()
            top_up()
            if device_jpeg:
                result = undistorter.jpeg(pending.result(), opts.quality)
            elif device_png:
                result = undistorter.png(pending.result(), [cv2.IMWRITE_PNG_COMPRESSION, opts.quality])
            else:
                result = undistorter(pending.result())
            if opts.name is not None:
                entry = "{}_{:04d}.{}".format(opts.name, counter, opts.srcformat)
                counter += 1
            stem = entry[:-4]
            if device_jpeg or device_png:
                ext = ".jpg" if device_jpeg else ".png"
                encodes.append(pool.submit(_write_bytes, os.path.join(opts.path_save, stem) + ext, result))
            else:
                encodes.append(pool.submit(_save, cv2, opts, os.path.join(opts.path_save, stem), stem, result))
            while len(encodes) > 2 * workers:
                encodes.popleft().result()
            written.append(entry)
        for job in encodes:
            job.result()      # surfaces an encoder exception, as the serial loop would
    return written


def main(argv=None):
    import cv2
    opts = make_parser().parse_args(argv)
    undistorter = build_undistorter(opts)
    for path, message in ((opts.path_read, "Original Image Read Path not exist"),
                          (opts.path_save, "Undistortion Image Save Path not exist")):
        if not os.path.exists(path):
            raise Exception(message)
    return run_directory(opts, undistorter, cv2)


if __name__ == "__main__":
    main()
