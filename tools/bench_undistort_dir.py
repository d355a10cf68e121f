#!/usr/bin/env python
"""Tools/undistort.py end to end on a directory (SURVEY 8f-3): images/s of the GPU tool (decode thread pool around the
device call, which undistorts and encodes the JPEG on the GPU; the pool writes the bytes) next to the reference's serial
loop (Tools/undistort.py:59-77: cv2.imread -> cv2.remap -> cv2.imwrite per file, restated in oracle/cv2_path.py terms)
on the same host.  ``files_byte_identical``: every file of the reference loop's sample equals the GPU tool's file byte
for byte.  One JSON line.

    python tools/bench_undistort_dir.py [--files 400] [--workers 16]
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=400)
    ap.add_argument("--workers", type=int, default=16)
    a = ap.parse_args()
    from cameracalibration_b200.Tools import undistort as T
    from oracle import cv2_path as C
    from tests.helpers import Fixtures
    fx = Fixtures()
    src = tempfile.mkdtemp(prefix="bevk_und_src_")
    dst = tempfile.mkdtemp(prefix="bevk_und_dst_")
    ref_dst = tempfile.mkdtemp(prefix="bevk_und_ref_")
    try:
        blob = bytes(fx._jpg["front"])                      # the reference's data/front/front.jpg, 1280x1024
        for i in range(a.files):
            with open(os.path.join(src, f"img_{i:05d}.jpg"), "wb") as f:
                f.write(blob)
        opts = T.make_parser().parse_args(["-load", "0", "-path_read", src + "/", "-path_save", dst + "/", "-workers", str(a.workers)])
        und = T.build_undistorter(opts)
        T.run_directory(T.make_parser().parse_args(["-load", "0", "-path_read", src + "/", "-path_save", dst + "/", "-workers", "2",
                                                    "-name", "warm"]), und, cv2)                      # warm-up (map build, pools)
        t0 = time.perf_counter()
        written = T.run_directory(opts, und, cv2)
        dt = time.perf_counter() - t0
        # the reference's loop on a sample of the files
        K, D = np.array(T._SAMPLE_K).reshape(3, 3), np.array(T._SAMPLE_D).reshape(4, 1)
        P = C.dst_camera_matrix(K, 1280, 1024, 1, 1)
        m1, m2 = C.undistort_maps(K, D, P, 1280, 1024)
        sample = sorted(os.listdir(src))[:max(20, a.files // 10)]
        t1 = time.perf_counter()
        for name in sample:
            img = cv2.imread(os.path.join(src, name))
            out = cv2.remap(img, m1, m2, interpolation=cv2.INTER_LINEAR)
            cv2.imwrite(os.path.join(ref_dst, name), out, [cv2.IMWRITE_JPEG_QUALITY, 100])
        dr = time.perf_counter() - t1
        same = bool((cv2.imread(os.path.join(dst, sample[0])) == cv2.imread(os.path.join(ref_dst, sample[0]))).all())
        identical = all(open(os.path.join(dst, n), "rb").read() == open(os.path.join(ref_dst, n), "rb").read() for n in sample)
        print(json.dumps({"tool": "Tools/undistort.py on a directory of 1280x1024 JPEGs (decode + undistort + encode, quality 100)",
                          "files": len(written), "workers": a.workers, "gpu_tool_images_per_s": len(written) / dt,
                          "reference_loop_images_per_s": len(sample) / dr, "reference_sample": len(sample),
                          "cv2_threads": cv2.getNumThreads(), "os_cpu_count": os.cpu_count(), "outputs_identical": same,
                          "files_byte_identical": identical}))
    finally:
        for d in (src, dst, ref_dst):
            shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
