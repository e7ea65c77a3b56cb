"""Writes tests/golden/ingest_cases.npz: raw camera frames of every source format and size class, with the gray image
the device must write into the stream's ring block (tests/ingest_ref.py), for the GPU tests, which must not need cv2.

Run from the repository root: python tests/golden/make_ingest.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import ingest_ref as ir  # noqa: E402

# the context's frame is 48 x 32; (source w, h, stream image w, h) per size class, UYVY widths even
CONTEXT = (48, 32)
SIZES = [(48, 32, 48, 32),   # same size: conversion only
         (96, 64, 48, 32),   # exact 2x
         (76, 51, 48, 32),   # downscale
         (20, 13, 48, 32),   # upscale
         (70, 40, 32, 24),   # stream image smaller than the context's
         (58, 41, 33, 27)]   # odd sizes


def main():
    rng = np.random.default_rng(20261016)
    out = {"context": np.array(CONTEXT, np.int32)}
    k = 0
    for fmt in (ir.SRC_GRAY8, ir.SRC_RGB24, ir.SRC_UYVY):
        for sw, sh, dw, dh in SIZES:
            raw = rng.integers(0, 256, (sh, sw * ir.BPP[fmt]), dtype=np.uint8)
            out["case_%d" % k] = np.array([fmt, sw, sh, dw, dh], np.int32)
            out["raw_%d" % k] = raw
            out["gray_%d" % k] = ir.ingest(fmt, raw, sw, sh, dw, dh)
            k += 1
    out["count"] = np.array(k)
    np.savez_compressed(os.path.join(HERE, "ingest_cases.npz"), **out)


if __name__ == "__main__":
    main()
