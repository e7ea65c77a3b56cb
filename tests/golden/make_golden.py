"""Generates tests/golden/*.npz from the original SceneLib2 sources:

    SL2_REFERENCE_SRC=<checkout> python tests/golden/make_golden.py
    SL2_REFERENCE_SRC=<checkout> SL2_RECORD_REFERENCE=1 python -m pytest tests -k reference   # ref_*.npz

* known_patches.npy  : the four 11x11 templates shipped as data/known_patch{0..3}.pgm
                       (input fixtures of BASELINE config C1).
* a1_ref_kat.npz     : correlate2_warning known-answer vectors produced by the REFERENCE's own
                       improc.cpp (oracle/_ref/libsl2ref.so), incl. sigma = 0 branches.
* a11_ref_kat.npz    : SearchMultipleOverlappingEllipses::search known answers from the
                       REFERENCE's own source, incl. border-clamped and overlapping ellipses.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import pyoracle as po  # noqa: E402
from scenelib2_b200 import synth  # noqa: E402


def read_pgm(path):
    with open(path, "rb") as f:
        data = f.read()
    toks, pos = [], 0
    while len(toks) < 4:
        while data[pos:pos + 1].isspace():
            pos += 1
        if data[pos:pos + 1] == b"#":
            while data[pos:pos + 1] != b"\n":
                pos += 1
            continue
        s = pos
        while not data[pos:pos + 1].isspace():
            pos += 1
        toks.append(data[s:pos])
    assert toks[0] == b"P5"
    w, h = int(toks[1]), int(toks[2])
    return np.frombuffer(data[pos + 1:pos + 1 + w * h], np.uint8).reshape(h, w).copy()


def main():
    po.build(force=True)
    assert po.ref() is not None, "oracle/_ref not built: set SL2_REFERENCE_SRC"
    kp = np.stack([read_pgm(os.path.join(os.environ["SL2_REFERENCE_SRC"], "data", "known_patch%d.pgm" % i))
                   for i in range(4)])
    np.save(os.path.join(HERE, "known_patches.npy"), kp)

    rng = np.random.default_rng(20260923)
    # ---- A1 KATs --------------------------------------------------------------------------
    cases = []
    for B in (11, 15):
        img = synth.make_texture(rng, 64, 80)
        for k in range(24):
            patch = rng.integers(0, 256, (B, B), dtype=np.uint8)
            if k % 6 == 1:
                patch[:] = 255                       # sigma0 = 0, max intensity
            if k % 6 == 2:
                patch = img[10:10 + B, 20:20 + B].copy()  # exact match -> 0
            im = img.copy()
            x1, y1 = int(rng.integers(0, 80 - B)), int(rng.integers(0, 64 - B))
            if k % 6 == 3:
                im[y1:y1 + B, x1:x1 + B] = 7         # sigma1 = 0
            if k % 6 == 4:
                im[:] = 255
                patch[:] = 255                       # both sigma 0, overflow check of sums
            if k % 6 == 2:
                x1, y1 = 20, 10
            c, s0, s1 = po.correlate2_warning(patch, im, x1, y1, use_ref=True)
            cases.append((B, patch, im, x1, y1, c, s0, s1))
    np.savez_compressed(
        os.path.join(HERE, "a1_ref_kat.npz"),
        B=np.array([c[0] for c in cases]),
        patch=np.array([np.pad(c[1], ((0, 15 - c[0]), (0, 15 - c[0]))) for c in cases]),
        image=np.array([c[2] for c in cases]),
        xy=np.array([[c[3], c[4]] for c in cases]),
        out=np.array([[c[5], c[6], c[7]] for c in cases]))

    # ---- A11 KATs -------------------------------------------------------------------------
    img = synth.make_texture(rng, 120, 160)
    img[40:70, 50:90] = 128                          # flat plateau: ties + low sigma penalty
    B = 11
    patch = img[80:91, 100:111].copy()
    K = 12
    centres = np.array([[105.3, 85.2], [103.9, 86.7], [108.0, 84.0], [3.2, 4.1], [157.5, 117.9],
                        [70.5, 55.5], [60.0, 50.0], [105.5, 85.5], [20.0, 100.0], [100.0, 10.0],
                        [140.2, 60.6], [105.0, 85.0]])
    pu = []
    for k in range(K):
        a, b = rng.uniform(3, 14), rng.uniform(3, 14)
        th = rng.uniform(0, np.pi)
        R = np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]])
        S = R @ np.diag([a * a / 9, b * b / 9]) @ R.T
        Si = np.linalg.inv(S)
        pu.append([Si[0, 0], Si[0, 1], Si[1, 1]])
    pu = np.array(pu)
    ru, rv, rf, _ = po.smoe_search(img, patch, pu, centres, use_ref=True)
    np.savez_compressed(os.path.join(HERE, "a11_ref_kat.npz"), image=img, patch=patch,
                        centres=centres, puinv3=pu, res_u=ru, res_v=rv, res_flag=rf)
    print("golden vectors written")


if __name__ == "__main__":
    main()
