"""CPU checks of relocalisation (sl2_relocalise): the restatement of tests/relocalise_ref.py (P3P, consensus,
hypothesis sequence) and the C ABI layout of its two structs."""
import ctypes as C
import hashlib
import math
import os
import subprocess

import numpy as np
import pytest

import relocalise_ref as rr
import scenelib2_b200.lib as mirror
from model_cases import quat_to_R
from scenelib2_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAMS = {"C1": synth.camera_params(320, 240), "C3": synth.camera_params(640, 480)}  # with their kd1


def random_pose(rng):
    q = rng.standard_normal(4)
    q /= np.linalg.norm(q)
    return rng.uniform(-1.0, 1.0, 3), q if q[0] >= 0 else -q


def pose_error(xp, r, q):
    return max(float(np.abs(np.asarray(xp[:3]) - r).max()), float(np.abs(np.asarray(xp[3:7]) - q).max()))


def test_p3p_recovers_exact_poses():
    """2000 exact configurations per camera: points 0.3-3 m in front of a camera at a random pose, seen at their exact
    (unrounded) projections.  One returned pose is the true one: within 1e-9 except where Kneip's parametrisation is
    singular (theta -> 0, where cos(theta) carries the angle 1 / sin(theta) times less precisely; at most 0.1 % of the
    configurations), and within 1e-7 everywhere."""
    rng = np.random.default_rng(20071014)
    for name, cam8 in CAMS.items():
        errs = []
        for _ in range(2000):
            r, q = random_pose(rng)
            R = quat_to_R(q)
            pix = np.stack([rng.uniform(20, cam8[0] - 20, 3), rng.uniform(20, cam8[1] - 20, 3)], axis=1)
            yw = synth.unproject(cam8, pix, rng.uniform(0.3, 3.0, 3)) @ R.T + r
            z = synth.project(cam8, (yw - r) @ R)
            sols = rr.p3p(yw, rr.unproject(cam8, z))
            assert 1 <= len(sols) <= 4
            errs.append(min(pose_error(s, r, q) for s in sols))
        errs = np.array(errs)
        print("%s: median %.2e, worst %.2e, above 1e-9: %d" % (name, np.median(errs), errs.max(), (errs > 1e-9).sum()))
        assert errs.max() <= 1e-7 and (errs > 1e-9).sum() <= 2, name


def test_p3p_degenerate_triples_give_no_pose():
    cam8 = CAMS["C1"]
    b = rr.unproject(cam8, np.array([[100.0, 80.0], [200.0, 150.0], [160.0, 60.0]]))
    line = np.array([[0.0, 0.0, 1.0], [0.1, 0.2, 1.5], [0.2, 0.4, 2.0]])
    assert rr.p3p(line, b) == []                                     # collinear points
    dup = np.array([[0.0, 0.0, 1.0], [0.0, 0.0, 1.0], [0.3, 0.1, 1.2]])
    assert rr.p3p(dup, b) == []                                      # coincident points
    pts = np.array([[0.0, 0.0, 1.0], [0.3, 0.0, 1.0], [0.0, 0.3, 1.2]])
    assert rr.p3p(pts, b[[0, 0, 2]]) == []                           # the same bearing twice
    assert rr.p3p(pts, np.full((3, 3), np.nan)) == []                # outside the camera model
    out = rr.relocalise(cam8, pts, np.array([[100.0, 80.0], [100.0, 80.0], [160.0, 60.0]]), 2.0, 4)
    assert out["win"] == -1 and np.isnan(out["pose"]).all() and out["status"] == 0


@pytest.mark.parametrize("outliers", [0.0, 0.3, 0.6])
def test_consensus_recovers_the_pose(outliers):
    """40 map points seen at their rounded projections (the search's integer pixels), a fraction replaced by random
    pixels: the winner and the refined pose keep exactly the true matches and the pose is recovered to the rounding."""
    rng = np.random.default_rng(int(outliers * 10) + 7)
    cam8 = CAMS["C1"]
    r, q = random_pose(rng)
    R = quat_to_R(q)
    k = 40
    pix = np.stack([rng.uniform(30, 290, k), rng.uniform(30, 210, k)], axis=1)
    y = synth.unproject(cam8, pix, rng.uniform(0.5, 2.5, k)) @ R.T + r
    z = np.round(synth.project(cam8, (y - r) @ R))
    bad = rng.permutation(k)[:int(round(outliers * k))]
    z[bad] = np.stack([rng.integers(10, 310, bad.size), rng.integers(10, 230, bad.size)], axis=1)
    truth = np.ones(k, bool)
    truth[bad] = False
    truth &= np.sqrt(((z - synth.project(cam8, (y - r) @ R)) ** 2).sum(1)) <= 2.0  # a random pixel may land right
    out = rr.relocalise(cam8, y, z, 2.0, 10)
    assert out["status"] == 1
    assert (out["mask"] == truth).all()
    assert pose_error(out["pose"], r, q) < 5e-3
    assert out["rms"] <= 0.5 * math.sqrt(2.0)


def test_hypothesis_sequence_is_pinned():
    assert rr.splitmix64(0) == 0xE220A8397B1DCDAF  # splitmix64's first output from state 0
    h = hashlib.sha256()
    for k in (3, 4, 7, 50, 100, 256):
        for i in range(rr.HYPOTHESES):
            t = rr.triple(i, k)
            assert len(set(t)) == 3 and all(0 <= v < k for v in t)
            h.update(np.array(t, np.int32).tobytes())
    assert h.hexdigest() == "f8370cc84dd008288f86beec78c67115a07425197a1223382ce90f40bdb02267", h.hexdigest()


def test_reloc_abi_layout(tmp_path):
    """sl2_reloc_params / sl2_reloc_result and the constants as the host C compiler reads include/sl2b200.h."""
    cases = [("sl2_reloc_params", mirror.Sl2RelocParams), ("sl2_reloc_result", mirror.Sl2RelocResult)]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "sl2b200.h"', "int main(void) {",
             '  printf("SL2_RELOC_HYPOTHESES %d\\n", SL2_RELOC_HYPOTHESES);',
             '  printf("SL2_RELOC_GN_ITERS %d\\n", SL2_RELOC_GN_ITERS);']
    for st, M in cases:
        lines.append('  printf("%s.sizeof %%zu\\n", sizeof(%s));' % (st, st))
        lines += ['  printf("%s.%s %%zu %%zu\\n", offsetof(%s, %s), sizeof(((%s *)0)->%s));' % (st, f, st, f, st, f)
                  for f, _ in M._fields_]
    lines += ["  return 0;", "}"]
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines) + "\n")
    subprocess.check_call([os.environ.get("CC", "cc"), "-std=c99", "-I", os.path.join(ROOT, "include"), "-o",
                           str(exe), str(src)])
    out = {ln.split()[0]: tuple(int(v) for v in ln.split()[1:])
           for ln in subprocess.check_output([str(exe)], text=True).splitlines()}
    assert out["SL2_RELOC_HYPOTHESES"] == (mirror.SL2_RELOC_HYPOTHESES,) == (rr.HYPOTHESES,)
    assert out["SL2_RELOC_GN_ITERS"] == (mirror.SL2_RELOC_GN_ITERS,) == (rr.GN_ITERS,)
    for st, M in cases:
        assert out[st + ".sizeof"] == (C.sizeof(M),)
        for f, t in M._fields_:
            assert out[st + "." + f] == (getattr(M, f).offset, C.sizeof(t)), (st, f)
    dt = mirror.RELOC_RESULT_DTYPE
    assert dt.itemsize == C.sizeof(mirror.Sl2RelocResult)
    for f, _ in mirror.Sl2RelocResult._fields_:
        assert out["sl2_reloc_result." + f] == (dt.fields[f][1], dt.fields[f][0].itemsize), f
