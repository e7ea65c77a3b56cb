"""Generates tests/golden/c1_trajectory_1000.npz: SURVEY 8(c)(iv), a 1 000-step C1 trajectory (20 features, 10
selected per frame, ellipses from the EKF's own S_i, known patches).  Frames: 32 synthetic frames walked forwards
and backwards, so consecutive frames always differ by one step of the bounded random walk.

    SL2_REFERENCE_SRC=<checkout> python tests/golden/make_c1_trajectory.py   # oracle/_ref is built from it

The fixture is an output of THE REFERENCE'S OWN CODE: monoslam.cpp / kalman.cpp / feature.cpp / models / improc
compiled unmodified against the stand-ins of oracle/stubs_arith (oracle/_ref/libsl2refmodels.so, driven through
MonoSLAM::Init / GoOneStep by oracle/ref_slam_shim.cpp).  The CPU oracle (tests/test_oracle_slam.py) and the CUDA
path (tests/test_gpu_step.py) are tested against it: the hash of every frame's selection ranks / flags / match
positions must be identical, the camera state agrees numerically.  (`python make_c1_trajectory.py --oracle`
regenerates it from the oracle instead; the integer hash is the same.)
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

STEPS, RING, EVERY = 1000, 32, 100


def frame_index(t):
    k = t % (2 * RING - 2)
    return k if k < RING else 2 * RING - 2 - k


def make_slam(oracle, sc, use_ref=False, workdir=None):
    if use_ref:
        import tempfile
        return oracle.RefSlam(sc, workdir or tempfile.mkdtemp(prefix="sl2ref_"))
    from test_oracle_slam import make_oracle_slam
    return make_oracle_slam(oracle, sc)


def run(oracle, use_ref=False, workdir=None):
    from scenelib2_b200 import synth
    kp = np.load(os.path.join(HERE, "known_patches.npy"))
    sc = synth.make_scene("C1", n_frames=RING, known_patches=kp)
    s = make_slam(oracle, sc, use_ref, workdir)
    hz = hashlib.sha256()
    xs, diag, nfeat = [], [], []
    for t in range(STEPS):
        s.step(sc.frames[frame_index(t)])
        f = s.features()
        hz.update(np.ascontiguousarray(f["select_rank"], np.int32).tobytes())
        hz.update(np.ascontiguousarray(f["flags"], np.uint8).tobytes())
        ok = (f["flags"] & 2) > 0
        hz.update(np.ascontiguousarray(f["z"][ok], np.float64).tobytes())
        if (t + 1) % EVERY == 0:
            x, P = s.get_state()
            xs.append(x[:13].copy())
            diag.append(np.diag(P)[:13].copy())
            nfeat.append(s.num_features)
    f = s.features()
    x, P = s.get_state()
    return dict(xv=np.array(xs), Pxx_diag=np.array(diag), nfeat=np.array(nfeat), x_final=x,
                P_diag_final=np.diag(P).copy(), attempted=f["attempted"], successful=f["successful"],
                integer_hash=np.frombuffer(hz.digest(), np.uint8).copy())


if __name__ == "__main__":
    from oracle import pyoracle as po
    po.build()
    use_ref = "--oracle" not in sys.argv
    assert not use_ref or po.ref_models() is not None, "oracle/_ref/libsl2refmodels.so missing: set SL2_REFERENCE_SRC"
    out = run(po, use_ref=use_ref)
    out["source"] = np.array("reference sources + oracle/stubs_arith" if use_ref else "oracle")
    np.savez_compressed(os.path.join(HERE, "c1_trajectory_1000.npz"), **out)
    print("written from", out["source"], "; features left:", out["nfeat"][-1], "successful:", out["successful"].sum())
