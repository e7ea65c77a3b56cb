"""What the patch normals buy: tracking the rendered orbit of tests/warp_scene.py and the slanted plane of
tests/normals_scene.py with the planar patch warp, with and without the normal estimates, in one context (stream 0:
warp only, stream 1: warp and normals).  Numbers measured on an H100 80GB HBM3 at a 700 W power limit are in
DESIGN.md §4."""
import numpy as np
import pytest

import normals_scene
import warp_scene
from test_gpu_warp import scene_ctx

PRM = dict(max_iterations=8, sigma0=0.5, sigma_i=8.0, sigma_step=0.02)


def track(sc, n_true):
    """Per step and stream the fraction of selected features matched and the map size; per step the median angle
    (degrees) between stream 1's estimated normals and the plane's; the final states."""
    ctx = scene_ctx([sc, sc])
    try:
        for s in range(2):
            ctx.set_stream_warp(s, 1)
        ctx.set_stream_normals(1, **PRM)
        T = len(sc.frames) - 1
        frac, nfeat, angle = np.zeros((T, 2)), np.zeros((T, 2), np.int64), np.zeros(T + 1)
        angle[0] = np.median([normals_scene.normal_angle_deg(sc.y[k], sc.xp_org[k], (0.0, 0.0), n_true)
                              for k in range(len(sc.y))])
        for t in range(1, T + 1):
            ctx.set_frames(0, np.stack([sc.frames[t]] * 2))
            ctx.step(0)
            ctx.sync()
            for s in range(2):
                f = ctx.features(s)
                sel = f["select_rank"] >= 0
                frac[t - 1, s] = ((f["flags"] & 2) > 0)[sel].sum() / max(1, sel.sum())
                nfeat[t - 1, s] = ctx.num_features(s)
            m = ctx.num_features(1)
            x, _ = ctx.get_state(1)
            th = ctx.patch_normals(1, np.arange(m))["theta"]
            y = x[13:13 + 3 * m].reshape(m, 3)
            xo = sc.xp_org[:m]  # every feature was first seen from frame 0
            angle[t] = np.median([normals_scene.normal_angle_deg(y[k], xo[k], th[k], n_true) for k in range(m)])
        return frac, nfeat, angle, [ctx.get_state(s)[0] for s in range(2)]
    finally:
        ctx.close()


def report(name, sc, frac, nfeat, angle, states):
    truth = sc.poses[-1]
    out = dict(name=name, min_plain=float(frac[:, 0].min()), min_normals=float(frac[:, 1].min()),
               nfeat_end=nfeat[-1].tolist(), angle_start=float(angle[0]), angle_end=float(angle[-1]))
    for s, x in enumerate(states):
        out["pos_err_%d" % s] = float(np.linalg.norm(x[:3] - truth[:3]))
        out["ang_err_%d" % s] = warp_scene.angle_deg(x[3:7], truth[3:])
    out["short"] = np.nonzero(frac[:, 1] < 0.9)[0].tolist()
    print(out)
    return out


@pytest.mark.gpu
def test_orbit_normals_converge_and_match_at_least_as_often():
    sc = warp_scene.make_warp_scene("orbit")
    n_true = np.array([0.0, 0.0, -1.0])  # the plane z = PLANE_Z, on the cameras' side
    frac, nfeat, angle, states = track(sc, n_true)
    r = report("orbit", sc, frac, nfeat, angle, states)
    # measured: 15.3 -> 0.7 degrees; lowest matched fraction 0.875 against the plain warp's 0.872 (the 0.90 of roll
    # and approach is not reached: steps 35, 36, 39 and 40 fall short)
    assert r["angle_end"] < 2.0 and r["angle_end"] < 0.5 * r["angle_start"], angle
    assert frac[:, 1].min() >= frac[:, 0].min() and frac[:, 1].sum() >= frac[:, 0].sum()
    assert nfeat[-1, 1] >= nfeat[-1, 0]


@pytest.mark.gpu
def test_slanted_plane_normals_keep_tracking():
    sc = normals_scene.make_slanted_scene()
    n_true = normals_scene.plane_normal(normals_scene.TILT)
    frac, nfeat, angle, states = track(sc, n_true)
    r = report("slanted", sc, frac, nfeat, angle, states)
    # measured: 44.5 -> 0.3 degrees; lowest matched fraction 0.84 (0.52 plain), 29 of 32 features kept (21 plain),
    # final pose 6.7 mm / 0.18 degrees off (68 mm / 2.0 degrees plain)
    assert r["angle_end"] < 2.0 and r["angle_end"] < 0.5 * r["angle_start"], angle
    assert r["min_normals"] >= 0.8 and r["pos_err_1"] <= 0.02 and r["ang_err_1"] <= 1.0, r
    assert frac[:, 1].min() >= frac[:, 0].min() and frac[:, 1].sum() >= frac[:, 0].sum()
    assert nfeat[-1, 1] >= nfeat[-1, 0]
