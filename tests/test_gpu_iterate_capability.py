"""What the iterated update buys on a rendered lateral translation (tests/warp_scene.py's renderer): a band-limited
texture on a plane 2 m in front of a 320 x 240 camera that translates 0.3 m sideways over 30 steps.  The map holds 40
settled features (1 mm sigma, as the warp scenes) and 8 appended ones whose covariance is shaped like a converted
depth ray: depth sigma 40 % along the ray through their template's centre, 1 % across it, cross terms to the camera
position as a converted ray has them; each estimate is off its true depth by one sigma.  Four streams of one context
track it: the iteration off and on (N = 3, tol = 1e-3), with the consensus off, and both again with the consensus and
the rescue on.  Reported: the appended features' mean depth error at the end and the mean camera position NEES over
the run.  The numbers are recorded in DESIGN.md section 3."""
import numpy as np
import pytest

import warp_scene
from scenelib2_b200 import synth
from test_gpu_warp import scene_ctx

STEPS = 30
NEW = 8
DEPTH_SIGMA = 0.4
NEES_RATIO_MAX = 0.6  # measured 0.43


def lateral_scene(seed=0, n_settled=40, margin=70):
    rng = np.random.default_rng(0x17E4 + seed)
    cam8 = warp_scene.CAM.copy()
    B, half = 11, 5
    tex = warp_scene.make_texture(rng, 4.0)
    t = np.arange(STEPS + 1) * warp_scene.DT
    vx = 0.3 / (STEPS * warp_scene.DT)
    w = np.radians(0.5) / (STEPS * warp_scene.DT)  # a little roll: the motion model's Jacobian needs |omega| > 0
    poses = np.zeros((STEPS + 1, 7))
    poses[:, 0] = vx * t
    for k, tk in enumerate(t):
        poses[k, 3:] = warp_scene.quat_axis([0, 0, 1], w * tk)
    frames = np.stack([warp_scene.render(cam8, p, tex, rng) for p in poses])
    N = n_settled + NEW
    pix = synth._feature_pixels(rng, int(cam8[0]), int(cam8[1]), N, margin)
    d = warp_scene.rays(cam8, poses[0])[pix[:, 1], pix[:, 0]]
    depth = (warp_scene.PLANE_Z - poses[0, 2]) / d[:, 2]
    y_true = poses[0, :3] + depth[:, None] * d
    patches = np.stack([frames[0][py - half:py + half + 1, px - half:px + half + 1] for px, py in pix])
    y = y_true.copy()
    x0 = np.concatenate([poses[0], [vx, 0.0, 0.0], [0.0, 0.0, w], y.ravel()])
    n = x0.size
    sd = np.concatenate([np.full(3, 1e-3), np.full(4, 1e-3), np.full(3, 1e-2), np.full(3, 1e-2), np.full(n - 13, 1e-3)])
    P0 = np.diag(sd * sd)
    for i in range(n_settled, N):  # converted depth rays: y = r + depth ray, depth off by one sigma
        p = 13 + 3 * i
        ray = d[i] / np.linalg.norm(d[i])
        dist = np.linalg.norm(y_true[i] - poses[0, :3])
        sign = 1.0 if (i % 2) else -1.0
        y[i] = poses[0, :3] + (dist * (1.0 + sign * DEPTH_SIGMA)) * ray
        x0[p:p + 3] = y[i]
        P0[p:p + 3, :] = P0[0:3, :]
        P0[:, p:p + 3] = P0[:, 0:3]
        P0[p:p + 3, p:p + 3] = P0[0:3, 0:3] + (DEPTH_SIGMA * dist) ** 2 * np.outer(ray, ray) + \
            (0.01 * dist) ** 2 * (np.eye(3) - np.outer(ray, ray))
    for i in range(n_settled, N):  # the appended rays share the camera's uncertainty
        for j in range(n_settled, N):
            if i != j:
                P0[13 + 3 * i:16 + 3 * i, 13 + 3 * j:16 + 3 * j] = P0[0:3, 0:3]
    sc = warp_scene.WarpScene(name="lateral", cam8=cam8, boxsize=B, poses=poses, v=np.array([vx, 0, 0]),
                              omega=np.array([0, 0, w]), frames=frames, y=y, xp_org=np.tile(poses[0], (N, 1)),
                              patches=patches, pix=pix, x0=x0, P0=0.5 * (P0 + P0.T))
    return sc, y_true


SETTINGS = [("off", 0, 0.0), ("iterated", 3, 1e-3), ("off+consensus+rescue", 0, 0.0),
            ("iterated+consensus+rescue", 3, 1e-3)]


def track(sc, y_true):
    ctx = scene_ctx([sc] * 4, n_select=16)
    try:
        for s, (name, N, tol) in enumerate(SETTINGS):
            ctx.set_stream_iterated(s, N, tol)
            if "consensus" in name:
                ctx.set_stream_consensus(s, 2.5)
                ctx.set_stream_rescue(s, 5.991)
        n_all = len(sc.y)
        nees = np.zeros((STEPS, 4))
        iters = np.zeros(4)
        for t in range(1, STEPS + 1):
            ctx.set_frames(0, np.stack([sc.frames[t]] * 4))
            ctx.step(0)
            ctx.sync()
            iters += ctx.iterated_results()[0]
            for s in range(4):
                x, P = ctx.get_state(s)
                e = x[:3] - sc.poses[t, :3]
                nees[t - 1, s] = float(e @ np.linalg.solve(P[:3, :3], e))
        out = {}
        for s, (name, _, _) in enumerate(SETTINGS):
            x, _ = ctx.get_state(s)
            kept = ctx.num_features(s) == n_all
            derr = None
            if kept:
                yn = x[13:].reshape(-1, 3)[n_all - NEW:]
                r0 = sc.poses[0, :3]
                derr = float(np.mean(np.abs(np.linalg.norm(yn - r0, axis=1) -
                                            np.linalg.norm(y_true[n_all - NEW:] - r0, axis=1))))
            out[name] = dict(depth_err_m=derr, mean_nees=float(nees[:, s].mean()), kept_map=kept,
                             mean_iterations=float(iters[s] / STEPS),
                             end_pos_err_m=float(np.linalg.norm(x[:3] - sc.poses[-1, :3])))
        return out
    finally:
        ctx.close()


@pytest.mark.gpu
def test_appended_depth_rays_on_a_rendered_lateral_translation():
    sc, y_true = lateral_scene()
    out = track(sc, y_true)
    print("iterate capability", out)
    for name in out:
        assert out[name]["kept_map"] and np.isfinite(out[name]["mean_nees"]), name
    assert out["iterated"]["mean_iterations"] > 0
    # Measured on an H100 (DESIGN.md section 3): the camera position NEES fell from 9.6 to 4.2 (3 for a consistent
    # filter), with and without the consensus and the rescue, which rejected nothing here; the appended features'
    # depth error (4.5 -> 5.2 cm) and the end position error (2.4 -> 6.1 mm) did not improve.  The threshold holds
    # the consistency gain with a margin; the accuracy numbers are reported, not claimed.
    for a, b in (("iterated", "off"), ("iterated+consensus+rescue", "off+consensus+rescue")):
        assert out[a]["mean_nees"] <= NEES_RATIO_MAX * out[b]["mean_nees"], (a, out[a], out[b])
