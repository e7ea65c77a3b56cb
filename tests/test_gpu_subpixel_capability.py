"""What the sub-pixel refinement buys on a rendered trajectory (tests/warp_scene.py): a band-limited texture on a plane
seen by a 320 x 240 camera that rolls by 40 degrees over 40 steps, so every feature's true projection moves by
fractions of a pixel from frame to frame.  Three streams of one context track it with the warp on: the refinement
off, on, and on with sd lowered to the refined matches' error.  The numbers are recorded in DESIGN.md section 4."""
import numpy as np
import pytest

import warp_scene
from camera_ref import camera_points, project_point
from test_gpu_warp import scene_ctx

SD_LOW = 0.5  # px: sd of the third stream, near the refined matches' radial error measured here


def track(sc):
    ctx = scene_ctx([sc, sc, sc])
    try:
        for s in range(3):
            ctx.set_stream_warp(s, 1)
        ctx.set_stream_subpixel(1, 1)
        ctx.set_stream_subpixel(2, 1)
        ctx.set_stream_config(2, sd=SD_LOW)
        N = len(sc.y)
        err = [[], [], []]      # per stream: match - true projection of every successful match
        ref_err, pos = [], np.zeros((len(sc.frames) - 1, 3))
        for t in range(1, len(sc.frames)):
            ctx.set_frames(0, np.stack([sc.frames[t]] * 3))
            ctx.step(0)
            ctx.sync()
            truth = project_point(sc.cam8, camera_points(sc.poses[t], sc.y))
            for s in range(3):
                f = ctx.features(s)
                pos[t - 1, s] = np.linalg.norm(ctx.get_state(s)[0][:3] - sc.poses[t, :3])
                if ctx.num_features(s) != N:
                    continue
                ok = (f["flags"] & 2) > 0
                err[s].append(f["z"][ok] - truth[ok])
                if s == 1:
                    ref_err.append(f["z"][ok & ((f["flags"] & 8) > 0)] - truth[ok & ((f["flags"] & 8) > 0)])
        rms = [float(np.sqrt((np.concatenate(e) ** 2).mean())) for e in err]
        rms_refined = float(np.sqrt((np.concatenate(ref_err) ** 2).mean()))
        return rms, rms_refined, pos
    finally:
        ctx.close()


@pytest.mark.gpu
def test_refined_matches_and_trajectory_on_a_rendered_roll():
    sc = warp_scene.make_warp_scene("roll", steps=40)
    rms, rms_refined, pos = track(sc)
    traj = pos.mean(axis=0)
    print("subpixel capability", dict(rms_px=rms, rms_refined_px=rms_refined, mean_pos_err_m=traj.tolist(),
                                      end_pos_err_m=pos[-1].tolist()))
    assert rms[1] <= 0.75 * rms[0]
    assert traj[1] <= 1.05 * traj[0]
    assert traj[2] < traj[0]
