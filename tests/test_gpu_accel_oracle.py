"""The accelerometer in whole steps: the fused step against the CPU oracle whose predict is the accelerometer's when a
sample is pending (tests/accel_oracle.cpp), and the capability it exists for, on a rendered jolt (tests/accel_scene.py)
whose samples are drawn from the true specific force through R_ac, the bias and cov."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import accel_oracle as ao
import scenelib2_b200 as sl2
from accel_scene import GRAVITY, accel_samples, make_jolt_scene
from gpu_util import check_streams_against_oracle, ctx_from_scenes, step_frames, update_variant
from warp_scene import angle_deg

R_AC = Rotation.from_euler("zyx", [90.0, 20.0, -10.0], degrees=True).as_matrix()
BIAS = np.array([0.05, -0.08, 0.03])
COV = np.diag([4e-4, 4e-4, 4e-4])
SD_A = 0.5


@pytest.mark.gpu
def test_whole_step_parity_with_the_oracle_through_a_cull():
    """20 fused steps of two streams with the accelerometer on, each checked against the oracle: selection, flags,
    matches and counters exactly, predictions and state at the suite's tolerances (1e-8), the accelerometer's status
    exactly and its a at 1e-6.  Three templates of each map are random bytes, never found: both streams cull.  Every fourth step
    of stream 1 has no sample (the reference prediction)."""
    T = 20
    scenes = [update_variant(30, 30, bad=3, stream_id=s, n_frames=T) for s in range(2)]
    for sc in scenes:
        sc.n_select = 12
    ctx = ctx_from_scenes(scenes)
    oracles = [ao.slam_from_scene(sc) for sc in scenes]
    rng = np.random.default_rng(21)
    g = np.array([0.0, 0.0, -9.81])
    try:
        for s, o in enumerate(oracles):
            ctx.set_stream_accel(s, 1, R_ac=R_AC, bias=BIAS, cov=COV, gravity=g, sd_a=SD_A)
            o.set_accel(R_AC, BIAS, COV, g, SD_A)
        for t in range(T):
            forces = np.zeros((2, 3))
            valid = np.array([1, t % 4 != 3], np.uint8)
            for s in range(2):
                x, _ = ctx.get_state(s)
                Rq = Rotation.from_quat(x[[4, 5, 6, 3]] / np.linalg.norm(x[3:7])).as_matrix()
                forces[s] = R_AC @ (Rq.T @ (rng.normal(0, 2.0, 3) - g)) + BIAS
                if valid[s]:
                    oracles[s].sample(forces[s])
            ctx.set_accel_samples(0, forces, valid)
            step_frames(ctx, np.stack([sc.frames[t] for sc in scenes]))
            check_streams_against_oracle(ctx, oracles, [0, 1], lambda s: scenes[s], t)
            a, status = ctx.accel_results()
            for s, o in enumerate(oracles):
                ao_a, st = o.result()
                assert status[s] == st == (1 if valid[s] else 0), (t, s)
                assert np.abs(a[s] - ao_a).max() <= 1e-6 * max(1.0, np.abs(ao_a).max()), (t, s, a[s], ao_a)
        assert all(ctx.num_features(s) < 30 for s in range(2))  # the never-found features were culled
    finally:
        ctx.close()


def _jolt_ctx(sc):
    cfg = sl2.default_config()
    cfg.width, cfg.height = int(sc.cam8[0]), int(sc.cam8[1])
    cfg.fku, cfg.fkv, cfg.u0, cfg.v0, cfg.kd1, cfg.sd = [float(v) for v in sc.cam8[2:8]]
    cfg.boxsize = sc.boxsize
    cfg.max_features = len(sc.patches)
    cfg.number_of_features_to_select = sc.n_select
    cfg.delta_t = sc.delta_t
    ctx = sl2.Context(cfg)
    n = len(sc.patches)
    ctx.set_features(0, sc.x0[13:].reshape(n, 3), sc.xp_org, sc.patches)
    ctx.set_state(0, sc.x0, sc.P0)
    return ctx


def run_jolt(sc, setting, samples, device):
    """Steps 1..T of the jolt on the device (device=True) or the accelerometer oracle: per step the matched fraction
    of the selected features; the final x."""
    run = _jolt_ctx(sc) if device else ao.slam_from_scene(sc)
    frac = []
    try:
        if setting is not None:
            if device:
                run.set_stream_accel(0, 1, **setting)
            else:
                run.set_accel(setting["R_ac"], setting["bias"], setting["cov"], setting["gravity"], setting["sd_a"])
        for t in range(1, len(sc.frames)):
            if setting is not None:
                if device:
                    run.set_accel_samples(0, samples[t - 1][None])
                else:
                    run.sample(samples[t - 1])
            if device:
                run.set_frames(0, sc.frames[t][None])
                run.step(0)
                run.sync()
                f = run.features(0)
            else:
                run.step(sc.frames[t])
                f = run.features()
            sel, ok = (f["flags"] & 1) > 0, (f["flags"] & 2) > 0
            frac.append(ok[sel].sum() / max(sel.sum(), 1))
        x, _ = run.get_state(0) if device else run.get_state()
    finally:
        if device:
            run.close()
    return np.array(frac), x


def jolt_settings():
    good = dict(R_ac=R_AC, bias=BIAS, cov=COV, gravity=GRAVITY, sd_a=SD_A)
    return good, dict(good, gravity=-GRAVITY), dict(good, R_ac=R_AC.T)


def pose_error(sc, x):
    return float(np.linalg.norm(x[:3] - sc.poses[-1, :3])), float(angle_deg(x[3:7], sc.poses[-1, 3:]))


@pytest.mark.gpu
def test_the_accelerometer_carries_the_features_through_a_jolt():
    """A shove of about 3.6 g nearly along the plane for two frames and back for two, 0.5 m from it.  The bounds come
    from the CPU oracle with the accelerometer's predict (the same calls with device=False, run here too): with the accelerometer on every
    step matches all its selected features; off, some step matches fewer than half; with gravity's sign flipped or
    R_ac transposed the track degrades (some step under half, or a final position error over ten times the good
    run's)."""
    sc = make_jolt_scene()
    good, flipped, transposed = jolt_settings()
    z = accel_samples(sc, R_AC, BIAS, COV)
    for device in (False, True):
        f_on, x = run_jolt(sc, good, z, device)
        f_off, _ = run_jolt(sc, None, z, device)
        pos, ang = pose_error(sc, x)
        assert (f_on == 1.0).all(), (device, f_on)
        assert pos <= 0.01 and ang <= 1.0, (device, pos, ang)
        assert f_off.min() < 0.5, (device, f_off)
        bad_runs = [run_jolt(sc, bad, z, device) for bad in (flipped, transposed)]
        for f_bad, xb in bad_runs:
            assert f_bad.min() < 0.5 or pose_error(sc, xb)[0] > 10 * pos, (device, f_bad, pose_error(sc, xb))
        print("jolt %s: on" % ("device" if device else "oracle"), np.round(f_on, 2).tolist(),
              "off", np.round(f_off, 2).tolist(), "pos_mm %.3f ang_deg %.4f" % (1000 * pos, ang),
              "gravity flipped / R_ac transposed", [np.round(f, 2).tolist() for f, _ in bad_runs],
              [np.round(pose_error(sc, xb), 4).tolist() for _, xb in bad_runs])
