"""The gyroscope update in whole steps: the fused step against the CPU oracle with the update inserted between its
predict and its selection (tests/gyro_oracle.cpp), and the capability it exists for, on a rendered hand-held "whip"
(tests/gyro_scene.py) whose samples are drawn from the true rates through R_gc, the bias and cov."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation
from scipy.stats import chi2

import gyro_oracle as go
import scenelib2_b200 as sl2
from gpu_util import check_streams_against_oracle, ctx_from_scenes, step_frames, update_variant
from gyro_scene import gyro_samples, make_whip_scene
from warp_scene import angle_deg

R_GC = Rotation.from_euler("zyx", [90.0, 20.0, -10.0], degrees=True).as_matrix()
BIAS = np.array([0.01, -0.02, 0.005])
COV = np.diag([4e-4, 4e-4, 4e-4])


@pytest.mark.gpu
def test_whole_step_parity_with_the_oracle_through_a_cull():
    """20 fused steps of two streams with the gyro on, each checked against the oracle: selection, flags, matches and
    counters exactly, predictions and state at the suite's tolerances, and the gyro's status and NIS.  Three templates
    of each map are random bytes, never found: both streams cull."""
    T = 20
    scenes = [update_variant(30, 30, bad=3, stream_id=s, n_frames=T) for s in range(2)]
    for sc in scenes:
        sc.n_select = 12
    ctx = ctx_from_scenes(scenes)
    oracles = [go.slam_from_scene(sc) for sc in scenes]
    rng = np.random.default_rng(20)
    try:
        for s, o in enumerate(oracles):
            ctx.set_stream_gyro(s, 1, R_gc=R_GC, bias=BIAS, cov=COV)
            o.set_gyro(R_GC, BIAS, COV)
        for t in range(T):
            rates = np.zeros((2, 3))
            for s in range(2):
                x, _ = ctx.get_state(s)
                rates[s] = R_GC @ (x[10:13] + rng.normal(0, 0.05, 3)) + BIAS
                oracles[s].sample(rates[s])
            ctx.set_gyro_samples(0, rates)
            step_frames(ctx, np.stack([sc.frames[t] for sc in scenes]))
            check_streams_against_oracle(ctx, oracles, [0, 1], lambda s: scenes[s], t)
            nis, status = ctx.gyro_results()
            for s, o in enumerate(oracles):
                q, st = o.result()
                assert status[s] == st == 1, (t, s)
                assert abs(nis[s] - q) <= 1e-6 * max(1.0, q), (t, s, nis[s], q)
        assert all(ctx.num_features(s) < 30 for s in range(2))  # the never-found features were culled
    finally:
        ctx.close()


def _whip_ctx(sc):
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


def _run(sc, setting, samples, device):
    """Steps 1..T of the whip on the device (device=True) or the gyro oracle: per step the matched fraction of the
    selected features and the gyro NIS; the final x."""
    run = _whip_ctx(sc) if device else go.slam_from_scene(sc)
    frac, nis = [], []
    try:
        if setting is not None:
            if device:
                run.set_stream_gyro(0, 1, **setting)
            else:
                run.set_gyro(setting["R_gc"], setting["bias"], setting["cov"])
        for t in range(1, len(sc.frames)):
            if setting is not None:
                if device:
                    run.set_gyro_samples(0, samples[t - 1][None])
                else:
                    run.sample(samples[t - 1])
            if device:
                run.set_frames(0, sc.frames[t][None])
                run.step(0)
                run.sync()
                f = run.features(0)
                nis.append(float(run.gyro_results()[0][0]))
            else:
                run.step(sc.frames[t])
                f = run.features()
                nis.append(run.result()[0])
            sel, ok = (f["flags"] & 1) > 0, (f["flags"] & 2) > 0
            frac.append(ok[sel].sum() / max(sel.sum(), 1))
        x, _ = run.get_state(0) if device else run.get_state()
    finally:
        if device:
            run.close()
    return np.array(frac), np.array(nis), x


@pytest.mark.gpu
def test_the_gyro_carries_the_features_through_a_whip():
    """A yaw-rate step of 2 rad/s within one frame and back.  The bounds were set from the CPU oracle with the update
    inserted (the same calls with device=False, run here too): with the gyro on every step matches all its selected
    features and the final pose is within 1.3 mm and 0.03 degrees; with the gyro off the whip step and the step after
    it match none.  The device is held to: on, >= 90 % matched on every step and the final pose within 2 cm and 1
    degree; off, under 50 % on the whip step; a wrong extrinsic (R_gc transposed) under 50 % after the whip.  The NIS
    of the steps away from the whip is below the 99 % band's upper edge of chi^2 with 3 degrees of freedom; the whip
    steps, a 10 sigma event for the motion model's 6 rad/s^2, are far above it."""
    sc = make_whip_scene()
    z = gyro_samples(sc, R_GC, BIAS, COV)
    good = dict(R_gc=R_GC, bias=BIAS, cov=COV)
    wrong = dict(R_gc=R_GC.T, bias=BIAS, cov=COV)
    w = sc.whip - 1  # index of the whip step in the per-step arrays
    for device in (False, True):
        f_on, nis, x = _run(sc, good, z, device)
        f_off, _, _ = _run(sc, None, z, device)
        f_wrong, _, _ = _run(sc, wrong, z, device)
        assert (f_on >= 0.9).all(), (device, f_on)
        assert np.linalg.norm(x[:3] - sc.poses[-1, :3]) <= 0.02, device
        assert angle_deg(x[3:7], sc.poses[-1, 3:]) <= 1.0, device
        assert f_off[w] < 0.5, (device, f_off)
        assert f_wrong[w + 1:].min() < 0.5, (device, f_wrong)
        calm = np.delete(nis, [w, w + 1])
        assert calm.mean() <= chi2.ppf(0.995, 3 * calm.size) / calm.size, (device, nis)
        assert nis[w] > chi2.ppf(0.995, 3) and nis[w + 1] > chi2.ppf(0.995, 3), (device, nis)
        if device:
            print("whip device: on", np.round(f_on, 2).tolist(), "off", np.round(f_off, 2).tolist(), "wrong",
                  np.round(f_wrong, 2).tolist(), "nis", np.round(nis, 3).tolist(),
                  "pos_cm %.3f" % (100 * np.linalg.norm(x[:3] - sc.poses[-1, :3])),
                  "ang_deg %.4f" % angle_deg(x[3:7], sc.poses[-1, 3:]))
