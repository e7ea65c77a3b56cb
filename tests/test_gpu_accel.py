"""The accelerometer on the device (sl2_set_stream_accel, csrc/ekf.cu accel_model / motion_model / predict_kernel):
bit parity with the restatement (tests/accel_ref.py) on the device's own pre-step state, the truth's bound
(tests/accel_truth.py), the fused step against the staged path, off-path identity and launch counts, every launch path,
samples, snapshots and arguments."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import accel_ref as ar
import accel_truth as at
import gyro_ref as gr
import scenelib2_b200 as sl2
from gpu_util import CAMS_320, assert_same_bytes, large_variant, ring_block, stream_result
from scenelib2_b200 import synth
from test_gpu_gyro import setting as gyro_setting

SEED = 120
GRAVITY = np.array([0.0, -9.81, 0.0])


def make_ctx(scenes, max_features=None, groups=1, frame_slots=1):
    cfg = sl2.config_for_scene(scenes[0], num_streams=len(scenes), frame_slots=frame_slots,
                               max_features=max_features or max(sc.n_features for sc in scenes))
    ctx = sl2.Context(cfg)
    ctx.set_step_groups(groups)
    for s, sc in enumerate(scenes):
        ctx.set_stream_config(s, sl2.stream_config_for_scene(sc))
        sl2.load_scene(ctx, s, sc)
    return ctx


def frames_at(ctx, scenes, t):
    H, W = ctx.cfg.height, ctx.cfg.width
    rng = np.random.default_rng(t)
    return np.stack([ring_block(sc.frames[t % len(sc.frames)], H, W, rng) for sc in scenes])


def setting(s):
    """Stream s's accelerometer: a rotation of its own, a bias, a correlated covariance ((m/s^2)^2), gravity along the
    world's y axis and sd_a."""
    rng = np.random.default_rng(SEED + s)
    R = Rotation.random(random_state=SEED + s).as_matrix() if s % 3 else np.eye(3)
    Q = Rotation.random(random_state=SEED + 100 + s).as_matrix()
    cov = Q @ np.diag([4e-4, 2e-4, 1e-4]) @ Q.T
    cov = 0.5 * (cov + cov.T)
    return dict(R_ac=R, bias=rng.normal(0, 0.05, 3), cov=cov, gravity=GRAVITY, sd_a=[1.0, 0.5, 0.0, 2.0][s % 4])


def turn_on(ctx, s):
    ctx.set_stream_accel(s, 1, **setting(s))


def force_for(ctx, s, a_world, k=None):
    """The reading of stream s's accelerometer (setting k, default s) when the camera accelerates at a_world:
    R_ac R(q)^T (a - g) + b."""
    g = setting(s if k is None else k)
    x, _ = ctx.get_state(s)
    Rq = np.array(ar.quat_to_R(*x[3:7]))
    return g["R_ac"] @ (Rq.T @ (a_world - g["gravity"])) + g["bias"]


def samples(ctx, t, B, streams):
    """A sample per stream: for the streams listed, the reading of an acceleration of a few m/s^2; the others get
    some force."""
    rng = np.random.default_rng(2000 + t)
    f = rng.normal(0, 5.0, (B, 3))
    for s in streams:
        f[s] = force_for(ctx, s, rng.normal(0, 3.0, 3))
    return f


def step(ctx, scenes, t, forces=None, valid=None, slot=0):
    if forces is not None:
        ctx.set_accel_samples(slot, forces, valid)
    ctx.set_frames(slot, frames_at(ctx, scenes, t))
    ctx.step(slot)
    ctx.sync()


def results(ctx, s):
    a, st = ctx.accel_results(s, 1)
    return a[0].tobytes(), int(st[0])


def device_skeleton(probe, blob):
    """The device's reference prediction parts (fv, F, Gn) of the stream in `blob`, read back exactly: with Pxx = 0
    and column 13 + k of the panel = e_k, sl2_ekf_predict leaves Q in P'[:13, :13] and F[:, k] in P'[:13, 13 + k]."""
    probe.load_stream(0, blob)
    x, _ = probe.get_state(0)
    n = x.size
    assert n >= 26, "the probe needs five features"
    Pp = np.zeros((n, n))
    for k in range(13):
        Pp[k, 13 + k] = Pp[13 + k, k] = 1.0
    probe.set_state(0, x, Pp)
    probe.ekf_predict(0)
    x2, P2 = probe.get_state(0)
    F = np.array(P2[:13, 13:26])
    dt = F[0, 7]
    Gn = np.zeros((13, 6))
    Gn[3:7, 3:6] = F[3:7, 10:13]
    for i in range(3):
        Gn[i, i], Gn[7 + i, i], Gn[10 + i, 3 + i] = dt, 1.0, 1.0
    _, Q = ar.covariance_passes(np.zeros((13, 13)), F, Gn, dt)
    assert Q.tobytes() == np.ascontiguousarray(P2[:13, :13]).tobytes()  # the skeleton reproduces the device's Q
    return (x2[:13].copy(), F, Gn), dt


# ---- the device against the restatement, the truth and the staged path ----------------------------------------------
def _parity_scenes(kind):
    if kind == "cap256":
        return [large_variant(256, 100, stream_id=0, n_frames=8)], 0, 256
    if kind == "stream2":
        scenes = [synth.make_scene("C4", stream_id=s, n_frames=8) for s in range(3)]
        return scenes, 2, None
    return [synth.make_scene(kind.split("+")[0], n_frames=8)], 0, None


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["C1", "C2", "C3", "C4", "cap256", "stream2", "C2+gyro"])
def test_prediction_equals_the_restatement_and_the_fused_step_the_staged(kind):
    """Every step: the staged prediction of the device's own pre-step state equals the restatement bit for bit (x, P,
    a, status) and the truth within its bound (with the gyro on, then the gyro update equals gyro_ref's); the staged
    step then equals the fused step byte for byte, its results included."""
    scenes, s, cap = _parity_scenes(kind)
    gyro = kind.endswith("+gyro")
    T = 6
    ctx = make_ctx(scenes, max_features=cap)
    if kind == "stream2":  # stream 2 with a camera of its own
        cam = CAMS_320[1]
        sc = ctx.stream_config(2)
        sc.fku, sc.fkv, sc.u0, sc.v0, sc.kd1, sc.sd = [float(v) for v in cam[2:8]]
        sc.delta_t = 1 / 25.0
        ctx.set_stream_config(2, sc)
    clone = make_ctx([scenes[s]], max_features=cap or ctx.cfg.max_features)
    probe = make_ctx([scenes[s]], max_features=cap or ctx.cfg.max_features)
    try:
        turn_on(ctx, s)
        clone.set_stream_accel(0, 1, **setting(s))
        if gyro:
            ctx.set_stream_gyro(s, 1, **gyro_setting(s))
            clone.set_stream_gyro(0, 1, **gyro_setting(s))
        if len(scenes) > 1:
            turn_on(ctx, 0)
        g = setting(s)
        for t in range(T):
            forces = samples(ctx, t, len(scenes), range(len(scenes)))
            rates = np.random.default_rng(t).normal(0, 0.3, (len(scenes), 3))
            blob = ctx.save_stream(s)
            sk, dt = device_skeleton(probe, blob)
            clone.load_stream(0, blob)
            x, P = clone.get_state(0)
            want_x, want_P, want_a, want_st = ar.predict(x, P, dt, g, forces[s], sk)
            clone.accel_predict(0, forces[s])
            xg, Pg = clone.get_state(0)
            a, st = clone.accel_results(0, 1)
            assert st[0] == want_st == 1, t
            assert xg.tobytes() == want_x.tobytes() and Pg.tobytes() == want_P.tobytes(), t
            assert a[0].tobytes() == np.array(want_a).tobytes(), t
            tr = at.predict(x, P, dt, g, forces[s], sk)
            assert max(at.errors(xg, Pg, x, P, dt, g, forces[s], tr)) <= at.OPS, t
            if gyro:
                gs = gyro_setting(s)
                wx, wP, _, wst = gr.update(xg, Pg, gs["R_gc"], gs["bias"], gs["cov"], rates[s])
                clone.gyro_update(0, rates[s])
                xg2, Pg2 = clone.get_state(0)
                assert wst == 1 and xg2.tobytes() == wx.tobytes() and Pg2.tobytes() == wP.tobytes(), t
                ctx.set_gyro_samples(0, rates)
            # the rest of the step on the staged path, then the fused step
            frames = frames_at(ctx, scenes, t)
            clone.set_frame(0, 0, frames[s])
            clone.predict_measurements(0)
            clone.make_measurements(0, 0)
            clone.ekf_update_measured(0)
            ctx.set_accel_samples(0, forces)
            ctx.set_frames(0, frames)
            ctx.step(0)
            ctx.sync()
            assert_same_bytes(stream_result(clone, 0, jacobians=True), stream_result(ctx, s, jacobians=True), t)
            assert results(ctx, s) == results(clone, 0), t
    finally:
        for c in (ctx, clone, probe):
            c.close()


# ---- off means off -------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("groups", [1, 2])
def test_off_streams_unchanged_and_no_launch_added(groups):
    B, T = 4, 5
    scenes = [synth.make_scene("C2", stream_id=s, n_frames=T) for s in range(B)]
    never, toggled, on = (make_ctx(scenes, groups=groups) for _ in range(3))
    try:
        turn_on(toggled, 1)
        toggled.set_stream_accel(1, 0, **setting(1))
        on_streams = [1] if groups == 1 else [0, 1, 3]
        for s in on_streams:
            turn_on(on, s)
        for t in range(T):
            on.set_accel_samples(0, samples(on, t, B, on_streams))
            n0, t0, o0 = never.launch_count(), toggled.launch_count(), on.launch_count()
            for c in (never, toggled, on):
                step(c, scenes, t)
            assert toggled.launch_count() - t0 == never.launch_count() - n0
            assert on.launch_count() - o0 == never.launch_count() - n0
            for s in range(B):
                assert_same_bytes(stream_result(toggled, s, jacobians=True), stream_result(never, s, jacobians=True),
                                  (t, s))
                if s not in on_streams:
                    assert_same_bytes(stream_result(on, s, jacobians=True), stream_result(never, s, jacobians=True),
                                      (t, s))
            assert [results(on, s)[1] for s in on_streams] == [1] * len(on_streams)
            assert toggled.accel_results()[1].tolist() == [0] * B
            assert never.save_streams() == toggled.save_streams()
        assert stream_result(on, 1)["x"].tobytes() != stream_result(never, 1)["x"].tobytes()
    finally:
        for c in (never, toggled, on):
            c.close()


# ---- every launch path gives the same bytes --------------------------------------------------------------------------
@pytest.mark.gpu
def test_serial_two_groups_async_and_single_stream_agree():
    import torch
    B, T = 4, 6
    scenes = [synth.make_scene("C2", stream_id=s, n_frames=T) for s in range(B)]
    serial, grouped, asyn = make_ctx(scenes), make_ctx(scenes, groups=2), make_ctx(scenes, frame_slots=2)
    alone = make_ctx(scenes[1:2])
    ctxs = (serial, grouped, asyn)
    try:
        for c in ctxs:
            for s in range(B):
                if s != 2:  # one stream stays off
                    turn_on(c, s)
        alone.set_stream_accel(0, 1, **setting(1))
        H, W = serial.cfg.height, serial.cfg.width
        host = torch.zeros((2, B, H, W), dtype=torch.uint8, pin_memory=True)
        xv = torch.zeros((2, B, 13), dtype=torch.float64, pin_memory=True)
        for t in range(T):
            forces = samples(serial, t, B, [0, 1, 3])
            valid = np.array([1, 1, 1, t % 3 != 1], np.uint8)  # stream 3 misses a sample now and then
            step(serial, scenes, t, forces, valid)
            step(grouped, scenes, t, forces, valid)
            step(alone, scenes[1:2], t, forces[1:2], valid[1:2])
            asyn.wait_slot(t % 2)
            asyn.set_accel_samples(t % 2, forces, valid)
            host[t % 2].numpy()[:] = frames_at(asyn, scenes, t)
            asyn.step_host_async(t % 2, host[t % 2].data_ptr(), xv[t % 2].data_ptr())
            asyn.wait_slot(t % 2)
            asyn.sync()
            for c in (grouped, asyn):
                for s in range(B):
                    assert_same_bytes(stream_result(c, s, jacobians=True), stream_result(serial, s, jacobians=True),
                                      (t, s))
                assert [results(c, s) for s in range(B)] == [results(serial, s) for s in range(B)]
            assert_same_bytes(stream_result(alone, 0, jacobians=True), stream_result(serial, 1, jacobians=True), t)
            assert results(alone, 0) == results(serial, 1)
            assert results(serial, 3)[1] == (1 if t % 3 != 1 else 0)
    finally:
        for c in ctxs + (alone,):
            c.close()


@pytest.mark.gpu
def test_a_stream_is_the_same_alone_and_in_a_264_stream_mixed_batch():
    B, pos, T = 264, 173, 5
    pool = [synth.make_scene("C4", stream_id=s, n_frames=T) for s in range(16)]
    own = pool[5]
    others = [pool[(s * 7) % 16] for s in range(B)]
    others[pos] = own
    alone, batch = make_ctx([own]), make_ctx(others)
    rng = np.random.default_rng(264)
    try:
        alone.set_stream_accel(0, 1, **setting(pos))
        turn_on(batch, pos)
        for s in rng.choice(B, 80, replace=False):
            s = int(s)
            if s == pos:
                continue
            k = s % 4
            if k == 0:
                turn_on(batch, s)
            elif k == 1:
                batch.set_stream_gyro(s, 1, **gyro_setting(s))
            elif k == 2:
                batch.set_stream_warp(s, 1)
            else:
                batch.set_stream_selection(s, sl2.lib.SL2_SELECT_INFORMATION, 0.5)
        for t in range(T):
            forces = np.random.default_rng(t).normal(0, 5.0, (B, 3))
            forces[pos] = samples(batch, t, B, [pos])[pos]
            batch.set_gyro_samples(0, np.random.default_rng(100 + t).normal(0, 0.3, (B, 3)))
            step(alone, [own], t, forces[pos:pos + 1])
            step(batch, others, t, forces)
            assert_same_bytes(stream_result(batch, pos, jacobians=True), stream_result(alone, 0, jacobians=True), t)
            assert results(batch, pos) == results(alone, 0)
    finally:
        alone.close()
        batch.close()


# ---- samples ---------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_a_sample_is_used_once_and_turning_on_clears_stale_samples():
    """A step without a sample is the reference prediction: byte-identical to a context without the feature."""
    T = 4
    sc = synth.make_scene("C2", n_frames=T)
    a, b = make_ctx([sc]), make_ctx([sc])
    try:
        for c in (a, b):
            turn_on(c, 0)
        f = samples(a, 0, 1, [0])
        step(a, [sc], 0, f)
        step(b, [sc], 0, f)
        assert results(a, 0)[1] == 1
        blob = a.save_stream(0)
        step(a, [sc], 1)  # no new sample: the reference prediction
        assert results(a, 0) == (np.zeros(3).tobytes(), 0)
        off = make_ctx([sc])
        off.load_stream(0, blob)
        step(off, [sc], 1)
        assert_same_bytes(stream_result(a, 0, jacobians=True), stream_result(off, 0, jacobians=True), "used once")
        off.close()
        # a sample written while the stream is off is stale once it is turned on
        b.set_stream_accel(0, 0, **setting(0))
        b.set_accel_samples(0, f)
        ref = make_ctx([sc])
        ref.load_stream(0, b.save_stream(0))
        turn_on(b, 0)
        step(b, [sc], 1)
        step(ref, [sc], 1)
        assert results(b, 0) == (np.zeros(3).tobytes(), 0)
        assert_same_bytes(stream_result(b, 0, jacobians=True), stream_result(ref, 0, jacobians=True), "stale")
        ref.close()
    finally:
        a.close()
        b.close()


@pytest.mark.gpu
def test_a_still_camera_reads_its_gravity_and_stays_finite():
    """A camera at rest reading -R_ac R(q)^T g + b for 30 steps: a is near 0 at every step."""
    sc = synth.make_scene("C2", n_frames=1)
    sc.frames = [sc.frames[0]] * 30
    ctx = make_ctx([sc])
    try:
        ctx.set_stream_accel(0, 1, **setting(1))  # a rotated R_ac
        x, P = ctx.get_state(0)
        x[7:10] = 0.0
        x[10:13] = [1e-3, -1e-3, 5e-4]  # omega = 0 exactly is the motion Jacobian's 0 / 0
        ctx.set_state(0, x, P)
        for t in range(30):
            step(ctx, [sc], 0, force_for(ctx, 0, np.zeros(3), k=1)[None])
            x, P = ctx.get_state(0)
            assert np.isfinite(x).all() and np.isfinite(P).all(), t
            a, st = ctx.accel_results(0, 1)
            assert st[0] == 1 and np.abs(a[0]).max() <= 1e-9, (t, a)
    finally:
        ctx.close()


# ---- snapshots -------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_snapshots_do_not_carry_the_setting_and_continue_bit_for_bit():
    T = 8
    scenes = [synth.make_scene("C2", stream_id=s, n_frames=T) for s in range(2)]
    run, plain, cont = make_ctx(scenes), make_ctx(scenes), make_ctx(scenes)
    try:
        for c in (run, cont):
            turn_on(c, 0)
        for t in range(4):
            step(run, scenes, t, samples(run, t, 2, [0]))
            step(plain, scenes, t)
        assert plain.save_stream(1) == run.save_stream(1)
        blob = run.save_stream(0)
        assert sl2.read_snapshot(blob)["version"] == sl2.lib.SL2_SNAPSHOT_VERSION
        assert len(blob) == len(plain.save_stream(0))
        cont.load_streams(run.save_streams())
        assert cont.stream_accel(0)["on"] == 1  # a load leaves the slot's setting
        for t in range(4, T):
            f = samples(run, t, 2, [0])
            step(run, scenes, t, f)
            step(cont, scenes, t, f)
            assert run.save_streams() == cont.save_streams(), t
    finally:
        for c in (run, plain, cont):
            c.close()


# ---- arguments -------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_rejected_arguments_change_nothing_and_launch_nothing():
    import ctypes as C
    sc = synth.make_scene("C2", n_frames=2)
    ctx = make_ctx([sc, sc])
    try:
        L, h = ctx.L, ctx.h
        before = ctx.stream_accel(0)
        assert before["on"] == 0 and (before["R_ac"] == np.eye(3)).all() and (before["cov"] == np.eye(3)).all()
        assert (before["gravity"] == 0).all() and before["sd_a"] == 4.0
        assert L.sl2_set_accel_samples(h, 0, 0, 1, np.zeros(3).ctypes.data, None) == -3  # no stream on yet
        turn_on(ctx, 0)
        good = ctx.stream_accel(0)
        x0, P0 = ctx.get_state(0)
        n0 = ctx.launch_count()

        def accel(**kw):
            a = sl2.lib.Sl2StreamAccel()
            a.on, a.reserved, a.sd_a = kw.get("on", 1), kw.get("reserved", 0), kw.get("sd_a", good["sd_a"])
            a.R_ac[:] = list(np.asarray(kw.get("R", good["R_ac"]), np.float64).ravel())
            a.bias[:] = list(np.asarray(kw.get("b", good["bias"]), np.float64).ravel())
            a.cov[:] = list(np.asarray(kw.get("cov", good["cov"]), np.float64).ravel())
            a.gravity[:] = list(np.asarray(kw.get("g", good["gravity"]), np.float64).ravel())
            return a

        R = good["R_ac"]
        bad_cov = good["cov"].copy()
        bad_cov[0, 1] = np.nextafter(bad_cov[0, 1], 1.0)
        refused = [dict(on=2), dict(on=-1), dict(reserved=1), dict(R=R * (1 + 1e-8)), dict(R=-R),
                   dict(R=np.diag([1.0, 1.0, -1.0])), dict(b=[np.nan, 0, 0]), dict(R=np.full((3, 3), np.inf)),
                   dict(g=[0, np.inf, 0]), dict(sd_a=-1e-300), dict(sd_a=np.nan), dict(cov=bad_cov),
                   dict(cov=np.diag([1.0, 0.0, 1.0])), dict(cov=np.diag([1.0, -1.0, 1.0])),
                   dict(cov=[[1, 2, 0], [2, 1, 0], [0, 0, 1]])]
        for kw in refused:
            assert L.sl2_set_stream_accel(h, 0, C.byref(accel(**kw))) == -1, kw
        assert L.sl2_set_stream_accel(h, 2, C.byref(accel())) == -1
        assert L.sl2_set_stream_accel(h, -1, C.byref(accel())) == -1
        assert L.sl2_set_stream_accel(h, 0, None) == -1
        assert L.sl2_get_stream_accel(h, 0, None) == -1
        forces = np.zeros((2, 3))
        forces[1, 0] = np.nan
        assert L.sl2_set_accel_samples(h, 0, 0, 2, forces.ctypes.data, None) == -1
        assert L.sl2_set_accel_samples(h, 1, 0, 1, forces.ctypes.data, None) == -1  # slot
        assert L.sl2_set_accel_samples(h, 0, 1, 2, forces.ctypes.data, None) == -1  # range
        assert L.sl2_set_accel_samples(h, 0, 0, 1, None, None) == -1
        assert L.sl2_accel_predict(h, 0, forces[1].ctypes.data) == -1
        assert L.sl2_accel_predict(h, 0, None) == -1
        assert L.sl2_accel_predict(h, 1, np.zeros(3).ctypes.data) == -3  # stream 1 is off
        assert L.sl2_get_accel_results(h, 1, 2, None, None) == -1
        assert ctx.launch_count() == n0
        after = ctx.stream_accel(0)
        assert all((after[k] == good[k]).all() for k in ("R_ac", "bias", "cov", "gravity")) and after["on"] == 1
        assert after["sd_a"] == good["sd_a"]
        x1, P1 = ctx.get_state(0)
        assert x1.tobytes() == x0.tobytes() and P1.tobytes() == P0.tobytes()
        assert L.sl2_set_accel_samples(h, 0, 0, 2, forces.ctypes.data, np.array([1, 0], np.uint8).ctypes.data) == 0
        # a skipped step: a force whose f - b overflows runs the reference prediction
        blob = ctx.save_stream(0)
        ctx.set_stream_accel(0, 1, **dict(setting(0), bias=np.array([-0.85e308, 0.85e308, -0.85e308])))
        ctx.accel_predict(0, np.array([1.7e308, -1.7e308, 1.7e308]))
        assert results(ctx, 0) == (np.zeros(3).tobytes(), 2)
        ref = make_ctx([sc])
        ref.load_stream(0, blob)
        ref.ekf_predict(0)
        assert_same_bytes(stream_result(ctx, 0), stream_result(ref, 0), "skipped")
        ref.close()
    finally:
        ctx.close()
