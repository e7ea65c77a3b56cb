"""The gyroscope update on the device (sl2_set_stream_gyro, csrc/gyro.cu): bit parity with the restatement
(tests/gyro_ref.py) fed the device's own predicted state, the truth's bound (tests/gyro_truth.py), the fused step
against the staged path, off-path identity and launch counts, every launch path, samples, snapshots and arguments."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import gyro_ref as gr
import gyro_truth as gt
import scenelib2_b200 as sl2
from gpu_util import CAMS_320, assert_same_bytes, large_variant, ring_block, stream_result
from scenelib2_b200 import synth

SEED = 90


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
    """Stream s's gyro: a rotation of its own, a bias and a correlated covariance (rad/s)."""
    rng = np.random.default_rng(SEED + s)
    R = Rotation.random(random_state=SEED + s).as_matrix() if s % 3 else np.eye(3)
    Q = Rotation.random(random_state=SEED + 100 + s).as_matrix()
    cov = Q @ np.diag([4e-4, 2e-4, 1e-4]) @ Q.T
    cov = 0.5 * (cov + cov.T)
    return dict(R_gc=R, bias=rng.normal(0, 0.01, 3), cov=cov)


def turn_on(ctx, s):
    ctx.set_stream_gyro(s, 1, **setting(s))


def samples(ctx, t, B, streams):
    """A sample per stream: for the streams listed, R_gc (omega + a turn of its own) + b with omega the stream's
    current estimate; the others get some rate."""
    rng = np.random.default_rng(1000 + t)
    rates = rng.normal(0, 0.3, (B, 3))
    for s in streams:
        g = setting(s)
        x, _ = ctx.get_state(s)
        rates[s] = g["R_gc"] @ (x[10:13] + rng.normal(0, 0.4, 3)) + g["bias"]
    return rates


def step(ctx, scenes, t, rates=None, valid=None, slot=0):
    if rates is not None:
        ctx.set_gyro_samples(slot, rates, valid)
    ctx.set_frames(slot, frames_at(ctx, scenes, t))
    ctx.step(slot)
    ctx.sync()


def results(ctx, s):
    nis, st = ctx.gyro_results(s, 1)
    return float(nis[0]), int(st[0])


# ---- the device against the restatement, the truth and the staged path ----------------------------------------------
def _parity_scenes(kind):
    if kind == "cap256":
        return [large_variant(256, 100, stream_id=0, n_frames=8)], 0, 256
    if kind == "stream2":
        scenes = [synth.make_scene("C4", stream_id=s, n_frames=8) for s in range(3)]
        return scenes, 2, None
    return [synth.make_scene(kind, n_frames=8)], 0, None


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["C1", "C2", "C3", "C4", "cap256", "stream2"])
def test_update_equals_the_restatement_and_the_fused_step_the_staged(kind):
    """Every step: the staged update of the device's own predicted x and P (a clone of the stream after
    sl2_ekf_predict) equals the restatement bit for bit (x, P, NIS, status) and the truth within its bound; the staged
    step then equals the fused step byte for byte, its gyro results included."""
    scenes, s, cap = _parity_scenes(kind)
    T = 6
    ctx = make_ctx(scenes, max_features=cap)
    if kind == "stream2":  # stream 2 with a camera of its own
        cam = CAMS_320[1]
        sc = ctx.stream_config(2)
        sc.fku, sc.fkv, sc.u0, sc.v0, sc.kd1, sc.sd = [float(v) for v in cam[2:8]]
        ctx.set_stream_config(2, sc)
    clone = make_ctx([scenes[s]], max_features=cap or ctx.cfg.max_features)
    try:
        turn_on(ctx, s)
        clone.set_stream_gyro(0, 1, **setting(s))
        if len(scenes) > 1:
            turn_on(ctx, 0)
        g = setting(s)
        applied = 0
        for t in range(T):
            rates = samples(ctx, t, len(scenes), range(len(scenes)))
            clone.load_stream(0, ctx.save_stream(s))
            clone.ekf_predict(0)
            x, P = clone.get_state(0)
            want_x, want_P, want_q, want_st = gr.update(x, P, g["R_gc"], g["bias"], g["cov"], rates[s])
            clone.gyro_update(0, rates[s])
            xg, Pg = clone.get_state(0)
            q, st = results(clone, 0)
            assert st == want_st == 1, t
            assert xg.tobytes() == want_x.tobytes() and Pg.tobytes() == want_P.tobytes(), t
            assert np.float64(q).tobytes() == np.float64(want_q).tobytes(), t
            tr = gt.update(x, P, g["R_gc"], g["bias"], g["cov"], rates[s])
            assert max(gt.errors(xg, Pg, q, tr)) <= gt.bound(tr, x, g["R_gc"], g["bias"], rates[s]), t
            applied += 1
            # the rest of the step on the staged path, then the fused step
            frames = frames_at(ctx, scenes, t)
            clone.set_frame(0, 0, frames[s])
            clone.predict_measurements(0)
            clone.make_measurements(0, 0)
            clone.ekf_update_measured(0)
            ctx.set_gyro_samples(0, rates)
            ctx.set_frames(0, frames)
            ctx.step(0)
            ctx.sync()
            assert_same_bytes(stream_result(clone, 0, jacobians=True), stream_result(ctx, s, jacobians=True), t)
            assert results(ctx, s) == (q, st), t
        assert applied == T
    finally:
        ctx.close()
        clone.close()


# ---- off means off -------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("groups", [1, 2])
def test_off_streams_unchanged_and_three_launches_per_group(groups):
    B, T = 4, 5
    scenes = [synth.make_scene("C2", stream_id=s, n_frames=T) for s in range(B)]
    never, toggled, on = (make_ctx(scenes, groups=groups) for _ in range(3))
    try:
        turn_on(toggled, 1)
        toggled.set_stream_gyro(1, 0, **setting(1))
        on_streams = [1] if groups == 1 else [0, 1, 3]
        for s in on_streams:
            turn_on(on, s)
        extra = 3 * (1 if groups == 1 else 2)
        for t in range(T):
            rates = samples(on, t, B, on_streams)
            on.set_gyro_samples(0, rates)
            n0, t0, o0 = never.launch_count(), toggled.launch_count(), on.launch_count()
            for c in (never, toggled, on):
                step(c, scenes, t)
            assert toggled.launch_count() - t0 == never.launch_count() - n0
            assert on.launch_count() - o0 == never.launch_count() - n0 + extra
            for s in range(B):
                assert_same_bytes(stream_result(toggled, s, jacobians=True), stream_result(never, s, jacobians=True),
                                  (t, s))
                if s not in on_streams:
                    assert_same_bytes(stream_result(on, s, jacobians=True), stream_result(never, s, jacobians=True),
                                      (t, s))
            assert [results(on, s)[1] for s in on_streams] == [1] * len(on_streams)
            assert toggled.gyro_results()[1].tolist() == [0] * B
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
        alone.set_stream_gyro(0, 1, **setting(1))
        H, W = serial.cfg.height, serial.cfg.width
        host = torch.zeros((2, B, H, W), dtype=torch.uint8, pin_memory=True)
        xv = torch.zeros((2, B, 13), dtype=torch.float64, pin_memory=True)
        for t in range(T):
            rates = samples(serial, t, B, [0, 1, 3])
            valid = np.array([1, 1, 1, t % 3 != 1], np.uint8)  # stream 3 misses a sample now and then
            step(serial, scenes, t, rates, valid)
            step(grouped, scenes, t, rates, valid)
            step(alone, scenes[1:2], t, rates[1:2], valid[1:2])
            asyn.wait_slot(t % 2)
            asyn.set_gyro_samples(t % 2, rates, valid)
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
        alone.set_stream_gyro(0, 1, **setting(pos))
        turn_on(batch, pos)
        for s in rng.choice(B, 80, replace=False):
            s = int(s)
            if s == pos:
                continue
            k = s % 4
            if k == 0:
                turn_on(batch, s)
            elif k == 1:
                batch.set_stream_consensus(s, 2.5)
            elif k == 2:
                batch.set_stream_warp(s, 1)
            else:
                batch.set_stream_selection(s, sl2.lib.SL2_SELECT_INFORMATION, 0.5)
        for t in range(T):
            rates = np.random.default_rng(t).normal(0, 0.3, (B, 3))
            rates[pos] = samples(batch, t, B, [pos])[pos]
            step(alone, [own], t, rates[pos:pos + 1])
            step(batch, others, t, rates)
            assert_same_bytes(stream_result(batch, pos, jacobians=True), stream_result(alone, 0, jacobians=True), t)
            assert results(batch, pos) == results(alone, 0)
    finally:
        alone.close()
        batch.close()


# ---- samples ---------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_a_sample_is_used_once_and_turning_on_clears_stale_samples():
    T = 4
    sc = synth.make_scene("C2", n_frames=T)
    a, b = make_ctx([sc]), make_ctx([sc])
    try:
        for c in (a, b):
            turn_on(c, 0)
        z = samples(a, 0, 1, [0])
        step(a, [sc], 0, z)
        step(b, [sc], 0, z)
        assert results(a, 0)[1] == 1
        blob = a.save_stream(0)
        step(a, [sc], 1)  # no new sample: the step does no gyro update
        assert results(a, 0) == (0.0, 0)
        off = make_ctx([sc])
        off.load_stream(0, blob)
        step(off, [sc], 1)
        assert_same_bytes(stream_result(a, 0, jacobians=True), stream_result(off, 0, jacobians=True), "used once")
        off.close()
        # a sample written while the stream is off is stale once it is turned on
        b.set_stream_gyro(0, 0, **setting(0))
        b.set_gyro_samples(0, z)
        ref = make_ctx([sc])
        ref.load_stream(0, b.save_stream(0))
        turn_on(b, 0)
        step(b, [sc], 1)
        step(ref, [sc], 1)
        assert results(b, 0) == (0.0, 0)
        assert_same_bytes(stream_result(b, 0, jacobians=True), stream_result(ref, 0, jacobians=True), "stale")
        ref.close()
    finally:
        a.close()
        b.close()


@pytest.mark.gpu
def test_a_still_camera_with_zero_readings_stays_finite():
    """A camera at rest (v = 0) reading zero rates for 30 steps.  It starts from a small non-zero omega, not from
    omega = 0: at omega = 0 exactly the motion Jacobian (dqomegadt_by_domega, as in the reference) divides 0 by 0 in
    the prediction, with or without a gyro.  The zero readings then pull omega towards 0 without reaching it."""
    sc = synth.make_scene("C2", n_frames=1)
    sc.frames = [sc.frames[0]] * 30
    ctx = make_ctx([sc])
    try:
        ctx.set_stream_gyro(0, 1, cov=np.eye(3) * 1e-4)
        x, P = ctx.get_state(0)
        x[7:10] = 0.0
        x[10:13] = [1e-3, -1e-3, 5e-4]  # omega = 0 exactly is the motion Jacobian's 0 / 0, with or without a gyro
        ctx.set_state(0, x, P)
        for t in range(30):
            step(ctx, [sc], 0, np.zeros((1, 3)))
            x, P = ctx.get_state(0)
            assert np.isfinite(x).all() and np.isfinite(P).all(), t
            assert results(ctx, 0)[1] == 1, t
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
            rates = samples(run, t, 2, [0])
            step(run, scenes, t, rates)
            step(plain, scenes, t)
        assert plain.save_stream(1) == run.save_stream(1)
        blob = run.save_stream(0)
        assert sl2.read_snapshot(blob)["version"] == sl2.lib.SL2_SNAPSHOT_VERSION
        assert len(blob) == len(plain.save_stream(0))
        cont.load_streams(run.save_streams())
        assert cont.stream_gyro(0)["on"] == 1  # a load leaves the slot's setting
        for t in range(4, T):
            rates = samples(run, t, 2, [0])
            step(run, scenes, t, rates)
            step(cont, scenes, t, rates)
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
        before = ctx.stream_gyro(0)
        assert before["on"] == 0 and (before["R_gc"] == np.eye(3)).all() and (before["cov"] == np.eye(3)).all()
        # no stream on yet: samples are refused
        assert L.sl2_set_gyro_samples(h, 0, 0, 1, np.zeros(3).ctypes.data, None) == -3
        turn_on(ctx, 0)
        good = ctx.stream_gyro(0)
        x0, P0 = ctx.get_state(0)
        n0 = ctx.launch_count()

        def gyro(**kw):
            g = sl2.lib.Sl2StreamGyro()
            g.on, g.reserved = kw.get("on", 1), kw.get("reserved", 0)
            g.R_gc[:] = list(np.asarray(kw.get("R", good["R_gc"]), np.float64).ravel())
            g.bias[:] = list(np.asarray(kw.get("b", good["bias"]), np.float64).ravel())
            g.cov[:] = list(np.asarray(kw.get("cov", good["cov"]), np.float64).ravel())
            return g

        R = good["R_gc"]
        bad_cov = good["cov"].copy()
        bad_cov[0, 1] = np.nextafter(bad_cov[0, 1], 1.0)
        refused = [dict(on=2), dict(on=-1), dict(reserved=1), dict(R=R * (1 + 1e-8)), dict(R=-R),
                   dict(R=np.diag([1.0, 1.0, -1.0])), dict(b=[np.nan, 0, 0]), dict(R=np.full((3, 3), np.inf)),
                   dict(cov=bad_cov), dict(cov=np.diag([1.0, 0.0, 1.0])), dict(cov=np.diag([1.0, -1.0, 1.0])),
                   dict(cov=[[1, 2, 0], [2, 1, 0], [0, 0, 1]])]
        for kw in refused:
            assert L.sl2_set_stream_gyro(h, 0, C.byref(gyro(**kw))) == -1, kw
        assert L.sl2_set_stream_gyro(h, 2, C.byref(gyro())) == -1
        assert L.sl2_set_stream_gyro(h, -1, C.byref(gyro())) == -1
        assert L.sl2_set_stream_gyro(h, 0, None) == -1
        assert L.sl2_get_stream_gyro(h, 0, None) == -1
        rates = np.zeros((2, 3))
        rates[1, 0] = np.nan
        assert L.sl2_set_gyro_samples(h, 0, 0, 2, rates.ctypes.data, None) == -1
        assert L.sl2_set_gyro_samples(h, 1, 0, 1, rates.ctypes.data, None) == -1  # slot
        assert L.sl2_set_gyro_samples(h, 0, 1, 2, rates.ctypes.data, None) == -1  # range
        assert L.sl2_set_gyro_samples(h, 0, 0, 1, None, None) == -1
        assert L.sl2_gyro_update(h, 0, rates[1].ctypes.data) == -1
        assert L.sl2_gyro_update(h, 0, None) == -1
        assert L.sl2_gyro_update(h, 1, np.zeros(3).ctypes.data) == -3  # stream 1 is off
        assert L.sl2_get_gyro_results(h, 1, 2, None, None) == -1
        assert ctx.launch_count() == n0
        after = ctx.stream_gyro(0)
        assert all((after[k] == good[k]).all() for k in ("R_gc", "bias", "cov")) and after["on"] == 1
        x1, P1 = ctx.get_state(0)
        assert x1.tobytes() == x0.tobytes() and P1.tobytes() == P0.tobytes()
        # a valid sample for stream 0 next to an invalid NaN one for stream 1 is accepted
        assert L.sl2_set_gyro_samples(h, 0, 0, 2, rates.ctypes.data, np.array([1, 0], np.uint8).ctypes.data) == 0
        # a skipped update: a non-positive-definite S leaves the state exactly
        x, P = ctx.get_state(0)
        P[11, 11] = -1.0
        ctx.set_state(0, x, P)
        ctx.gyro_update(0, np.zeros(3))
        assert results(ctx, 0) == (0.0, 2)
        x2, P2 = ctx.get_state(0)
        assert x2.tobytes() == x.tobytes() and P2.tobytes() == np.asfortranarray(P).tobytes()
    finally:
        ctx.close()
