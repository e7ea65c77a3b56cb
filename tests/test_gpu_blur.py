"""The exposure blur on the device (sl2_set_stream_blur, sl2_blur_templates; csrc/warp.cu warp_kernel<BOX, true>):
byte for byte against the NumPy restatement (tests/blur_ref.py) fed the device's own exposure poses, fused against
staged, isolation of blur-off streams and the launch count, snapshots and rejected arguments, the measure stage
against the oracle's search over the restatement's templates, and one stream of a 264-stream batch against a single
stream."""
import numpy as np
import pytest

import blur_ref
import scenelib2_b200 as sl2
from gpu_util import assert_same_bytes, stream_result
from test_gpu_warp import cam8_of, ctx_for, envelope_features, frames_at, look_at, scene, scene_ctx

EXPOSURE = 1.0 / 60.0


class DevicePoses:
    """The device's pose at time s of a state x (13): the motion model's prediction over dt = |s| (v and omega negated
    for s < 0, which forms exactly r + v s and omega s), read back from a one-feature context."""

    def __init__(self):
        sc = sl2.default_config()
        sc.max_features = 1
        sc.number_of_features_to_select = 1
        self.ctx = sl2.Context(sc)
        self.ctx.set_features(0, np.array([[0.0, 0.0, 2.0]]), np.array([[0.0, 0, 0, 1, 0, 0, 0]]),
                              np.zeros((1, sc.boxsize, sc.boxsize), np.uint8))
        self.cache = {}

    def __call__(self, x, s):
        key = (np.asarray(x, np.float64)[:13].tobytes(), float(s))
        if key not in self.cache:
            xs = np.concatenate([np.asarray(x, np.float64)[:13], [0.0, 0.0, 2.0]])
            if s < 0:
                xs[7:13] = -xs[7:13]
            self.ctx.set_state(0, xs, np.eye(16))
            self.ctx.set_stream_config(0, delta_t=abs(float(s)))
            self.ctx.ekf_predict(0)
            self.cache[key] = self.ctx.get_state(0)[0][:7].copy()
        return self.cache[key]

    def close(self):
        self.ctx.close()


def moving_state(xp, rng, rate):
    axis = rng.standard_normal(3)
    return np.concatenate([xp, rng.standard_normal(3) * 0.5, axis / np.linalg.norm(axis) * rate])


def check(ctx, s, cam8, y, xo, T, x, warp, poses, idx=None, theta=None):
    idx = np.arange(len(y)) if idx is None else np.asarray(idx)
    b = ctx.stream_blur(s)
    out, valid, K = ctx.blur_templates(s, idx, x)
    want, wv, wk = blur_ref.blur_templates(cam8, T[idx], y[idx], xo[idx], x, b["exposure"], b["offset"], warp,
                                           None if theta is None else theta[idx], pose_fn=poses)
    assert (valid == wv).all() and (K == wk).all() and out.tobytes() == want.tobytes()
    return valid, K


# ---- 1. the staged form against the restatement -------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["C1", "C2", "C3", "C4"])
def test_blur_templates_equal_the_restatement(name):
    n = 128
    ctx, cam8 = ctx_for(name, n)
    poses = DevicePoses()
    rng = np.random.default_rng(ord(name[1]))
    B = ctx.cfg.boxsize
    try:
        ks = set()
        for warp in (0, 1):
            ctx.set_stream_warp(0, warp)
            for offset, rate in ((0.0, 3.0), (-EXPOSURE / 2, 1.0), (0.004, 12.0), (0.0, 0.0)):
                ctx.set_stream_blur(0, 1, EXPOSURE, offset)
                xp = look_at(rng.uniform(-1, 1, 3), rng.uniform(-1, 1, 3) + [0, 0, 3.0], rng.uniform(-np.pi, np.pi))
                xp[3:7] *= rng.choice([1.0, 1.001, 0.97])
                y, xo = envelope_features(cam8, xp, n, rng)
                T = rng.integers(0, 256, (n, B, B), dtype=np.uint8)
                ctx.set_features(0, y, xo, T)
                valid, K = check(ctx, 0, cam8, y, xo, T, moving_state(xp, rng, rate), warp, poses)
                ks |= set(K.tolist())
                assert (valid == 2).sum() >= 0.8 * n
            # exposure 0: the warp's bytes or the stored template
            ctx.set_stream_blur(0, 1, 0.0, 0.0)
            x = moving_state(xp, rng, 3.0)
            out, valid, K = ctx.blur_templates(0, np.arange(n), x)
            want, wv = ctx.warp_templates(0, np.arange(n), x[:7]) if warp else (T, np.zeros(n, np.uint8))
            keep = wv == 1 if warp else np.ones(n, bool)
            assert (out[keep] == want[keep]).all() and (K[valid == 2] == 1).all()
            # a blur-off stream: what the search of the stream sees without the blur
            ctx.set_stream_blur(0, 0, EXPOSURE, 0.0)
            out, valid, K = ctx.blur_templates(0, np.arange(n), x)
            assert (K == 0).all() and (valid <= 1).all()
            assert out.tobytes() == (want if warp else T).tobytes()
        assert 1 in ks and 32 in ks and any(1 < k < 32 for k in ks), ks
    finally:
        ctx.close()
        poses.close()


@pytest.mark.gpu
def test_capacity_256_a_stream_with_its_own_camera_and_normals():
    n = 256
    ctx, cam8 = ctx_for("C1", n, num_streams=3)
    poses = DevicePoses()
    rng = np.random.default_rng(256)
    try:
        xp = look_at(np.zeros(3), np.array([0.1, -0.1, 2.0]), 0.2)
        y, xo = envelope_features(cam8, xp, n, rng)
        T = rng.integers(0, 256, (n, 11, 11), dtype=np.uint8)
        ctx.set_features(2, y, xo, T)
        ctx.set_features(0, y[::-1], xo[::-1], T[::-1])
        ctx.set_stream_config(2, ctx.stream_config(2), kd1=3e-5, fku=240.0)  # stream 2's own camera
        cam2 = cam8_of(ctx, 2)
        ctx.set_stream_blur(2, 1, EXPOSURE, -EXPOSURE / 2)
        x = moving_state(xp, rng, 3.0)
        for warp in (0, 1):
            ctx.set_stream_warp(2, warp)
            check(ctx, 2, cam2, y, xo, T, x, warp, poses, idx=np.arange(128, 256))
            check(ctx, 2, cam2, y, xo, T, x, warp, poses, idx=[255, 0, 200, 128, 127])
        # normals on, with seeded tilts
        ctx.set_stream_normals(2, 2)
        theta = rng.uniform(-0.3, 0.3, (n, 2))
        theta[::7] = 0.0
        ctx.set_patch_normals(2, np.arange(n), theta, np.tile([0.1, 0.0, 0.1], (n, 1)))
        check(ctx, 2, cam2, y, xo, T, x, 1, poses, idx=np.arange(0, 256, 3), theta=theta)
    finally:
        ctx.close()
        poses.close()


# ---- 2. fused equals staged; isolation and launches ------------------------------------------------------------------
def run_staged(ctx, scenes, t):
    ctx.set_frames(0, frames_at(scenes, t))
    for s in range(len(scenes)):
        ctx.ekf_predict(s)
        ctx.predict_measurements(s)
        ctx.make_measurements(s, 0)
        ctx.ekf_update_measured(s)


@pytest.mark.gpu
@pytest.mark.parametrize("groups", [1, 2])
def test_fused_equals_staged(groups):
    scenes = [scene("roll"), scene("approach")]
    fused, staged = scene_ctx(scenes), scene_ctx(scenes)
    try:
        fused.set_step_groups(groups)
        for c in (fused, staged):
            c.set_stream_blur(0, 1, EXPOSURE, 0.0)
            c.set_stream_blur(1, 1, EXPOSURE, -EXPOSURE / 2)
            c.set_stream_warp(1, 1)
            c.set_stream_subpixel(0, 1)
            c.set_stream_consensus(1, 2.5)
        for t in range(1, 9):
            fused.set_frames(0, frames_at(scenes, t))
            fused.step(0)
            fused.sync()
            run_staged(staged, scenes, t)
            for s in range(2):
                assert_same_bytes(stream_result(staged, s, jacobians=True), stream_result(fused, s, jacobians=True),
                                  (t, s))
    finally:
        fused.close()
        staged.close()


@pytest.mark.gpu
def test_blur_off_streams_are_untouched_and_launches_rise_only_without_the_warp():
    scenes = [scene("roll"), scene("approach"), scene("orbit"), scene("roll")]
    plain, mixed, toggled = scene_ctx(scenes), scene_ctx(scenes), scene_ctx(scenes)
    try:
        for c in (plain, mixed, toggled):
            c.set_step_groups(2)  # groups {0, 1} and {2, 3}
            c.set_stream_warp(2, 1)  # group B warps anyway
        mixed.set_stream_blur(1, 1, EXPOSURE, 0.0)  # group A: blur without the warp, one more launch
        mixed.set_stream_blur(3, 1, EXPOSURE, 0.0)  # group B: no more launches
        for s in range(4):
            toggled.set_stream_blur(s, 1, EXPOSURE, 0.0)
            toggled.set_stream_blur(s, 0, EXPOSURE, 0.0)
        for t in range(1, 7):
            l0, m0, g0 = plain.launch_count(), mixed.launch_count(), toggled.launch_count()
            for c in (plain, mixed, toggled):
                c.set_frames(0, frames_at(scenes, t))
                c.step(0)
                c.sync()
            assert (mixed.launch_count() - m0) - (plain.launch_count() - l0) == 1, t
            assert toggled.launch_count() - g0 == plain.launch_count() - l0
            for s in range(4):
                assert_same_bytes(stream_result(toggled, s, jacobians=True), stream_result(plain, s, jacobians=True),
                                  ("toggled", s, t))
            for s in (0, 2):
                assert_same_bytes(stream_result(mixed, s, jacobians=True), stream_result(plain, s, jacobians=True),
                                  ("mixed", s, t))
    finally:
        for c in (plain, mixed, toggled):
            c.close()


@pytest.mark.gpu
def test_host_steps_equal_the_fused_step():
    sc = scene("roll")
    a, b, h = scene_ctx([sc]), scene_ctx([sc]), scene_ctx([sc])
    try:
        for c in (a, b, h):
            c.set_stream_blur(0, 1, EXPOSURE, 0.0)
        xv = np.zeros(13)
        for t in range(1, 6):
            frame = np.ascontiguousarray(sc.frames[t])
            a.set_frames(0, frame[None])
            a.step(0)
            a.sync()
            b.step_host(0, frame.ctypes.data, xv.ctypes.data)
            h.step_host_async(0, frame.ctypes.data, xv.ctypes.data)
            h.wait_slot(0)
            for c in (b, h):
                assert_same_bytes(stream_result(a, 0, jacobians=True), stream_result(c, 0, jacobians=True), t)
    finally:
        for c in (a, b, h):
            c.close()


# ---- 3. snapshots and rejected arguments ---------------------------------------------------------------------------
@pytest.mark.gpu
def test_snapshots_do_not_carry_the_setting_and_bad_arguments_change_nothing():
    sc = scene("roll")
    on, off = scene_ctx([sc, sc]), scene_ctx([sc, sc])
    try:
        on.set_stream_blur(0, 1, EXPOSURE, 0.0)
        for t in range(1, 4):
            for c in (on, off):
                c.set_frames(0, frames_at([sc, sc], t))
                c.step(0)
                c.sync()
        assert on.save_stream(1) == off.save_stream(1)
        off.load_stream(1, on.save_stream(0))
        assert off.stream_blur(1)["on"] == 0 and on.stream_blur(0)["on"] == 1
        on.load_stream(0, off.save_stream(0))
        assert on.stream_blur(0) == dict(on=1, exposure=EXPOSURE, offset=0.0)
        before = [stream_result(on, s) for s in range(2)]
        launches = on.launch_count()
        bad = [dict(on=2), dict(on=-1), dict(reserved=1), dict(exposure=-1e-3), dict(exposure=np.nan),
               dict(exposure=np.inf), dict(offset=np.nan), dict(offset=-np.inf)]
        for kw in bad:
            args = dict(on=1, exposure=EXPOSURE, offset=0.0)
            args.update(kw)
            with pytest.raises(sl2.Sl2Error):
                on.set_stream_blur(0, **args)
        with pytest.raises(sl2.Sl2Error):
            on.set_stream_blur(2, 1, EXPOSURE)
        assert on.L.sl2_get_stream_blur(on.h, 0, None) == -1
        assert on.stream_blur(0) == dict(on=1, exposure=EXPOSURE, offset=0.0)
        x = on.get_state(0)[0][:13].copy()
        for i, v in ((2, np.nan), (9, np.inf), (12, np.nan)):
            xb = x.copy()
            xb[i] = v
            with pytest.raises(sl2.Sl2Error):
                on.blur_templates(0, [0, 1], xb)
        xb = x.copy()
        xb[3:7] = 0.0
        with pytest.raises(sl2.Sl2Error):
            on.blur_templates(0, [0], xb)
        for idx in ([len(sc.y)], [-1]):
            with pytest.raises(sl2.Sl2Error):
                on.blur_templates(0, idx, x)
        assert on.launch_count() == launches
        for s in range(2):
            assert_same_bytes(stream_result(on, s), before[s], s)
        for c in (on, off):  # and later steps go on as if nothing was asked
            c.set_frames(0, frames_at([sc, sc], 4))
            c.step(0)
            c.sync()
    finally:
        on.close()
        off.close()


# ---- 4. the measure stage against the oracle's search over the restatement's templates ------------------------------
def blur_scene_ctx(S, n_select=16):
    import blur_scene as bs
    sc = bs.make_blur_scene() if "blur" not in BLUR_SCENES else BLUR_SCENES["blur"]
    BLUR_SCENES["blur"] = sc
    cfg = sl2.default_config()
    cfg.num_streams = S
    cfg.width, cfg.height = int(sc.cam8[0]), int(sc.cam8[1])
    cfg.boxsize = sc.boxsize
    cfg.max_features = len(sc.y)
    cfg.number_of_features_to_select = n_select
    cfg.fku, cfg.fkv, cfg.u0, cfg.v0, cfg.kd1, cfg.sd = [float(v) for v in sc.cam8[2:8]]
    cfg.delta_t = sc.delta_t
    ctx = sl2.Context(cfg)
    for s in range(S):
        ctx.set_features(s, sc.y, sc.xp_org, sc.patches)
        ctx.set_state(s, sc.x0, sc.P0)
    return ctx, sc


BLUR_SCENES = {}


def setup_blur_stream(ctx, s, warp, offset, gyro=True):
    import blur_scene as bs
    ctx.set_stream_blur(s, 1, bs.EXPOSURE, offset)
    ctx.set_stream_warp(s, warp)
    ctx.set_stream_gyro(s, int(gyro), cov=np.eye(3) * 1e-4)
    ctx.set_stream_subpixel(s, 1)
    ctx.set_stream_consensus(s, 2.5)


@pytest.mark.gpu
@pytest.mark.parametrize("gyro", [False, True])
def test_measure_stage_equals_the_oracle_search_of_blurred_templates(gyro):
    """Two streams (warp on and off) over 20 steps, sub-pixel refinement and consensus on, with and without the gyro:
    at every staged step the search's scores and matches equal the oracle's search of blur_ref's templates at the
    device's predicted state (the staged path, whose predicted state can be read between its calls), and the fused
    steps of a twin context, which cull from step 10, equal the staged ones up to their first cull (the staged entry
    points do not cull)."""
    import blur_scene as bs
    from oracle import pyoracle as po
    fused, sc = blur_scene_ctx(2)
    for s, (warp, off) in enumerate(((1, bs.OFFSET), (0, 0.0))):
        setup_blur_stream(fused, s, warp, off, gyro)
    results = []
    try:
        for t in range(1, 21):
            if gyro:
                fused.set_gyro_samples(0, np.tile(sc.omega[t - 1], (2, 1)))
            fused.set_frames(0, np.stack([sc.frames[t]] * 2))
            fused.step(0)
            fused.sync()
            results.append([stream_result(fused, s, jacobians=True) for s in range(2)])
    finally:
        fused.close()
    staged, _ = blur_scene_ctx(2)
    steps = []  # per staged step and stream: the predicted state, the blur setting and the snapshot after the search
    try:
        for s, (warp, off) in enumerate(((1, bs.OFFSET), (0, 0.0))):
            setup_blur_stream(staged, s, warp, off, gyro)
        culled, compared = 0, 0
        for t in range(1, 21):
            staged.set_frames(0, np.stack([sc.frames[t]] * 2))
            for s in range(2):
                nf = staged.num_features(s)
                staged.ekf_predict(s)
                if gyro:
                    staged.gyro_update(s, sc.omega[t - 1])
                staged.predict_measurements(s)
                x, _ = staged.get_state(s)
                staged.make_measurements(s, 0)
                steps.append((t, s, x, staged.stream_blur(s), sl2.read_snapshot(staged.save_stream(s))))
                staged.ekf_update_measured(s)
                culled += nf - staged.num_features(s)
            # the staged entry points cull at their own point of the step, so fused and staged agree up to the
            # first cull
            if not culled and all(len(results[t - 1][s]["x"]) == len(sc.x0) for s in range(2)):
                for s in range(2):
                    assert_same_bytes(stream_result(staged, s, jacobians=True), results[t - 1][s], (t, s))
                compared = t
    finally:
        staged.close()
    assert compared >= 5, compared
    # the oracle's search over the restatement's templates, fed the device's exposure poses (read once the staged
    # context is done, from a context of their own)
    poses = DevicePoses()
    try:
        blurred = 0
        for t, s, x, b, snap in steps:
            nsel = snap["nsel"]
            jf = snap["job_feat"][:nsel]
            if nsel == 0:
                continue
            y = x[13:].reshape(-1, 3)
            T, valid, K = blur_ref.blur_templates(sc.cam8, snap["templates"][jf], y[jf], snap["xp_org"][jf], x,
                                                  b["exposure"], b["offset"], s == 0, pose_fn=poses)
            blurred += int((valid == 2).sum())
            u, v, found, best = po.elliptical_search(sc.frames[t], T, snap["job_centre"][:nsel],
                                                     snap["job_puinv"][:nsel])
            assert snap["best"][jf].tobytes() == best.tobytes(), (t, s)
            ok = snap["found"][jf].astype(bool)
            assert not (ok & ~found.astype(bool)).any(), (t, s)  # the consensus only removes matches
            assert (snap["z_uv"][jf][ok] == np.stack([u, v], axis=1)[ok]).all(), (t, s)
        assert blurred > 100, blurred
        print("measure stage: gyro", gyro, "blurred jobs", blurred, "culled", culled, "fused = staged to step", compared)
    finally:
        poses.close()


# ---- 5. one stream of a large mixed batch, and a single (PDL) stream -------------------------------------------------
@pytest.mark.gpu
def test_stream_173_of_264_equals_a_single_stream():
    import blur_scene as bs
    big, sc = blur_scene_ctx(264)
    one, _ = blur_scene_ctx(1)
    try:
        for s in range(264):
            if s % 3 == 0:
                big.set_stream_warp(s, 1)
            if s % 4 == 1:
                big.set_stream_blur(s, 1, bs.EXPOSURE, 0.0)
        setup_blur_stream(big, 173, 1, bs.OFFSET)
        setup_blur_stream(one, 0, 1, bs.OFFSET)
        for t in range(1, 11):
            big.set_gyro_samples(0, np.tile(sc.omega[t - 1], (264, 1)))
            one.set_gyro_samples(0, sc.omega[t - 1][None])
            big.set_frames(0, np.stack([sc.frames[t]] * 264))
            one.set_frames(0, sc.frames[t][None])
            for c in (big, one):
                c.step(0)
                c.sync()
            assert_same_bytes(stream_result(one, 0, jacobians=True), stream_result(big, 173, jacobians=True), t)
    finally:
        big.close()
        one.close()
