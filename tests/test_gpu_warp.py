"""The planar patch warp on the device (sl2_set_stream_warp, sl2_warp_templates; csrc/warp.cu warp_kernel): byte for
byte against the NumPy restatement (tests/warp_ref.py), the measure stage against the oracle's search fed the
restatement's templates, fused against staged, isolation of warp-off streams, snapshots, rejected arguments, and the
tracking it buys on rendered scenes (tests/warp_scene.py)."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import scenelib2_b200 as sl2
import warp_ref
import warp_scene
from gpu_util import assert_same_bytes, stream_result
from oracle import pyoracle as po
from scenelib2_b200 import synth

TAU = 2.5  # px: the match consensus radius of the combined runs


def cam8_of(ctx, s):
    c = ctx.stream_config(s)
    return np.array([c.width, c.height, c.fku, c.fkv, c.u0, c.v0, c.kd1, c.sd], np.float64)


def look_at(pos, target, roll):
    """The pose at pos whose optical axis (camera z) points at target, rolled by `roll` radians about it."""
    z = (target - pos) / np.linalg.norm(target - pos)
    a = np.array([1.0, 0.0, 0.0]) if abs(z[0]) < 0.9 else np.array([0.0, 1.0, 0.0])
    x = np.cross(a, z)
    x /= np.linalg.norm(x)
    R = np.stack([x, np.cross(z, x), z], axis=1) @ Rotation.from_rotvec([0, 0, roll]).as_matrix()
    qx, qy, qz, qw = Rotation.from_matrix(R).as_quat()
    return np.concatenate([pos, [qw, qx, qy, qz]])


def envelope_features(cam8, xp, n, rng):
    """n features seen from xp at random pixels 30 px inside the image, each first seen from a pose inside the
    visibility envelope: distance ratio in [0.55, 1.8], viewing direction turned by up to 40 degrees, any roll, with the
    feature up to 10 degrees off that camera's axis."""
    y, xo = np.zeros((n, 3)), np.zeros((n, 7))
    for k in range(n):
        y[k] = warp_ref_point(cam8, xp, rng)
        view = xp[:3] - y[k]
        turn = Rotation.from_rotvec(rng.standard_normal(3) * 1.0).as_matrix()
        axis = np.cross(view, turn @ view)
        ang = np.radians(rng.uniform(0, 40))
        dirn = Rotation.from_rotvec(axis / np.linalg.norm(axis) * ang).as_matrix() @ view
        pos = y[k] + dirn * rng.uniform(0.55, 1.8)
        off = Rotation.from_rotvec(rng.standard_normal(3) * np.radians(4)).as_matrix() @ (y[k] - pos)
        xo[k] = look_at(pos, pos + off, rng.uniform(-np.pi, np.pi))
    return y, xo


def warp_ref_point(cam8, xp, rng, margin=30):
    u, v = rng.uniform(margin, cam8[0] - 1 - margin), rng.uniform(margin, cam8[1] - 1 - margin)
    c0, c1 = warp_ref.unproject_point(cam8, u, v)
    zc = np.array([float(c0), float(c1), 1.0]) * rng.uniform(0.5, 3.0)
    return xp[:3] + np.array(warp_ref.rrw(xp)).T @ zc


def ctx_for(name, n, num_streams=1, **kw):
    sc = synth.make_scene(name, n_frames=1)
    cfg = sl2.config_for_scene(sc, num_streams=num_streams, max_features=n, **kw)
    return sl2.Context(cfg), sc.cam8


def check_against_restatement(ctx, s, cam8, y, xo, T, xp, idx=None):
    idx = np.arange(len(y)) if idx is None else np.asarray(idx)
    out, valid = ctx.warp_templates(s, idx, xp)
    want, wvalid = warp_ref.warp_templates(cam8, T[idx], y[idx], xo[idx], xp)
    assert (valid == wvalid).all() and out.tobytes() == want.tobytes()
    return valid


# ---- 1. the staged form against the restatement -------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["C1", "C3"])  # box 11 / 320 x 240, box 15 / 640 x 480, both with kd1 != 0
def test_warp_templates_equal_the_restatement(name):
    n = 200
    ctx, cam8 = ctx_for(name, n)
    rng = np.random.default_rng(11 if name == "C1" else 15)
    B = ctx.cfg.boxsize
    try:
        warped = 0
        for _ in range(3):
            xp = look_at(rng.uniform(-1, 1, 3), rng.uniform(-1, 1, 3) + [0, 0, 3.0], rng.uniform(-np.pi, np.pi))
            y, xo = envelope_features(cam8, xp, n, rng)
            T = rng.integers(0, 256, (n, B, B), dtype=np.uint8)
            ctx.set_features(0, y, xo, T)
            warped += int(check_against_restatement(ctx, 0, cam8, y, xo, T, xp).sum())
            # identity: every feature seen from its own xp_org
            check_against_restatement(ctx, 0, cam8, y, xo, T, xo[7], idx=[7])
            out, valid = ctx.warp_templates(0, [3, 9], xo[3])
            assert valid[0] == 1 and out[0].tobytes() == T[3].tobytes()
            # the camera turned away from the features: whatever each pixel gives, the same as the restatement
            away = look_at(xp[:3], 2 * xp[:3] - y.mean(axis=0), 0.3)
            check_against_restatement(ctx, 0, cam8, y, xo, T, away, idx=np.arange(20))
        assert warped >= 0.9 * 3 * n, warped
        # invalid by construction (tests/test_warp.py): a fronto-parallel plane behind the camera, and the camera in
        # the plane; the stored bytes, valid = 0
        y = np.array([[0.0, 0.0, 2.0]] * 2)
        xo = np.array([[0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0]] * 2)
        T = rng.integers(0, 256, (2, B, B), dtype=np.uint8)
        ctx.set_features(0, y, xo, T)
        c45 = np.cos(np.pi / 4)
        for bad in ([0, 0, 0, 0, 0, 1.0, 0], [-1.0, 0, 2.0, c45, 0, c45, 0]):
            v = check_against_restatement(ctx, 0, cam8, y, xo, T, np.array(bad))
            assert not v.any()
        out, valid = ctx.warp_templates(0, [], xp)
        assert out.shape == (0, B, B) and valid.shape == (0,)
    finally:
        ctx.close()


@pytest.mark.gpu
def test_capacity_256_and_a_stream_other_than_0():
    n = 256
    ctx, cam8 = ctx_for("C1", n, num_streams=3)
    rng = np.random.default_rng(256)
    try:
        xp = look_at(np.zeros(3), np.array([0.1, -0.1, 2.0]), 0.2)
        y, xo = envelope_features(cam8, xp, n, rng)
        T = rng.integers(0, 256, (n, 11, 11), dtype=np.uint8)
        ctx.set_features(2, y, xo, T)
        ctx.set_features(0, y[::-1], xo[::-1], T[::-1])
        v = check_against_restatement(ctx, 2, cam8, y, xo, T, xp, idx=np.arange(128, 256))
        assert v.sum() >= 100
        check_against_restatement(ctx, 2, cam8, y, xo, T, xp, idx=[255, 0, 200, 128, 127])
        ctx.set_stream_config(2, ctx.stream_config(2), kd1=3e-5, fku=240.0)  # stream 2's own camera
        check_against_restatement(ctx, 2, cam8_of(ctx, 2), y, xo, T, xp, idx=np.arange(0, 256, 3))
    finally:
        ctx.close()


# ---- rendered scenes in a context --------------------------------------------------------------------------------
def scene_ctx(scenes, max_features=None, n_select=None):
    sc = scenes[0]
    cfg = sl2.default_config()
    cfg.num_streams = len(scenes)
    cfg.width, cfg.height = int(sc.cam8[0]), int(sc.cam8[1])
    cfg.boxsize = sc.boxsize
    N = len(sc.y)
    cfg.max_features = max_features or N
    cfg.number_of_features_to_select = n_select or min(N, sl2.lib.SL2_MAX_MEASURED)
    cfg.search_tile_radius = 20
    cfg.fku, cfg.fkv, cfg.u0, cfg.v0, cfg.kd1, cfg.sd = [float(v) for v in sc.cam8[2:8]]
    cfg.delta_t = warp_scene.DT
    ctx = sl2.Context(cfg)
    for s, scn in enumerate(scenes):
        ctx.set_features(s, scn.y, scn.xp_org, scn.patches)
        ctx.set_state(s, scn.x0, scn.P0)
    return ctx


def frames_at(scenes, t):
    return np.stack([sc.frames[t] for sc in scenes])


SCENES = {}


def scene(kind):
    if kind not in SCENES:
        SCENES[kind] = warp_scene.make_warp_scene(kind)
    return SCENES[kind]


# ---- 2. the measure stage against the oracle's search with the restatement's templates ----------------------------
@pytest.mark.gpu
def test_measure_stage_equals_the_oracle_search_of_templates_warped_at_non_unit_q():
    """The search of a warp-on stream reads the restatement's templates at the predicted x[0:7], whose |q| drifts from
    1 (x is never renormalised), so the rays go through RRW^-1 and not RRW^T."""
    sc = scene("roll")
    ctx = scene_ctx([sc])
    cam8 = sc.cam8
    drift = 0.0
    try:
        ctx.set_stream_warp(0, 1)
        assert ctx.get_stream_warp(0) == 1
        for t in range(1, 13):
            ctx.set_frame(0, 0, sc.frames[t])
            ctx.ekf_predict(0)
            ctx.predict_measurements(0)
            x, _ = ctx.get_state(0)
            drift = max(drift, abs(float(np.dot(x[3:7], x[3:7])) - 1.0))
            cnt = ctx.make_measurements(0, 0)
            snap = sl2.read_snapshot(ctx.save_stream(0))
            nsel = snap["nsel"]
            jf = snap["job_feat"][:nsel]
            assert nsel > 0 and (jf >= 0).all()
            y = x[13:].reshape(-1, 3)
            wt, _ = warp_ref.warp_templates(cam8, sc.patches[jf], y[jf], snap["xp_org"][jf], x[:7])
            u, v, found, best = po.elliptical_search(sc.frames[t], wt, snap["job_centre"][:nsel],
                                                     snap["job_puinv"][:nsel])
            assert (snap["h"][jf] == snap["job_centre"][:nsel]).all()
            ok = found.astype(bool)
            assert (snap["found"][jf] == found).all(), t
            assert (snap["z_uv"][jf][ok] == np.stack([u, v], axis=1)[ok]).all(), t
            assert snap["best"][jf].tobytes() == best.tobytes(), t
            assert cnt == int(found.sum())
            ctx.ekf_update_measured(0)
        assert drift > 0.0
    finally:
        ctx.close()


# ---- 3. fused equals staged, with the consensus and two step groups -------------------------------------------------
@pytest.mark.gpu
def test_fused_equals_staged_with_consensus_and_two_groups():
    scenes = [scene("roll"), scene("approach")]
    fused, staged = scene_ctx(scenes), scene_ctx(scenes)
    try:
        fused.set_step_groups(2)
        for c in (fused, staged):
            for s in range(2):
                c.set_stream_warp(s, 1)
                c.set_stream_consensus(s, TAU)
        for t in range(1, 9):
            fused.set_frames(0, frames_at(scenes, t))
            fused.step(0)
            fused.sync()
            staged.set_frames(0, frames_at(scenes, t))
            for s in range(2):
                staged.ekf_predict(s)
                staged.predict_measurements(s)
                staged.make_measurements(s, 0)
                staged.ekf_update_measured(s)
            for s in range(2):
                assert_same_bytes(stream_result(staged, s, jacobians=True), stream_result(fused, s, jacobians=True),
                                  (t, s))
    finally:
        fused.close()
        staged.close()


# ---- 4. isolation and launches ---------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_warp_off_streams_are_untouched_and_one_launch_per_group():
    scenes = [scene("roll"), scene("approach"), scene("orbit"), scene("roll")]
    plain, mixed, toggled = scene_ctx(scenes), scene_ctx(scenes), scene_ctx(scenes)
    try:
        for c in (plain, mixed, toggled):
            c.set_step_groups(2)  # groups {0, 1} and {2, 3}
        mixed.set_stream_warp(1, 1)
        mixed.set_stream_warp(3, 1)
        for s in range(4):
            toggled.set_stream_warp(s, 1)
            toggled.set_stream_warp(s, 0)
        assert toggled.launch_count() == plain.launch_count()
        for t in range(1, 8):
            if t == 4:
                mixed.set_stream_warp(3, 0)  # only group A has a stream on from here
            l0, m0, g0 = plain.launch_count(), mixed.launch_count(), toggled.launch_count()
            for c in (plain, mixed, toggled):
                c.set_frames(0, frames_at(scenes, t))
                c.step(0)
                c.sync()
            extra = (mixed.launch_count() - m0) - (plain.launch_count() - l0)
            assert extra == (2 if t < 4 else 1), (t, extra)
            assert toggled.launch_count() - g0 == plain.launch_count() - l0
            for s in range(4):
                assert_same_bytes(stream_result(toggled, s, jacobians=True), stream_result(plain, s, jacobians=True),
                                  ("toggled", s, t))
            for s in (0, 2):
                assert_same_bytes(stream_result(mixed, s, jacobians=True), stream_result(plain, s, jacobians=True),
                                  ("mixed", s, t))
        assert [mixed.get_stream_warp(s) for s in range(4)] == [0, 1, 0, 0]
    finally:
        for c in (plain, mixed, toggled):
            c.close()


# ---- 5. snapshots ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_snapshots_do_not_carry_the_setting():
    sc = scene("roll")
    on, off, ref_on, ref_off = (scene_ctx([sc, sc]) for _ in range(4))
    try:
        on.set_stream_warp(0, 1)
        ref_on.set_stream_warp(1, 1)
        for t in range(1, 5):  # both slots of `on` and `off` hold the same stream: stream 0 of `on` runs warped
            for c in (on, off):
                c.set_frames(0, frames_at([sc, sc], t))
                c.step(0)
                c.sync()
        b_on, b_off = on.save_stream(0), off.save_stream(0)
        assert b_on != b_off  # the warped run differs ...
        assert on.save_stream(1) == off.save_stream(1)  # ... and the setting itself changes no snapshot byte
        # the stream saved from a warp-on slot into a warp-off slot, and the reverse; the loads leave the settings
        off.load_stream(1, b_on)
        on.load_stream(0, b_off)
        assert [on.get_stream_warp(s) for s in range(2)] == [1, 0] and off.get_stream_warp(1) == 0
        # references: stream 0 of ref_off continues b_on unwarped, stream 1 of ref_on continues b_off warped
        ref_off.load_stream(0, b_on)
        ref_on.load_stream(1, b_off)
        for t in range(5, 9):
            for c in (on, off, ref_on, ref_off):
                c.set_frames(0, frames_at([sc, sc], t))
                c.step(0)
                c.sync()
            assert_same_bytes(stream_result(off, 1), stream_result(ref_off, 0), ("on -> off", t))
            assert_same_bytes(stream_result(on, 0), stream_result(ref_on, 1), ("off -> on", t))
    finally:
        for c in (on, off, ref_on, ref_off):
            c.close()


# ---- 6. rejected arguments -------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_rejected_arguments_change_nothing():
    sc = scene("roll")
    ctx = scene_ctx([sc, sc])
    N, B = len(sc.y), sc.boxsize
    try:
        ctx.set_stream_warp(1, 1)
        before = [stream_result(ctx, s) for s in range(2)]
        launches = ctx.launch_count()
        for s, v in ((-1, 1), (2, 1), (0, 2), (1, -1), (0, 255)):
            with pytest.raises(sl2.Sl2Error):
                ctx.set_stream_warp(s, v)
        with pytest.raises(sl2.Sl2Error):
            ctx.get_stream_warp(2)
        assert ctx.L.sl2_get_stream_warp(ctx.h, 0, None) == -1
        assert [ctx.get_stream_warp(s) for s in range(2)] == [0, 1]
        xp = sc.poses[0].copy()
        bad_xp = [np.where(np.arange(7) == 2, np.nan, xp), np.where(np.arange(7) == 5, np.inf, xp),
                  np.concatenate([xp[:3], np.zeros(4)])]
        for x in bad_xp:
            with pytest.raises(sl2.Sl2Error):
                ctx.warp_templates(0, [0, 1], x)
        for idx in ([N], [-1], [0, N + 3]):
            with pytest.raises(sl2.Sl2Error):
                ctx.warp_templates(0, idx, xp)
        with pytest.raises(sl2.Sl2Error):
            ctx.warp_templates(2, [0], xp)
        out = np.full((2, B, B), 7, np.uint8)
        valid = np.full(2, 9, np.uint8)
        fi = np.array([0, 1], np.int32)
        L = ctx.L
        assert L.sl2_warp_templates(ctx.h, 0, N + 1, fi.ctypes.data, xp.ctypes.data, out.ctypes.data,
                                    valid.ctypes.data) == -1
        assert L.sl2_warp_templates(ctx.h, 0, -1, fi.ctypes.data, xp.ctypes.data, out.ctypes.data, None) == -1
        for args in ((None, xp.ctypes.data, out.ctypes.data), (fi.ctypes.data, None, out.ctypes.data),
                     (fi.ctypes.data, xp.ctypes.data, None)):
            assert L.sl2_warp_templates(ctx.h, 0, 2, *args, valid.ctypes.data) == -1
        assert (out == 7).all() and (valid == 9).all()
        assert ctx.launch_count() == launches
        for s in range(2):
            assert_same_bytes(stream_result(ctx, s), before[s], s)
    finally:
        ctx.close()


# ---- 7. the capability: tracking through roll, approach and orbit ---------------------------------------------------
def track(sc):
    """The scene's trajectory tracked by one context whose stream 0 has the warp off and stream 1 on: per step and
    stream the fraction of selected features matched, and the map sizes; the final states."""
    ctx = scene_ctx([sc, sc])
    try:
        ctx.set_stream_warp(1, 1)
        frac, nfeat = np.zeros((len(sc.frames) - 1, 2)), np.zeros((len(sc.frames) - 1, 2), np.int64)
        for t in range(1, len(sc.frames)):
            ctx.set_frames(0, np.stack([sc.frames[t]] * 2))
            ctx.step(0)
            ctx.sync()
            for s in range(2):
                f = ctx.features(s)
                sel = f["select_rank"] >= 0
                frac[t - 1, s] = ((f["flags"] & 2) > 0)[sel].sum() / max(1, sel.sum())
                nfeat[t - 1, s] = ctx.num_features(s)
        return frac, nfeat, [ctx.get_state(s)[0] for s in range(2)]
    finally:
        ctx.close()


CAPABILITY = {}


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["roll", "approach"])
def test_warp_keeps_tracking_where_the_stored_templates_fail(kind):
    sc = scene(kind)
    frac, nfeat, (x_off, x_on) = track(sc)
    truth = sc.poses[-1]
    pos_err = float(np.linalg.norm(x_on[:3] - truth[:3]))
    ang_err = warp_scene.angle_deg(x_on[3:7], truth[3:])
    CAPABILITY[kind] = dict(min_on=frac[:, 1].min(), end_off=frac[-1, 0], pos_err=pos_err, ang_err=ang_err)
    print(kind, CAPABILITY[kind])
    assert frac[:, 1].min() >= 0.9, frac[:, 1]
    assert (nfeat[:, 1] == len(sc.y)).all()
    assert pos_err <= 0.02 and ang_err <= 1.0, (pos_err, ang_err)
    assert frac[-1, 0] < 0.5, frac[:, 0]


@pytest.mark.gpu
def test_orbit_warp_matches_at_least_as_often():
    """The orbit views the plane obliquely, where the assumed normal (towards the first camera) differs from the
    plane's by up to the feature's angle off the frame-0 axis: the warp helps without reaching the roll and approach's
    rates (DESIGN.md §4).  It never matches fewer features than the stored templates, and keeps the map."""
    sc = scene("orbit")
    frac, nfeat, (x_off, x_on) = track(sc)
    truth = sc.poses[-1]
    pos_err = float(np.linalg.norm(x_on[:3] - truth[:3]))
    ang_err = warp_scene.angle_deg(x_on[3:7], truth[3:])
    print("orbit", dict(on=frac[:, 1].round(2).tolist(), off=frac[:, 0].round(2).tolist(), pos_err=pos_err,
                        ang_err=ang_err, nfeat=nfeat[-1].tolist()))
    assert frac[:, 1].sum() >= frac[:, 0].sum()
    assert nfeat[-1, 1] >= nfeat[-1, 0]
