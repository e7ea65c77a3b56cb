"""The iterated EKF update on the device (sl2_set_stream_iterated; csrc/iterate.cu iterate_kernel and the iteration's
upd_hp / upd_chol passes): x, P and the results of sl2_ekf_update_measured against the update from its definition
(tests/iterate_truth.py), a tolerance that stops at once against the plain update byte for byte, off streams against
a context without the feature, the launch count, fused against staged, two step groups, a snapshot continued in an
iterated slot, the other per-stream features on together, and rejected arguments."""
import numpy as np
import pytest

import iterate_ref as ref
import iterate_truth as tr
import scenelib2_b200 as sl2
import update_truth as ut
from gpu_util import CAMS_320, assert_same_bytes, ctx_from_scenes, large_variant, stream_result
from rescue_scene import rescue_scene
from rescue_truth import Ext
from test_gpu_update_accuracy import C, FLOOR

pytestmark = pytest.mark.gpu


def staged_measure(ctx, s, slot=0):
    ctx.ekf_predict(s)
    ctx.predict_measurements(s)
    ctx.make_measurements(s, slot)


def device_rows(ctx, s):
    """x0, P0 and the measured rows of stream s after its measurement: feats (rank order), z, Rvar and L_0 (h, Hxp,
    Hy) as the prediction left them; cam8 of the stream."""
    x0, P0 = ctx.get_state(s)
    f = ctx.features(s)
    J, Jy, R, _ = ctx.feature_jacobians(s)
    sel = np.flatnonzero((f["flags"] & 3) == 3)
    feats = [int(i) for i in sel[np.argsort(f["select_rank"][sel])]]
    Hxp = np.array([J[i].reshape(13, 2).T[:, :7] for i in feats])
    Hy = np.array([Jy[i].reshape(3, 2).T for i in feats])
    sc = ctx.stream_config(s)
    cam8 = np.array([sc.width, sc.height, sc.fku, sc.fkv, sc.u0, sc.v0, sc.kd1, sc.sd], np.float64)
    return x0, P0, feats, f["z"][feats], R[feats, 0], (f["h"][feats], Hxp, Hy), cam8


def scene_cases():
    yield "C1", rescue_scene("C1", new=(1, 3), sigma=0.08)
    yield "C2", rescue_scene("C2", new=(0, 2, 5), sigma=0.08)
    yield "C3", rescue_scene("C3", new=(1, 4), sigma=0.08)
    yield "C4", rescue_scene("C4", new=(0, 3, 7, 9), sigma=0.08)
    yield "cap256", large_variant(256, 256)
    yield "own_camera", rescue_scene("C2", new=(0, 2), sigma=0.08, camera=CAMS_320[1])


@pytest.mark.parametrize("N", [1, 2, 3])
def test_measured_update_matches_the_truth(N):
    for name, sc in scene_cases():
        ctx = ctx_from_scenes([sc])
        ctx.set_stream_iterated(0, N, 0.0)
        ctx.set_frames(0, sc.frames[0][None])
        staged_measure(ctx, 0)
        x0, P0, feats, z, Rvar, L0, cam8 = device_rows(ctx, 0)
        assert len(feats) > 0, name
        ctx.ekf_update_measured(0)
        xg, Pg = ctx.get_state(0)
        it, st, _ = ctx.iterated_results(0, 1)
        t = tr.iterated_truth(Ext, cam8, x0, P0, feats, z, Rvar, N, 0.0, L0)
        assert (int(it[0]), int(st[0])) == (t["iterations"], t["status"]), name
        fin = tr.final_truth(x0, P0, feats, t["L"], z, Rvar)
        # the yardstick: the same definition in FP64 (the restatement's iteration, then a LAPACK update at its
        # linearisation), whose tables carry their own rounding like the device's
        r = ref.iterated(cam8, x0, P0, feats, z, Rvar, N, 0.0, L0)
        assert (r["iterations"], r["status"]) == (t["iterations"], t["status"]), name
        K = len(feats)
        Hxv = np.zeros((2 * K, 13))
        h, Hxp, Hy = r["L"]
        Hxv[:, :7] = Hxp.reshape(2 * K, 7)
        ch = ut.chol64_update(x0, P0, feats, Hxv, Hy.reshape(2 * K, 3), [np.eye(2) * v for v in Rvar],
                              (z - h).reshape(-1))
        ex, eP = ut.update_err(xg, Pg, fin.x, fin.P)
        cx, cP = ut.update_err(ch.x, ch.P, fin.x, fin.P)
        assert ex <= max(C * cx, FLOOR) and eP <= max(C * cP, FLOOR), (name, N, ex, cx, eP, cP)
        assert np.abs(Pg - Pg.T).max() == 0.0
        # the getters keep the step's prediction
        assert ctx.features(0)["h"][feats].tobytes() == L0[0].tobytes()
        ctx.close()


# A tolerance between the truth's steps, so that the iteration converges at a pass i >= 1 and the final update reads
# L_i: the decision, the reported delta_i and the state after the final update against the truth.  A case whose delta_i
# and the smallest earlier step lie within a factor of 1.01 of each other is skipped (the band around tol; the device's
# deltas differ from the truth's by far less, see the check of last_delta).
DELTA_RTOL = 1e-6
BAND = 1.01


def test_convergence_decision_matches_the_truth():
    checked = 0
    for name, sc in scene_cases():
        ctx = ctx_from_scenes([sc])
        ctx.set_frames(0, sc.frames[0][None])
        ctx.set_stream_iterated(0, 4, 0.0)
        staged_measure(ctx, 0)
        x0, P0, feats, z, Rvar, L0, cam8 = device_rows(ctx, 0)
        t0 = tr.iterated_truth(Ext, cam8, x0, P0, feats, z, Rvar, 4, 0.0, L0)
        d = [float(v) for v in t0["deltas"]]
        pick = next((i for i in range(1, len(d)) if d[i] * BAND < min(d[:i])), None)
        if pick is None:
            continue
        tol = float(np.sqrt(d[pick] * min(d[:pick])))
        ctx.set_stream_iterated(0, 4, tol)
        ctx.ekf_update_measured(0)
        it, st, dl = ctx.iterated_results(0, 1)
        t = tr.iterated_truth(Ext, cam8, x0, P0, feats, z, Rvar, 4, tol, L0)
        assert (t["iterations"], t["status"]) == (pick, 1)
        assert (int(it[0]), int(st[0])) == (pick, 1), name
        assert abs(dl[0] - d[pick]) <= DELTA_RTOL * d[pick], (name, dl[0], d[pick])
        fin = tr.final_truth(x0, P0, feats, t["L"], z, Rvar)
        r = ref.iterated(cam8, x0, P0, feats, z, Rvar, 4, tol, L0)
        assert (r["iterations"], r["status"]) == (pick, 1)
        K = len(feats)
        Hxv = np.zeros((2 * K, 13))
        h, Hxp, Hy = r["L"]
        Hxv[:, :7] = Hxp.reshape(2 * K, 7)
        ch = ut.chol64_update(x0, P0, feats, Hxv, Hy.reshape(2 * K, 3), [np.eye(2) * v for v in Rvar],
                              (z - h).reshape(-1))
        xg, Pg = ctx.get_state(0)
        ex, eP = ut.update_err(xg, Pg, fin.x, fin.P)
        cx, cP = ut.update_err(ch.x, ch.P, fin.x, fin.P)
        assert ex <= max(C * cx, FLOOR) and eP <= max(C * cP, FLOOR), (name, ex, cx, eP, cP)
        checked += 1
        ctx.close()
    assert checked >= 3


def _run(scenes, T, setup=None, groups=1, records=0):
    ctx = ctx_from_scenes(scenes)
    if groups > 1:
        ctx.set_step_groups(groups)
    if records:
        ctx.enable_records(records)
    if setup:
        setup(ctx)
    out = []
    for t in range(T):
        ctx.set_frames(0, np.stack([sc.frames[t] for sc in scenes]))
        ctx.step(0)
        ctx.sync()
    for s in range(len(scenes)):
        out.append(stream_result(ctx, s))
    return ctx, out


def _scenes(k=4, T=6):
    return [rescue_scene("C2", stream_id=s, new=(0, 3), sigma=0.06, n_frames=T) for s in range(k)]


def test_large_tol_is_byte_identical_to_the_plain_update():
    scenes = _scenes(2)
    on, a = _run(scenes, 6, lambda c: [c.set_stream_iterated(s, 3, 1e300) for s in range(2)], records=8)
    off, b = _run(scenes, 6, records=8)
    for s in range(2):
        assert_same_bytes(a[s], b[s], s)
    assert on.records().tobytes() == off.records().tobytes()
    it, st, _ = on.iterated_results()
    assert (it == 0).all() and (st == 1).all()


def test_off_streams_and_launch_count():
    scenes = _scenes(3)
    on, a = _run(scenes, 1, lambda c: c.set_stream_iterated(1, 2, 0.0))
    off, b = _run(scenes, 1)
    for s in (0, 2):
        assert_same_bytes(a[s], b[s], s)
    assert on.iterated_results()[1].tolist() == [0, 2, 0]
    for ctx in (on, off):
        ctx.set_frames(0, np.stack([sc.frames[1] for sc in scenes]))
    l0, l1 = on.launch_count(), off.launch_count()
    on.step(0), off.step(0)
    on.sync(), off.sync()
    assert (on.launch_count() - l0) - (off.launch_count() - l1) == 3 * 2


def _iter_setting(s):
    """A per-stream mix: N = 1, 2, 3 in turn, tol 0 on odd streams and 1e-3 on even ones."""
    return 1 + s % 3, (0.0 if s % 2 else 1e-3)


def run_regime(regime, scs, T):
    B = len(scs)
    ctx = ctx_from_scenes(scs)
    for s in range(B):
        ctx.set_stream_iterated(s, *_iter_setting(s))
    if regime == "groups":
        ctx.set_step_groups(2)
    results = []
    for t in range(T):
        fr = np.stack([sc.frames[t] for sc in scs])
        if regime == "host_async":
            ctx.step_host_async(0, fr.ctypes.data, 0)
            ctx.wait_slot(0)
        elif regime == "host":
            ctx.step_host(0, fr.ctypes.data, 0)
        else:
            ctx.set_frames(0, fr)
            ctx.step(0)
        ctx.sync()
        results.append(ctx.iterated_results())
    return [stream_result(ctx, s, jacobians=True) for s in range(B)], results


def test_every_launch_regime_gives_the_same_bytes():
    """Serial order, two step groups, the host step and the async host step of 4 streams; and stream 2 alone in a
    context of its own, whose launches cover one camera stream and so run with programmatic dependent launch
    (sl2_use_pdl: fewer than SL2_PDL_AUTO_STREAMS = 2 streams)."""
    T = 6
    scs = _scenes(4, T=T)
    base, rb = run_regime("serial", scs, T)
    assert any((st == 1).any() for _, st, _ in rb) and any((it > 0).any() for it, _, _ in rb)
    for regime in ("groups", "host", "host_async"):
        got, rg = run_regime(regime, scs, T)
        for s in range(4):
            assert_same_bytes(got[s], base[s], (regime, s))
        for a, b in zip(rg, rb):
            assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b)), regime
    ctx = ctx_from_scenes([scs[2]])
    ctx.set_stream_iterated(0, *_iter_setting(2))
    for t in range(T):
        ctx.set_frame(0, 0, scs[2].frames[t])
        ctx.step(0)
        ctx.sync()
    assert_same_bytes(stream_result(ctx, 0, jacobians=True), base[2], "single stream (PDL)")


def test_a_stream_of_a_large_mixed_batch():
    """Stream 173 of a 264-stream context whose streams mix settled C4 maps with maps holding uncertain new features,
    and iteration settings (every third stream on, each with its own N and tol), has the bytes of the same stream alone
    in a context."""
    T = 4
    B, pick = 264, 173
    scs = [rescue_scene("C4", stream_id=s, n_frames=T, new=(0, 3) if s % 2 else (), sigma=0.06) for s in range(B)]
    ctx = ctx_from_scenes(scs)
    for s in range(0, B, 3):
        ctx.set_stream_iterated(s, *_iter_setting(s))
    ctx.set_stream_iterated(pick, 3, 0.0)
    for t in range(T):
        ctx.set_frames(0, np.stack([sc.frames[t] for sc in scs]))
        ctx.step(0)
    ctx.sync()
    alone = ctx_from_scenes([scs[pick]])
    alone.set_stream_iterated(0, 3, 0.0)
    for t in range(T):
        alone.set_frame(0, 0, scs[pick].frames[t])
        alone.step(0)
    alone.sync()
    assert_same_bytes(stream_result(ctx, pick, jacobians=True), stream_result(alone, 0, jacobians=True), "pick")
    assert ctx.iterated_results(pick, 1)[0].tolist() == alone.iterated_results(0, 1)[0].tolist() == [3]


def test_fused_equals_staged():
    """Every step of the fused step against predict, measure and sl2_ekf_update_measured; the scene's features are all
    found, so nothing reaches the cull's threshold in these steps (asserted)."""
    T = 5
    sc = rescue_scene("C2", n_frames=T, new=(0, 3), sigma=0.06)
    fused, staged = ctx_from_scenes([sc]), ctx_from_scenes([sc])
    for c in (fused, staged):
        c.set_stream_iterated(0, 2, 1e-4)
    for t in range(T):
        fused.set_frame(0, 0, sc.frames[t])
        fused.step(0)
        fused.sync()
        staged.set_frame(0, 0, sc.frames[t])
        staged_measure(staged, 0)
        staged.ekf_update_measured(0)
        assert fused.num_features(0) == staged.num_features(0) == sc.n_features, t
        assert_same_bytes(stream_result(fused, 0, jacobians=True), stream_result(staged, 0, jacobians=True), t)
        assert all(a.tobytes() == b.tobytes() for a, b in zip(fused.iterated_results(), staged.iterated_results()))


def test_snapshot_continues_in_an_iterated_slot():
    scenes = _scenes(2, T=6)
    a, _ = _run(scenes, 3, lambda c: [c.set_stream_iterated(s, 2, 0.0) for s in range(2)])
    b = ctx_from_scenes(scenes)
    b.set_stream_iterated(0, 2, 0.0)
    b.set_stream_iterated(1, 2, 0.0)
    b.load_streams(a.save_streams())
    for t in range(3, 6):
        fr = np.stack([sc.frames[t] for sc in scenes])
        for c in (a, b):
            c.set_frames(0, fr)
            c.step(0)
            c.sync()
    for s in range(2):
        assert_same_bytes(stream_result(a, s), stream_result(b, s), s)


def test_with_every_other_stream_feature_on():
    scenes = _scenes(2, T=6)

    def setup(c):
        for s in range(2):
            c.set_stream_consensus(s, 2.5)
            c.set_stream_rescue(s, 5.991)
            c.set_stream_subpixel(s, 1)
            c.set_stream_warp(s, 1)
            c.set_stream_gyro(s, 1)
            c.set_stream_iterated(s, 2, 1e-3)
    ctx, out = _run(scenes, 4, setup)
    _, out2 = _run(scenes, 4, setup, groups=2)
    for s in range(2):
        assert np.isfinite(out[s]["x"]).all() and np.isfinite(out[s]["P"]).all()
        assert_same_bytes(out[s], out2[s], s)
    assert set(ctx.iterated_results()[1].tolist()) <= {1, 2, 3}


def test_rejected_arguments_change_nothing():
    """Rejected settings leave the setting, and so the steps that follow, as they were: a context that received them
    runs byte for byte like one that did not."""
    scs = _scenes(2, T=3)
    ctx, ref_ctx = ctx_from_scenes(scs), ctx_from_scenes(scs)
    for c in (ctx, ref_ctx):
        c.set_stream_iterated(0, 2, 0.5)
    for bad in ((-1, 0.0, 0), (9, 0.0, 0), (2, float("nan"), 0), (2, -1.0, 0), (2, float("inf"), 0), (2, 0.0, 1)):
        for s in (0, 1):
            with pytest.raises(sl2.Sl2Error):
                ctx.set_stream_iterated(s, *bad[:2], reserved=bad[2])
        assert ctx.stream_iterated(0) == (2, 0.5) and ctx.stream_iterated(1) == (0, 0.0)
    with pytest.raises(sl2.Sl2Error):
        ctx.set_stream_iterated(2, 1, 0.0)
    with pytest.raises(sl2.Sl2Error):
        ctx.iterated_results(0, 3)
    for t in range(3):
        for c in (ctx, ref_ctx):
            c.set_frames(0, np.stack([sc.frames[t] for sc in scs]))
            c.step(0)
            c.sync()
    for s in range(2):
        assert_same_bytes(stream_result(ctx, s, jacobians=True), stream_result(ref_ctx, s, jacobians=True), s)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(ctx.iterated_results(), ref_ctx.iterated_results()))
