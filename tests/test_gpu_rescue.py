"""The consensus rescue on the device (sl2_set_stream_rescue, csrc/rescue.cu rescue_kernel and the second update) on
settled maps with uncertain new features and distractors (tests/rescue_scene.py).  A match is correct iff
z = pix + shift[t]."""
import math

import numpy as np
import pytest

import rescue_oracle as ro
import rescue_ref
import rescue_truth as rt
import scenelib2_b200 as sl2
from gpu_util import (assert_same_bytes, assert_state_close, check_streams_against_oracle, ctx_from_scenes,
                      large_variant, step_frames, stream_result)
from rescue_scene import rescue_scene

TAU = 2.5
CHI2 = 5.991


def _cam8(ctx, s):
    c = ctx.stream_config(s)
    return np.array([c.width, c.height, c.fku, c.fkv, c.u0, c.v0, c.kd1, c.sd], np.float64)


def _scene(name="C2", stream_id=0, T=8, nf=None, new=None, wrong=None, sigma=0.03):
    nf = nf or (50 if name == "C2" else 100)
    new = range(nf - 8, nf) if new is None else new
    wrong = [3, nf // 2] if wrong is None else wrong
    return rescue_scene(name, stream_id=stream_id, n_frames=T, n_features=nf, new=new, sigma=sigma, wrong=wrong)


def _rank_order(f, mask):
    idx = np.flatnonzero((f["select_rank"] >= 0) & mask)
    return idx[np.argsort(f["select_rank"][idx])]


def staged_update_1(clone, blob, frame):
    """The stream of `blob` in the one-stream context `clone` (consensus on, rescue off) through the staged predict,
    search, consensus and update 1: -> x', P', the rejected features in rank order and their z."""
    clone.load_stream(0, blob)
    clone.set_frame(0, 0, frame)
    clone.ekf_predict(0)
    clone.predict_measurements(0)
    clone.make_measurements(0, 0)
    f = clone.features(0)
    J, Jy, R, nu = clone.feature_jacobians(0)
    x0, P0 = clone.get_state(0)
    inl = _rank_order(f, (f["flags"] & 2) > 0)
    rej = _rank_order(f, (f["flags"] & 4) > 0)
    pre = dict(x=x0, P=P0, inl=inl, S=f["S"][inl].reshape(-1, 2, 2).transpose(0, 2, 1), nu=nu[inl], z_inl=f["z"][inl])
    clone.ekf_update_measured(0)
    x, P = clone.get_state(0)
    return x, P, rej, f["z"][rej], pre


# ---- off means off -------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_off_streams_unchanged_and_six_launches_per_group():
    T = 6
    scenes = [_scene(stream_id=s, T=T) for s in range(4)]
    never, toggled, on = (ctx_from_scenes(scenes) for _ in range(3))
    try:
        for c in (never, toggled, on):
            for s in range(4):
                c.set_stream_consensus(s, TAU if s != 3 else 0.0)
        toggled.set_stream_rescue(1, CHI2)
        toggled.set_stream_rescue(1, 0.0)
        on.set_stream_rescue(1, CHI2)
        on.set_stream_rescue(3, CHI2)  # consensus off: unaffected
        rescued_any = False
        for t in range(T):
            n0, t0, o0 = never.launch_count(), toggled.launch_count(), on.launch_count()
            fs = np.stack([sc.frames[t] for sc in scenes])
            for c in (never, toggled, on):
                step_frames(c, fs)
            assert toggled.launch_count() - t0 == never.launch_count() - n0
            assert on.launch_count() - o0 == never.launch_count() - n0 + 6
            for s in range(4):
                assert_same_bytes(stream_result(toggled, s, jacobians=True), stream_result(never, s, jacobians=True),
                                  (t, s))
                if s != 1:
                    assert_same_bytes(stream_result(on, s, jacobians=True), stream_result(never, s, jacobians=True),
                                      (t, s))
            if stream_result(on, 1)["x"].tobytes() != stream_result(never, 1)["x"].tobytes():
                rescued_any = True
        assert rescued_any
    finally:
        for c in (never, toggled, on):
            c.close()


# ---- the device's decisions against the restatement ----------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["C2", "C4"])
def test_decisions_equal_the_restatement(name):
    T = 6
    sc = _scene(name, T=T)
    ctx, clone = ctx_from_scenes([sc]), ctx_from_scenes([sc])
    try:
        ctx.set_stream_consensus(0, TAU)
        ctx.set_stream_rescue(0, CHI2)
        clone.set_stream_consensus(0, TAU)
        cam8 = _cam8(ctx, 0)
        seen = 0
        for t in range(T):
            x, P, rej, z, _ = staged_update_1(clone, ctx.save_stream(0), sc.frames[t])
            ok, q, preds = rescue_ref.gate(cam8, x, P, 13 + 3 * rej, z, CHI2)
            step_frames(ctx, sc.frames[t][None])
            f = ctx.features(0)
            got = ((f["flags"][rej] & 2) > 0) if rej.size else np.zeros(0, bool)
            assert (got == ok).all(), (t, rej, q)
            assert ((f["flags"][rej[~ok]] & 4) > 0).all()
            for j in np.flatnonzero(ok):
                assert f["h"][rej[j]].tobytes() == preds[j]["h"].tobytes()
                assert f["S"][rej[j]].tobytes() == preds[j]["S"].T.reshape(4).tobytes()
            seen += int(ok.sum())
        assert seen > 0
    finally:
        ctx.close()
        clone.close()


@pytest.mark.gpu
def test_chi2_knife_edge_on_the_device():
    sc = _scene("C2", T=2)
    ctx, clone = ctx_from_scenes([sc]), ctx_from_scenes([sc])
    try:
        clone.set_stream_consensus(0, TAU)
        blob = ctx.save_stream(0)
        x, P, rej, z, _ = staged_update_1(clone, blob, sc.frames[0])
        _, q, _ = rescue_ref.gate(_cam8(ctx, 0), x, P, 13 + 3 * rej, z, CHI2)
        j = int(np.flatnonzero(np.isfinite(q))[0])
        for chi2, want in ((q[j], True), (np.nextafter(q[j], -np.inf), False)):
            ctx.load_stream(0, blob)
            ctx.set_stream_consensus(0, TAU)
            ctx.set_stream_rescue(0, chi2)
            step_frames(ctx, sc.frames[0][None])
            assert bool(ctx.features(0)["flags"][rej[j]] & 2) == want
    finally:
        ctx.close()
        clone.close()


# ---- the whole step against the rescue oracle -----------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["C2", "C4"])
def test_whole_step_matches_the_rescue_oracle(name):
    T = 20
    sc = _scene(name, T=T, new=range(40, 48) if name == "C2" else range(92, 100))
    ctx = ctx_from_scenes([sc])
    o = ro.slam_from_scene(sc, TAU, CHI2)
    try:
        ctx.set_stream_consensus(0, TAU)
        ctx.set_stream_rescue(0, CHI2)
        rescued = 0
        for t in range(T):
            step_frames(ctx, sc.frames[t][None])
            check_streams_against_oracle(ctx, [o], [0], lambda s: sc, t)
            rescued += len(o.rescued())
        assert rescued > 0
        # through a cull: the distractors' features were deleted (the second update's finish counted the cull)
        assert o.num_features < sc.n_features
        assert not set(o.features()["label"].tolist()) & {3, sc.n_features // 2}
    finally:
        ctx.close()


# ---- records --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_records_hold_the_sums_of_both_updates():
    T = 4
    sc = _scene("C2", T=T)
    ctx, clone = ctx_from_scenes([sc]), ctx_from_scenes([sc])
    try:
        ctx.set_stream_consensus(0, TAU)
        ctx.set_stream_rescue(0, CHI2)
        clone.set_stream_consensus(0, TAU)
        ctx.enable_records(T)
        cam8 = _cam8(ctx, 0)
        two = 0
        for t in range(T):
            x, P, rej, z, pre = staged_update_1(clone, ctx.save_stream(0), sc.frames[t])
            ok, _, preds = rescue_ref.gate(cam8, x, P, 13 + 3 * rej, z, CHI2)
            step_frames(ctx, sc.frames[t][None])
            r = ctx.records(0, 1, 1)[0, 0]
            # update 1 in NumPy: S1 = H P H^T + R of the inliers, from the device's own S blocks and the cross terms
            k1 = pre["inl"].size
            nis1, ld1 = 0.0, 0.0
            if k1:
                S1 = _joint_S(cam8, pre["x"], pre["P"], pre["inl"])
                nu1 = pre["nu"].reshape(-1)
                nis1 = float(nu1 @ np.linalg.solve(S1, nu1))
                ld1 = float(np.linalg.slogdet(S1)[1])
            res = rej[ok]
            nis2, ld2 = 0.0, 0.0
            if res.size:
                two += 1
                S2 = _joint_S(cam8, x, P, res)
                nu2 = np.concatenate([z[j] - preds[j]["h"] for j in np.flatnonzero(ok)])
                nis2 = float(nu2 @ np.linalg.solve(S2, nu2))
                ld2 = float(np.linalg.slogdet(S2)[1])
            assert r["m"] == 2 * (k1 + res.size) and r["nmeas"] == k1 + res.size, t
            assert abs(r["nis"] - (nis1 + nis2)) <= 1e-9 * max(1.0, nis1 + nis2), (t, r["nis"], nis1 + nis2)
            assert abs(r["logdet_s"] - (ld1 + ld2)) <= 1e-9 * max(1.0, abs(ld1 + ld2)), t
        assert two > 0
    finally:
        ctx.close()
        clone.close()


def _joint_S(cam8, x, P, feats):
    """H P H^T + R of the features `feats` (rank order) predicted at x, P (the restatement's Jacobians)."""
    n = x.size
    H = np.zeros((2 * len(feats), n))
    R = np.zeros(2 * len(feats))
    for a, i in enumerate(feats):
        p = rescue_ref.predict(cam8, x, x[13 + 3 * i:16 + 3 * i], P, 13 + 3 * i)
        H[2 * a:2 * a + 2, 0:7] = p["dxp"]
        H[2 * a:2 * a + 2, 13 + 3 * i:16 + 3 * i] = p["dy"]
        R[2 * a:2 * a + 2] = p["var"]
    return H @ P @ H.T + np.diag(R)


# ---- staged equals fused, snapshots, launch regimes --------------------------------------------------------------------
@pytest.mark.gpu
def test_staged_equals_fused():
    T = 6
    sc = _scene("C2", T=T)
    fused, staged = ctx_from_scenes([sc]), ctx_from_scenes([sc])
    try:
        for c in (fused, staged):
            c.set_stream_consensus(0, TAU)
            c.set_stream_rescue(0, CHI2)
        for t in range(T):
            step_frames(fused, sc.frames[t][None])
            staged.set_frame(0, 0, sc.frames[t])
            staged.ekf_predict(0)
            staged.predict_measurements(0)
            staged.make_measurements(0, 0)
            staged.ekf_update_measured(0)
            # no feature reaches minimum_attempted_measurements_of_feature in T < 10 steps: the fused step's cull
            # deletes nothing, so every step is compared
            assert_same_bytes(stream_result(staged, 0, jacobians=True), stream_result(fused, 0, jacobians=True), t)
        assert fused.num_features(0) == sc.n_features
    finally:
        fused.close()
        staged.close()


@pytest.mark.gpu
def test_same_bytes_in_every_launch_regime():
    """serial, two step groups, sl2_step_host_async and a single stream (PDL) give the same bytes."""
    T = 5
    scenes = [_scene(stream_id=s, T=T) for s in range(3)]
    results = {}
    for regime in ("serial", "groups", "async", "single"):
        if regime == "single":
            ctx = ctx_from_scenes([scenes[1]])
        else:
            ctx = ctx_from_scenes(scenes)
        try:
            ns = 1 if regime == "single" else 3
            for s in range(ns):
                ctx.set_stream_consensus(s, TAU)
                ctx.set_stream_rescue(s, CHI2)
            if regime == "groups":
                ctx.set_step_groups(2)
            for t in range(T):
                fs = np.stack([scenes[1].frames[t]] if ns == 1 else [sc.frames[t] for sc in scenes])
                if regime == "async":
                    fs = np.ascontiguousarray(fs, np.uint8)
                    xv = np.zeros((ns, 13))
                    ctx.step_host_async(0, fs.ctypes.data, xv.ctypes.data)
                    ctx.wait_slot(0)
                    ctx.sync()
                else:
                    step_frames(ctx, fs)
            results[regime] = stream_result(ctx, 0 if ns == 1 else 1, jacobians=True)
        finally:
            ctx.close()
    for regime in ("groups", "async", "single"):
        assert_same_bytes(results[regime], results["serial"], regime)


@pytest.mark.gpu
def test_snapshots_continue_bit_for_bit():
    T = 8
    sc = _scene("C2", T=T)
    a, b = ctx_from_scenes([sc, sc]), ctx_from_scenes([sc, sc])
    try:
        for c in (a, b):
            for s in range(2):
                c.set_stream_consensus(s, TAU)
            c.set_stream_rescue(0, CHI2)
        for t in range(T):
            if t == 3:
                b.load_streams(a.save_streams())
            step_frames(a, np.stack([sc.frames[t]] * 2))
            step_frames(b, np.stack([sc.frames[t]] * 2))
            if t >= 3:
                for s in range(2):
                    assert_same_bytes(stream_result(a, s, jacobians=True), stream_result(b, s, jacobians=True),
                                      (t, s))
    finally:
        a.close()
        b.close()


# ---- arguments ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_rejected_arguments_change_nothing_and_launch_nothing():
    sc = _scene("C2", T=2)
    ctx = ctx_from_scenes([sc, sc])
    try:
        ctx.set_stream_rescue(1, 3.0)
        before = [stream_result(ctx, s) for s in range(2)]
        n0 = ctx.launch_count()
        for s, v in ((-1, 1.0), (2, 1.0), (0, -1.0), (1, -1e-300), (0, float("nan")), (1, float("inf")),
                     (0, float("-inf"))):
            with pytest.raises(sl2.Sl2Error):
                ctx.set_stream_rescue(s, v)
        assert ctx.stream_rescue(0) == 0.0 and ctx.stream_rescue(1) == 3.0
        with pytest.raises(sl2.Sl2Error):
            ctx.stream_rescue(2)
        assert ctx.launch_count() == n0
        for s in range(2):
            assert_same_bytes(stream_result(ctx, s), before[s], s)
        ctx.set_stream_rescue(0, -0.0)
        assert math.copysign(1.0, ctx.stream_rescue(0)) == 1.0
        assert ctx.launch_count() == n0
    finally:
        ctx.close()


# ---- what it is for ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_capability_uncertain_features_are_kept():
    """C4 map, 8 new features with sigma 3 cm, distractors on two settled features (bounds from the rescue oracle on
    the CPU, tests/test_rescue.py).  The oracle stepped alongside names the features the cull kept."""
    T = 15
    new, wrong = set(range(92, 100)), {5, 50}
    out = {}
    for chi2 in (0.0, CHI2):
        sc = _scene("C4", T=T + 1, new=range(92, 100), wrong=[5, 50])
        ctx = ctx_from_scenes([sc])
        o = ro.slam_from_scene(sc, TAU, chi2)
        try:
            ctx.set_stream_consensus(0, TAU)
            ctx.set_stream_rescue(0, chi2)
            rows = []
            for t in range(T):
                step_frames(ctx, sc.frames[t][None])
                o.step(sc.frames[t])
                assert ctx.num_features(0) == o.num_features, t
                lab = o.features()["label"]
                f = ctx.features(0)
                rows.append(dict(rej_new=sum(1 for i, l in enumerate(lab) if l in new and f["flags"][i] & 4),
                                 in_new=sum(1 for i, l in enumerate(lab) if l in new and f["flags"][i] & 2),
                                 in_wrong=sum(1 for i, l in enumerate(lab) if l in wrong and f["flags"][i] & 2)))
            lab = o.features()["label"]
            idx = [i for i, l in enumerate(lab) if l in new]
            _, P = ctx.get_state(0)
            sig = [math.sqrt(np.trace(P[13 + 3 * i:16 + 3 * i, 13 + 3 * i:16 + 3 * i]) / 3) for i in idx]
            out[chi2] = (rows, sig)
        finally:
            ctx.close()
    (off, sig_off), (on, sig_on) = out[0.0], out[CHI2]
    assert off[0]["rej_new"] >= 5 and on[0]["rej_new"] == 0 and on[0]["in_new"] >= 6
    assert len(sig_off) <= 6 and len(sig_on) == 8 and max(sig_on) < 0.02
    assert all(r["in_wrong"] == 0 for r in on)


# ---- the kernel's shape edges against the restatement and the truth --------------------------------------------------
# (features, distractors) whose step 0 has exactly k matches rejected by the consensus (set from the consensus oracle,
# which the device's consensus equals bit for bit): k crosses the warps of rescue_kernel's gather and match loop.
SHAPES = {2: (40, 2), 3: (40, 3), 31: (96, 32), 32: (100, 32), 33: (100, 33), 64: (128, 69), 65: (128, 70)}


def shape_scene(k):
    nf, d = SHAPES[k]
    return rescue_scene(None, sc=large_variant(nf, nf, n_frames=2), wrong=np.linspace(1, nf - 2, d).round().astype(int),
                        spread=True)


@pytest.mark.gpu
@pytest.mark.parametrize("k", sorted(SHAPES))
def test_decisions_at_the_shape_edges(k):
    """chi2 is set to the median q of the step, so that both outcomes and the knife edge occur; the device's decisions,
    h and S equal the restatement's, and equal the truth's wherever the truth's q lies outside q_band of chi2."""
    sc = shape_scene(k)
    ctx, clone = ctx_from_scenes([sc]), ctx_from_scenes([sc])
    try:
        ctx.set_stream_consensus(0, TAU)
        clone.set_stream_consensus(0, TAU)
        cam8 = _cam8(ctx, 0)
        x, P, rej, z, pre = staged_update_1(clone, ctx.save_stream(0), sc.frames[0])
        assert rej.size == k
        pos = (13 + 3 * rej).astype(np.int32)
        _, q, _ = rescue_ref.gate(cam8, x, P, pos, z, 0.0)
        chi2 = float(np.sort(q[np.isfinite(q)])[(k - 1) // 2])
        ok, _, preds = rescue_ref.gate(cam8, x, P, pos, z, chi2)
        assert 0 < ok.sum() <= k
        ctx.set_stream_rescue(0, chi2)
        step_frames(ctx, sc.frames[0][None])
        f = ctx.features(0)
        assert (((f["flags"][rej] & 2) > 0) == ok).all()
        for j in np.flatnonzero(ok):
            assert f["h"][rej[j]].tobytes() == preds[j]["h"].tobytes()
            assert f["S"][rej[j]].tobytes() == preds[j]["S"].T.reshape(4).tobytes()
        q_t, ok_t, cond = rt.truth(cam8, pre["x"], pre["P"], pre["inl"], pre["z_inl"], rej, z, chi2)
        q_t = np.array([float(v) for v in q_t])
        band = np.array([rt.q_band(v, x.size, 2 * pre["inl"].size, cond) for v in q_t])
        assert (np.abs(q - q_t) <= band).all()
        far = np.abs(q_t - chi2) > band
        assert far.sum() >= k - 1 and (ok[far] == ok_t[far]).all()
    finally:
        ctx.close()
        clone.close()


@pytest.mark.gpu
def test_capacity_256_with_128_selected():
    """A map of 256 features, 128 of them in view and all selected, 24 distractors; chi2 large enough to take back
    every rejected match in front of the camera: the second update runs at its largest m2, the record sums m1 + m2 rows.
    Two fused steps against the rescue oracle."""
    sc = rescue_scene(None, sc=large_variant(256, 128, n_frames=3), wrong=np.linspace(1, 126, 24).round().astype(int),
                      spread=True)
    ctx = ctx_from_scenes([sc], max_features=256)
    o = ro.slam_from_scene(sc, TAU, 1e12)
    try:
        ctx.set_stream_consensus(0, TAU)
        ctx.set_stream_rescue(0, 1e12)
        ctx.enable_records(2)
        for t in range(2):
            step_frames(ctx, sc.frames[t][None])
            o.step(sc.frames[t])
            f, fo = ctx.features(0), o.features()
            assert ctx.num_features(0) == o.num_features
            for key in ("select_rank", "flags", "attempted", "successful"):
                assert (f[key] == fo[key]).all(), (t, key)
            ok = (fo["flags"] & 2) > 0
            assert (f["z"][ok] == fo["z"][ok]).all()
            # the second update here takes back ~11 px distractor matches, whose innovations are several times a
            # correct match's: the rounding difference between the device's update and the oracle's dense one reaches
            # h about that many times farther than on the suite's steps (H_ATOL_STEP = 1e-11 px)
            assert float(np.abs(f["h"] - fo["h"]).max()) <= 1e-10
            assert_state_close(*ctx.get_state(0), *o.get_state())
            assert int((f["select_rank"] >= 0).sum()) == 128
            nres = len(o.rescued())
            assert nres >= 16
            r = ctx.records(0, 1, 1)[0, 0]
            assert r["m"] == 2 * int(((f["flags"] & 2) > 0).sum()) and r["nmeas"] == r["m"] // 2
    finally:
        ctx.close()


@pytest.mark.gpu
def test_position_173_of_a_264_stream_mixed_context():
    """Stream 173 (consensus and rescue on) of a 264-stream context in which the settings vary from stream to stream
    (one CTA per stream per launch, no PDL, the batched launch shapes) has the bytes of the same stream alone in a
    context (PDL)."""
    T, B, pick = 3, 264, 173
    tiles = [_scene("C4", stream_id=u, T=T) for u in range(6)]
    scenes = [tiles[s % len(tiles)] for s in range(B)]
    big = ctx_from_scenes(scenes)
    one = ctx_from_scenes([scenes[pick]])
    try:
        for s in range(B):
            big.set_stream_consensus(s, TAU if s % 3 != 1 else 0.0)
            big.set_stream_rescue(s, CHI2 if s % 4 != 2 else 0.0)
        assert big.stream_consensus(pick) == TAU and big.stream_rescue(pick) == CHI2
        one.set_stream_consensus(0, TAU)
        one.set_stream_rescue(0, CHI2)
        o = ro.slam_from_scene(scenes[pick], TAU, CHI2)
        rescued = 0
        for t in range(T):
            step_frames(big, np.stack([sc.frames[t] for sc in scenes]))
            step_frames(one, scenes[pick].frames[t][None])
            a, b = stream_result(big, pick, jacobians=True), stream_result(one, 0, jacobians=True)
            assert_same_bytes(a, b, t)
            o.step(scenes[pick].frames[t])
            rescued += len(o.rescued())
        assert rescued > 0
    finally:
        big.close()
        one.close()
