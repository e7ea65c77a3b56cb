"""The mutual-information selection on the device (sl2_set_stream_selection; csrc/select.cu select_kernel): its
decisions bit for bit against the NumPy restatement (tests/selection_ref.py) fed the device's own prediction, the
constructed knife-edge, degenerate and duplicate cases, whole steps against the CPU oracle extended by the selection
(tests/selection_oracle.py), the off path and the launch count, fused against staged, a stream's independence of its
batch position, snapshots, rejected arguments, and what it buys, with margins set on the CPU: more information per row
on a clustered map and fewer rows with a threshold."""
import numpy as np
import pytest

import scenelib2_b200 as sl2
import selection_ref as sr
import selection_oracle as so
from gpu_util import (assert_same_bytes, camera, check_streams_against_oracle, large_variant, ring_block,
                      step_frames, stream_result, update_variant)
from scenelib2_b200 import synth

INFO, TRACE = sl2.lib.SL2_SELECT_INFORMATION, sl2.lib.SL2_SELECT_TRACE
TAU = 2.5  # px: the match consensus radius of the combined runs
MARGINS = {}


def make_ctx(scenes, max_features=None, groups=1, W=None, H=None):
    cfg = sl2.config_for_scene(scenes[0], num_streams=len(scenes),
                               max_features=max_features or max(sc.n_features for sc in scenes))
    if W:
        cfg.width, cfg.height = W, H
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


def step(ctx, scenes, t):
    ctx.set_frames(0, frames_at(ctx, scenes, t))
    ctx.step(0)
    ctx.sync()


def kmax(ctx):
    return min(ctx.cfg.max_features, sl2.lib.SL2_MAX_MEASURED)


def candidates(ctx, s, mode, min_bits):
    """The trace rule's candidates of stream s at its current state, from the device: a trace prediction with n_select
    = kmax gives the ranks when it selects every candidate; otherwise every feature must be visible and the ranking is
    restated from the device's S.  Leaves the stream's setting as (mode, min_bits)."""
    n_sel = ctx.stream_config(s).number_of_features_to_select
    ctx.set_stream_selection(s, TRACE)
    ctx.set_stream_config(s, number_of_features_to_select=kmax(ctx))
    nvis = ctx.predict_measurements(s)
    snap = sl2.read_snapshot(ctx.save_stream(s))
    ctx.set_stream_config(s, number_of_features_to_select=n_sel)
    ctx.set_stream_selection(s, mode, min_bits)
    rank = snap["sel_rank"]
    nf = len(rank)
    if snap["nsel"] < kmax(ctx):
        feats = np.flatnonzero(rank >= 0)
        return feats, rank[feats], nvis
    assert nvis == nf, "a stream with more candidates than kmax must see its whole map"
    feats, rho = sr.trace_candidates(snap["S"], np.ones(nf, bool))
    top = feats[np.argsort(rho)][:kmax(ctx)]
    assert (rank[top] == np.arange(len(top))).all()  # the restated ranking agrees with the device's
    return feats, rho, nvis


def check_stream(ctx, s, min_bits=0.0, case=None):
    """One staged prediction of stream s by information, against the restatement fed the device's prediction."""
    feats, rho, nvis = candidates(ctx, s, INFO, min_bits)
    assert ctx.predict_measurements(s) == nvis
    snap = sl2.read_snapshot(ctx.save_stream(s))
    nf = len(snap["sel_rank"])
    n_sel = ctx.stream_config(s).number_of_features_to_select
    x, P = snap["x"], snap["P"]
    t = 2.0 ** (2 * min_bits)
    picks, info = sr.information_select(P, feats, rho, snap["S"], snap["dh_dxp"], snap["dh_dy"], snap["Rvar"],
                                        n_sel, t)
    k = len(picks)
    assert snap["nsel"] == k and snap["nvisible"] == nvis and snap["nmeas"] == 0
    want_rank = np.full(nf, -1, np.int32)
    want_rank[picks] = np.arange(k)
    assert (snap["sel_rank"] == want_rank).all()
    jf = snap["job_feat"]
    assert (jf[:k] == picks).all() and (jf[k:] == -1).all()
    assert snap["job_centre"][:k].tobytes() == snap["h"][picks].tobytes()
    ovr = np.array(ctx.cfg.search_override[:], np.float64)
    if ovr[0] > 0:
        want = np.tile(ovr, (k, 1))
    else:
        S = snap["S"][picks]
        want = np.stack(sr.sinv_from_S(S[:, 0], S[:, 1], S[:, 3]), axis=1)
    assert snap["job_puinv"][:k].tobytes() == want.tobytes()
    if case is not None:
        MARGINS[case] = sr.margins(info, t) + (k, len(feats))
        print(case, "picks", k, "of", len(feats), "margins (winner, threshold)", MARGINS[case][:2])
    return picks, info


# ---- 2. bit-exact decisions --------------------------------------------------------------------------------------
CASES = [("C1", 10, 0.0), ("C2", 1, 0.0), ("C2", 2, 0.0), ("C2", 10, 0.5), ("C2", 50, 0.0), ("C4", 10, 0.0),
         ("C4", 100, 1.0), ("C3", 10, 0.0), ("C3", 100, 0.5)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,n_select,min_bits", CASES)
def test_decisions_equal_the_restatement(name, n_select, min_bits):
    sc = synth.make_scene(name, n_frames=6)
    ctx = make_ctx([sc])
    try:
        ctx.set_stream_config(0, number_of_features_to_select=n_select)
        ctx.set_stream_selection(0, INFO, min_bits)
        for t in range(1, 5):  # settle the map through fused steps that select by information
            step(ctx, [sc], t)
        ctx.ekf_predict(0)
        check_stream(ctx, 0, min_bits, (name, n_select, min_bits))
    finally:
        ctx.close()


@pytest.mark.gpu
def test_capacity_256_with_256_visible_and_128_picks():
    sc = large_variant(256, 256, n_select=128)
    ctx = make_ctx([sc])
    try:
        ctx.set_stream_selection(0, INFO)
        step(ctx, [sc], 1)
        ctx.ekf_predict(0)
        picks, _ = check_stream(ctx, 0, 0.0, ("cap256", 128, 0.0))
        assert len(picks) == 128
    finally:
        ctx.close()


@pytest.mark.gpu
def test_stream_2_of_three_with_its_own_camera():
    scenes = [synth.make_scene("C2", stream_id=s, n_frames=6) for s in range(2)]
    scenes.append(synth.make_scene("C2", stream_id=2, n_frames=6,
                                   camera=camera(288, 224, focal=1.1, shift=(-6.0, 4.0), kd1=2.0, sd=1.5)))
    scenes[2].n_select = 10
    ctx = make_ctx(scenes, W=320, H=240)
    try:
        ctx.set_stream_selection(2, INFO, 0.5)
        for t in range(1, 4):
            step(ctx, scenes, t)
        ctx.ekf_predict(2)
        check_stream(ctx, 2, 0.5, ("stream2", 10, 0.5))
    finally:
        ctx.close()


@pytest.mark.gpu
def test_without_correlation_information_selects_like_trace():
    """P_xx = 0, P_xy = 0 and P_yy block-diagonal: no pick changes another candidate's C, so where the order of
    det(S_i) / R_i^2 equals the trace order (checked by the restatement), both rules select the same, ties included."""
    sc = synth.make_scene("C2", n_frames=2, n_features=12)
    nf = sc.n_features
    P = np.zeros_like(sc.P0)
    # a factor 16 between features, every c B B^T well above R: the det order follows the trace order (with c B B^T
    # near R, a larger R raises the trace and lowers det / R^2, and the orders part)
    for j in range(nf):
        P[13 + 3 * j:16 + 3 * j, 13 + 3 * j:16 + 3 * j] = np.eye(3) * (1e-3 * 16.0 ** ((5 * j) % nf))
    ctx = make_ctx([sc])
    try:
        agree = 0
        for n_select in (1, 2, 10, 12):
            ctx.set_state(0, sc.x0, P)
            ctx.set_stream_config(0, number_of_features_to_select=n_select)
            feats, rho, _ = candidates(ctx, 0, INFO, 0.0)
            snap_t = sl2.read_snapshot(ctx.save_stream(0))
            qdet = (snap_t["S"][:, 0] * snap_t["S"][:, 3] - snap_t["S"][:, 1] * snap_t["S"][:, 1]) / (
                snap_t["Rvar"] * snap_t["Rvar"])
            by_det = [feats[a] for a in sorted(range(len(feats)), key=lambda a: (-qdet[feats[a]], rho[a]))]
            picks, info = check_stream(ctx, 0)
            assert picks == by_det[:n_select]  # the top n_select by det(S_i) / R_i^2
            for d in info:  # no pick changed another candidate's C
                live = ~np.isnan(d["qall"])
                assert (d["qall"][live] == qdet[feats][live]).all()
            if by_det == list(feats[np.argsort(rho)]):
                agree += 1
                assert picks == list(feats[np.argsort(rho)][:n_select])  # = the trace rule's selection
        assert agree == 4, "the scene no longer orders det(S_i) / R_i^2 like trace(S_i)"
    finally:
        ctx.close()


# ---- 1. off means off, and the launch count ------------------------------------------------------------------------
@pytest.mark.gpu
def test_off_streams_are_untouched_and_one_launch_per_group():
    scenes = [synth.make_scene("C4", stream_id=s, n_frames=8) for s in range(4)]
    plain, mixed, toggled = (make_ctx(scenes, groups=2) for _ in range(3))  # groups {0, 1} and {2, 3}
    try:
        mixed.set_stream_selection(1, INFO, 0.5)
        mixed.set_stream_selection(3, INFO)
        for s in range(4):
            toggled.set_stream_selection(s, INFO, 1.0)
            toggled.set_stream_selection(s, TRACE)
        assert toggled.launch_count() == plain.launch_count() == mixed.launch_count()
        for t in range(1, 8):
            if t == 4:
                mixed.set_stream_selection(3, TRACE)  # only group {0, 1} selects by information from here
            counts = [c.launch_count() for c in (plain, mixed, toggled)]
            for c in (plain, mixed, toggled):
                step(c, scenes, t)
            d = [c.launch_count() - n for c, n in zip((plain, mixed, toggled), counts)]
            assert d[1] - d[0] == (2 if t < 4 else 1) and d[2] == d[0], (t, d)
            for s in range(4):
                assert_same_bytes(stream_result(toggled, s, jacobians=True), stream_result(plain, s, jacobians=True),
                                  ("toggled", s, t))
            for s in (0, 2):
                assert_same_bytes(stream_result(mixed, s, jacobians=True), stream_result(plain, s, jacobians=True),
                                  ("mixed", s, t))
            assert plain.save_streams() == toggled.save_streams()
        assert [mixed.get_stream_selection(s) for s in range(4)] == [(0, 0.0), (1, 0.5), (0, 0.0), (0, 0.0)]
        # one more launch per sl2_predict_measurements of an information stream, none for a trace stream
        for s, extra in ((0, 0), (1, 1)):
            n0, p0 = mixed.launch_count(), plain.launch_count()
            mixed.predict_measurements(s)
            plain.predict_measurements(s)
            assert (mixed.launch_count() - n0) - (plain.launch_count() - p0) == extra
    finally:
        for c in (plain, mixed, toggled):
            c.close()


@pytest.mark.gpu
def test_rejected_arguments_change_nothing():
    scenes = [synth.make_scene("C2", stream_id=s, n_frames=2) for s in range(2)]
    ctx = make_ctx(scenes)
    try:
        ctx.set_stream_selection(1, INFO, 0.25)
        before = [stream_result(ctx, s) for s in range(2)]
        launches = ctx.launch_count()
        bad = [(-1, INFO, 0.0, 0), (2, INFO, 0.0, 0), (0, 2, 0.0, 0), (0, -1, 0.0, 0), (0, INFO, 0.0, 1),
               (0, INFO, -0.5, 0), (0, INFO, np.nan, 0), (0, INFO, np.inf, 0), (0, TRACE, 0.5, 0),
               (1, TRACE, 1e-300, 0)]
        for s, mode, bits, res in bad:
            with pytest.raises(sl2.Sl2Error):
                ctx.set_stream_selection(s, mode, bits, reserved=res)
        with pytest.raises(sl2.Sl2Error):
            ctx.get_stream_selection(2)
        assert ctx.L.sl2_set_stream_selection(ctx.h, 0, None) == -1
        assert ctx.L.sl2_get_stream_selection(ctx.h, 0, None) == -1
        assert [ctx.get_stream_selection(s) for s in range(2)] == [(0, 0.0), (1, 0.25)]
        assert ctx.launch_count() == launches
        for s in range(2):
            assert_same_bytes(stream_result(ctx, s), before[s], s)
        ctx.set_stream_selection(0, INFO, -0.0)  # -0 is 0
        assert ctx.get_stream_selection(0) == (1, 0.0)
    finally:
        ctx.close()


# ---- 5. paths and placement -----------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_fused_equals_staged_with_consensus_warp_and_two_groups():
    scenes = [synth.make_scene("C2", stream_id=s, n_frames=9) for s in range(2)]
    for sc in scenes:
        sc.n_select = 12
    fused, staged = make_ctx(scenes, groups=2), make_ctx(scenes)
    try:
        for c in (fused, staged):
            for s in range(2):
                c.set_stream_selection(s, INFO, 0.5 * s)
                c.set_stream_consensus(s, TAU)
                c.set_stream_warp(s, 1)
        for t in range(1, 9):
            step(fused, scenes, t)
            staged.set_frames(0, frames_at(staged, scenes, t))
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


@pytest.mark.gpu
def test_a_stream_is_the_same_alone_and_in_a_264_stream_batch():
    B, pos = 264, 173
    pool = [synth.make_scene("C4", stream_id=s, n_frames=7) for s in range(16)]
    own = pool[5]
    others = [pool[(s * 7) % 16] for s in range(B)]
    rng = np.random.default_rng(264)
    others[pos] = own
    alone, batch = make_ctx([own]), make_ctx(others)
    try:
        alone.set_stream_selection(0, INFO, 0.5)
        batch.set_stream_selection(pos, INFO, 0.5)
        for s in rng.choice(B, 60, replace=False):  # other streams mixed in on both rules
            if s != pos:
                batch.set_stream_selection(int(s), INFO, float(rng.integers(0, 3)) * 0.5)
        for t in range(1, 7):
            step(alone, [own], t)
            step(batch, others, t)
            assert_same_bytes(stream_result(batch, pos, jacobians=True), stream_result(alone, 0, jacobians=True), t)
    finally:
        alone.close()
        batch.close()


@pytest.mark.gpu
def test_snapshots_do_not_carry_the_setting():
    scenes = [synth.make_scene("C2", stream_id=s, n_frames=9) for s in range(2)]
    on, off, ref_on, ref_off, cont, reload = (make_ctx(scenes) for _ in range(6))
    try:
        for c in (on, cont, reload):
            c.set_stream_selection(0, INFO, 0.5)
        ref_on.set_stream_selection(1, INFO, 0.5)
        for t in range(1, 5):
            for c in (on, off, cont):
                step(c, scenes, t)
        b_on, b_off = on.save_stream(0), off.save_stream(0)
        # saved from an information slot and loaded into another: continues bit for bit like the uninterrupted run
        reload.load_streams([b_on, on.save_stream(1)])
        for t in range(5, 9):
            for c in (cont, reload):
                step(c, scenes, t)
            assert_same_bytes(stream_result(reload, 0, jacobians=True), stream_result(cont, 0, jacobians=True),
                              ("reload", t))
            assert reload.save_stream(0) == cont.save_stream(0)
        assert b_on != b_off
        assert on.save_stream(1) == off.save_stream(1)
        off.load_stream(1, b_on)  # an information run continues under the trace rule, and the reverse
        on.load_stream(0, b_off)
        assert on.get_stream_selection(0) == (1, 0.5) and off.get_stream_selection(1) == (0, 0.0)
        ref_off.load_stream(0, b_on)
        ref_on.load_stream(1, b_off)
        for t in range(5, 9):
            step(on, scenes, t)
            step(off, scenes[:1] + scenes[:1], t)  # stream 1 of `off` now holds stream 0's map
            step(ref_on, scenes[:1] + scenes[:1], t)  # stream 1 of `ref_on` holds stream 0's map
            step(ref_off, scenes, t)
            assert_same_bytes(stream_result(off, 1), stream_result(ref_off, 0), ("info -> trace", t))
            assert_same_bytes(stream_result(on, 0), stream_result(ref_on, 1), ("trace -> info", t))
    finally:
        for c in (on, off, ref_on, ref_off, cont, reload):
            c.close()


# ---- 5. whole-step parity with the oracle extended by the selection, through a cull --------------------------------
@pytest.mark.gpu
def test_whole_step_parity_with_the_oracle_through_a_cull():
    """22 fused steps of two streams, every one checked against the CPU oracle selecting by information
    (tests/selection_oracle.cpp): the selection ranks, flags, matches and counters exactly, the predictions and the
    state at the suite's tolerances.  Three templates of each map are random bytes, never found: both streams cull."""
    T = 22
    scenes = [update_variant(30, 30, bad=3, stream_id=s, n_frames=T) for s in range(2)]
    settings = [(30, 0.0), (8, 0.5)]  # (n_select, min_bits): every candidate with information, then a real choice
    for sc, (n_sel, _) in zip(scenes, settings):
        sc.n_select = n_sel
    ctx = make_ctx(scenes)
    oracles = [so.slam_from_scene(sc, INFO, bits) for sc, (_, bits) in zip(scenes, settings)]
    try:
        for s, (_, bits) in enumerate(settings):
            ctx.set_stream_selection(s, INFO, bits)
        for t in range(T):
            step_frames(ctx, np.stack([sc.frames[t] for sc in scenes]))
            check_streams_against_oracle(ctx, oracles, [0, 1], lambda s: scenes[s], t)
        assert all(ctx.num_features(s) < 30 for s in range(2))  # the never-found features were culled
    finally:
        ctx.close()


# ---- 4. constructed cases on the device --------------------------------------------------------------------------
def constructed_ctx(nf, y=None, P=None, n_select=None, max_features=None):
    """A one-stream context on a C2 scene of nf features with the map y and covariance P set directly: the staged
    prediction then sees exactly this P (no motion step)."""
    sc = synth.make_scene("C2", n_frames=2, n_features=nf)
    if n_select is not None:
        sc.n_select = n_select
    ctx = make_ctx([sc], max_features=max_features)
    x = sc.x0.copy()
    if y is not None:
        x[13:] = np.asarray(y).reshape(-1)
        ctx.set_features(0, np.asarray(y).reshape(nf, 3), sc.xp_org, sc.patches)
    ctx.set_state(0, x, sc.P0 if P is None else P)
    return ctx, sc


def block(P, j, v):
    P[13 + 3 * j:16 + 3 * j, 13 + 3 * j:16 + 3 * j] = v


@pytest.mark.gpu
def test_knife_edge_and_degenerate_C_on_the_device():
    """P_xx = 0 and P_xy = 0.  Features whose P_yy is 0 have S = R I exactly, so q = 1 = t at min_bits = 0: never
    picked.  Features with a P_yy of 1e-18 .. 1e-14 have q a few doubles above 1 or exactly 1: picked exactly when the
    restatement says.  A negative P_yy gives C00 < 0 with a large positive q, a NaN P_yy a NaN C: never picked."""
    nf = 40
    sc = synth.make_scene("C2", n_frames=2, n_features=nf)
    P = np.zeros_like(sc.P0)
    kinds = {}
    for j in range(nf):
        if j % 8 == 0:
            kinds[j] = "zero"
        elif j % 8 == 1:
            block(P, j, np.eye(3) * 10.0 ** (-18 + (j // 8)))
            kinds[j] = "tiny"
        elif j % 8 == 2:
            block(P, j, -np.eye(3) * 1e-2)
            kinds[j] = "negative"
        elif j % 8 == 3:
            block(P, j, np.eye(3) * np.nan)
            kinds[j] = "nan"
        else:
            block(P, j, np.eye(3) * 1e-4 * (1 + j % 5))
            kinds[j] = "normal"
    ctx, _ = constructed_ctx(nf, P=P, n_select=nf, max_features=50)
    try:
        picks, info = check_stream(ctx, 0, 0.0, ("knife edge", nf, 0.0))
        snap = sl2.read_snapshot(ctx.save_stream(0))
        S, Rv = snap["S"], snap["Rvar"]
        q = (S[:, 0] * S[:, 3] - S[:, 1] * S[:, 1]) / (Rv * Rv)
        for j, k in kinds.items():
            if k == "zero":
                assert q[j] == 1.0 and j not in picks
            if k in ("negative", "nan"):
                assert not (S[j, 0] > 0.0) and j not in picks
            if k == "normal":
                assert j in picks
        tiny = [j for j, k in kinds.items() if k == "tiny"]
        assert any(q[j] > 1.0 and q[j] - 1.0 < 1e-12 for j in tiny)  # picked a few doubles above t
        for j in tiny:
            assert (j in picks) == (q[j] > 1.0)
    finally:
        ctx.close()


@pytest.mark.gpu
def test_a_duplicate_is_not_the_next_pick_on_the_device():
    """Feature 1 is feature 0 again (the same y, P rows and template) with the largest variance of the map: one twin is
    the first pick, and the other is not the second while independent candidates remain."""
    nf = 30
    sc = synth.make_scene("C2", n_frames=2, n_features=nf)
    y = sc.x0[13:].reshape(nf, 3).copy()
    y[1] = y[0]
    P = sc.P0.copy()
    y0, y1 = slice(13, 16), slice(16, 19)
    P[y0, :] *= 5.0
    P[:, y0] *= 5.0
    P[y1, :] = P[y0, :]
    P[:, y1] = P[:, y0]
    ctx, _ = constructed_ctx(nf, y=y, P=P, n_select=10)
    try:
        picks, info = check_stream(ctx, 0, 0.0, ("duplicate", 10, 0.0))
        assert picks[0] in (0, 1) and picks[1] not in (0, 1)
        feats, _, _ = candidates(ctx, 0, INFO, 0.0)
        twin = 1 - picks[0]
        q_twin = info[1]["qall"][list(feats).index(twin)]
        assert 1.0 <= q_twin < 4.0 < info[1]["q"]
    finally:
        ctx.close()


# ---- capability -----------------------------------------------------------------------------------------------------
def dense_update(snap, feats):
    """The posterior of an update with the rows of `feats` from the snapshot's P and Jacobians, on the CPU: the rows'
    information 1/2 log2 det S_sel / det R_sel (bits) and log det of the camera position block of P+ (natural log)."""
    P = snap["P"]
    n = P.shape[0]
    H = np.zeros((2 * len(feats), n))
    for r, f in enumerate(feats):
        H[2 * r:2 * r + 2, :7] = snap["dh_dxp"][f]
        H[2 * r:2 * r + 2, 13 + 3 * f:16 + 3 * f] = snap["dh_dy"][f]
    Rr = np.repeat(snap["Rvar"][list(feats)], 2)
    S = H @ P @ H.T + np.diag(Rr)
    bits = 0.5 * (np.linalg.slogdet(S)[1] - np.log(Rr).sum()) / np.log(2)
    Pp = P - P @ H.T @ np.linalg.solve(S, H @ P)
    return float(bits), float(np.linalg.slogdet(Pp[:3, :3])[1])


def device_update(ctx, s, snap, feats):
    """The device's EKF update (sl2_ekf_update, nu = 0) with the rows of `feats`: log det of the camera position
    block of its posterior."""
    k = len(feats)
    if k:
        jf = np.asarray(feats, np.int32)
        Hxv = np.zeros((2 * k, 13))
        Hxv[:, :7] = np.concatenate([snap["dh_dxp"][f] for f in jf])
        Hy = np.concatenate([snap["dh_dy"][f] for f in jf])
        Rb = np.stack([np.eye(2) * snap["Rvar"][f] for f in jf])
        ctx.ekf_update(s, jf, Hxv, Hy, Rb, np.zeros(2 * k))
    _, P = ctx.get_state(s)
    return float(np.linalg.slogdet(P[:3, :3])[1])


LOGDET_ATOL = 1e-6  # the device's update against NumPy's dense one, on log det of a 3 x 3 block near -30


@pytest.mark.gpu
def test_clustered_map_information_beats_trace():
    """Eight features in one clump of the image share a large common offset (variance 0.05^2 m^2 per axis on top of
    the prior): they have the largest traces.  With n_select = 6 the trace rule measures six of them, the information
    rule at most two.  The margins come from the CPU: the restatement's picks and a dense update of the device's
    predicted P give the information rule more bits and a smaller posterior camera-position log det; the device's
    picks equal the restatement's and its updates reproduce the CPU's log dets."""
    nf, cl = 50, [3, 9, 14, 20, 27, 33, 40, 46]
    sc = synth.make_scene("C2", n_frames=2, n_features=nf)
    rng = np.random.default_rng(8)
    y = sc.x0[13:].reshape(nf, 3).copy()
    for f in cl:  # a clump: within 5 mm of feature 3
        y[f] = y[cl[0]] + rng.uniform(-0.005, 0.005, 3)
    P = sc.P0.copy()
    for a in cl:
        for b in cl:
            P[13 + 3 * a:16 + 3 * a, 13 + 3 * b:16 + 3 * b] += 0.05 ** 2 * np.eye(3)
    ctx, _ = constructed_ctx(nf, y=y, P=P, n_select=6)
    try:
        x0, P0 = ctx.get_state(0)
        ctx.set_stream_selection(0, TRACE)
        ctx.predict_measurements(0)
        snap_t = sl2.read_snapshot(ctx.save_stream(0))
        trace = [int(f) for f in snap_t["job_feat"][:snap_t["nsel"]]]
        info_picks, _ = check_stream(ctx, 0, 0.0, ("cluster", 6, 0.0))  # device == restatement, bit for bit
        snap = sl2.read_snapshot(ctx.save_stream(0))
        assert sorted(trace) == sorted(set(trace) & set(cl)) and len(trace) == 6
        assert len(set(info_picks) & set(cl)) <= 2 and len(info_picks) == 6
        bits_t, ld_t = dense_update(snap, trace)
        bits_i, ld_i = dense_update(snap, info_picks)
        print("cluster: trace", trace, bits_t, ld_t, "information", info_picks, bits_i, ld_i)
        assert bits_i > bits_t and ld_i < ld_t  # the CPU's margins
        dev_i = device_update(ctx, 0, snap, info_picks)
        ctx.set_state(0, x0, P0)
        dev_t = device_update(ctx, 0, snap, trace)
        assert abs(dev_i - ld_i) <= LOGDET_ATOL and abs(dev_t - ld_t) <= LOGDET_ATOL, (dev_i, ld_i, dev_t, ld_t)
        assert dev_t - dev_i > 0.5 * (ld_t - ld_i)
    finally:
        ctx.close()


def settled(scenes, steps):
    """Contexts of `scenes` stepped `steps` times under the trace rule, then saved: the settled maps."""
    ctx = make_ctx(scenes)
    try:
        for t in range(1, steps + 1):
            step(ctx, scenes, t)
        return ctx.save_streams()
    finally:
        ctx.close()


@pytest.mark.gpu
def test_threshold_gives_fewer_rows_on_settled_maps():
    """Settled C4 maps (10 trace steps), n_select = 100.  Per stream and setting the device's picks equal the
    restatement's, and the device's update reproduces the dense CPU update of those rows (LOGDET_ATOL): the posterior
    camera log dets are the CPU's.  min_bits = 1 measures fewer than 2 n_select rows; min_bits = 0 measures every
    candidate the trace rule measures except those whose conditional measurement adds no information (q <= 1 when
    the picks stop)."""
    scenes = [synth.make_scene("C4", stream_id=s, n_frames=12) for s in range(2)]
    blobs = settled(scenes, 10)
    ctx = make_ctx(scenes)
    try:
        for s in range(2):
            rows = {}
            for mode, bits in ((TRACE, 0.0), (INFO, 0.0), (INFO, 1.0)):
                ctx.load_streams([blobs[s]], s)
                ctx.ekf_predict(s)
                x0, P0 = ctx.get_state(s)
                if mode == TRACE:
                    ctx.set_stream_selection(s, TRACE)
                    ctx.predict_measurements(s)
                    snap = sl2.read_snapshot(ctx.save_stream(s))
                    picks, info = [int(f) for f in snap["job_feat"][:snap["nsel"]]], None
                else:
                    picks, info = check_stream(ctx, s, bits, ("threshold", s, bits))
                    snap = sl2.read_snapshot(ctx.save_stream(s))
                b_cpu, ld_cpu = dense_update(snap, picks)
                ctx.set_state(s, x0, P0)
                ld_dev = device_update(ctx, s, snap, picks)
                assert abs(ld_dev - ld_cpu) <= LOGDET_ATOL, (s, mode, bits, ld_dev, ld_cpu)
                rows[(mode, bits)] = (picks, info, b_cpu, ld_cpu)
                print("threshold", s, mode, bits, "m", 2 * len(picks), "bits", b_cpu, "camera log det", ld_cpu)
            tr, i0, i1 = rows[(TRACE, 0.0)], rows[(INFO, 0.0)], rows[(INFO, 1.0)]
            assert 2 * len(i1[0]) < 2 * 100 and len(i1[0]) < len(tr[0])
            assert set(i0[0]) <= set(tr[0])
            if len(i0[0]) < len(tr[0]):
                stop = i0[1][-1]
                assert stop["stop"] and not (np.nan_to_num(stop["qall"], nan=0.0) > 1.0).any()
    finally:
        ctx.close()
