"""The match consensus on the device (sl2_set_stream_consensus, csrc/consensus.cu consensus_kernel) on scenes with
distractors: a feature's template pasted at a fixed offset inside its search ellipse while its true location is
occluded, so that the patch search returns a confident wrong match.  A match is correct iff z = pix + shift[t]."""
import dataclasses
import math

import numpy as np
import pytest

import consensus_oracle as co
import scenelib2_b200 as sl2
from consensus_ref import restated
from consensus_truth import consensus_truth
from gpu_util import (CAMS_320, assert_same_bytes, check_streams_against_oracle, ctx_from_scenes, large_variant,
                      oracle_slam_from_scene, step_frames, stream_result)
from oracle import pyoracle as po
from scenelib2_b200 import synth
from scenelib2_b200.lib import SL2_MAX_MEASURED

TAU = 2.5          # px: the synthetic camera moves by whole pixels, correct matches sit within ~1 px of a hypothesis
OFFSET = (9, -6)   # px: where a distractor pastes the template, inside the 20 px ellipse


def distractor_scene(name, stream_id=0, n_frames=12, n_features=None, persistent=(), transient=(), camera=None,
                     sc=None):
    """synth scene whose frames carry distractors: for every feature f of `persistent` (every frame) and of
    `transient` ({f: frames}), the true location is covered with fresh noise and the template is pasted at
    pix + shift[t] + OFFSET.  meta["wrong"][t] = the features with a distractor in frame t."""
    if sc is None:
        sc = synth.make_scene(name, stream_id=stream_id, n_frames=n_frames, n_features=n_features, camera=camera)
    rng = np.random.default_rng(777 + stream_id)
    B = sc.boxsize
    half = (B - 1) // 2
    frames = sc.frames.copy()
    wrong = [set() for _ in range(len(frames))]
    for f in persistent:
        for t in range(len(frames)):
            wrong[t].add(f)
    for f, ts in dict(transient).items():
        for t in ts:
            wrong[t].add(f)
    for t, fs in enumerate(wrong):
        for f in fs:  # occlude first, then paste, so that no paste is covered by another feature's occlusion
            u, v = sc.pix[f] + sc.shifts[t]
            frames[t, v - half - 2:v + half + 3, u - half - 2:u + half + 3] = rng.integers(0, 256, (B + 4, B + 4))
        for f in fs:
            u, v = sc.pix[f] + sc.shifts[t] + OFFSET
            frames[t, v - half:v + half + 1, u - half:u + half + 1] = sc.patches[f]
    # a converged map: feature sigmas / 10, camera sigmas x 2.  A one-point hypothesis then moves the camera (and every
    # prediction with it) rather than only its own feature, which is what lets matches outvote each other
    d = np.concatenate([np.full(13, 2.0), np.full(sc.n - 13, 0.1)])
    sc.P0 = d[:, None] * sc.P0 * d[None, :]
    sc.frames = frames
    sc.meta["wrong"] = wrong
    return sc


def truth(sc, t):
    return sc.pix + sc.shifts[t]


def consensus_inputs(ctx, s):
    """After the staged predict / search of stream s (consensus off): x, P, and the step's matches M in rank order
    with what the consensus reads of them."""
    x, P = ctx.get_state(s)
    f = ctx.features(s)
    J, Jy, R, _ = ctx.feature_jacobians(s)
    sel = np.flatnonzero((f["select_rank"] >= 0) & ((f["flags"] & 2) > 0))
    M = sel[np.argsort(f["select_rank"][sel])]
    k = M.size
    dxp = J[M].reshape(k, 13, 2).transpose(0, 2, 1)[:, :, :7]
    dy = Jy[M].reshape(k, 3, 2).transpose(0, 2, 1)
    S = f["S"][M].reshape(k, 2, 2).transpose(0, 2, 1)
    return dict(x=x, P=P, M=M, pos=(13 + 3 * M).astype(np.int32), z=f["z"][M], h=f["h"][M], S=S, dh_dxp=dxp,
                dh_dy=dy, R=R[M])


def staged_clone(clone, blob, frame):
    """The stream of `blob` in the one-stream context `clone` (consensus off), predicted and searched on `frame`."""
    clone.load_stream(0, blob)
    clone.set_frame(0, 0, frame)
    clone.ekf_predict(0)
    clone.predict_measurements(0)
    clone.make_measurements(0, 0)
    return consensus_inputs(clone, 0)


def expected(cam8, inp, tau):
    return co.consensus(cam8, inp["x"], inp["P"], inp["pos"], inp["z"], inp["h"], inp["S"], inp["dh_dxp"],
                        inp["dh_dy"], tau)


def rejected_now(ctx, s):
    f = ctx.features(s)
    return set(np.flatnonzero((f["select_rank"] >= 0) & ((f["flags"] & 4) > 0)).tolist())


def min_margin(cam8, inp, tau):
    """The smallest |d2 - fl(tau tau)| over every (hypothesis, match) pair of the step (restated on the host)."""
    _, _, _, d2 = restated(cam8, inp["x"], inp["P"], inp["pos"], inp["z"], inp["h"], inp["S"], inp["dh_dxp"],
                           inp["dh_dy"], tau)
    d = np.abs(d2[~np.isnan(d2)] - tau * tau)
    return float(d.min()) if d.size else np.inf


def _cam8(ctx, s):
    c = ctx.stream_config(s)
    return np.array([c.width, c.height, c.fku, c.fkv, c.u0, c.v0, c.kd1, c.sd], np.float64)


# ---- 1. off means off ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_off_means_off_and_one_launch_per_group():
    scenes = [distractor_scene("C2", stream_id=s, n_frames=6, n_features=30, persistent=[3, 11]) for s in range(4)]
    plain, mixed = ctx_from_scenes(scenes), ctx_from_scenes(scenes)
    try:
        for c in (plain, mixed):
            c.enable_records(8)
            c.set_step_groups(2)  # groups {0, 1} and {2, 3}
        mixed.set_stream_consensus(1, TAU)
        mixed.set_stream_consensus(3, TAU)
        for t in range(6):
            if t == 3:
                mixed.set_stream_consensus(3, 0.0)  # only group A has a stream on from here
            l0, m0 = plain.launch_count(), mixed.launch_count()
            frames = np.stack([sc.frames[t] for sc in scenes])
            step_frames(plain, frames)
            step_frames(mixed, frames)
            extra = (mixed.launch_count() - m0) - (plain.launch_count() - l0)
            assert extra == (2 if t < 3 else 1), (t, extra)
            for s in (0, 2):
                assert_same_bytes(stream_result(mixed, s, jacobians=True), stream_result(plain, s, jacobians=True),
                                  ("stream", s, "step", t))
        for s in (0, 2):
            assert mixed.records(s, 1).tobytes() == plain.records(s, 1).tobytes()
        assert mixed.stream_consensus(1) == TAU and mixed.stream_consensus(0) == 0.0
    finally:
        plain.close()
        mixed.close()


# ---- 2. decisions bit-exact against the test oracle on the device's own inputs; 4. it does its job ---------------
CASES = {
    "C1": dict(name="C1", n_features=20, persistent=[5], transient={9: range(2, 5), 14: range(6, 8)}),
    "C2": dict(name="C2", n_features=40, persistent=[4, 17], transient={25: range(1, 4), 33: range(5, 9)}),
    "C4": dict(name="C4", n_features=100, persistent=[7, 40, 71], transient={20: range(0, 3), 90: range(4, 9)}),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_decisions_bit_exact_and_wrong_matches_rejected(case):
    kw = dict(CASES[case])
    T = 9  # below minimum_attempted_measurements_of_feature: no cull renumbers the features
    sc = distractor_scene(kw.pop("name"), n_frames=T, **kw)
    ctx, clone, off = ctx_from_scenes([sc]), ctx_from_scenes([sc]), ctx_from_scenes([sc])
    cam8 = _cam8(ctx, 0)
    err_on, err_off = [], []
    try:
        ctx.set_stream_consensus(0, TAU)
        checked = rejections = 0
        for t in range(T):
            inp = staged_clone(clone, ctx.save_stream(0), sc.frames[t])
            keep, _, _ = expected(cam8, inp, TAU)
            step_frames(ctx, sc.frames[t][None])
            step_frames(off, sc.frames[t][None])
            assert rejected_now(ctx, 0) == set(inp["M"][~keep].tolist()), t
            rejections += int((~keep).sum())
            # the matches that are wrong by the scene's ground truth
            z = inp["z"].astype(np.int64)
            bad = (z != truth(sc, t)[inp["M"]]).any(axis=1)
            if (~bad).sum() >= 3:
                assert rejected_now(ctx, 0) == set(inp["M"][bad].tolist()), (t, inp["M"][bad])
                checked += 1
            # prediction error of the features without a distractor this step, after the step
            clean = np.setdiff1d(np.arange(sc.n_features), list(sc.meta["wrong"][t]))
            for c, acc in ((ctx, err_on), (off, err_off)):
                h = c.features(0)["h"]
                acc.append(np.abs(h[clean] - truth(sc, t)[clean]).mean())
        assert checked >= T - 1 and rejections > 0
        on, offm = float(np.mean(err_on)), float(np.mean(err_off))
        print("%s: mean |h - truth| of the untouched features: on %.4f px, off %.4f px" % (case, on, offm))
        assert on < offm
    finally:
        for c in (ctx, clone, off):
            c.close()


@pytest.mark.gpu
def test_tau_knife_edge_on_the_device():
    sc = distractor_scene("C2", n_frames=2, n_features=40, persistent=[4, 17])
    ctx, clone = ctx_from_scenes([sc]), ctx_from_scenes([sc])
    cam8 = _cam8(ctx, 0)
    try:
        blob = ctx.save_stream(0)
        inp = staged_clone(clone, blob, sc.frames[0])
        keep, sup, win = expected(cam8, inp, TAU)
        assert win >= 0
        _, _, _, d2 = restated(cam8, inp["x"], inp["P"], inp["pos"], inp["z"], inp["h"], inp["S"], inp["dh_dxp"],
                               inp["dh_dy"], TAU)
        j = int(np.nanargmax(np.where(keep & (np.arange(keep.size) != win), d2[win], np.nan)))
        s = math.sqrt(d2[win, j])
        taus = [s]
        for _ in range(2):
            taus = [np.nextafter(taus[0], 0.0)] + taus + [np.nextafter(taus[-1], np.inf)]
        seen = set()
        for tau in taus:
            ctx.load_stream(0, blob)
            ctx.set_stream_consensus(0, float(tau))
            step_frames(ctx, sc.frames[0][None])
            k2, _, _ = expected(cam8, inp, float(tau))
            assert rejected_now(ctx, 0) == set(inp["M"][~k2].tolist()), tau
            seen.add(float(tau) * float(tau) >= d2[win, j])
        assert seen == {False, True}
    finally:
        ctx.close()
        clone.close()


# ---- 3. whole-step parity with the oracle running the same consensus, through a cull ---------------------------------
@pytest.mark.gpu
def test_whole_step_parity_with_the_oracle_through_a_cull():
    T = 22
    sc = distractor_scene("C2", n_frames=T, n_features=30, persistent=[6], transient={12: range(3, 6)})
    ctx, clone = ctx_from_scenes([sc]), ctx_from_scenes([sc])
    o = co.slam_from_scene(sc, TAU)
    cam8 = _cam8(ctx, 0)
    try:
        ctx.set_stream_consensus(0, TAU)
        margin = np.inf
        for t in range(T):
            margin = min(margin, min_margin(cam8, staged_clone(clone, ctx.save_stream(0), sc.frames[t]), TAU))
            step_frames(ctx, sc.frames[t][None])
            check_streams_against_oracle(ctx, [o], [0], lambda s: sc, t)
        assert ctx.num_features(0) < sc.n_features  # the persistent distractor's feature was culled
        assert margin > 1e-6, margin  # no decision of the run within reach of a last-bit difference
    finally:
        ctx.close()
        clone.close()


# ---- 5. batch invariance on the 264-stream C4 shape -------------------------------------------------------------------
@pytest.mark.gpu
def test_batch_invariance_c4_shape():
    import torch
    U, B, T = 8, 264, 4
    scenes = [distractor_scene("C4", stream_id=u, n_frames=T, camera=CAMS_320[u % 4], persistent=[3, 50],
                               transient={20: range(1, 3)}) for u in range(U)]
    on = lambda u: u % 2 == 0  # noqa: E731
    H, W = scenes[0].height, scenes[0].width  # the largest image: the ring's block

    def make(us):
        """a context of the ring's frame size whose stream s runs scene us[s] with that scene's camera"""
        c = sl2.Context(sl2.config_for_scene(scenes[0], num_streams=len(us), frame_slots=2))
        for s, u in enumerate(us):
            sl2.load_scene(c, s, scenes[u])
            c.set_stream_config(s, sl2.stream_config_for_scene(scenes[u]))
            if on(u):
                c.set_stream_consensus(s, TAU)
        return c

    def frame_set(us, t):
        out = np.zeros((len(us), H, W), np.uint8)
        for s, u in enumerate(us):
            f = scenes[u].frames[t]
            out[s, :f.shape[0], :f.shape[1]] = f
        return out

    us = [s % U for s in range(B)]
    results = {}
    for path in ("serial", "groups", "async"):
        ctx = make(us)
        try:
            if path == "groups":
                ctx.set_step_groups(2)
            host = torch.empty((B, H, W), dtype=torch.uint8, pin_memory=True)
            xv = torch.empty((B, 13), dtype=torch.float64, pin_memory=True)
            for t in range(T):
                if path == "async":
                    ctx.wait_slot(t % 2)
                    host.numpy()[:] = frame_set(us, t)
                    ctx.step_host_async(t % 2, host.data_ptr(), xv.data_ptr())
                    ctx.wait_slot(t % 2)
                else:
                    ctx.set_frames(t % 2, frame_set(us, t))
                    ctx.step(t % 2)
            ctx.sync()
            first = {}
            for s in range(B):
                r = stream_result(ctx, s, jacobians=True)
                u = s % U
                if u in first:
                    assert_same_bytes(r, first[u], (path, "stream", s, "vs first of scene", u))
                else:
                    first[u] = r
            results[path] = first
        finally:
            ctx.close()
    for u in range(U):  # a single-stream context: the PDL chain
        c = make([u])
        try:
            for t in range(T):
                step_frames(c, frame_set([u], t))
            results.setdefault("single", {})[u] = stream_result(c, 0, jacobians=True)
        finally:
            c.close()
    for path in ("groups", "async", "single"):
        for u in range(U):
            assert_same_bytes(results[path][u], results["serial"][u], (path, "scene", u))
    assert any((r["flags"] & 4).any() for u, r in results["serial"].items() if on(u))


# ---- 6. staged equals fused ----------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_staged_equals_fused():
    T = 8
    sc = distractor_scene("C2", n_frames=T, n_features=40, persistent=[4, 17], transient={25: range(1, 4)})
    fused, staged = ctx_from_scenes([sc]), ctx_from_scenes([sc])
    try:
        for c in (fused, staged):
            c.set_stream_consensus(0, TAU)
        for t in range(T):
            step_frames(fused, sc.frames[t][None])
            staged.set_frame(0, 0, sc.frames[t])
            staged.ekf_predict(0)
            staged.predict_measurements(0)
            cnt = staged.make_measurements(0, 0)
            f = staged.features(0)
            assert cnt == int(((f["select_rank"] >= 0) & ((f["flags"] & 2) > 0)).sum()), t
            staged.ekf_update_measured(0)
            assert_same_bytes(stream_result(staged, 0, jacobians=True), stream_result(fused, 0, jacobians=True), t)
    finally:
        fused.close()
        staged.close()


# ---- 7. the kernel's largest shape: capacity 256, k = 128 ----------------------------------------------------------
@pytest.mark.gpu
def test_capacity_256_with_128_matches():
    T = 3
    sc = large_variant(256, 128, n_frames=T)
    sc = distractor_scene(None, sc=sc, persistent=[10, 60, 100])
    ctx = ctx_from_scenes([sc], max_features=256)
    o = co.slam_from_scene(sc, TAU)
    try:
        ctx.set_stream_consensus(0, TAU)
        for t in range(T):
            step_frames(ctx, sc.frames[t][None])
            check_streams_against_oracle(ctx, [o], [0], lambda s: sc, t)
            f = ctx.features(0)
            assert int((f["select_rank"] >= 0).sum()) == 128
        assert rejected_now(ctx, 0)
    finally:
        ctx.close()


# ---- 8. snapshots and records ----------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_snapshot_with_rejections_and_records():
    T = 6
    sc = distractor_scene("C2", n_frames=T, n_features=40, persistent=[4, 17])
    ctx, other, clone = ctx_from_scenes([sc]), ctx_from_scenes([sc, sc]), ctx_from_scenes([sc])
    try:
        ctx.enable_records(T)
        ctx.set_stream_consensus(0, TAU)
        other.set_stream_consensus(1, TAU)
        other.set_stream_consensus(0, 1.0)
        for t in range(T):
            inp = staged_clone(clone, ctx.save_stream(0), sc.frames[t])
            keep, _, _ = expected(_cam8(ctx, 0), inp, TAU)
            step_frames(ctx, sc.frames[t][None])
            rec = ctx.records(0, 1)[0, -1]
            acc = inp["M"][keep]
            assert rec["nmeas"] == acc.size and rec["m"] == 2 * acc.size
            # S = H P H^T + R and nu over the rows that entered the update
            n = inp["x"].size
            H = np.zeros((2 * acc.size, n))
            for q, j in enumerate(np.flatnonzero(keep)):
                H[2 * q:2 * q + 2, :7] = inp["dh_dxp"][j]
                H[2 * q:2 * q + 2, inp["pos"][j]:inp["pos"][j] + 3] = inp["dh_dy"][j]
            Rm = np.kron(np.diag(inp["R"][keep][:, 0]), np.eye(2))
            S = H @ inp["P"] @ H.T + Rm
            nu = (inp["z"][keep] - inp["h"][keep]).ravel()
            nis = float(nu @ np.linalg.solve(S, nu))
            logdet = float(np.linalg.slogdet(S)[1])
            assert abs(rec["nis"] - nis) <= 1e-9 * max(1.0, abs(nis)), (t, rec["nis"], nis)
            assert abs(rec["logdet_s"] - logdet) <= 1e-9 * max(1.0, abs(logdet)), (t, rec["logdet_s"], logdet)
            if t == 2:
                assert rejected_now(ctx, 0)
                f = ctx.features(0)
                blob = ctx.save_stream(0)
                assert (sl2.read_snapshot(blob)["found"] == 2).sum() == ((f["flags"] & 4) > 0).sum() > 0
                other.load_stream(1, blob)
                assert other.stream_consensus(1) == TAU  # the load leaves the slot's setting
                other.load_stream(0, blob)
                assert other.stream_consensus(0) == 1.0
                other.set_stream_consensus(0, TAU)
            if t > 2:
                step_frames(other, np.stack([sc.frames[t]] * 2))
                for s in (0, 1):
                    assert_same_bytes(stream_result(other, s, jacobians=True), stream_result(ctx, 0, jacobians=True),
                                      (t, s))
    finally:
        for c in (ctx, other, clone):
            c.close()


# ---- 9. rejected setter arguments ---------------------------------------------------------------------------------
@pytest.mark.gpu
def test_rejected_setter_arguments_change_nothing():
    sc = distractor_scene("C2", n_frames=2, n_features=20)
    ctx = ctx_from_scenes([sc, sc])
    try:
        ctx.set_stream_consensus(1, 3.0)
        before = [stream_result(ctx, s) for s in range(2)]
        for s, v in ((-1, 1.0), (2, 1.0), (0, -1.0), (1, -1e-300), (0, float("nan")), (1, float("inf")),
                     (0, float("-inf"))):
            with pytest.raises(sl2.Sl2Error):
                ctx.set_stream_consensus(s, v)
        assert ctx.stream_consensus(0) == 0.0 and ctx.stream_consensus(1) == 3.0
        with pytest.raises(sl2.Sl2Error):
            ctx.stream_consensus(2)
        for s in range(2):
            assert_same_bytes(stream_result(ctx, s), before[s], s)
        ctx.set_stream_consensus(0, -0.0)
        assert math.copysign(1.0, ctx.stream_consensus(0)) == 1.0
    finally:
        ctx.close()


# ---- 10. the device against the consensus from its definition, at the kernel's shape edges --------------------------
# The device exposes only its rejections: the rejected set must be the complement of the truth winner's inlier set
# (consensus_truth, np.longdouble) whenever no decision of the step lies within D2_BAND of fl(tau tau), besides equal
# to the test oracle's bit for bit.  D2_BAND is test_consensus_truth.D2_BOUND, set from the CPU cases.
D2_BAND = 1e-10
K_SHAPES = (2, 3, 8, 9, 16, 17, 31, 32, 33, 63, 64, 65)   # CONS_WARPS = 8 hypotheses, 32 matches per word


def truth_of(cam8, inp, tau=TAU):
    return consensus_truth(cam8, inp["x"], inp["P"], inp["pos"], inp["z"], inp["h"], inp["S"], inp["dh_dxp"],
                           inp["dh_dy"], tau, prec="ld")


def staged_inputs(ctx, clone, streams, frame_of):
    """The consensus inputs of each stream of `streams` on frame_of(s), staged in the one-stream `clone` under that
    stream's camera and selection count, with the test oracle's decisions and the truth: {s: (inp, keep, truth)}."""
    out = {}
    for s in streams:
        clone.set_stream_config(0, ctx.stream_config(s))
        inp = staged_clone(clone, ctx.save_stream(s), frame_of(s))
        cam8 = _cam8(ctx, s)
        out[s] = (inp, expected(cam8, inp, TAU)[0], truth_of(cam8, inp))
    return out


def check_rejections(ctx, s, inp, keep, tr, where):
    """-> True when the truth was unambiguous and the device's rejections were held to it."""
    got = rejected_now(ctx, s)
    assert got == set(inp["M"][~keep].tolist()), (where, "oracle")
    if tr.margin <= D2_BAND * max(1.0, TAU * TAU):
        print("%s: a decision within %.1e px^2 of tau^2; only the oracle compared" % (where, tr.margin))
        return False
    assert got == set(inp["M"][~tr.keep].tolist()), (where, "truth", tr.winner, tr.support)
    return True


def matched_count(sc, n_select, t=0):
    """How many of the n_select features the oracle (and so the device) finds in frame t of the scene."""
    o = oracle_slam_from_scene(po, dataclasses.replace(sc, n_select=n_select))
    o.predict()
    o.select()
    o.measure(sc.frames[t])
    f = o.features()
    return int(((f["select_rank"] >= 0) & ((f["flags"] & 2) > 0)).sum())


def shape_scene(k, stream_id=0, n_frames=2):
    """C4 camera, k + 8 features (at least 12) in view, distractors on every fourth feature (every ninth from k = 64
    on, where the grid is dense), and the smallest n_select at which exactly k matches are found in frame 0."""
    nf = max(k + 8, 12)
    sc = large_variant(nf, nf, stream_id=stream_id, n_frames=n_frames)
    sc = distractor_scene(None, sc=sc, persistent=range(1, nf, 4 if k < 64 else 9))
    for n in range(k, min(nf, SL2_MAX_MEASURED) + 1):
        if matched_count(sc, n) >= k:
            break
    assert matched_count(sc, n) == k, (k, n)
    sc.n_select = n
    return sc


def run_against_truth(scenes, T, max_features=None, tau_streams=None, expect_k=None):
    """Fused steps of a context of `scenes` with the consensus on, each step held to the oracle and the truth.
    -> (steps held to the truth, [the k of every step and stream])"""
    ctx, clone = ctx_from_scenes(scenes, max_features=max_features), ctx_from_scenes(scenes[:1],
                                                                                     max_features=max_features)
    held, ks = 0, []
    try:
        streams = range(len(scenes))
        for s in streams:
            ctx.set_stream_consensus(s, TAU)
        for t in range(T):
            staged = staged_inputs(ctx, clone, streams, lambda s: scenes[s].frames[t])
            step_frames(ctx, np.stack([sc.frames[t] for sc in scenes]))
            for s, (inp, keep, tr) in staged.items():
                ks.append(inp["M"].size)
                if expect_k is not None and t == 0:
                    assert inp["M"].size == expect_k[s], (s, inp["M"].size, expect_k[s])
                held += check_rejections(ctx, s, inp, keep, tr, ("step", t, "stream", s, "k", inp["M"].size))
        return held, ks, ctx.get_state(0)[0]
    finally:
        ctx.close()
        clone.close()


@pytest.mark.gpu
@pytest.mark.parametrize("k", K_SHAPES)
def test_shapes_against_the_truth(k):
    sc = shape_scene(k)
    held, ks, _ = run_against_truth([sc], 2, expect_k=[k])
    assert held >= 1, ks


@pytest.mark.gpu
def test_rank_order_is_a_permutation_of_map_order():
    sc = shape_scene(40)
    ctx, clone = ctx_from_scenes([sc]), ctx_from_scenes([sc])
    try:
        inp = staged_clone(clone, ctx.save_stream(0), sc.frames[0])
        assert (np.diff(inp["M"]) < 0).any() and (inp["M"] != np.sort(inp["M"])).sum() > inp["M"].size // 2
    finally:
        ctx.close()
        clone.close()
    assert run_against_truth([sc], 2)[0] >= 1


@pytest.mark.gpu
def test_capacity_256_matches_past_index_128():
    """ld = 784: features 0..127 out of view, 40 of 128..255 measured."""
    sc = large_variant(256, 256, n_frames=2)
    sc.x0 = sc.x0.copy()
    sc.x0[13:13 + 3 * 128] += np.tile([3.0, 0.0, 0.0], 128)
    sc = distractor_scene(None, sc=sc, persistent=range(129, 256, 5))
    sc.n_select = next(n for n in range(40, 129) if matched_count(sc, n) >= 40)
    ctx, clone = ctx_from_scenes([sc], max_features=256), ctx_from_scenes([sc], max_features=256)
    try:
        inp = staged_clone(clone, ctx.save_stream(0), sc.frames[0])
        assert inp["M"].size == 40 and inp["M"].min() >= 128 and inp["P"].shape[0] == 13 + 3 * 256
    finally:
        ctx.close()
        clone.close()
    assert run_against_truth([sc], 2, max_features=256)[0] >= 1


@pytest.mark.gpu
def test_c3_camera_against_the_truth():
    """640 x 480, kd1 = 2.25e-6, 15 x 15 templates, 100 features selected."""
    sc = distractor_scene("C3", n_frames=2, persistent=range(2, 100, 6))
    held, ks, _ = run_against_truth([sc], 2)
    assert held >= 1 and max(ks) > 64, ks


@pytest.mark.gpu
def test_non_unit_q_after_fused_steps():
    """x is never renormalised (quirk Q1): after some fused steps |q| != 1 and the truth's pose model sees it.  Nine
    steps: the tenth would cull the distractors' features and renumber the map under the comparison."""
    sc = distractor_scene("C2", n_frames=9, n_features=40, persistent=[4, 17], transient={25: range(2, 6)})
    held, ks, x = run_against_truth([sc], 9)
    dq = abs(float(np.linalg.norm(x[3:7])) - 1.0)
    print("| |q| - 1 | after 9 fused steps: %.3e" % dq)
    assert dq > 0.0 and held >= 8, (dq, held)


@pytest.mark.gpu
def test_264_streams_each_with_its_own_k():
    """One C4-camera scene in 264 streams whose selection counts give every k from 2 to 65 that the scene allows, in a
    scrambled order (no two neighbours alike): each stream's decisions are held to its own k."""
    B = 264
    sc = shape_scene(65)
    n_for = {}
    for n in range(2, sc.n_select + 1):
        n_for.setdefault(matched_count(sc, n), n)
    kv = sorted(k for k in n_for if k >= 2)
    ks = [kv[(37 * s) % len(kv)] for s in range(B)]
    assert len(kv) >= 50 and all(a != b for a, b in zip(ks, ks[1:]))
    ctx, clone = ctx_from_scenes([sc] * B), ctx_from_scenes([sc])
    held = 0
    try:
        for s in range(B):
            ctx.set_stream_config(s, number_of_features_to_select=n_for[ks[s]])
            ctx.set_stream_consensus(s, TAU)
        staged = staged_inputs(ctx, clone, range(B), lambda s: sc.frames[0])
        step_frames(ctx, np.stack([sc.frames[0]] * B))
        for s, (inp, keep, tr) in staged.items():
            assert inp["M"].size == ks[s], (s, inp["M"].size, ks[s])
            held += check_rejections(ctx, s, inp, keep, tr, ("stream", s, "k", ks[s]))
    finally:
        ctx.close()
        clone.close()
    assert held >= B - 4, held
