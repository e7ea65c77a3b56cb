"""The mutual-information selection on the device (csrc/select.cu select_kernel) against the greedy selection from its
definition (tests/selection_truth.py) under the derived bound (tests/selection_cases.py): every constructed problem, the
kernel's shape edges (candidates V across the 128-thread stride and the warp edges), both sides of the factor store's
switch from shared memory to the context scratch, a mixed launch and a 264-stream context stepped both fused and staged.  Each run is also held to the restatement bit
for bit (test_gpu_selection.check_stream), and the predicted P the kernel reads is bit-symmetric.  The kernel does not
report q: the device is held to the truth through its picks, stop and job slots, and the q that is held to the bound
is the restatement's on the device's arrays, which picks as the device does bit for bit."""
import hashlib

import numpy as np
import pytest

import scenelib2_b200 as sl2
import selection_cases as sc
import selection_truth as st
from gpu_util import assert_same_bytes, stream_result
from test_gpu_selection import INFO, TRACE, candidates, check_stream

NXV = 13
V_EDGES = [1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256]
CONSTRUCTIONS = sc.constructions()
XP_ORG = np.array([0.0, 0, 0, 1, 0, 0, 0])
_TRUTHS = {}
STATS = {"decisions": 0, "inside": 0, "worst": 0.0}


def context(cap, num_streams=1):
    cfg = sl2.config_for_scene(sl2.synth.make_scene("C2", n_frames=1, n_features=1), num_streams=num_streams,
                               max_features=cap)
    return sl2.Context(cfg)


def install(ctx, s, pb, n_select=None, mode=INFO):
    """Problem pb in stream s: CAM8, the map and P set directly (no motion step), the selection setting."""
    c = sc.CAM8
    ctx.set_stream_config(s, width=int(c[0]), height=int(c[1]), fku=c[2], fkv=c[3], u0=c[4], v0=c[5], kd1=c[6],
                          sd=c[7], number_of_features_to_select=pb.n_select if n_select is None else n_select)
    V = len(pb.y)
    patches = np.random.default_rng(V).integers(0, 256, (V, 11, 11), dtype=np.uint8)
    ctx.set_features(s, pb.y, np.tile(XP_ORG, (V, 1)), patches)
    ctx.set_state(s, pb.x, pb.P)
    ctx.set_stream_selection(s, mode, pb.min_bits if mode == INFO else 0.0)


def truth_of(snap, feats, rho, n_select, t):
    """The truth's run on the device's arrays, followed along its own picks; cached per input bytes (a shorter run
    of the same problem is its prefix)."""
    key = hashlib.sha1(b"".join(np.ascontiguousarray(a).tobytes() for a in (
        snap["P"], snap["dh_dxp"], snap["dh_dy"], snap["Rvar"], np.asarray(feats), np.asarray(rho),
        np.array([t])))).hexdigest()
    have = _TRUTHS.get(key)
    if have is None or (have[0] < n_select and (len(have[1]) == have[0])):
        tr = st.Truth(snap["P"], snap["dh_dxp"], snap["dh_dy"], snap["Rvar"], feats, rho)
        have = (n_select, tr.run(n_select, t, bound=sc.q_bound))
        _TRUTHS[key] = have
    return have[1][:n_select]


def assert_symmetric(P, moved):
    """The P the kernel reads is bit-symmetric, except, after a motion step (`moved`), in its 13 x 13 camera block:
    the motion step forms F P_xx Fᵀ + Q entry by entry, and, as in the reference, its triangles are made equal only
    by the update's symmetrisation.  There they may differ by that rounding alone: two orders of a sum of 13 x 13
    products differ by at most 2 γ_169 (|F| |P_xx| |F|ᵀ), within 512 u sqrt(P_ii P_jj) for the F of a frame period
    (|F| within a few percent of I)."""
    D = P.view(np.uint64) != np.ascontiguousarray(P.T).view(np.uint64)  # bits: a NaN block equals itself
    if moved:
        D[:NXV, :NXV] = False
        Pxx = P[:NXV, :NXV]
        scale = np.sqrt(np.outer(np.diag(Pxx), np.diag(Pxx)))
        assert (np.abs(Pxx - Pxx.T) <= 512 * sc.U * scale).all(), "P_xx triangles differ by more than rounding"
    assert not D.any(), "the predicted P is not bit-symmetric"


def check_truth(ctx, s, pb, n_select=None, moved=False):
    """Stream s by information against the restatement (bit for bit) and the truth: every decided decision equal,
    the exact problems equal throughout; P bit-symmetric (assert_symmetric).  Returns the snapshot and the device's
    picks."""
    n_select = pb.n_select if n_select is None else n_select
    picks, info = check_stream(ctx, s, pb.min_bits)
    snap = sl2.read_snapshot(ctx.save_stream(s))
    assert_symmetric(snap["P"], moved)
    feats, rho, _ = candidates(ctx, s, INFO, pb.min_bits)
    index = {int(f): k for k, f in enumerate(feats)}
    got = [index[f] for f in picks]
    nmax = min(n_select, len(feats))
    got_stop = got + ([-1] if len(got) < nmax else [])
    ds = truth_of(snap, feats, rho, n_select, pb.t)
    # the truth's own run: equal wherever it is decided, up to the first decision inside the bound (after it the
    # device may legitimately condition on another pick)
    for r, d in enumerate(ds):
        STATS["decisions"] += 1
        if not sc.decided(d, pb.t):
            STATS["inside"] += 1
            assert not pb.exact or got_stop[r] == d["pick"], (pb.name, r)
            if not pb.exact:
                break
        else:
            assert got_stop[r] == d["pick"], (pb.name, r, got_stop[r], d["pick"])
        live = d["live"] & np.isfinite(d["q"])
        if r < len(info):
            ratio = np.abs(info[r]["qall"][live] - d["q"][live]) / d["beta"][live, 0]
            STATS["worst"] = max(STATS["worst"], float(ratio.max()) if ratio.size else 0.0)
            assert (ratio <= 1.0).all(), (pb.name, r, float(ratio.max()))
    if pb.exact:
        assert [d["pick"] for d in ds] == got_stop[:len(ds)] and len(ds) == len(got_stop)
    return snap, picks


def report():
    print("truth decisions %d, inside the bound %d, worst |q_restated - q_truth| / bound on the device's arrays %.3g" % (
        STATS["decisions"], STATS["inside"], STATS["worst"]))


def selection_bytes(snap, k):
    """The first k picks' selection outputs: job slots and the ranks below k."""
    rank = snap["sel_rank"]
    return dict(job_feat=snap["job_feat"][:k], job_centre=snap["job_centre"][:k], job_puinv=snap["job_puinv"][:k],
                rank=np.where(rank < k, rank, -1))


# ---- 1. the constructed problems ---------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("k", range(len(CONSTRUCTIONS)))
def test_constructions_equal_the_truth(k):
    pb = CONSTRUCTIONS[k]
    ctx = context(max(len(pb.y), 128))  # above V: the candidates come from the device's own trace ranks
    try:
        install(ctx, 0, pb)
        snap, picks = check_truth(ctx, 0, pb)
        if pb.name == "ties":
            for a, b in sc.TIE_PAIRS:
                assert picks.index(a) + 1 == picks.index(b)
            lo, hi = sc.RHO_PAIR
            assert picks.index(hi) + 1 == picks.index(lo)
        print(pb.name, "picks", len(picks))
        report()
    finally:
        ctx.close()


# ---- 2. shape edges ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_shape_edges():
    ctx = context(256, num_streams=len(V_EDGES))
    try:
        for s, V in enumerate(V_EDGES):
            install(ctx, s, sc.dense(V, V, min(V, 128)))
        for s, V in enumerate(V_EDGES):
            pb = sc.dense(V, V, min(V, 128))
            for n in (min(V, 128), min(V, 3)):
                ctx.set_stream_config(s, number_of_features_to_select=n)
                _, picks = check_truth(ctx, s, pb, n)
                assert len(picks) == n, (V, n)
        report()
    finally:
        ctx.close()


# ---- 3. the factor store: shared memory and the context scratch ----------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cap,k_prefix,k_more", [(100, 22, 23), (128, 15, 16), (256, 15, 16)])
def test_both_sides_of_the_storage_boundary(cap, k_prefix, k_more):
    """sel_base_bytes(N) + 32 N npick > 113 KB moves the factors to the scratch: at capacity 100, 22 picks keep them
    in shared memory and 23 use the scratch; at capacity 128, 15 and 16.  At capacity 256 both pick counts use the
    scratch, and only the prefix property is tested.  Greedy selection is a prefix process: the first k_prefix picks
    and their job slots are byte-identical on both sides."""
    pb = sc.dense(cap + 1, cap, k_more)
    ctx = context(cap)
    try:
        install(ctx, 0, pb)
        out = {}
        for k in (k_prefix, k_more):
            ctx.set_stream_config(0, number_of_features_to_select=k)
            snap, picks = check_truth(ctx, 0, pb, k)
            assert len(picks) == k
            out[k] = selection_bytes(snap, k_prefix)
        assert_same_bytes(out[k_prefix], out[k_more], (cap, "prefix"))
        report()
    finally:
        ctx.close()


@pytest.mark.gpu
def test_a_mixed_launch_gives_the_bytes_of_the_stream_alone():
    """Capacity 128: a stream with 15 picks launched beside one with 16 has its factors in the scratch (the launch's
    largest pick count sets the store), alone in shared memory.  Its fused step gives the same bytes either way."""
    pa, pb = sc.dense(7, 128, 15), sc.dense(8, 128, 16)
    mixed, alone = context(128, 2), context(128, 2)
    frames = np.random.default_rng(3).integers(0, 256, (2, 240, 320), dtype=np.uint8)
    try:
        for c, mode in ((mixed, INFO), (alone, TRACE)):
            install(c, 0, pa)
            install(c, 1, pb, mode=mode)
            c.set_frames(0, frames)
            c.step(0)
            c.sync()
        assert_same_bytes(stream_result(mixed, 0, jacobians=True), stream_result(alone, 0, jacobians=True), "mixed")
        assert mixed.save_stream(0) == alone.save_stream(0)
    finally:
        mixed.close()
        alone.close()


# ---- 4. a 264-stream context ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cap,groups", [(256, 1), (128, 2)])
def test_a_264_stream_context_equals_the_truth(cap, groups):
    """264 streams take one fused step, whose selection runs as one launch per step group, and the same streams are
    stepped staged one at a time (ekf_predict, predict_measurements, make_measurements, ekf_update_measured): every
    stream's staged selection equals the truth of its own problem, and its fused step gives the staged bytes.  Streams
    cycle through the V edges up to the capacity.  Capacity 256, one group: n_select cycles through min(V, 128), 16
    and 15, every launch on the scratch.  Capacity 128, two groups: group A (streams 0..131) picks at most 15, so its
    launch keeps the factors in shared memory; group B mixes 16 and 15 picks, so its launch puts them in the scratch,
    while a 15-pick stream staged alone keeps them in shared memory."""
    B = 264
    edges = [V for V in V_EDGES if V <= cap]
    fused, staged = context(cap, B), context(cap, B)
    frames = np.random.default_rng(264).integers(0, 256, (B, 240, 320), dtype=np.uint8)
    try:
        fused.set_step_groups(groups)
        plan = []
        for s in range(B):
            V = edges[s % len(edges)]
            if cap == 256:
                n = [min(V, 128), min(V, 16), min(V, 15)][(s // len(edges)) % 3]
            else:
                n = min(V, 15) if s < (B + 1) // 2 else [min(V, 16), min(V, 15)][(s // len(edges)) % 2]
            plan.append(sc.dense(V, V, n))
            for c in (fused, staged):
                install(c, s, plan[s])
        assert cap == 256 or max(pb.n_select for pb in plan[(B + 1) // 2:]) == 16
        fused.set_frames(0, frames)
        fused.step(0)
        fused.sync()
        staged.set_frames(0, frames)
        for s in range(B):
            staged.ekf_predict(s)
            check_truth(staged, s, plan[s], moved=True)
            staged.predict_measurements(s)  # check_truth leaves the trace rule's prediction behind
            staged.make_measurements(s, 0)
            staged.ekf_update_measured(s)
            assert_same_bytes(stream_result(staged, s, jacobians=True), stream_result(fused, s, jacobians=True),
                              (cap, s, len(plan[s].y), plan[s].n_select))
        report()
    finally:
        fused.close()
        staged.close()
