"""The sub-pixel refinement on the device (sl2_set_stream_subpixel; csrc/subpixel.cu subpixel_kernel): its z and
refined flags bit for bit against the NumPy restatement (tests/subpixel_ref.py) on the device's own search results,
the isolation of off streams and the launch count, launch regimes, fused against staged, snapshots and rejected
arguments."""
import numpy as np
import pytest

import scenelib2_b200 as sl2
import subpixel_ref as ref
import subpixel_oracle as so
from gpu_util import (CAMS_320, assert_same_bytes, check_streams_against_oracle, ctx_from_scenes, large_variant,
                      ring_block, step_frames, stream_result)
from rescue_scene import rescue_scene
from scenelib2_b200 import synth

TAU = 2.5
CHI2 = 5.991

REFINED = 8  # sl2_get_features flags bit 3


def staged_measure(ctx, s, slot=0):
    ctx.ekf_predict(s)
    ctx.predict_measurements(s)
    ctx.make_measurements(s, slot)


def check_stream(on, off, s, frame, templates, width, height):
    """Stream s of `on` (refinement on) against `off` (the same state, refinement off) after the same measurement:
    every successful match's z and bit 3 equal the restatement fed off's integer match; everything else is off's.
    Returns the number of refined matches."""
    fo, ff = on.features(s), off.features(s)
    assert (fo["flags"] & (0xFF ^ REFINED)).tobytes() == ff["flags"].tobytes()
    zi = ff["z"]
    assert (zi == np.rint(zi)).all()
    n = 0
    for i in range(len(zi)):
        u, v = int(zi[i, 0]), int(zi[i, 1])
        if (ff["flags"][i] & 3) == 3:  # selected and successful
            zu, zv, ok = ref.refine(frame, width, height, templates[i], u, v)
            assert fo["z"][i].tobytes() == np.array([zu, zv]).tobytes(), i
            assert bool(fo["flags"][i] & REFINED) == ok, i
            n += ok
        elif not ff["flags"][i] & 1 and fo["flags"][i] & REFINED:
            # not selected: z and bit 3 keep the feature's last match, refined in an earlier step
            assert np.abs(fo["z"][i] - zi[i]).max() <= 0.5
        else:
            assert fo["z"][i].tobytes() == zi[i].tobytes() and not fo["flags"][i] & REFINED
    _, _, _, nu = on.feature_jacobians(s)
    sel = (fo["flags"] & 3) == 3
    assert nu[sel].tobytes() == (fo["z"] - fo["h"])[sel].tobytes()
    return n


def twins(sc, warp=False):
    on, off = ctx_from_scenes([sc]), ctx_from_scenes([sc])
    on.set_stream_subpixel(0, 1)
    if warp:
        on.set_stream_warp(0, 1)
        off.set_stream_warp(0, 1)
    return on, off


# ---- 1. decisions against the restatement, on the device's own search -------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,warp", [("C1", False), ("C2", False), ("C3", False), ("C4", False), ("C4", True)])
def test_decisions_equal_the_restatement(name, warp):
    T = 6
    sc = synth.make_scene(name, n_frames=T)
    on, off = twins(sc, warp)
    refined = 0
    for t in range(T):
        for c in (on, off):
            c.set_frame(0, 0, sc.frames[t])
            staged_measure(c, 0)
        if warp:
            fo = on.features(0)
            idx = np.arange(len(fo["flags"]))
            templates, _ = on.warp_templates(0, idx, on.get_state(0)[0][:7])
        else:
            templates = sc.patches
        refined += check_stream(on, off, 0, sc.frames[t], templates, sc.width, sc.height)
        on.ekf_update_measured(0)
        off.set_state(0, *on.get_state(0))
    assert refined >= T


def run_twins(on, off, frame_of, T, check):
    """T staged measurements of stream 0 of `on` and `off`, off taking on's state before each; check(t) after each."""
    refined = 0
    for t in range(T):
        for c in (on, off):
            c.set_frame(0, 0, frame_of(t))
            staged_measure(c, 0)
        refined += check(t)
        on.ekf_update_measured(0)
        off.set_state(0, *on.get_state(0))
    return refined


@pytest.mark.gpu
def test_decisions_at_capacity_256_with_128_selected():
    T = 4
    sc = large_variant(256, 128, n_frames=T)
    on, off = ctx_from_scenes([sc], max_features=256), ctx_from_scenes([sc], max_features=256)
    on.set_stream_subpixel(0, 1)

    def check(t):
        assert int((on.features(0)["select_rank"] >= 0).sum()) == 128
        return check_stream(on, off, 0, sc.frames[t], sc.patches, sc.width, sc.height)
    assert run_twins(on, off, lambda t: sc.frames[t], T, check) >= 4 * 100


@pytest.mark.gpu
def test_decisions_on_a_stream_with_its_own_smaller_camera():
    """The stream's image is 288 x 224 in a 320 x 240 ring block of noise: the refinement's edge test uses the stream's
    own width and height, so matches within one window of its right or bottom edge keep their integer position."""
    T = 6
    cam = CAMS_320[2]
    sc = synth.make_scene("C4", n_frames=T, camera=cam)
    W, H = int(cam[0]), int(cam[1])
    base = synth.make_scene("C4", n_frames=1)
    rng = np.random.default_rng(3)
    blocks = [ring_block(sc.frames[t], 240, 320, rng) for t in range(T)]
    on, off = ctx_from_scenes([base]), ctx_from_scenes([base])
    for c in (on, off):
        c.set_stream_config(0, width=W, height=H, fku=cam[2], fkv=cam[3], u0=cam[4], v0=cam[5], kd1=cam[6], sd=cam[7])
        sl2.load_scene(c, 0, sc)
    on.set_stream_subpixel(0, 1)

    def check(t):
        # the restatement sees the stream's own image: the block beyond it must not matter
        return check_stream(on, off, 0, blocks[t][:H, :W], sc.patches, W, H)
    assert run_twins(on, off, lambda t: blocks[t], T, check) >= T


# ---- 1b. whole steps against the oracle -----------------------------------------------------------------------------
@pytest.mark.gpu
def test_whole_steps_of_two_culling_streams_match_the_oracle():
    """20 fused steps of two streams with the refinement, the consensus and the rescue on, each with uncertain new
    features and two distractor templates that the cull deletes: selection, flags (bit 3 included), refined and
    integer z, counters exactly, h and S at the suite's step tolerances, state at 1e-8 (gpu_util)."""
    T = 20
    scs = [rescue_scene("C2", stream_id=s, n_frames=T, n_features=50, new=range(42, 50), sigma=0.03, wrong=[3, 25])
           for s in range(2)]
    ctx = ctx_from_scenes(scs)
    oracles = [so.slam_from_scene(sc, TAU, CHI2) for sc in scs]
    for s in range(2):
        ctx.set_stream_subpixel(s, 1)
        ctx.set_stream_consensus(s, TAU)
        ctx.set_stream_rescue(s, CHI2)
    refined = 0
    for t in range(T):
        step_frames(ctx, np.stack([sc.frames[t] for sc in scs]))
        check_streams_against_oracle(ctx, oracles, [0, 1], lambda s: scs[s], t)
        # the oracle's update, consensus and rescue read the refined z: a consumer reading the integer match would
        # leave the device's state far outside 1e-8
        refined += sum(int(((ctx.features(s)["flags"] & 10) == 10).sum()) for s in range(2))
    assert refined > 0
    for s in range(2):
        assert oracles[s].num_features < scs[s].n_features  # through a cull


@pytest.mark.gpu
def test_a_feature_appended_after_a_cull_starts_unrefined():
    T = 14
    sc = rescue_scene("C2", n_frames=T, n_features=50, wrong=[3, 25, 40, 48])
    ctx = ctx_from_scenes([sc])
    ctx.set_stream_subpixel(0, 1)
    for t in range(T):
        step_frames(ctx, sc.frames[t][None])
        if ctx.num_features(0) < sc.n_features:
            break
    nf = ctx.num_features(0)
    assert nf < sc.n_features
    before = ctx.features(0)
    assert (before["flags"] & 8).any()
    for _ in range(sc.n_features - nf):
        ctx.append_feature(0, sc.x0[13:16], sc.xp_org[0], sc.patches[0])
    f = ctx.features(0)
    assert not (f["flags"][nf:] & 8).any() and (f["z"][nf:] == np.rint(f["z"][nf:])).all()
    _, _, _, nu = ctx.feature_jacobians(0)
    assert (nu[nf:] == f["z"][nf:] - f["h"][nf:]).all()
    assert_same_bytes({k: v[:nf] for k, v in f.items()}, {k: v[:nf] for k, v in before.items()}, "kept")


# ---- 2. off means off; one launch per step group ----------------------------------------------------------------
@pytest.mark.gpu
def test_off_streams_are_untouched_and_launches_rise_by_one_per_group():
    T = 8
    scs = [synth.make_scene("C2", stream_id=s, n_frames=T) for s in range(2)]
    plain, mixed, toggled = ctx_from_scenes(scs), ctx_from_scenes(scs), ctx_from_scenes(scs)
    mixed.set_stream_subpixel(1, 1)
    toggled.set_stream_subpixel(0, 1)
    toggled.set_stream_subpixel(0, 0)
    assert mixed.get_stream_subpixel(1) == 1 and mixed.get_stream_subpixel(0) == 0
    frames = lambda t: np.stack([scs[s].frames[t] for s in range(2)])  # noqa: E731
    l0 = [c.launch_count() for c in (plain, mixed, toggled)]
    for t in range(T):
        for c in (plain, mixed, toggled):
            c.set_frames(0, frames(t))
            c.step(0)
            c.sync()
    dl = [c.launch_count() - l for c, l in zip((plain, mixed, toggled), l0)]
    assert dl[1] == dl[0] + T and dl[2] == dl[0]
    for s in range(2):
        assert_same_bytes(stream_result(toggled, s, jacobians=True), stream_result(plain, s, jacobians=True), s)
    assert_same_bytes(stream_result(mixed, 0, jacobians=True), stream_result(plain, 0, jacobians=True), "off")
    f1 = mixed.features(1)
    assert (f1["flags"] & REFINED).any()
    assert not (plain.features(1)["flags"] & REFINED).any()


# ---- 3. launch regimes -------------------------------------------------------------------------------------------
def run_regime(regime, scs, T):
    B = len(scs)
    ctx = ctx_from_scenes(scs)
    for s in range(B):
        ctx.set_stream_subpixel(s, 1)
        ctx.set_stream_consensus(s, 2.5)
        ctx.set_stream_rescue(s, 5.991)
    if regime == "groups":
        ctx.set_step_groups(2)
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
    return [stream_result(ctx, s, jacobians=True) for s in range(B)]


@pytest.mark.gpu
def test_every_launch_regime_gives_the_same_bytes():
    T = 10
    scs = [synth.make_scene("C4", stream_id=s, n_frames=T) for s in range(4)]
    base = run_regime("serial", scs, T)
    for regime in ("groups", "host", "host_async"):
        got = run_regime(regime, scs, T)
        for s in range(4):
            assert_same_bytes(got[s], base[s], (regime, s))
    single = run_regime("serial", [scs[2]], T)
    assert_same_bytes(single[0], base[2], "single")


@pytest.mark.gpu
def test_a_stream_of_a_large_mixed_batch():
    T = 6
    B, pick = 264, 173
    cfgs = ["C4", "C2"]
    scs = [synth.make_scene(cfgs[s % 2] if s != pick else "C4", stream_id=s, n_frames=T, n_features=100)
           for s in range(B)]
    ctx = ctx_from_scenes(scs)
    for s in range(0, B, 3):
        ctx.set_stream_subpixel(s, 1)
    ctx.set_stream_subpixel(pick, 1)
    ctx.set_stream_consensus(pick, 2.5)
    for t in range(T):
        ctx.set_frames(0, np.stack([sc.frames[t] for sc in scs]))
        ctx.step(0)
    ctx.sync()
    alone = ctx_from_scenes([scs[pick]])
    alone.set_stream_subpixel(0, 1)
    alone.set_stream_consensus(0, 2.5)
    for t in range(T):
        alone.set_frame(0, 0, scs[pick].frames[t])
        alone.step(0)
    alone.sync()
    assert_same_bytes(stream_result(ctx, pick, jacobians=True), stream_result(alone, 0, jacobians=True), "pick")


# ---- 4. fused against staged -------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["C1", "C4"])
def test_fused_equals_staged(name):
    T = 6
    sc = synth.make_scene(name, n_frames=T)
    fused, staged = ctx_from_scenes([sc]), ctx_from_scenes([sc])
    for c in (fused, staged):
        c.set_stream_subpixel(0, 1)
        c.set_stream_consensus(0, 2.5)
        c.set_stream_rescue(0, 5.991)
    for t in range(T):
        fused.set_frame(0, 0, sc.frames[t])
        fused.step(0)
        fused.sync()
        staged.set_frame(0, 0, sc.frames[t])
        staged_measure(staged, 0)
        staged.ekf_update_measured(0)
        a, b = stream_result(fused, 0, jacobians=True), stream_result(staged, 0, jacobians=True)
        if fused.num_features(0) != sc.n_features:
            break  # the fused step culled: the staged path has no cull
        assert_same_bytes(a, b, t)


# ---- 5. snapshots ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_snapshots_continue_and_read_back_the_integer_match():
    T, k = 10, 4
    sc = synth.make_scene("C4", n_frames=T)
    run, resumed = ctx_from_scenes([sc]), ctx_from_scenes([synth.make_scene("C2", n_frames=1, n_features=100)])
    run.set_stream_subpixel(0, 1)
    resumed.set_stream_subpixel(0, 1)
    for t in range(T):
        run.set_frame(0, 0, sc.frames[t])
        run.step(0)
        run.sync()
        if t == k - 1:
            assert (run.features(0)["flags"] & REFINED).any()
            resumed.load_stream(0, run.save_stream(0))
            f = resumed.features(0)
            assert not (f["flags"] & REFINED).any() and (f["z"] == np.rint(f["z"])).all()
            assert f["flags"].tobytes() == (run.features(0)["flags"] & (0xFF ^ REFINED)).tobytes()
        elif t >= k:
            resumed.set_frame(0, 0, sc.frames[t])
            resumed.step(0)
            resumed.sync()
            assert_same_bytes(stream_result(resumed, 0, jacobians=True), stream_result(run, 0, jacobians=True), t)


# ---- 6. arguments ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_rejected_arguments_change_nothing():
    sc = synth.make_scene("C2", n_frames=1)
    ctx = ctx_from_scenes([sc, sc])
    ctx.set_stream_subpixel(1, 1)
    for s, on in ((0, 2), (0, -1), (1, 7), (2, 1), (-1, 0)):
        with pytest.raises(sl2.lib.Sl2Error):
            ctx.set_stream_subpixel(s, on)
    assert ctx.get_stream_subpixel(0) == 0 and ctx.get_stream_subpixel(1) == 1
    with pytest.raises(sl2.lib.Sl2Error):
        ctx.get_stream_subpixel(2)
