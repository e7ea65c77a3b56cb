"""Stream recovery inside the fused step (sl2_set_stream_recovery; csrc/recover.cu) on kidnapped scenes.

The oracle is a host emulation built from existing entry points only: a context without the feature steps, reads the
step's nmeas from its record and applies the rule of include/sl2b200.h through tests/recovery_ref.py, turning the
selection off with number_of_features_to_select = 0 while the stream is lost and trying sl2_relocalise when a try is
due.  The device run must match it byte for byte at every step."""
import ctypes as C

import numpy as np
import pytest

import recovery_ref as rv
import scenelib2_b200 as sl2
from gpu_util import assert_same_bytes, ctx_from_scenes, large_variant, ring_block, step_frames, stream_result
from model_cases import quat_to_R
from scenelib2_b200 import synth
from test_gpu_relocalise import MIN_INLIERS, OMEGA, PXX, TAU, V, kidnap_pose, render

SETTING = dict(inlier_px=TAU, min_inliers=MIN_INLIERS, v=V, omega=OMEGA, Pxx=PXX)


def min_matches(sc):
    """A failed step: fewer matches than a third of the selection (a fresh texture still gives a large selection a few
    chance matches under a 20 px search ellipse)"""
    return max(4, sc.n_select // 3)


def scene(cfg):
    if cfg == "C2-50":
        return synth.make_scene("C2", n_frames=5, n_features=50)
    if cfg == "cap256":
        return large_variant(256, 256, n_frames=5)
    return synth.make_scene(cfg.split("-")[0], n_frames=5)


class Case:
    """A scene tracked for its 5 frames (saved as a blob), then `occluded` fresh textures (no template anywhere), then
    the kidnapped frame (every template pasted at its projection under a pose the prediction cannot reach)."""

    def __init__(self, sc, seed, occluded, kidnapped, cap=None, pad=0):
        self.sc, self.cap, self.pad = sc, cap, pad
        rng = np.random.default_rng(seed)
        ctx = self.context(1)
        try:
            for t in range(5):
                self.step(ctx, sc.frames[t])
            self.blob = ctx.save_stream(0)
            x, _ = ctx.get_state(0)
        finally:
            ctx.close()
        y = x[13:].reshape(-1, 3)
        with np.errstate(all="ignore"):
            before = synth.project(sc.cam8, (y - x[:3]) @ quat_to_R(x[3:7]))
            for _ in range(1000):
                r, q = kidnap_pose(x, rng)
                after = synth.project(sc.cam8, (y - r) @ quat_to_R(q))
                if np.nanmin(np.sqrt(((after - before) ** 2).sum(axis=1))) > 30.0:
                    break
        self.r, self.q, self.y = r, q, y
        kid, self.at = render(sc, y, r, q, rng)
        self.frames = [synth.make_texture(rng, sc.height, sc.width) for _ in range(occluded)] + [kid] * kidnapped

    def context(self, B, slots=2):
        cfg = sl2.config_for_scene(self.sc, num_streams=B, frame_slots=slots, max_features=self.cap)
        cfg.width, cfg.height = self.sc.width + self.pad, self.sc.height + 2 * self.pad  # a larger ring: own camera
        ctx = sl2.Context(cfg)
        for s in range(B):
            ctx.set_stream_config(s, sl2.stream_config_for_scene(self.sc))
            sl2.load_scene(ctx, s, self.sc)
        return ctx

    def ring(self, ctx, img, B):
        rng = np.random.default_rng(int(img[0, :8].sum()))
        H, W = ctx.cfg.height, ctx.cfg.width
        return np.stack([ring_block(img, H, W, rng) for _ in range(B)])

    def step(self, ctx, img, slot=0):
        step_frames(ctx, self.ring(ctx, img, ctx.cfg.num_streams), slot)

    def contexts(self, B=1):
        ctx = self.context(B)
        ctx.load_streams([self.blob] * B)
        ctx.enable_records(4)
        return ctx


def emulate(case, cfg, mode=sl2.lib.SL2_SELECT_TRACE):
    """The device run of stream 0 with recovery on against the host emulation, step for step.  Returns per step a
    dict: st (the restatement's state), tried, sel (the step selected), nf, got (the device's state) and rec (its
    step record)."""
    dev, emu = case.contexts(), case.contexts()
    out = []
    try:
        for c in (dev, emu):
            c.set_stream_selection(0, mode)
        dev.set_stream_recovery(0, cfg["lost_after"], cfg["min_matches"], cfg["retry_period"], **SETTING)
        n_select = case.sc.n_select
        st, last = rv.fresh(), np.zeros(1, sl2.lib.RELOC_RESULT_DTYPE)[0]
        for t, img in enumerate(case.frames):
            slot = t % 2
            sel = rv.selects(cfg, st)
            emu.set_stream_config(0, number_of_features_to_select=n_select if sel else 0)
            case.step(dev, img, slot)
            case.step(emu, img, slot)
            nmeas = int(emu.records(0, 1, 1)[0, -1]["nmeas"])

            def accept():
                nonlocal last
                res, _, _ = emu.relocalise([0], slot, TAU, MIN_INLIERS, V, OMEGA, PXX)
                last = res[0]
                return bool(res[0]["status"] == 1)
            st, tried = rv.end_of_step(cfg, st, nmeas, accept)
            got = dev.recovery_results(0, 1)[0]
            where = (case.sc.meta.get("variant"), t)
            assert {k: int(got[k]) for k in rv.FIELDS} == st, (where, got, st)
            assert got["last"].tobytes() == last.tobytes(), where
            assert_same_bytes(stream_result(dev, 0, jacobians=True), stream_result(emu, 0, jacobians=True), where)
            assert dev.records(0, 1, 4).tobytes() == emu.records(0, 1, 4).tobytes(), where
            rec = dev.records(0, 1, 1)[0, -1]
            if not sel:  # rule 4: nothing selected, nothing attempted
                f = dev.features(0)
                assert rec["nsel"] == 0 and rec["nmeas"] == 0 and (f["select_rank"] == -1).all(), where
            out.append(dict(st=st, tried=tried, sel=sel, nf=dev.num_features(0), got=got, rec=rec))
    finally:
        dev.close()
        emu.close()
    return out


# ---- the device equals the host emulation ----------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cfg", ["C1", "C2-50", "C4", "C3", "C4-info", "cap256", "C1-own-camera"])
def test_device_equals_host_emulation(cfg):
    cap = 256 if cfg == "cap256" else None
    case = Case(scene(cfg), 11, occluded=6, kidnapped=5, cap=cap, pad=32 if "own" in cfg else 0)
    mode = sl2.lib.SL2_SELECT_INFORMATION if "info" in cfg else sl2.lib.SL2_SELECT_TRACE
    rule = dict(lost_after=3, min_matches=min_matches(case.sc), retry_period=3)
    out = emulate(case, rule, mode)
    print(cfg, "nmeas", [int(o["rec"]["nmeas"]) for o in out])
    tried = [t for t, o in enumerate(out) if o["tried"]]
    assert [t for t, o in enumerate(out) if o["got"]["attempted"]] == tried
    declared = next(t for t, o in enumerate(out) if o["st"]["lost"] or o["st"]["recoveries"])
    # attempts exactly on the due steps: the declaring step, then every third step until one is accepted
    accepted = next(t for t, o in enumerate(out) if o["st"]["recoveries"])
    assert tried == list(range(declared, accepted + 1, 3)), tried
    assert accepted >= 6  # on the kidnapped frame, not on an occluded one
    assert out[-1]["sel"] and out[-1]["st"]["lost"] == 0


# ---- the map survives the loss ---------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_the_map_survives_a_long_occlusion():
    sc = synth.make_scene("C4", n_frames=5)
    case = Case(sc, 23, occluded=40, kidnapped=12)
    off = case.contexts()
    try:
        for t in range(40):
            case.step(off, case.frames[t], t % 2)
        assert off.num_features(0) < sc.n_features  # the cull deleted the features the loss kept failing
    finally:
        off.close()
    rule = dict(lost_after=3, min_matches=min_matches(sc), retry_period=5)
    out = emulate(case, rule)
    declared = next(t for t, o in enumerate(out) if o["st"]["lost"])
    nf = [o["nf"] for o in out]
    accepted = next(t for t, o in enumerate(out) if o["st"]["recoveries"])
    assert len(set(nf[declared:accepted + 1])) == 1  # nothing is culled once the stream is lost
    due = [t for t in range(declared, len(out)) if (t - declared) % 5 == 0]
    assert accepted == min(t for t in due if t >= 40)  # the first due step that shows the map
    # the accepted pose is within the bounds test_gpu_relocalise holds the relocalisation to, and tracking resumes
    pose = out[accepted]["got"]["last"]["pose"]
    ang = 8 * 0.5 * np.sqrt(2.0) / sc.cam8[2]
    depth = float(((case.y - case.r) @ quat_to_R(case.q))[:, 2].max())
    assert np.abs(pose[:3] - case.r).max() <= ang * depth
    assert 2 * np.arccos(min(1.0, abs(float(pose[3:] @ case.q)))) <= ang
    assert all(o["sel"] and o["rec"]["nmeas"] >= 4 for o in out[accepted + 1:])


# ---- selection ---------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mode", [sl2.lib.SL2_SELECT_TRACE, sl2.lib.SL2_SELECT_INFORMATION])
def test_a_lost_stream_selects_nothing(mode):
    case = Case(synth.make_scene("C2", n_frames=5, n_features=50), 31, occluded=6, kidnapped=0)
    rule = dict(lost_after=2, min_matches=min_matches(case.sc), retry_period=100)

    out = emulate(case, rule, mode)  # checks rule 4 at every step that entered lost
    assert [o["sel"] for o in out] == [True, True, False, False, False, False]
    assert all(o["rec"]["nvisible"] > 0 for o in out)  # features stay visible: only the selection stops


# ---- the default path ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_default_path_is_untouched():
    """Streams with recovery off are byte-identical to a context without the feature, a stream with recovery on that
    never fails is byte-identical to recovery off, and only a step group holding an on stream launches three more
    kernels per step."""
    sc = synth.make_scene("C4", n_frames=12)
    B = 4
    a, b = ctx_from_scenes([sc] * B, frame_slots=2), ctx_from_scenes([sc] * B, frame_slots=2)
    try:
        for c in (a, b):
            c.set_step_groups(2)
        a.set_stream_recovery(3, lost_after=2, min_matches=1, retry_period=1, **SETTING)  # group B only
        for t in range(12):
            la, lb = a.launch_count(), b.launch_count()
            step_frames(a, np.stack([sc.frames[t]] * B), t % 2)
            step_frames(b, np.stack([sc.frames[t]] * B), t % 2)
            assert a.launch_count() - la == b.launch_count() - lb + 3, t
            for s in range(B):
                assert_same_bytes(stream_result(a, s, jacobians=True), stream_result(b, s, jacobians=True), (t, s))
        r = a.recovery_results()
        assert (r["lost"] == 0).all() and (r["attempted"] == 0).all() and r["failed_steps"][3] == 0
        a.set_stream_recovery(3, 0)
        la, lb = a.launch_count(), b.launch_count()
        step_frames(a, np.stack([sc.frames[0]] * B), 0)
        step_frames(b, np.stack([sc.frames[0]] * B), 0)
        assert a.launch_count() - la == b.launch_count() - lb
    finally:
        a.close()
        b.close()


# ---- regimes ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_regimes_give_the_same_bytes():
    """Serial order, two step groups, sl2_step_host, sl2_step_host_async and a single stream (PDL) give the same bytes
    for a lost stream, and so does the lost stream at index 173 of a 264-stream context beside tracking streams."""
    import torch
    case = Case(synth.make_scene("C4", n_frames=5), 41, occluded=4, kidnapped=4)
    rule = dict(lost_after=2, min_matches=min_matches(case.sc), retry_period=2)
    sc = case.sc

    def run(B, lost, groups=1, how="step"):
        ctx = case.contexts(B)
        try:
            if groups > 1:
                ctx.set_step_groups(groups)
            ctx.set_stream_recovery(lost, **rule, **SETTING)
            trail = []
            xv = torch.zeros((2, B, 13), dtype=torch.float64).pin_memory()
            for t, img in enumerate(case.frames):
                # the lost stream sees the case's frames; every other stream keeps seeing its tracked scene
                frames = case.ring(ctx, sc.frames[4], B)
                frames[lost, :sc.height, :sc.width] = img
                if how == "step":
                    step_frames(ctx, frames, t % 2)
                else:
                    host = torch.from_numpy(np.ascontiguousarray(frames)).pin_memory()
                    if how == "host":
                        ctx.step_host(t % 2, host.data_ptr(), xv[t % 2].data_ptr())
                    else:
                        ctx.step_host_async(t % 2, host.data_ptr(), xv[t % 2].data_ptr())
                        ctx.wait_slot(t % 2)
                    x, _ = ctx.get_state(lost)
                    assert xv[t % 2, lost].numpy().tobytes() == x[:13].tobytes()
                trail.append((stream_result(ctx, lost, jacobians=True), ctx.recovery_results(lost, 1).tobytes(),
                              ctx.records(lost, 1, 1).tobytes()))
            others = [s for s in (0, B - 1) if s != lost]
            return trail, [stream_result(ctx, s) for s in others]
        finally:
            ctx.close()

    ref, _ = run(1, 0)
    assert any(np.frombuffer(r, sl2.lib.RECOVERY_RESULT_DTYPE)["recoveries"][0] for _, r, _ in ref)
    for name, kw in (("serial", dict(B=3, lost=1)), ("groups", dict(B=3, lost=2, groups=2)),
                     ("host", dict(B=2, lost=1, how="host")), ("async", dict(B=3, lost=1, groups=2, how="async")),
                     ("264", dict(B=264, lost=173, groups=2))):
        trail, others = run(**kw)
        for t, (a, b) in enumerate(zip(trail, ref)):
            assert_same_bytes(a[0], b[0], (name, t))
            assert a[1] == b[1] and a[2][8:] == b[2][8:], (name, t)  # records: the step index aside
        for o in others:  # the tracking streams beside it see the same frames
            assert_same_bytes(o, others[0], (name, "tracking streams"))


# ---- resets and rejected arguments ----------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_resets_return_the_stream_to_tracking():
    case = Case(synth.make_scene("C2", n_frames=5, n_features=50), 51, occluded=3, kidnapped=1)
    rule = dict(lost_after=1, min_matches=min_matches(case.sc), retry_period=50)
    ctx = case.contexts()
    try:
        x, P = ctx.get_state(0)
        sc = case.sc

        def lose():
            ctx.set_stream_recovery(0, **rule, **SETTING)
            for t in range(2):
                case.step(ctx, case.frames[t], t % 2)
            r = ctx.recovery_results(0, 1)[0]
            assert r["lost"] == 1 and r["lost_steps"] == 1, r
            return r

        def tracking(before, keep_past):
            """back to tracking; a reset other than the setter keeps the past (recoveries, the last try)"""
            r = ctx.recovery_results(0, 1)[0]
            assert r["lost"] == 0 and r["failed_steps"] == 0 and r["lost_steps"] == 0
            if keep_past:
                assert r["last"].tobytes() == before["last"].tobytes() and r["recoveries"] == before["recoveries"]
            else:
                assert not r["last"].tobytes().strip(b"\0") and r["recoveries"] == 0 and r["attempted"] == 0

        b = lose()
        ctx.set_stream_recovery(0, **rule, **SETTING)
        tracking(b, False)
        b = lose()
        ctx.load_stream(0, case.blob)
        tracking(b, True)
        b = lose()  # on the blob's map: the kidnapped frame shows it
        ctx.set_frames(0, case.ring(ctx, case.frames[-1], 1))
        res, _, _ = ctx.relocalise([0], 0, TAU, MIN_INLIERS, V, OMEGA, PXX)
        assert res[0]["status"] == 1
        tracking(b, True)
        b = lose()
        ctx.set_state(0, x, P)
        tracking(b, True)
        b = lose()
        sl2.load_scene(ctx, 0, sc)
        tracking(b, True)
        lose()
        ctx.set_stream_recovery(0, 0)  # off while lost: the next step selects again
        tracking(None, False)
        case.step(ctx, case.frames[0])
        assert ctx.records(0, 1, 1)[0, -1]["nsel"] > 0
        # rejected arguments leave the setting and the later steps unchanged
        ctx.set_stream_recovery(0, **rule, **SETTING)
        before = bytes(ctx.stream_recovery(0))
        asym = PXX.copy()
        asym[0, 1] = 1e-9
        bad = [dict(lost_after=-1), dict(min_matches=0), dict(retry_period=0), dict(reserved=1),
               dict(inlier_px=0.0), dict(min_inliers=3), dict(omega=(0.0, 0.0, 0.0)), dict(v=(np.nan, 0, 0)),
               dict(Pxx=asym)]
        for kw in bad:
            with pytest.raises(sl2.Sl2Error):
                ctx.set_stream_recovery(0, **{**rule, **SETTING, **kw})
            assert bytes(ctx.stream_recovery(0)) == before, kw
        L = ctx.L
        assert L.sl2_set_stream_recovery(ctx.h, 0, None) < 0
        assert L.sl2_set_stream_recovery(ctx.h, 1, C.byref(ctx.stream_recovery(0))) < 0
        assert L.sl2_set_stream_recovery(ctx.h, -1, C.byref(ctx.stream_recovery(0))) < 0
        assert L.sl2_get_recovery_results(ctx.h, 0, 1, None) < 0
        assert L.sl2_get_recovery_results(ctx.h, 0, 2, None) < 0
        # off with any reloc values is accepted (nothing of it is read)
        ctx.set_stream_recovery(0, 0, min_matches=0, retry_period=0, omega=(0.0, 0.0, 0.0))
        assert bytes(ctx.stream_recovery(0)) != before
        ctx.set_stream_recovery(0, **rule, **SETTING)
        lose()
        twin = case.contexts()
        try:
            twin.set_stream_recovery(0, **rule, **SETTING)
            for t in range(2):
                case.step(twin, case.frames[t], t % 2)
            ctx.load_stream(0, twin.save_stream(0))
            ctx.set_stream_recovery(0, **rule, **SETTING)
            twin.set_stream_recovery(0, **rule, **SETTING)
            for c in (ctx, twin):
                case.step(c, case.frames[2], 0)
            assert_same_bytes(stream_result(ctx, 0), stream_result(twin, 0), "after the rejected calls")
        finally:
            twin.close()
    finally:
        ctx.close()


# ---- an empty map -----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_a_lost_stream_with_an_empty_map_tries_and_stays_lost():
    case = Case(synth.make_scene("C1", n_frames=5), 61, occluded=4, kidnapped=0)
    ctx, twin = case.contexts(), case.contexts()
    try:
        b = case.sc.boxsize
        for c in (ctx, twin):
            c.set_features(0, np.zeros((0, 3)), np.zeros((0, 7)), np.zeros((0, b, b), np.uint8))
        ctx.set_stream_recovery(0, lost_after=1, min_matches=1, retry_period=1, **SETTING)
        for t, img in enumerate(case.frames):
            case.step(ctx, img, t % 2)
            case.step(twin, img, t % 2)
            r = ctx.recovery_results(0, 1)[0]
            assert r["lost"] == 1 and r["attempted"] == 1 and r["lost_steps"] == t and r["recoveries"] == 0
            assert r["last"]["status"] == 0 and r["last"]["matches"] == 0 and np.isnan(r["last"]["pose"]).all()
            assert_same_bytes(stream_result(ctx, 0), stream_result(twin, 0), t)  # the try writes nothing
    finally:
        ctx.close()
        twin.close()
