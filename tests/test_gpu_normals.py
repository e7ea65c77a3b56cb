"""The patch normals on the device (sl2_set_stream_normals, sl2_align_normals, sl2_get/set_patch_normals; csrc/normals.cu
normals_kernel, warp_kernel with normals on): bit for bit against the NumPy restatement (tests/normals_ref.py), the
fused step against the staged alignment, the default path and its launches, step groups, and the estimates' lifecycle
through the cull, deletion, appends, new maps, loads and the setter."""
import numpy as np
import pytest

import normals_ref
import normals_scene
import normals_truth
import warp_ref
import scenelib2_b200 as sl2
from gpu_util import assert_same_bytes, patch_snapshot_field, ring_block, stream_result
from rescue_scene import rescue_scene
from scenelib2_b200 import synth
from test_gpu_warp import cam8_of, scene_ctx

SL2_ERR_ARG, SL2_ERR_STATE = -1, -3  # include/sl2b200.h

PRM = dict(max_iterations=8, sigma0=0.5, sigma_i=8.0, sigma_step=0.02)


def prm_tuple(p=PRM):
    return (p["max_iterations"], p["sigma0"], p["sigma_i"], p["sigma_step"])


def check_alignment(ctx, s, slot, img, before, prm=PRM):
    """The fused step's alignment of stream s (the estimates `before` it, the step's frame `img` in ring slot `slot`)
    against sl2_align_normals from the same estimates and against the restatement; returns the statuses."""
    cam8 = cam8_of(ctx, s)
    nf = ctx.num_features(s)
    assert nf == len(before["theta"])
    idx = np.arange(nf)
    x, _ = ctx.get_state(s)
    f = ctx.features(s)
    y = x[13:13 + 3 * nf].reshape(nf, 3)
    xo, T = ctx_xp_org(ctx, s), ctx_patches(ctx, s)
    fused = ctx.patch_normals(s, idx)
    ctx.set_patch_normals(s, idx, before["theta"], before["cov"])
    ctx.align_normals(s, slot)
    got = ctx.patch_normals(s, idx)
    assert_same_bytes(fused, got, "fused vs staged, stream %d" % s, keys=["theta", "cov", "normal_w", "status"])
    for i in range(nf):
        if (f["flags"][i] & 3) != 3:
            assert got["status"][i] == 0
            assert got["theta"][i].tobytes() == before["theta"][i].tobytes()
            assert got["cov"][i].tobytes() == before["cov"][i].tobytes()
            continue
        (th, cv, acc, st), _ = normals_ref.align(cam8, img, T[i], y[i], xo[i], x[:7], f["z"][i], before["theta"][i],
                                                 before["cov"][i], prm_tuple(prm))
        assert got["status"][i] == st, (i, got["status"][i], st)
        assert np.array(th).tobytes() == got["theta"][i].tobytes(), (i, th, got["theta"][i])
        assert np.array(cv).tobytes() == got["cov"][i].tobytes(), (i, cv, got["cov"][i])
        assert got["count"][i] == acc and fused["count"][i] == before["count"][i] + acc
    ctx.set_patch_normals(s, idx, fused["theta"], fused["cov"])  # the fused step's estimates, counts reset
    return got["status"][:nf]


XP_ORG, PATCHES = {}, {}


def ctx_xp_org(ctx, s):
    return XP_ORG[id(ctx), s]


def ctx_patches(ctx, s):
    return PATCHES[id(ctx), s]


def load(ctx, s, y, xo, T, x0, P0):
    ctx.set_features(s, y, xo, T)
    ctx.set_state(s, x0, P0)
    XP_ORG[id(ctx), s] = np.asarray(xo, np.float64)
    PATCHES[id(ctx), s] = np.asarray(T, np.uint8)


def synth_ctx(name, num_streams=1, max_features=None, n_features=None):
    scs = [synth.make_scene(name, stream_id=s, n_frames=4, n_features=n_features) for s in range(num_streams)]
    cfg = sl2.config_for_scene(scs[0], num_streams=num_streams, max_features=max_features)
    ctx = sl2.Context(cfg)
    for s, sc in enumerate(scs):
        n = sc.n_features
        load(ctx, s, sc.x0[13:].reshape(n, 3), sc.xp_org, sc.patches, sc.x0, sc.P0)
    return ctx, scs


def slanted_ctx(num_streams=1, steps=12):
    sc = normals_scene.make_slanted_scene(steps=steps, end_deg=40.0 * steps / 40)
    ctx = scene_ctx([sc] * num_streams)
    for s in range(num_streams):
        XP_ORG[id(ctx), s] = sc.xp_org
        PATCHES[id(ctx), s] = sc.patches
    return ctx, sc


# ---- 1. sl2_align_normals against the restatement ------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["C1", "C2", "C3", "C4"])
def test_align_equals_the_restatement(name):
    ctx, scs = synth_ctx(name)
    try:
        ctx.set_stream_warp(0, 1)
        ctx.set_stream_normals(0, **PRM)
        aligned = 0
        for t in range(3):
            ctx.set_frames(0, scs[0].frames[t][None])
            before = ctx.patch_normals(0, np.arange(ctx.num_features(0)))
            ctx.step(0)
            ctx.sync()
            st = check_alignment(ctx, 0, 0, scs[0].frames[t], before)
            aligned += int((st > 0).sum())
        assert aligned > 0
    finally:
        ctx.close()


@pytest.mark.gpu
def test_align_on_the_slanted_plane_accepts_and_equals_the_restatement():
    ctx, sc = slanted_ctx()
    try:
        ctx.set_stream_warp(0, 1)
        ctx.set_stream_normals(0, **PRM)
        accepted = 0
        for t in range(1, 6):
            ctx.set_frames(0, sc.frames[t][None])
            before = ctx.patch_normals(0, np.arange(ctx.num_features(0)))
            ctx.step(0)
            ctx.sync()
            st = check_alignment(ctx, 0, 0, sc.frames[t], before)
            accepted += int((st == 1).sum())
        assert accepted >= len(sc.y)
    finally:
        ctx.close()


@pytest.mark.gpu
def test_capacity_256_and_a_stream_with_its_own_camera():
    """Stream 1 has its own 240 x 180 camera in a 320 x 240 context, with noise beyond its image in the ring block:
    the alignment's bounds are the stream's own.  A match moved next to its image's right edge (through a snapshot)
    makes the alignment's start invalid there, where the context's bounds would admit it."""
    ctx, scs = synth_ctx("C4", num_streams=2, max_features=256)
    try:
        small = synth.make_scene("C1", stream_id=1, n_frames=4, camera=synth.camera_params(240, 180))
        sc_cfg = ctx.stream_config(1)
        sc_cfg.width, sc_cfg.height = int(small.cam8[0]), int(small.cam8[1])
        sc_cfg.fku, sc_cfg.fkv, sc_cfg.u0, sc_cfg.v0, sc_cfg.kd1, sc_cfg.sd = [float(v) for v in small.cam8[2:8]]
        ctx.set_stream_config(1, sc_cfg)
        n = small.n_features
        load(ctx, 1, small.x0[13:].reshape(n, 3), small.xp_org, small.patches, small.x0, small.P0)
        H, W = scs[0].frames[0].shape
        rng = np.random.default_rng(240)
        for s in range(2):
            ctx.set_stream_warp(s, 1)
            ctx.set_stream_normals(s, **PRM)
        for t in range(2):
            fr = np.zeros((2, H, W), np.uint8)
            fr[0] = scs[0].frames[t]
            fr[1] = ring_block(small.frames[t], H, W, rng)
            ctx.set_frames(0, fr)
            before = [ctx.patch_normals(s, np.arange(ctx.num_features(s))) for s in range(2)]
            ctx.step(0)
            ctx.sync()
            for s in range(2):
                check_alignment(ctx, s, 0, fr[s], before[s])
        # the edge: feature i's match moved to u = 240 - 4, inside the context's 320 columns
        f = ctx.features(1)
        i = int(np.flatnonzero((f["flags"] & 3) == 3)[0])
        blob = patch_snapshot_field(ctx.save_stream(1), "z_uv", 2 * i, 240 - 4)
        ctx.load_stream(1, blob)
        assert ctx.features(1)["z"][i, 0] == 236.0
        before = ctx.patch_normals(1, np.arange(ctx.num_features(1)))
        ctx.align_normals(1, 0)
        got = ctx.patch_normals(1, [i])
        x, _ = ctx.get_state(1)
        (th, cv, acc, st), _ = normals_ref.align(small.cam8, small.frames[1], small.patches[i], x[13 + 3 * i:16 + 3 * i],
                                                 small.xp_org[i], x[:7], ctx.features(1)["z"][i], before["theta"][i],
                                                 before["cov"][i], prm_tuple())
        assert st == 3 and got["status"][0] == 3
        assert got["theta"][0].tobytes() == before["theta"][i].tobytes()
    finally:
        ctx.close()


# ---- 2. the warp through an estimated normal ------------------------------------------------------------------------
@pytest.mark.gpu
def test_warp_templates_through_set_normals_equal_the_restatement():
    ctx, sc = slanted_ctx()
    try:
        n = normals_scene.plane_normal(normals_scene.TILT)
        idx = np.arange(len(sc.y))
        ctx.set_stream_normals(0, **PRM)
        th = np.array([normals_scene.true_theta(sc.y[k], sc.xp_org[k], n) for k in idx])
        ctx.set_patch_normals(0, idx, th, np.tile([0.01, 0.0, 0.01], (len(idx), 1)))
        got = ctx.patch_normals(0, idx)
        assert got["theta"].tobytes() == th.tobytes() and (got["count"] == 0).all() and (got["status"] == 0).all()
        for k in idx:  # the unit normal the getter forms is the plane's
            assert abs(abs(got["normal_w"][k] @ n) - 1.0) < 1e-12
        for t in (4, 8, 12):
            out, valid = ctx.warp_templates(0, idx, sc.poses[t])
            for k in idx:
                want, wv = normals_ref.warp_template(sc.cam8, sc.patches[k], sc.y[k], sc.xp_org[k], sc.poses[t], th[k])
                assert valid[k] == wv and out[k].tobytes() == want.tobytes()
                # and the plane-to-plane view from its definition: the bytes of the truth's source positions, but
                # where the truth's sample lies within 1e-6 of a rounding boundary
                src = np.array(normals_truth.warp_source(sc.cam8, sc.boxsize, sc.y[k], sc.xp_org[k], sc.poses[t],
                                                         th[k]), np.float64).reshape(sc.boxsize, sc.boxsize, 2)
                v = unrounded_sample(sc.patches[k], src)
                edge = np.abs(v - np.floor(v) - 0.5) < 1e-6
                assert ((warp_ref.sample(sc.patches[k], src) == out[k]) | edge).all(), (t, k)
        # theta = 0 is the plain warp, byte for byte
        ctx.set_patch_normals(0, idx, np.zeros((len(idx), 2)), np.tile([0.25, 0.0, 0.25], (len(idx), 1)))
        on, _ = ctx.warp_templates(0, idx, sc.poses[8])
        ctx.set_stream_normals(0, max_iterations=0, sigma0=0.5, sigma_i=8.0, sigma_step=0.0)
        off, _ = ctx.warp_templates(0, idx, sc.poses[8])
        assert on.tobytes() == off.tobytes()
    finally:
        ctx.close()


def unrounded_sample(T, src):
    """warp_ref.sample before its rounding: the bilinear value at the clamped positions."""
    B = T.shape[0]
    Tf = T.astype(np.float64)
    sx = np.minimum(np.maximum(src[..., 0], 0.0), float(B - 1))
    sy = np.minimum(np.maximum(src[..., 1], 0.0), float(B - 1))
    x0 = np.minimum(np.floor(sx).astype(np.int64), B - 2)
    y0 = np.minimum(np.floor(sy).astype(np.int64), B - 2)
    fx, fy = sx - x0, sy - y0
    top = (1.0 - fx) * Tf[y0, x0] + fx * Tf[y0, x0 + 1]
    bot = (1.0 - fx) * Tf[y0 + 1, x0] + fx * Tf[y0 + 1, x0 + 1]
    return (1.0 - fy) * top + fy * bot


# ---- 3. the default path, launches, groups -------------------------------------------------------------------------
def run_steps(ctx, sc, steps, num_streams):
    for t in range(1, steps + 1):
        ctx.set_frames(0, np.stack([sc.frames[t]] * num_streams))
        ctx.step(0)
        ctx.sync()


@pytest.mark.gpu
def test_off_is_the_default_path_and_on_adds_one_launch_per_group():
    S, steps = 4, 5
    ctxs = [slanted_ctx(S)[0] for _ in range(3)]
    sc = normals_scene.make_slanted_scene(steps=12, end_deg=12.0)
    try:
        never, was_on, on = ctxs
        for c in ctxs:
            for s in range(S):
                c.set_stream_warp(s, 1)
        was_on.set_stream_normals(2, **PRM)
        was_on.set_stream_normals(2, max_iterations=0, sigma0=0.5, sigma_i=8.0, sigma_step=0.0)
        on.set_stream_normals(1, **PRM)
        counts = [0, 0, 0]
        for t in range(1, steps + 1):
            for j, c in enumerate(ctxs):
                l0 = c.launch_count()
                c.set_frames(0, np.stack([sc.frames[t]] * S))
                c.step(0)
                c.sync()
                counts[j] += c.launch_count() - l0
            if t == 1:
                # every estimate of the on stream was unestimated at this step's search: the fused step warped, searched
                # and updated exactly as the plain warp (the alignment only writes the estimates)
                assert_same_bytes(stream_result(never, 1, jacobians=True), stream_result(on, 1, jacobians=True),
                                  "first step of the on stream")
                assert (on.patch_normals(1, np.arange(len(sc.y)))["count"] > 0).any()
        for s in range(S):
            assert_same_bytes(stream_result(never, s), stream_result(was_on, s), "turned off, stream %d" % s)
        assert counts[1] == counts[0]
        assert counts[2] == counts[0] + steps
        # streams without normals in a context that has them are untouched
        for s in (0, 2, 3):
            assert_same_bytes(stream_result(never, s), stream_result(on, s), "off stream %d" % s)
    finally:
        for c in ctxs:
            c.close()


@pytest.mark.gpu
def test_two_step_groups_and_the_host_steps_give_the_same_bytes():
    S, steps = 4, 5
    sc = normals_scene.make_slanted_scene(steps=12, end_deg=12.0)
    ctxs = [slanted_ctx(S)[0] for _ in range(4)]
    try:
        for c in ctxs:
            for s in range(S):
                c.set_stream_warp(s, 1)
                c.set_stream_normals(s, **PRM)
        ctxs[1].set_step_groups(2)
        run_steps(ctxs[0], sc, steps, S)
        run_steps(ctxs[1], sc, steps, S)
        for c, host_async in ((ctxs[2], False), (ctxs[3], True)):
            for t in range(1, steps + 1):
                fr = np.ascontiguousarray(np.stack([sc.frames[t]] * S))
                if host_async:
                    c.step_host_async(0, fr.ctypes.data, 0)
                    c.wait_slot(0)
                else:
                    c.step_host(0, fr.ctypes.data, 0)
            c.sync()
        idx = np.arange(len(sc.y))
        for s in range(S):
            ref = ctxs[0].patch_normals(s, idx)
            for other in ctxs[1:]:
                assert_same_bytes(ref, other.patch_normals(s, idx), "normals, stream %d" % s)
                assert_same_bytes(stream_result(ctxs[0], s), stream_result(other, s), "stream %d" % s)
        assert (ref["count"] > 0).any()
    finally:
        for c in ctxs:
            c.close()


TAU, CHI2 = 2.5, 5.991  # the match consensus radius and the rescue's gate of the mixed runs


def pick_settings(ctx, s):
    """Stream 173's settings: warp, sub-pixel, consensus, rescue and normals."""
    ctx.set_stream_warp(s, 1)
    ctx.set_stream_subpixel(s, 1)
    ctx.set_stream_consensus(s, TAU)
    ctx.set_stream_rescue(s, CHI2)
    ctx.set_stream_normals(s, **PRM)


@pytest.mark.gpu
def test_a_stream_of_a_large_mixed_batch():
    """Stream 173 of a 264-stream context (the whole batch per launch, no programmatic dependent launch) with the warp,
    the sub-pixel refinement, the consensus, its rescue and the normals, among streams with every mix of them; stream
    172 has normals on and the warp off.  Stream 173 equals a one-stream context byte for byte at every step, and both,
    and stream 172, equal the restatement fed the refined matches.  The scene holds wrong matches the consensus rejects
    (never aligned) and uncertain new features whose matches the rescue takes back (aligned)."""
    T, B, pick = 4, 264, 173
    base = [synth.make_scene("C4", stream_id=u, n_frames=T + 1) for u in range(8)]
    sc_pick = rescue_scene("C4", stream_id=pick, n_frames=T + 1, n_features=100, new=range(92, 100), sigma=0.03,
                           wrong=[3, 50])
    scs = [sc_pick if s == pick else base[s % 8] for s in range(B)]
    cfg = sl2.config_for_scene(scs[0], num_streams=B)
    big = sl2.Context(cfg)
    alone = sl2.Context(sl2.config_for_scene(sc_pick, num_streams=1))
    twin = sl2.Context(sl2.config_for_scene(sc_pick, num_streams=1))  # the same without the rescue
    try:
        for s, sc in enumerate(scs):
            n = sc.n_features
            load(big, s, sc.x0[13:].reshape(n, 3), sc.xp_org, sc.patches, sc.x0, sc.P0)
        for c in (alone, twin):
            load(c, 0, sc_pick.x0[13:].reshape(100, 3), sc_pick.xp_org, sc_pick.patches, sc_pick.x0, sc_pick.P0)
        for s in range(B):
            if s % 4 == 0:
                big.set_stream_warp(s, 1)
            if s % 4 == 1:
                big.set_stream_consensus(s, TAU)
            if s % 3 == 2:
                big.set_stream_subpixel(s, 1)
            if s % 5 == 0:
                big.set_stream_normals(s, **PRM)
        big.set_stream_warp(pick - 1, 0)
        big.set_stream_normals(pick - 1, **PRM)
        pick_settings(big, pick)
        pick_settings(alone, 0)
        pick_settings(twin, 0)
        twin.set_stream_rescue(0, 0.0)
        seen = dict(rejected=0, rescued=0, refined=0, aligned_off_warp=0)
        for t in range(T):
            before = {s: big.patch_normals(s, np.arange(big.num_features(s))) for s in (pick - 1, pick)}
            before_alone = alone.patch_normals(0, np.arange(alone.num_features(0)))
            big.set_frames(0, np.stack([sc.frames[t] for sc in scs]))
            big.step(0)
            big.sync()
            for c in (alone, twin):
                c.set_frame(0, 0, sc_pick.frames[t])
                c.step(0)
                c.sync()
            idx = np.arange(alone.num_features(0))
            assert_same_bytes(stream_result(big, pick, jacobians=True), stream_result(alone, 0, jacobians=True),
                              "stream %d, step %d" % (pick, t))
            assert_same_bytes(big.patch_normals(pick, idx), alone.patch_normals(0, idx), "normals, step %d" % t)
            fa = alone.features(0)
            st = alone.patch_normals(0, idx)["status"]
            seen["rejected"] += int((fa["flags"] & 4).sum())
            assert (st[(fa["flags"] & 4) > 0] == 0).all()  # a match the consensus rejected is not aligned
            seen["refined"] += int(((fa["flags"] & 11) == 11).sum())
            if t == 0:  # the same inputs: rejected by the consensus without the rescue, found 1 with it
                rescued = ((twin.features(0)["flags"] & 4) > 0) & ((fa["flags"] & 2) > 0)
                seen["rescued"] = int(rescued.sum())
                assert (st[rescued] > 0).all()
            check_alignment(big, pick, 0, sc_pick.frames[t], before[pick])
            check_alignment(alone, 0, 0, sc_pick.frames[t], before_alone)
            st172 = check_alignment(big, pick - 1, 0, scs[pick - 1].frames[t], before[pick - 1])
            seen["aligned_off_warp"] += int((st172 > 0).sum())
        assert all(v > 0 for v in seen.values()), seen
    finally:
        for c in (big, alone, twin):
            c.close()


# ---- 4. lifecycle ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_estimates_move_with_their_features_and_reset_on_entry():
    ctx, sc = slanted_ctx()
    try:
        ctx.set_stream_warp(0, 1)
        ctx.set_stream_normals(0, **PRM)
        run_steps(ctx, sc, 3, 1)
        n = ctx.num_features(0)
        idx = np.arange(n)
        a = ctx.patch_normals(0, idx)
        assert (a["count"] > 0).any()
        ctx.delete_feature(0, 2)
        b = ctx.patch_normals(0, np.arange(n - 1))
        keep = np.delete(idx, 2)
        for k in ("theta", "cov", "count", "status"):
            assert b[k].tobytes() == a[k][keep].tobytes(), k
        # an appended feature starts unestimated
        x, _ = ctx.get_state(0)
        j = ctx.append_feature(0, sc.y[2], sc.xp_org[2], sc.patches[2])
        c = ctx.patch_normals(0, [j])
        assert (c["theta"] == 0).all() and (c["cov"][0] == [0.25, 0.0, 0.25]).all() and c["count"][0] == 0
        # the setter, a new map and a load reset the stream
        ctx.load_streams(ctx.save_streams(0, 1))
        d = ctx.patch_normals(0, np.arange(ctx.num_features(0)))
        assert (d["theta"] == 0).all() and (d["count"] == 0).all()
        run_steps(ctx, sc, 2, 1)
        ctx.set_features(0, sc.y, sc.xp_org, sc.patches)
        e = ctx.patch_normals(0, idx)
        assert (e["theta"] == 0).all() and (e["count"] == 0).all() and (e["cov"][:, 0] == 0.25).all()
        ctx.set_stream_normals(0, **dict(PRM, sigma0=0.3))
        assert (ctx.patch_normals(0, idx)["cov"][:, 0] == 0.09).all()
    finally:
        ctx.close()


@pytest.mark.gpu
def test_the_cull_moves_the_estimates():
    ctx, sc = slanted_ctx()
    try:
        ctx.set_stream_warp(0, 1)
        ctx.set_stream_normals(0, **PRM)
        run_steps(ctx, sc, 2, 1)
        n = len(sc.y)
        a = ctx.patch_normals(0, np.arange(n))
        # a frame that matches nothing, with min_attempts reached: the cull of the features that fail
        bad = np.zeros_like(sc.frames[0])
        ctx.set_frames(0, bad[None])
        for _ in range(12):
            ctx.step(0)
            ctx.sync()
            if ctx.num_features(0) < n:
                break
        m = ctx.num_features(0)
        assert m < n
        # the survivors keep their estimates in order (nothing was aligned on the blank frames)
        x, _ = ctx.get_state(0)
        y = x[13:13 + 3 * m].reshape(m, 3)
        kept = [int(np.argmin(np.abs(sc.y - yk).sum(axis=1))) for yk in y]
        assert kept == sorted(kept)
        b = ctx.patch_normals(0, np.arange(m))
        assert b["theta"].tobytes() == a["theta"][kept].tobytes()
        assert b["cov"].tobytes() == a["cov"][kept].tobytes()
    finally:
        ctx.close()


@pytest.mark.gpu
def test_rejected_arguments_change_nothing():
    ctx, sc = slanted_ctx()
    try:
        L, h = ctx.L, ctx.h
        bad = [dict(PRM, max_iterations=9), dict(PRM, max_iterations=-1), dict(PRM, sigma0=0.0),
               dict(PRM, sigma_i=float("nan")), dict(PRM, sigma_step=-1.0), dict(PRM, sigma0=float("inf"))]
        for b in bad:
            v = sl2.lib.Sl2StreamNormals(b["max_iterations"], 0, b["sigma0"], b["sigma_i"], b["sigma_step"])
            assert L.sl2_set_stream_normals(h, 0, sl2.lib.C.byref(v)) == SL2_ERR_ARG
        v = sl2.lib.Sl2StreamNormals(8, 1, 0.5, 8.0, 0.0)
        assert L.sl2_set_stream_normals(h, 0, sl2.lib.C.byref(v)) == SL2_ERR_ARG
        assert ctx.stream_normals(0)["max_iterations"] == 0
        assert L.sl2_align_normals(h, 0, 0) == SL2_ERR_STATE
        ctx.set_stream_normals(0, **PRM)
        idx = np.arange(len(sc.y))
        a = ctx.patch_normals(0, idx)
        for th, cv, ix in (([[np.nan, 0.0]], [[0.1, 0.0, 0.1]], [0]), ([[0.0, 0.0]], [[0.1, 0.2, 0.1]], [0]),
                           ([[0.0, 0.0]], [[-0.1, 0.0, 0.1]], [0]), ([[0.0, 0.0]], [[0.1, 0.0, 0.1]], [len(sc.y)])):
            with pytest.raises(sl2.Sl2Error):
                ctx.set_patch_normals(0, ix, th, cv)
        assert_same_bytes(a, ctx.patch_normals(0, idx), "after rejected sets")
        assert L.sl2_align_normals(h, 0, 5) == SL2_ERR_ARG
        assert L.sl2_align_normals(h, 3, 0) == SL2_ERR_ARG
        # later steps are those of a context that never saw the rejected calls
        clean, _ = slanted_ctx()
        try:
            clean.set_stream_normals(0, **PRM)
            for c in (ctx, clean):
                c.set_stream_warp(0, 1)
                run_steps(c, sc, 4, 1)
            assert_same_bytes(stream_result(ctx, 0, jacobians=True), stream_result(clean, 0, jacobians=True), "steps")
            assert_same_bytes(ctx.patch_normals(0, idx), clean.patch_normals(0, idx), "normals")
        finally:
            clean.close()
    finally:
        ctx.close()
