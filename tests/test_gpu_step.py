"""GPU parity, fused step (MonoSLAM::GoOneStep, monoslam.cpp:108-180) for several independent
camera streams in one context vs one CPU oracle per stream."""
import os

import numpy as np
import pytest

from gpu_util import (RTOL_NORTH_STAR, assert_state_close, check_streams_against_oracle, ctx_from_scenes,
                      oracle_slam_from_scene, sl2, state_err, step_frames, synth)

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _run(oracle, scenes, steps, slots=2):
    ctx = ctx_from_scenes(scenes, frame_slots=slots)
    oracles = [oracle_slam_from_scene(oracle, sc) for sc in scenes]
    worst = (0.0, 0.0)
    for t in range(steps):
        k = t % scenes[0].frames.shape[0]
        step_frames(ctx, np.stack([sc.frames[k] for sc in scenes]), t % slots)
        w = check_streams_against_oracle(ctx, oracles, range(len(scenes)), lambda s: scenes[s], k)
        worst = (max(worst[0], w[0]), max(worst[1], w[1]))
    ctx.close()
    return worst


def test_three_streams_c2_like(oracle):
    scenes = [synth.make_scene("C2", stream_id=s, n_frames=6, n_features=24, override=False)
              for s in range(3)]
    w = _run(oracle, scenes, 6)
    print("worst errors:", w)


def test_c1_reference_config(oracle):
    kp = np.load(os.path.join(G, "known_patches.npy"))
    scenes = [synth.make_scene("C1", stream_id=s, n_frames=5, known_patches=kp) for s in range(2)]
    _run(oracle, scenes, 8)


def test_bad_feature_is_culled_like_the_reference(oracle):
    sc = synth.make_scene("C2", n_frames=2, n_features=12)
    bad = sc.patches.copy()
    bad[3] = np.random.default_rng(0).integers(0, 256, bad[3].shape, dtype=np.uint8)
    sc.patches = bad
    good = synth.make_scene("C2", stream_id=1, n_frames=2, n_features=12)
    ctx_scenes = [sc, good]
    _run(oracle, ctx_scenes, 12)


def test_c4_full_size_two_frames(oracle):
    """BASELINE config C4: 320x240, N = 100 (n = 313, m = 200), fixed +-20 px search."""
    sc = synth.make_scene("C4", n_frames=2)
    assert sc.n == 313 and sc.search_override[0] > 0
    w = _run(oracle, [sc], 2)
    assert max(w) < RTOL_NORTH_STAR
    print("C4 worst errors:", w)


def test_c3_full_size_one_frame(oracle):
    sc = synth.make_scene("C3", n_frames=1)
    w = _run(oracle, [sc], 1, slots=1)
    print("C3 worst errors:", w)


def test_step_host_returns_camera_states(oracle):
    scenes = [synth.make_scene("C2", stream_id=s, n_frames=2, n_features=16) for s in range(2)]
    ctx = ctx_from_scenes(scenes)
    frames = np.ascontiguousarray(np.stack([sc.frames[0] for sc in scenes]))
    xv = np.zeros((2, 13))
    ctx.step_host(0, frames.ctypes.data, xv.ctypes.data)
    for s, sc in enumerate(scenes):
        o = oracle_slam_from_scene(oracle, sc)
        o.step(sc.frames[0])
        xo, Po = o.get_state()
        assert np.allclose(xv[s], xo[:13], rtol=1e-7, atol=1e-12)
    ctx.close()


def test_async_host_ring_matches_blocking(oracle):
    """sl2_step_host_async (copy of frame t+1 overlapped with the step of frame t) == blocking path."""
    import torch
    scenes = [synth.make_scene("C2", stream_id=s, n_frames=4, n_features=16) for s in range(3)]
    a = ctx_from_scenes(scenes, frame_slots=4)
    b = ctx_from_scenes(scenes, frame_slots=4)
    host = torch.empty((4, 3, 240, 320), dtype=torch.uint8, pin_memory=True)
    host.numpy()[:] = np.stack([np.stack([sc.frames[t] for sc in scenes]) for t in range(4)])
    xa = torch.zeros((4, 3, 13), dtype=torch.float64, pin_memory=True)
    xb = np.zeros((4, 3, 13))
    for t in range(4):
        a.step_host_async(t, host[t].data_ptr(), xa[t].data_ptr())
    for t in range(4):
        b.step_host(t, host[t].data_ptr(), xb[t].ctypes.data)
    a.wait_slot(3)
    a.sync()
    assert (xa.numpy() == xb).all()
    for s in range(3):
        xs, Ps = a.get_state(s)
        xt, Pt = b.get_state(s)
        assert (xs == xt).all() and (Ps == Pt).all()
    a.close()
    b.close()


def test_empty_map_and_invisible_features(oracle):
    """Edge cases of GoOneStep: a stream with no features at all, and one whose features are all
    outside the image (visibility test fails -> nothing selected, no update; monoslam.cpp:130-139)."""
    import scenelib2_b200 as sl2
    sc = synth.make_scene("C2", n_frames=2, n_features=8)
    far = synth.make_scene("C2", stream_id=1, n_frames=2, n_features=8)
    far.x0 = far.x0.copy()
    far.x0[13:] += np.tile([3.0, 0.0, 0.0], 8)          # all features far to the side of the view
    cfg = sl2.config_for_scene(sc, num_streams=3, frame_slots=1)
    ctx = sl2.Context(cfg)
    sl2.load_scene(ctx, 0, sc)
    sl2.load_scene(ctx, 1, far)
    ctx.set_features(2, np.zeros((0, 3)), np.zeros((0, 7)), np.zeros((0, 11, 11), np.uint8))
    x2 = np.zeros(13)
    x2[3], x2[12] = 1.0, 0.01
    ctx.set_state(2, x2, np.eye(13) * 1e-4)
    o0, o1 = oracle_slam_from_scene(oracle, sc), oracle_slam_from_scene(oracle, far)
    for t in range(2):
        step_frames(ctx, np.stack([sc.frames[t], far.frames[t], sc.frames[t]]))
        o0.step(sc.frames[t])
        o1.step(far.frames[t])
    assert_state_close(*ctx.get_state(0), *o0.get_state())
    assert_state_close(*ctx.get_state(1), *o1.get_state())
    f1 = ctx.features(1)
    assert (f1["select_rank"] == -1).all() and (f1["attempted"] == 0).all()
    x, P = ctx.get_state(2)
    assert ctx.num_features(2) == 0 and np.isfinite(P).all() and P.shape == (13, 13)
    # empty map: only the prediction acts (kalman.cpp:50-62)
    fv, F, Q = oracle.motion(x2, sc.delta_t)
    fv2, F2, Q2 = oracle.motion(fv, sc.delta_t)
    Pe = F2 @ (F @ (np.eye(13) * 1e-4) @ F.T + Q) @ F2.T + Q2
    Pe = 0.5 * (Pe + Pe.T)
    assert np.allclose(x, fv2, rtol=1e-12, atol=1e-15)
    assert np.abs(P - Pe).max() <= 1e-9 * np.abs(Pe).max()
    ctx.close()


def test_c4_many_streams_ground_truth_properties():
    """Full BASELINE size (C4: n = 313, m = 200) with 37 streams in one context, checked through
    size-independent properties instead of the oracle: every feature is found at its known ground-truth
    pixel (template position + frame shift), P stays exactly symmetric and positive semi-definite, and
    the map uncertainty never grows."""
    B, T = 37, 4
    scenes = [synth.make_scene("C4", stream_id=s, n_frames=T) for s in range(B)]
    ctx = ctx_from_scenes(scenes, frame_slots=2)
    tr_prev = [np.trace(sc.P0[13:, 13:]) for sc in scenes]
    for t in range(T):
        step_frames(ctx, np.stack([sc.frames[t] for sc in scenes]), t % 2)
        for s in (0, 7, 18, 36) if t < T - 1 else range(B):
            sc = scenes[s]
            f = ctx.features(s)
            assert ((f["flags"] & 3) == 3).all()                      # selected and successfully measured
            assert (f["z"] == sc.pix + sc.shifts[t]).all()            # ground truth, bit-exact
            x, P = ctx.get_state(s)
            assert np.abs(P - P.T).max() == 0.0
            tr = np.trace(P[13:, 13:])
            assert tr <= tr_prev[s] * (1 + 1e-12)
            tr_prev[s] = tr
            if t == T - 1:
                w = np.linalg.eigvalsh(P)
                assert w.min() > -1e-10 * w.max()
                assert abs(np.linalg.norm(x[3:7]) - 1.0) < 1e-2      # quaternion stays near unit (quirk Q1)
    ctx.close()


def test_maximum_map_size_fused_step(oracle):
    """SL2_MAX_FEATURES = 128 features per stream (n = 397, m = 256): the largest supported map."""
    sc = synth.make_scene("C4", n_frames=2, n_features=128)
    sc.n_select = 128
    assert sc.n == 397
    w = _run(oracle, [sc], 2)
    print("max-size worst errors:", w)


def test_long_run_does_not_drift_from_oracle(oracle):
    """40 consecutive frames (ring of 8) on a C2-sized map with the EKF's own search ellipses: the
    CUDA path and the oracle must keep making the same decisions (same selected set, same matches,
    same culling) and stay within the north-star tolerance at every frame, i.e. rounding
    differences do not accumulate."""
    sc = synth.make_scene("C2", n_frames=8, n_features=50, override=False)
    ctx = ctx_from_scenes([sc], frame_slots=2)
    o = oracle_slam_from_scene(oracle, sc)
    worst = 0.0
    for t in range(40):
        k = t % 8
        step_frames(ctx, sc.frames[k][None], t % 2)
        o.step(sc.frames[k])
        fg, fo = ctx.features(0), o.features()
        assert ctx.num_features(0) == o.num_features
        assert (fg["select_rank"] == fo["select_rank"]).all() and (fg["flags"] == fo["flags"]).all(), t
        ok = (fo["flags"] & 2) > 0
        assert (fg["z"][ok] == fo["z"][ok]).all(), t
        ex, eP = state_err(*ctx.get_state(0), *o.get_state())
        worst = max(worst, ex, eP)
        assert max(ex, eP) < 1e-7, (t, ex, eP)
    print("long run worst error:", worst)
    ctx.close()


def test_two_devices_in_one_process(oracle):
    """Two contexts on two GPUs driven from ONE process (each call selects its device itself)."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import scenelib2_b200 as sl2
    scenes = [synth.make_scene("C2", stream_id=s, n_frames=3, n_features=20) for s in range(2)]
    ctxs = []
    for dev, sc in enumerate(scenes):
        cfg = sl2.config_for_scene(sc, num_streams=1, frame_slots=1, device=dev)
        c = sl2.Context(cfg)
        sl2.load_scene(c, 0, sc)
        ctxs.append(c)
    oracles = [oracle_slam_from_scene(oracle, sc) for sc in scenes]
    for t in range(3):
        for c, sc in zip(ctxs, scenes):         # interleaved calls: device 0, device 1, ...
            c.set_frames(0, sc.frames[t][None])
            c.step(0)
        for c, sc, o in zip(ctxs, scenes, oracles):
            c.sync()
            o.step(sc.frames[t])
            assert (c.features(0)["z"] == o.features()["z"]).all()
            assert_state_close(*c.get_state(0), *o.get_state())
    for c in ctxs:
        c.close()


def test_staggered_stream_groups_match_serial_order():
    """sl2_set_step_groups: the fused step run as two staggered stream groups on internal CUDA streams
    gives bit-identical states to the serial kernel order, for back-to-back sl2_step calls, for the
    asynchronous host ring, and when other entry points are interleaved (they join the groups)."""
    import torch
    nS, T = 5, 6
    scenes = [synth.make_scene("C2", stream_id=s, n_frames=4, n_features=20) for s in range(nS)]
    ctxs = []
    for groups in (1, 2):
        c = ctx_from_scenes(scenes, frame_slots=4)
        c.set_step_groups(groups)
        ctxs.append(c)
    host = torch.empty((4, nS, 240, 320), dtype=torch.uint8, pin_memory=True)
    host.numpy()[:] = np.stack([np.stack([sc.frames[t] for sc in scenes]) for t in range(4)])
    xs = [torch.zeros((4, nS, 13), dtype=torch.float64, pin_memory=True) for _ in ctxs]
    for c in ctxs:                                   # device-resident frames, steps back to back
        for t in range(4):
            c.set_frames(t, host[t].numpy())
        for t in range(T):
            c.step(t % 4)
    for s in range(nS):                              # get_state joins the groups
        (x1, P1), (x2, P2) = ctxs[0].get_state(s), ctxs[1].get_state(s)
        assert (x1 == x2).all() and (P1 == P2).all(), s
    for c, xo in zip(ctxs, xs):                      # host ring on top of the same contexts
        for t in range(T):
            c.step_host_async(t % 4, host[t % 4].data_ptr(), xo[t % 4].data_ptr())
        c.sync()
    assert (xs[0].numpy() == xs[1].numpy()).all()
    for s in range(nS):
        (x1, P1), (x2, P2) = ctxs[0].get_state(s), ctxs[1].get_state(s)
        assert (x1 == x2).all() and (P1 == P2).all(), s
        f1, f2 = ctxs[0].features(s), ctxs[1].features(s)
        assert all((f1[k] == f2[k]).all() for k in ("z", "flags", "attempted", "successful"))
    for c in ctxs:
        c.close()


def test_c1_trajectory_1000_steps_matches_oracle_fixture():
    """The CUDA path over the 1 000-step C1 trajectory of tests/golden/c1_trajectory_1000.npz (an output of the
    REFERENCE'S OWN code, see tests/golden/make_c1_trajectory.py): selection ranks, found flags and match
    positions of EVERY step hash to the reference's value (bit-exact integer results over 10 000
    measurements); camera state within the north-star tolerance at every 100th step."""
    import hashlib
    import sys
    sys.path.insert(0, G)
    import make_c1_trajectory as gen
    k = np.load(os.path.join(G, "c1_trajectory_1000.npz"))
    kp = np.load(os.path.join(G, "known_patches.npy"))
    sc = synth.make_scene("C1", n_frames=gen.RING, known_patches=kp)
    ctx = ctx_from_scenes([sc], frame_slots=gen.RING)
    for t in range(gen.RING):
        ctx.set_frames(t, sc.frames[t:t + 1])
    hz = hashlib.sha256()
    xs = []
    for t in range(gen.STEPS):
        ctx.step(gen.frame_index(t))
        f = ctx.features(0)
        hz.update(np.ascontiguousarray(f["select_rank"], np.int32).tobytes())
        hz.update(np.ascontiguousarray(f["flags"], np.uint8).tobytes())
        ok = (f["flags"] & 2) > 0
        hz.update(np.ascontiguousarray(f["z"][ok], np.float64).tobytes())
        if (t + 1) % gen.EVERY == 0:
            x, P = ctx.get_state(0)
            xs.append((x[:13].copy(), np.diag(P)[:13].copy()))
    f = ctx.features(0)
    assert (np.frombuffer(hz.digest(), np.uint8) == k["integer_hash"]).all()
    assert (f["attempted"] == k["attempted"]).all() and (f["successful"] == k["successful"]).all()
    for i, (xv, pd) in enumerate(xs):
        np.testing.assert_allclose(xv, k["xv"][i], rtol=RTOL_NORTH_STAR, atol=1e-9)
        np.testing.assert_allclose(pd, k["Pxx_diag"][i], rtol=RTOL_NORTH_STAR, atol=1e-15)
    ctx.close()


def test_cuda_path_against_the_reference_source(oracle, reference, tmp_path):
    """The CUDA path vs the REFERENCE'S OWN MonoSLAM code (monoslam.cpp / kalman.cpp / feature.cpp / models /
    improc compiled unmodified against oracle/stubs_arith, oracle/_ref/libsl2refmodels.so; see
    oracle/ref_slam_shim.cpp), replayed from tests/golden: selection ranks, flags, match positions and counters identical on every frame,
    state and covariance within the test tolerance (C1, and a 24-feature scene where every feature is measured)."""
    kp = np.load(os.path.join(G, "known_patches.npy"))
    cases = [(synth.make_scene("C1", n_frames=10, known_patches=kp), 10),
             (synth.make_scene("C2", n_frames=4, n_features=24, override=False), 4)]
    for ci, (sc, steps) in enumerate(cases):
        ctx = ctx_from_scenes([sc], frame_slots=1)
        ref = reference.slam(sc, str(tmp_path / ("case%d" % ci)))
        for t in range(steps):
            ctx.set_frames(0, sc.frames[t:t + 1])
            ctx.step(0)
            ref.step(sc.frames[t])
            fg, fr = ctx.features(0), ref.features()
            assert ctx.num_features(0) == ref.num_features
            assert (fg["select_rank"] == fr["select_rank"]).all(), (ci, t)
            assert ((fg["flags"] & 1) == (fr["flags"] & 1)).all(), (ci, t)
            seen = fr["attempted"] > 0
            assert ((fg["flags"] & 2)[seen] == (fr["flags"] & 2)[seen]).all(), (ci, t)
            ok = (fr["flags"] & 2) > 0
            assert (fg["z"][ok] == fr["z"][ok]).all(), (ci, t)
            assert (fg["attempted"] == fr["attempted"]).all() and (fg["successful"] == fr["successful"]).all()
            xg, Pg = ctx.get_state(0)
            xr, Pr = ref.get_state()
            stored = np.isfinite(Pr)                          # the stored entries of the reference's P
            assert_state_close(xg, np.where(stored, Pg, 0.0), xr, np.where(stored, Pr, 0.0))
        ctx.close()


def test_c4_bench_shape_264_streams_against_oracle(oracle):
    """The shape bench.py runs (BASELINE C4, 264 camera streams in one context: 2 per SM of an H100), 3 frames, with the first,
    the two middle and the last stream compared with the oracle -- a stream-indexing bug above the sizes of the other
    tests (<= 37 streams) cannot hide.  The remaining streams are checked against the ground truth of the scene."""
    B, T, U = 264, 3, 8
    uniq = [synth.make_scene("C4", stream_id=u, n_frames=T) for u in range(U)]
    scene_of = lambda s: uniq[(s * 5) % U]          # neighbours get different scenes
    cfg_ctx = ctx_from_scenes([scene_of(s) for s in range(B)], frame_slots=2)
    picks = (0, 131, 132, 263)
    assert len({(s * 5) % U for s in picks}) == 4
    oracles = {s: oracle_slam_from_scene(oracle, scene_of(s)) for s in picks}
    for t in range(T):
        step_frames(cfg_ctx, np.stack([scene_of(s).frames[t] for s in range(B)]), t % 2)
        check_streams_against_oracle(cfg_ctx, oracles, picks, scene_of, t)
        for s in range(0, B, 7):
            sc = scene_of(s)
            f = cfg_ctx.features(s)
            assert ((f["flags"] & 3) == 3).all() and (f["z"] == sc.pix + sc.shifts[t]).all(), (t, s)
    # every stream that shares a scene must hold bit-identical results (same inputs, different CTA / SM / slab)
    ref = {}
    for s in range(B):
        x, P = cfg_ctx.get_state(s)
        key = (s * 5) % U
        if key in ref:
            assert (x == ref[key][0]).all() and (P == ref[key][1]).all(), s
        else:
            ref[key] = (x, P)
    cfg_ctx.close()


def test_c3_four_streams_four_frames_against_oracle(oracle):
    """BASELINE C3 (640x480, N = 100, 15x15 patch, +-40 px: the FP64-moment filter path of the search and the
    multi-tile window walk) through the FUSED step: 4 streams x 4 frames, all compared with the oracle."""
    B, T = 4, 4
    scenes = [synth.make_scene("C3", stream_id=s, n_frames=T) for s in range(B)]
    ctx = ctx_from_scenes(scenes, frame_slots=2)
    oracles = {s: oracle_slam_from_scene(oracle, scenes[s]) for s in range(B)}
    for t in range(T):
        step_frames(ctx, np.stack([sc.frames[t] for sc in scenes]), t % 2)
        check_streams_against_oracle(ctx, oracles, range(B), lambda s: scenes[s], t)
    ctx.close()


def _ellipse_membership(cx, cy, S4, W, H, B):
    """Candidate set of MonoSLAM::elliptical_search (monoslam.cpp:401-454) for a predicted centre and S (column-major
    2x2), op for op in IEEE double like the oracle / the kernel: {(u, v)} inside the 3-sigma ellipse and the box."""
    import math
    s00, s10, s11 = float(S4[0]), float(S4[1]), float(S4[3])
    l00 = math.sqrt(s00)
    l10 = s10 / l00
    l11 = math.sqrt(s11 - l10 * l10)
    x00 = 1.0 / l00
    x10 = (0.0 - l10 * x00) / l11
    x11 = 1.0 / l11
    p00, p01, p11 = x00 * x00 + x10 * x10, x10 * x11, x11 * x11
    hw = int(3.0 / math.sqrt(p00 - p01 * p01 / p11))
    hh = int(3.0 / math.sqrt(p11 - p01 * p01 / p00))
    uc, vc = int(cx + 0.5), int(cy + 0.5)
    half = (B - 1) // 2
    us, uf, vs, vf = -hw, hw, -hh, hh
    if uc + us - half < 0: us = half - uc
    if uc + uf - half > W - B: uf = W - B - uc + half
    if vc + vs - half < 0: vs = half - vc
    if vc + vf - half > H - B: vf = H - B - vc + half
    if uf < us or vf < vs:
        return set()
    du = np.arange(us, uf + 1, dtype=np.float64)[:, None]
    dv = np.arange(vs, vf + 1, dtype=np.float64)[None, :]
    q = ((p00 * du) * du + ((2.0 * p01) * du) * dv) + (p11 * dv) * dv
    iu, iv = np.nonzero(q < 9.0)
    return {(uc + us + int(a), vc + vs + int(b)) for a, b in zip(iu, iv)}


def test_h2_ellipse_boundary_flips_are_counted(oracle):
    """SURVEY H2: device sin/cos/acos differ from glibc by ulps, so S_i (hence the ellipse Sinv) can differ in the last
    bits from the oracle's and a candidate exactly on the ellipse boundary could enter or leave the search region.
    Count it: over a C1 run (ellipses from the EKF's own S_i, 10 selected per frame) and a C2 run with EKF ellipses,
    the candidate sets built from the device's (h, S) and from the oracle's are compared feature by feature."""
    kp = np.load(os.path.join(G, "known_patches.npy"))
    cases = [("C1", synth.make_scene("C1", n_frames=8, known_patches=kp), 120),
             ("C2", synth.make_scene("C2", n_frames=8, n_features=50, override=False), 24)]
    report = []
    for name, sc, steps in cases:
        ctx = ctx_from_scenes([sc], frame_slots=1)
        o = oracle_slam_from_scene(oracle, sc)
        ellipses = cands = flips = bit_diff = 0
        for t in range(steps):
            k = t % sc.frames.shape[0]
            step_frames(ctx, sc.frames[k][None])
            o.step(sc.frames[k])
            fg, fo = ctx.features(0), o.features()
            assert (fg["select_rank"] == fo["select_rank"]).all() and (fg["flags"] == fo["flags"]).all()
            for i in np.nonzero(fo["select_rank"] >= 0)[0]:
                ellipses += 1
                same = (fg["S"][i] == fo["S"][i]).all() and (fg["h"][i] == fo["h"][i]).all()
                if same:
                    continue                      # identical bits in, identical candidate set out
                bit_diff += 1
                a = _ellipse_membership(fg["h"][i][0], fg["h"][i][1], fg["S"][i], sc.width, sc.height, sc.boxsize)
                b = _ellipse_membership(fo["h"][i][0], fo["h"][i][1], fo["S"][i], sc.width, sc.height, sc.boxsize)
                cands += len(b)
                flips += len(a ^ b)
        report.append((name, steps, ellipses, bit_diff, cands, flips))
        ctx.close()
    for r in report:
        print("H2 %s: %d steps, %d ellipses, %d with last-bit differences in (h, S), %d candidates in those, "
              "%d boundary flips" % r)
    # a flip would not be an error by itself (the match positions above are compared bit-exactly anyway); it has to be
    # rare enough to be explained by boundary pixels: fewer than one candidate in 10^4
    for r in report:
        assert r[5] <= max(1, r[4] // 10000), r
