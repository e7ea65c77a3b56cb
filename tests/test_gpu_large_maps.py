"""Maps of more than 128 features per camera stream (up to SL2_MAX_FEATURES = 256, n <= 781), of which at most
SL2_MAX_MEASURED = 128 are measured per step (m <= 256).

The measurement tables of the update (H, R, nu, S and its Cholesky factor in shared memory, the upd_solve
instantiation, the rows of the G scratch) are sized by min(capacity, 128); everything that scales with the map (H P
column chunks of upd_hp, upd_solve column groups, upd_syrk tiles, predict / finish / cull loops) walks n in HBM.
"""
import os
import subprocess

import numpy as np
import pytest

from gpu_util import (assert_same_bytes, assert_state_close, ctx_from_scenes, large_variant, oracle_slam_from_scene,
                      random_measurements, record_oracle, run_regimes, step_frames, stream_result, synth)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T = 12           # frames per run; the bad features are culled by the 10th step
N_SELECT = 128   # SL2_MAX_MEASURED: the largest selection a map above 128 features may ask for

# capacity -> variants (nf, in view, bad, the edge the variant exists for).  Features from index `in view` on are
# moved out of the view (never selected); the `bad` ones (spread over the features in view) never match, so
# K = in_view - bad measurements per step (at most 128) and the bad ones are culled at step 10.
VARIANTS = {
    129: [(129, 129, 0, "nf = 129, n = 400: K = 128 of 129 selected"),
          (101, 101, 0, "K mod 4 = 1"),
          (3, 3, 3, "K = 0, culled to an empty map"),
          (129, 0, 0, "K = 0, whole map out of view")],
    210: [(210, 128, 0, "n = 643: three upd_hp column chunks, K = 128"),
          (145, 120, 0, "n = 448: nu alone in its syrk tile"),
          (209, 127, 0, "n = 640: exactly two upd_hp chunks, nu alone in its tile, K mod 4 = 3"),
          (166, 126, 0, "n + 1 = 512: nu is the last column of a tile, K mod 4 = 2"),
          (210, 128, 100, "cull: n 643 -> 343 crosses 640 and 397"),
          (150, 0, 0, "K = 0, whole map out of view")],
    256: [(256, 128, 0, "n = 781, m = 256"),
          (230, 125, 0, "n + 1 = 704: nu is the last column of a tile, K mod 4 = 1"),
          (256, 10, 0, "K = 10 on a 256-feature map (the reference's regime)"),
          (256, 128, 118, "cull 256 -> 138 features: n 781 -> 427"),
          (130, 110, 30, "cull 130 -> 100 features: n 403 -> 313 crosses 397 and 320"),
          (4, 4, 4, "K = 0, culled to an empty map"),
          (200, 0, 0, "K = 0, whole map out of view")],
}


def designed(v):
    """(K, nf before the cull, nf after it)."""
    nf, vis, bad, _ = v
    return min(vis - bad, N_SELECT), nf, nf - bad


def variant_scenes(cap):
    return [large_variant(nf, vis, bad, stream_id=i) for i, (nf, vis, bad, _) in enumerate(VARIANTS[cap])]


def regimes(nsm, U):
    """(name, B, step groups): the batched launch regimes of the update (upd_hp2 is never chosen above 102
    features: the batch regimes here run upd_hp with one CTA per stream)."""
    return [("small", U, 1), ("walk", nsm, 1), ("batch", 2 * nsm, 1), ("groups", 2 * nsm, 2)]


@pytest.mark.parametrize("cap", sorted(VARIANTS))
def test_large_map_update_shapes_against_oracle(oracle, cap):
    """Every regime of one capacity above 128: checked streams against the oracle at every step, every stream
    bit-identical to the first stream of its variant, every variant bit-identical across regimes."""
    import torch
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    scenes = variant_scenes(cap)
    traj = record_oracle(oracle, scenes, T)
    for v, rec in zip(VARIANTS[cap], traj):                  # the run is the designed one
        K, nf0, nf1 = designed(v)
        assert int(((rec[0]["f"]["flags"] & 3) == 3).sum()) == K, v
        assert rec[0]["nf"] == nf0 and rec[-1]["nf"] == nf1, v
    regs = regimes(nsm, len(scenes))
    _, worst = run_regimes(scenes, cap, regs, T, (8, T - 1), traj)
    for name, B, _ in regs:
        print("\ncap %3d %-7s B = %3d  worst state %.2e  covariance %.2e" % (cap, name, B, *worst[name]))


@pytest.mark.parametrize("name, nf", [("C4", 100), ("C4", 128), ("C1", 20)])
def test_capacity_does_not_change_results(name, nf):
    """The same scenes in a context of capacity nf and one of capacity 256: bit-identical x, P and per-feature
    outputs at every step (every product's summation order is set by m and the column, not by ld or the capacity)."""
    import scenelib2_b200 as sl2
    kp = np.load(os.path.join(ROOT, "tests", "golden", "known_patches.npy")) if name == "C1" else None
    scenes = [synth.make_scene(name, stream_id=s, n_frames=6, n_features=nf, known_patches=kp) for s in range(3)]
    small = ctx_from_scenes(scenes, max_features=nf)
    large = ctx_from_scenes(scenes, max_features=sl2.lib.SL2_MAX_FEATURES)
    try:
        for t in range(6):
            for c in (small, large):
                step_frames(c, np.stack([sc.frames[t] for sc in scenes]))
            for s in range(len(scenes)):
                assert_same_bytes(stream_result(large, s, jacobians=True), stream_result(small, s, jacobians=True),
                                  (name, nf, "step", t, "stream", s))
    finally:
        small.close()
        large.close()


def _oracle_from_ctx(oracle, ctx, s, sc):
    """An oracle holding the stream's current map and state (its counters start at zero)."""
    x, P = ctx.get_state(s)
    nf = ctx.num_features(s)
    cfg = oracle.make_config(width=sc.width, height=sc.height, fku=sc.cam8[2], fkv=sc.cam8[3], u0=sc.cam8[4],
                             v0=sc.cam8[5], kd1=sc.cam8[6], sd=sc.cam8[7], delta_t=sc.delta_t, n_select=sc.n_select,
                             boxsize=sc.boxsize, search_override=sc.search_override)
    o = oracle.Slam(cfg)
    for i in range(nf):
        o.add_feature(x[13 + 3 * i:16 + 3 * i], sc.meta["xp_now"][i], sc.meta["patch_now"][i])
    o.set_state(x, P)
    return o


def _step_both(ctx, o, frame):
    step_frames(ctx, frame[None])
    o.step(frame)
    fg, fo = ctx.features(0), o.features()
    assert ctx.num_features(0) == o.num_features
    assert (fg["select_rank"] == fo["select_rank"]).all() and (fg["flags"] == fo["flags"]).all()
    ok = (fo["flags"] & 2) > 0
    assert (fg["z"][ok] == fo["z"][ok]).all()
    (xg, Pg), (xo, Po) = ctx.get_state(0), o.get_state()
    # known features appended without Pcol have zero variance (no natural scale): their rows must match exactly
    live = np.diag(Po) > 0
    assert_state_close(xg[live], Pg[np.ix_(live, live)], xo[live], Po[np.ix_(live, live)])
    assert np.array_equal(xg[~live], xo[~live]) and np.array_equal(Pg[~live], Po[~live])
    assert np.abs(Pg - Pg.T).max() == 0.0
    return int(ok.sum())


def test_map_grows_and_shrinks_through_128(oracle):
    """120 features uploaded, grown to 256 by sl2_append_feature (with and without Pcol) with fused steps in between,
    then features deleted at the front, the middle and the end; every step against the oracle, the grown map against
    the same map uploaded whole, and the full map refuses a further append."""
    import scenelib2_b200 as sl2
    full = large_variant(256, 128, stream_id=7, n_frames=8)
    cfg = sl2.config_for_scene(full, num_streams=1, frame_slots=1, max_features=256)

    # grown without steps, Pcol from the prior: the same bits as the map uploaded whole, and the same next steps
    a, b = sl2.Context(cfg), sl2.Context(cfg)
    n0 = 13 + 3 * 120
    a.set_features(0, full.x0[13:n0].reshape(120, 3), full.xp_org[:120], full.patches[:120])
    a.set_state(0, full.x0[:n0], full.P0[:n0, :n0])
    for i in range(120, 256):
        n = 13 + 3 * i
        assert a.append_feature(0, full.x0[n:n + 3], full.xp_org[i], full.patches[i], full.P0[:n + 3, n:n + 3]) == i
    with pytest.raises(sl2.Sl2Error) as e:                  # the map is full: SL2_ERR_STATE
        a.append_feature(0, full.x0[13:16], full.xp_org[0], full.patches[0])
    assert "error -3" in str(e.value)
    sl2.load_scene(b, 0, full)
    (xa, Pa), (xb, Pb) = a.get_state(0), b.get_state(0)
    assert a.num_features(0) == 256 and np.array_equal(xa, xb) and np.array_equal(Pa, Pb)
    for t in range(2):
        for c in (a, b):
            c.set_frames(0, full.frames[t][None])
            c.step(0)
        assert_same_bytes(stream_result(a, 0), stream_result(b, 0), ("grown vs whole", t))
    a.close()
    b.close()

    # grown with steps in between: 120 -> 200 (known features, Pcol = NULL) -> 256 (Pcol with only the 3x3 block)
    c = sl2.Context(cfg)
    c.set_features(0, full.x0[13:n0].reshape(120, 3), full.xp_org[:120], full.patches[:120])
    c.set_state(0, full.x0[:n0], full.P0[:n0, :n0])
    full.meta["xp_now"], full.meta["patch_now"] = list(full.xp_org), list(full.patches)
    o = _oracle_from_ctx(oracle, c, 0, full)
    t = 0
    for lo, hi, with_pcol in ((120, 200, False), (200, 256, True)):
        for _ in range(2):
            _step_both(c, o, full.frames[t])
            t += 1
        for i in range(lo, hi):
            n = c.state_size(0)
            pcol = None
            if with_pcol:
                pcol = np.zeros((n + 3, 3))
                pcol[n:, :] = full.P0[13 + 3 * i:16 + 3 * i, 13 + 3 * i:16 + 3 * i]
            y = full.x0[13 + 3 * i:16 + 3 * i]
            assert c.append_feature(0, y, full.xp_org[i], full.patches[i], pcol) == i
        x, P = c.get_state(0)
        assert x.size == 13 + 3 * hi and np.array_equal(x[13 + 3 * lo:], full.x0[13 + 3 * lo:13 + 3 * hi])
        assert np.abs(P - P.T).max() == 0.0
        o = _oracle_from_ctx(oracle, c, 0, full)
    measured = [_step_both(c, o, full.frames[t + k]) for k in range(2)]
    assert measured[-1] > 100, measured
    t += 2

    # shrink: the first, a middle and the last feature
    for idx in (0, 127, 253):
        x0, P0 = c.get_state(0)
        nf = c.num_features(0)
        c.delete_feature(0, idx)
        keep = np.r_[0:13, [13 + 3 * f + k for f in range(nf) if f != idx for k in range(3)]]
        x1, P1 = c.get_state(0)
        assert c.num_features(0) == nf - 1 and np.array_equal(x1, x0[keep]) and np.array_equal(P1, P0[np.ix_(keep, keep)])
        del full.meta["xp_now"][idx], full.meta["patch_now"][idx]
    o = _oracle_from_ctx(oracle, c, 0, full)
    for k in range(2):
        _step_both(c, o, full.frames[t + k])
    c.close()


def test_staged_path_at_capacity_256(oracle):
    """sl2_predict_measurements -> sl2_make_measurements -> sl2_ekf_update_measured on a 256-feature map, and
    sl2_ekf_update with host rows at m = 256 on n = 781 against the dense update of kalman.cpp; m = 258 is refused."""
    sc = large_variant(256, 128, stream_id=3, n_frames=3)
    ctx = ctx_from_scenes([sc], max_features=256)
    o = oracle_slam_from_scene(oracle, sc)
    for t in range(3):
        ctx.set_frame(0, 0, sc.frames[t])
        ctx.ekf_predict(0)
        nv = ctx.predict_measurements(0)
        cnt = ctx.make_measurements(0, 0)
        ctx.ekf_update_measured(0)
        o.predict()
        assert nv == o.select()
        assert cnt == o.measure(sc.frames[t]) and cnt == 128
        o.update()
        o.normalise()
        o.finish()
        fg, fo = ctx.features(0), o.features()
        assert (fg["z"] == fo["z"]).all() and (fg["flags"] == fo["flags"]).all()
        assert (fg["attempted"] == fo["attempted"]).all() and (fg["successful"] == fo["successful"]).all()
        assert_state_close(*ctx.get_state(0), *o.get_state())
    ctx.close()

    sc = synth.make_scene("C4", n_frames=1, n_features=256)
    ctx = ctx_from_scenes([sc], max_features=256)
    rng = np.random.default_rng(256128)
    n = sc.n
    assert n == 781
    feats, Hxv, Hy, R, nu, H, Rfull = random_measurements(rng, n, 256, 128)
    ctx.ekf_update(0, feats, Hxv, Hy, R, nu)
    xg, Pg = ctx.get_state(0)
    xo, Po = oracle.kalman_update_dense(sc.x0, sc.P0, H, Rfull, nu)
    J = np.eye(n)
    J[:13, :13] = oracle.dxvnorm_by_dxv(xo[:13])
    Po = J @ Po @ J.T
    Po = 0.5 * (Po + Po.T)
    ex, eP = assert_state_close(xg, Pg, xo, Po)
    assert np.abs(Pg - Pg.T).max() == 0.0
    print("update n=781 m=256: state err %.2e cov err %.2e" % (ex, eP))
    f2, Hx2, Hy2, R2, nu2, _, _ = random_measurements(rng, n, 256, 129)
    with pytest.raises(Exception) as e:
        ctx.ekf_update(0, f2, Hx2, Hy2, R2, nu2)
    assert "bad m" in str(e.value)
    ctx.close()


def test_large_map_against_the_reference_source(oracle, reference, tmp_path):
    """The CUDA path vs the REFERENCE'S OWN MonoSLAM code on a 200-feature map (n = 613) in a context of capacity 256,
    EKF ellipses, 10 of 200 selected by trace S (a selection that changes from step to step), replayed from
    tests/golden as test_cuda_path_against_the_reference_source does: selection ranks, flags, match positions and
    counters identical on every step, state and covariance within the test tolerance."""
    import scenelib2_b200 as sl2
    kp = np.load(os.path.join(ROOT, "tests", "golden", "known_patches.npy"))
    sc = synth.make_scene("C1", n_frames=8, known_patches=kp, n_features=200)
    assert sc.n_select == 10 and sc.search_override == (0.0, 0.0, 0.0) and sc.n == 613
    ctx = ctx_from_scenes([sc], frame_slots=1, max_features=sl2.lib.SL2_MAX_FEATURES)
    ref = reference.slam(sc, str(tmp_path / "ref"))
    selections = set()
    for t in range(8):
        ctx.set_frames(0, sc.frames[t:t + 1])
        ctx.step(0)
        ref.step(sc.frames[t])
        fg, fr = ctx.features(0), ref.features()
        assert ctx.num_features(0) == ref.num_features == 200
        assert (fg["select_rank"] == fr["select_rank"]).all(), t
        assert ((fg["flags"] & 1) == (fr["flags"] & 1)).all(), t
        seen = fr["attempted"] > 0
        assert ((fg["flags"] & 2)[seen] == (fr["flags"] & 2)[seen]).all(), t
        ok = (fr["flags"] & 2) > 0
        assert (fg["z"][ok] == fr["z"][ok]).all(), t
        assert (fg["attempted"] == fr["attempted"]).all() and (fg["successful"] == fr["successful"]).all()
        xg, Pg = ctx.get_state(0)
        xr, Pr = ref.get_state()
        stored = np.isfinite(Pr)                          # the stored entries of the reference's P
        assert_state_close(xg, np.where(stored, Pg, 0.0), xr, np.where(stored, Pr, 0.0))
        selections.add(tuple(np.nonzero(fr["select_rank"] >= 0)[0]))
    assert len(selections) > 1, "the selection must change between steps"
    ctx.close()


def test_headless_with_150_known_features(tmp_path, oracle):
    """The C++ shim reads 150 known features f1 .. f150 and creates a context with device.max_features = 150."""
    kp = np.load(os.path.join(ROOT, "tests", "golden", "known_patches.npy"))
    sc = synth.make_scene("C1", n_frames=6, known_patches=kp, n_features=150)
    Pxx = np.diag([4e-4] * 3 + [2e-5] * 4 + [1e-3] * 3 + [1e-3] * 3)
    sc.P0 = np.zeros_like(sc.P0)
    sc.P0[:13, :13] = Pxx
    cfg = synth.write_reference_case(str(tmp_path), sc, Pxx)
    assert "device.max_features = 150;" in open(cfg).read()
    exe = os.path.join(ROOT, "scenelib2_b200", "host", "sl2_headless")
    out = tmp_path / "out.txt"
    r = subprocess.run([exe, cfg, str(tmp_path / "frames.raw"), "320", "240", "6", str(out)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    vals = np.loadtxt(str(out))
    n = int(vals[0])
    xg, Pg = vals[1:1 + n], vals[1 + n:].reshape(n, n).T
    o = oracle_slam_from_scene(oracle, sc)
    for t in range(6):
        o.step(sc.frames[t])
    xo, Po = o.get_state()
    assert n == o.n == 13 + 3 * 150
    d = np.sqrt(np.abs(np.diag(Po))) + 1e-12
    assert (np.abs(Pg - Po) <= 1e-6 * d[:, None] * d[None, :] + 1e-18).all()
    assert np.allclose(xg, xo, rtol=1e-7, atol=1e-10)
    assert "measured 10" in r.stdout
