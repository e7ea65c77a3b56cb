"""The device's closed-form models (predict_kernel and particle_predict_kernel, ekf.cu) at general camera poses and
viewpoints: the motion model's fv, F and Q and the normalisation Jacobian read out exactly and compared with the
reference's stored outputs, the measurement model (h, dh/dxv, dh/dy, R, S), the depth-particle prediction (h, S^-1,
det S) and the visibility gates against the oracle bit for bit, per-feature xp_org through deletions, appends and
culls, and a fused run in a rigidly moved world.

The CPU tests at the top check that the inputs reach what the GPU tests claim to cover."""
import collections

import numpy as np
import pytest

import model_cases as mc
from gpu_util import (RTOL_TEST, check_streams_against_oracle, ctx_from_scenes, oracle_slam_from_scene,
                      rigid_transform_scene, sl2, state_err, step_frames, synth, untransform_state)
from ref_golden import Reference

# motion-model entries that contain sin/cos: device sin/cos may differ from glibc by 1-2 ulp (SURVEY H2); on an H100
# with CUDA 12.9 all 200 cases came out bit-identical (scaled difference 0), the bound allows a few ulp
MOTION_TRIG_TOL = 1e-15
ANGLE_EXACT_MARGIN = 1e-12      # below this the angle gate (acos) may flip between the device and glibc
TRANSFORMS = [([1e-3, 0.48, -0.6, 0.64], [0.7, -1.3, 2.1]),      # near-180 degree rotation: q_w.w ~ 0
              ([0.8, 0.3, -0.4, 0.3], [-0.2, 0.5, 0.1]),
              ([0.2, -0.1, 0.9, -0.4], [3.0, 0.0, -1.0])]
GENERAL_OMEGA = [0.05, -0.08, 0.03]
# The moved world is equivariant only while |q| = 1: the reference never renormalises q in x (quirk Q1), so after an
# update |q| - 1 is ~1e-6 .. 1e-4, and for q = s u its rotation matrix (math_util / sl2_model.cuh quat_to_R) is
# (1 - s^2) I + s^2 R(u), whose (1 - s^2) I part acts in world axes.  h then moves by 1e-4 px after the second step
# and ~5e-3 px after the twelfth, enough to reorder two features of nearly equal trace S.  So the moved and unmoved
# runs are compared on the first step only; later steps are compared with the oracle, stream by stream.
EQUIVARIANT_STEPS = 1


def _tangent_prior(oracle, sc):
    """sc with P0 <- J P0 J^T, J = dxvnorm_by_dxv: no prior variance along |q|, so that the first update leaves
    |q| = 1 to first order and the moved world stays close to equivariant (see EQUIVARIANT_STEPS)."""
    J = np.eye(sc.n)
    J[:13, :13] = oracle.dxvnorm_by_dxv(sc.x0[:13])
    P = J @ sc.P0 @ J.T
    sc.P0 = 0.5 * (P + P.T)
    return sc


def _cfg(cam8, nf, n_select=None, dt=0.033333333, streams=1, override=(0.0, 0.0, 0.0)):
    cfg = sl2.default_config()
    cfg.num_streams, cfg.frame_slots = streams, 1
    cfg.width, cfg.height = int(cam8[0]), int(cam8[1])
    cfg.fku, cfg.fkv, cfg.u0, cfg.v0, cfg.kd1, cfg.sd = [float(v) for v in cam8[2:8]]
    cfg.max_features = nf
    cfg.number_of_features_to_select = nf if n_select is None else n_select
    cfg.delta_t = dt
    for i in range(3):
        cfg.search_override[i] = override[i]
    return cfg


def _load(ctx, s, x, P, xp_org):
    nf = xp_org.shape[0]
    B = ctx.cfg.boxsize
    ctx.set_features(s, x[13:].reshape(nf, 3), xp_org, np.zeros((nf, B, B), np.uint8))
    ctx.set_state(s, x, P)


def _oracle_slam(oracle, cam8, x, P, xp_org, n_select, boxsize=11):
    cfg = oracle.make_config(width=int(cam8[0]), height=int(cam8[1]), fku=cam8[2], fkv=cam8[3], u0=cam8[4],
                             v0=cam8[5], kd1=cam8[6], sd=cam8[7], n_select=n_select, boxsize=boxsize)
    o = oracle.Slam(cfg)
    for i in range(xp_org.shape[0]):
        o.add_feature(x[13 + 3 * i:16 + 3 * i], xp_org[i], np.zeros((boxsize, boxsize), np.uint8))
    o.set_state(x, P)
    return o


def _device_feature(ctx, s):
    """Per feature: h, dh/dxv (2 x 13), dh/dy (2 x 3), R (2 x 2), S (2 x 2) of the last measurement prediction."""
    f = ctx.features(s)
    J, Jy, R, _ = ctx.feature_jacobians(s)
    return [(f["h"][i], J[i].reshape(13, 2).T, Jy[i].reshape(3, 2).T, R[i].reshape(2, 2).T,
             f["S"][i].reshape(2, 2).T) for i in range(len(f["h"]))]


def _predict_feature(oracle, cam8, x, P, i):
    b = slice(13 + 3 * i, 16 + 3 * i)
    return oracle.predict_feature(cam8, x[:13], x[b], P[:13, :13], P[:13, b], P[b, b])


def _assert_feature_bits(dev, orc, what):
    for name, a, b in zip(("h", "dh_dxv", "dh_dy", "R", "S"), dev, orc):
        assert np.array_equal(a, b), (what, name, a, b)


# ---- CPU: the inputs reach what the GPU tests claim ---------------------------------------------------------------
def _stream_codes(oracle, st):
    x, P, xo = st["x"], st["P"], st["xp_org"]
    out = []
    for i in range(xo.shape[0]):
        y = x[13 + 3 * i:16 + 3 * i]
        h = _predict_feature(oracle, st["cam8"], x, P, i)[0]
        ratio, angle = mc.gates(x[:7], y, xo[i])
        out.append((oracle.visibility_test(st["cam8"], x[:7], y, xo[i], h), h, ratio, angle))
    return out


def test_viewpoint_streams_reach_every_gate(oracle):
    """Every failure code of visibility_test (1, 2, 4, 8, 16) alone and in combinations, and cases within a pixel
    (search bound) or a small margin (distance ratio 2 and 1/2, angle 45 degrees) on both sides of every gate; exact
    trace-S ties; map sizes 1 .. 128."""
    streams = mc.viewpoint_streams()
    codes = collections.Counter()
    near = collections.Counter()
    ties = 0
    for st in streams:
        W, H = st["cam8"][0], st["cam8"][1]
        for (code, h, ratio, angle), d in zip(_stream_codes(oracle, st), st["design"]):
            codes[code] += 1
            for c, lim in ((0, mc.BOUND), (0, W - 1 - mc.BOUND), (1, mc.BOUND), (1, H - 1 - mc.BOUND)):
                if abs(h[c] - lim) < 1:
                    near["pixel %s %s" % ("uv"[c], "out" if (h[c] < lim) == (lim == mc.BOUND) else "in")] += 1
            for lim in (2.0, 0.5):
                if abs(ratio / lim - 1) < 1e-3:
                    near["ratio %.1f %s" % (lim, "out" if (ratio > lim) == (lim == 2.0) else "in")] += 1
            if abs(angle - mc.ANGLE_MAX) < 1e-3:
                m = abs(angle - mc.ANGLE_MAX)
                key = "< 1e-12" if m < ANGLE_EXACT_MARGIN else ">= 1e-12"
                near["angle %s %s" % ("out" if angle > mc.ANGLE_MAX else "in", key)] += 1
            ties += d[0] == "tie"
    print("\nvisibility code : features")
    for c in sorted(codes):
        print("  %2d : %d" % (c, codes[c]))
    print("near-threshold cases:")
    for k in sorted(near):
        print("  %-22s %d" % (k, near[k]))
    for bit in (1, 2, 4, 8, 16):
        assert codes[bit] > 0, bit                              # each gate alone
    assert codes[0] > 100 and sum(v for c, v in codes.items() if bin(c).count("1") >= 2) > 50
    for k in ("pixel u in", "pixel u out", "pixel v in", "pixel v out", "ratio 2.0 in", "ratio 2.0 out",
              "ratio 0.5 in", "ratio 0.5 out", "angle in >= 1e-12", "angle out >= 1e-12", "angle in < 1e-12",
              "angle out < 1e-12"):
        assert near[k] > 0, k
    assert ties >= 40
    assert sorted(len(st["xp_org"]) for st in streams)[:3] == [1, 2, 3] and max(len(st["xp_org"]) for st in streams) == 128


def test_rigid_transform_scene_on_the_oracle(oracle):
    """A rigidly moved world tracks the same frames on the oracle: h within 1e-10 px, S within 1e-10 relative, and
    selection, flags and match positions identical over a few whole steps (for this scene); x and P mapped back agree
    within RTOL_TEST after the first step (later, see EQUIVARIANT_STEPS)."""
    base = synth.make_scene("C2", n_frames=4, n_features=24, override=False)
    base.x0[10:13] = GENERAL_OMEGA
    _tangent_prior(oracle, base)
    for q_w, t_w in TRANSFORMS:
        moved = rigid_transform_scene(base, q_w, t_w)
        a, b = oracle_slam_from_scene(oracle, base), oracle_slam_from_scene(oracle, moved)
        for o in (a, b):
            o.predict()
            o.select()
        fa, fb = a.features(), b.features()
        assert np.abs(fa["h"] - fb["h"]).max() <= 1e-10
        assert (np.abs(fa["S"] - fb["S"]).max(axis=1) / np.abs(fa["S"]).max(axis=1)).max() <= 1e-10
        assert (fa["select_rank"] == fb["select_rank"]).all()
        a, b = oracle_slam_from_scene(oracle, base), oracle_slam_from_scene(oracle, moved)
        for t in range(4):
            a.step(base.frames[t])
            b.step(moved.frames[t])
            fa, fb = a.features(), b.features()
            for k in ("select_rank", "flags", "z"):
                assert (fa[k] == fb[k]).all(), (q_w, t, k)
            if t < EQUIVARIANT_STEPS:
                xb, Pb = untransform_state(*b.get_state(), *moved.meta["rigid"])
                assert max(state_err(xb, Pb, *a.get_state())) <= RTOL_TEST


# ---- GPU: motion model and normalisation, read out exactly ---------------------------------------------------------
def _readout_state(xv, nf=5):
    """x = [xv | 0], P = [[0, E], [E^T, 0]] with E = [I13 | 0]: after a predict Pxx = Q, P[:13, 13:26] = F and
    x[:13] = fv; after a normalisation P[:13, 13:26] = dxvnorm_by_dxv, all bit for bit."""
    n = 13 + 3 * nf
    x = np.zeros(n)
    x[:13] = xv
    P = np.zeros((n, n))
    P[:13, 13:26] = np.eye(13)
    P[13:26, :13] = np.eye(13)
    return x, P


EXACT_ROWS = np.r_[0:3, 7:13]              # no sin/cos in fv or F on these rows, nor in Q off rows / columns 3..6


def _motion_errors(dev, ref):
    """Bit identity on the sin/cos-free entries; the largest scaled difference |d|.max() / max(1, |ref|.max())
    elsewhere."""
    (fv, F, Q), (fr, Fr, Qr) = dev, ref
    assert np.array_equal(fv[EXACT_ROWS], fr[EXACT_ROWS])
    assert np.array_equal(F[EXACT_ROWS], Fr[EXACT_ROWS])
    assert np.array_equal(Q[np.ix_(EXACT_ROWS, EXACT_ROWS)], Qr[np.ix_(EXACT_ROWS, EXACT_ROWS)])
    return max(np.abs(a - b).max() / max(1.0, np.abs(b).max()) for a, b in zip(dev, ref))


@pytest.mark.gpu
def test_motion_model_and_normalisation_match_reference_outputs(oracle):
    """predict_kernel's fv, F, Q on the inputs of test_motion_model_matches_reference_source (general omega, non-unit
    q, three dt, control input) against the reference's stored outputs and the oracle; upd_finish's quirk-Q2
    normalisation Jacobian bit-identical to the stored dxvnorm_by_dxv, x left un-normalised (quirk Q1)."""
    ref = Reference("test_motion_model_matches_reference_source", oracle)
    ctxs = {}
    worst_ref = worst_orc = 0.0
    for xv, dt, u in mc.motion_cases():
        if dt not in ctxs:
            ctxs[dt] = sl2.Context(_cfg(mc.CAMS[0], 5, dt=dt))
            _load(ctxs[dt], 0, *_readout_state(xv)[:2], np.tile(xv[:7], (5, 1)))
        ctx = ctxs[dt]
        x, P = _readout_state(xv)
        ctx.set_state(0, x, P)
        ctx.ekf_predict(0, u if u.any() else None)
        xg, Pg = ctx.get_state(0)
        dev = (xg[:13], Pg[:13, 13:26], Pg[:13, :13])
        assert np.array_equal(Pg[13:26, :13], dev[1].T) and not Pg[26:].any() and not Pg[:, 26:].any()
        worst_ref = max(worst_ref, _motion_errors(dev, ref.call("motion", xv, dt, u)))
        worst_orc = max(worst_orc, _motion_errors(dev, oracle.motion(xv, dt, u)))
        Jr, xn = ref.call("dxvnorm_by_dxv", xv)
        ctx.set_state(0, x, P)
        ctx.normalise_state(0)
        xg, Pg = ctx.get_state(0)
        assert np.array_equal(Pg[:13, 13:26], Jr) and np.array_equal(Pg[13:26, :13], Jr.T)
        assert np.array_equal(Pg[3:7, 16:20], Jr[3:7, 3:7]) and not Pg[:13, :13].any()
        assert np.array_equal(xg, x) and np.array_equal(xn, xv)
    ref.close()
    for c in ctxs.values():
        c.close()
    print("\nmotion model, scaled worst on sin/cos entries: vs reference %.2e, vs oracle %.2e" % (worst_ref, worst_orc))
    assert worst_ref <= MOTION_TRIG_TOL and worst_orc <= MOTION_TRIG_TOL


def _nan_product(A, B):
    """A B as the kernels sum it, with NaN * 0 = NaN kept (no BLAS)."""
    return (A[:, :, None] * B[None, :, :]).sum(axis=1)


@pytest.mark.gpu
def test_motion_model_at_zero_omega(oracle):
    """omega = 0 exactly: neither dqomegadt_by_domega of the reference (motion_model.cpp:290-349) nor the device's has
    a branch for |omega| = 0, so dq/domega is 0/0.  The device's readout must hold the oracle's F and Q as the
    predict's products carry them, NaN positions included; fv is finite and exact."""
    xv = np.array([0.1, -0.2, 0.3, 0.9, 0.1, -0.3, 0.2, 0.05, 0.0, -0.1, 0.0, 0.0, 0.0])
    u = np.array([0.3, -0.1, 0.2])
    dt = 1 / 30.0
    ctx = sl2.Context(_cfg(mc.CAMS[0], 5, dt=dt))
    x, P = _readout_state(xv)
    _load(ctx, 0, x, P, np.tile(xv[:7], (5, 1)))
    ctx.ekf_predict(0, u)
    xg, Pg = ctx.get_state(0)
    fo, Fo, Qo = oracle.motion(xv, dt, u)
    assert np.isnan(Fo).any() and np.isfinite(fo).all()
    assert np.array_equal(xg[:13], fo)
    F_read = _nan_product(Fo, np.eye(13))
    Q_read = _nan_product(_nan_product(Fo, np.zeros((13, 13))), Fo.T) + Qo
    assert np.array_equal(Pg[:13, 13:26], F_read, equal_nan=True)
    assert np.array_equal(Pg[:13, :13], Q_read, equal_nan=True)
    assert np.isfinite(Pg[np.ix_(EXACT_ROWS, EXACT_ROWS)]).all() and np.isfinite(Pg[EXACT_ROWS, 13:26]).all()
    ctx.close()


# ---- GPU: measurement model against the reference's stored outputs -------------------------------------------------
@pytest.mark.gpu
def test_measurement_model_matches_reference_outputs(oracle):
    """The 300 cases of test_measurement_model_matches_reference_source, one stream each (one feature, n_select = 1)
    in one context per camera: h, dh/dxv, dh/dy, R and S bit-identical to oracle.predict_feature (never-fused ops in
    the oracle's order, no transcendental functions) and within 1e-13 of the reference; selected exactly when the
    reference's visibility code is 0."""
    cases = list(mc.measurement_cases())
    per_cam = [[c for k, c in enumerate(cases) if k % 2 == j] for j in range(2)]
    ctxs = [sl2.Context(_cfg(mc.CAMS[j], 1, streams=len(per_cam[j]))) for j in range(2)]
    dev = []
    for k, (cam8, xv, y, P, xp_org) in enumerate(cases):
        ctx, s = ctxs[k % 2], k // 2
        _load(ctx, s, np.concatenate([xv, y]), P, xp_org[None])
        nv = ctx.predict_measurements(s)
        dev.append((nv, ctx.features(s)["select_rank"][0], _device_feature(ctx, s)[0]))
    ref = Reference("test_measurement_model_matches_reference_source", oracle)
    worst = 0.0
    codes = collections.Counter()
    for (cam8, xv, y, P, xp_org), (nv, rank, d) in zip(cases, dev):
        a = oracle.predict_feature(cam8, xv, y, P[:13, :13], P[:13, 13:], P[13:, 13:])
        b = ref.call("predict_feature", cam8, xv, y, P[:13, :13], P[:13, 13:], P[13:, 13:])
        _assert_feature_bits(d, a, "measurement")
        for x, r in zip(d, b):
            if np.isfinite(r).all():
                worst = max(worst, np.abs(x - r).max() / max(1.0, np.abs(r).max()))
        assert np.isfinite(a[0]).all()
        code = ref.call("visibility_test", cam8, xv[:7], y, xp_org, a[0])
        codes[code] += 1
        assert (nv == 1) == (rank == 0) == (code == 0), (code, nv, rank)
    ref.close()
    for c in ctxs:
        c.close()
    print("\nmeasurement model vs reference: scaled worst %.2e; visibility codes %s" % (worst, sorted(codes.items())))
    assert worst <= 1e-13
    assert codes[0] > 0 and len(codes) >= 5


# ---- GPU: particle prediction against the reference's stored outputs -----------------------------------------------
def _device_particles(ctx, xv, ypi, P, lam):
    """h, S^-1 (00, 01, 11) and det S of the depth particles lam of the ray ypi, predicted on the device by
    sl2_measure_partial_features from the camera state xv, P[:13, :13] of stream 0 and the ray's blocks of P."""
    _load(ctx, 0, np.concatenate([xv, ypi[:3]]), P[:16, :16], xv[None, :7])
    B = ctx.cfg.boxsize
    out = ctx.measure_partial_features(0, 0, np.zeros((1, B, B), np.uint8), ypi[None], P[None, :13, 13:],
                                       P[None, 13:, 13:], lam[None], 0.05, np.full((1, lam.size), 1.0 / lam.size))
    return out["h"][0], out["Sinv3"][0], out["detS"][0]


PARTICLE_OUTPUTS = (("h", 0), ("Sinv3", 2), ("detS", 3))    # positions in the result of predict_particles


@pytest.mark.gpu
def test_particle_prediction_matches_reference_outputs(oracle):
    """The 120 rays of test_particle_prediction_matches_reference_source (both cameras, camera poses with a non-unit
    q, 9 depths each): every particle's h, S^-1 and det S bit-identical to oracle.predict_particles and within 1e-13
    of the reference."""
    ctxs = [sl2.Context(_cfg(cam8, 1)) for cam8 in mc.CAMS]
    ref = Reference("test_particle_prediction_matches_reference_source", oracle)
    worst = 0.0
    for k, (cam8, xv, ypi, P, lam) in enumerate(mc.particle_cases()):
        dev = _device_particles(ctxs[k % 2], xv, ypi, P, lam)
        args = (cam8, xv, ypi, lam, P[:13, :13], P[:13, 13:], P[13:, 13:])
        a, r = oracle.predict_particles(*args), ref.call("predict_particles", *args)
        for d, (name, i) in zip(dev, PARTICLE_OUTPUTS):
            assert d.tobytes() == a[i].tobytes(), (k, name, d, a[i])
            worst = max(worst, np.abs(d - r[i]).max() / max(1.0, np.abs(r[i]).max()))
    ref.close()
    for c in ctxs:
        c.close()
    print("\nparticle prediction vs reference: scaled worst %.2e" % worst)
    assert worst <= 1e-13


@pytest.mark.gpu
def test_particle_prediction_at_zero_norm_q(oracle):
    """A camera quaternion of zero norm: Eigen's inverse() returns the zero quaternion (its squaredNorm > 0 guard),
    so the rotation matrix is the identity and the prediction is finite; the device must give the oracle's bits."""
    cam8, xv, ypi, P, lam = next(mc.particle_cases())
    xv = xv.copy()
    xv[3:7] = 0.0
    ctx = sl2.Context(_cfg(cam8, 1))
    dev = _device_particles(ctx, xv, ypi, P, lam)
    ctx.close()
    a = oracle.predict_particles(cam8, xv, ypi, lam, P[:13, :13], P[:13, 13:], P[13:, 13:])
    for d, (name, i) in zip(dev, PARTICLE_OUTPUTS):
        assert np.isfinite(a[i]).all() and d.tobytes() == a[i].tobytes(), (name, d, a[i])


# ---- GPU: viewpoint gates, selection and xp_org bookkeeping --------------------------------------------------------
def _compare_stream(oracle, ctx, s, st, n_select, expect_flips=False):
    """predict_measurements on stream s against a fresh oracle Slam of the same map: every feature's fields bit for
    bit, and nvisible and the selection ranks exactly.  Visibility may differ only where the view angle is within
    ANGLE_EXACT_MARGIN of 45 degrees (acos); returns the number of such flips (then the ranks are not compared)."""
    x, P, xo, cam8 = st["x"], st["P"], st["xp_org"], st["cam8"]
    nv = ctx.predict_measurements(s)
    fg = ctx.features(s)
    assert len(fg["h"]) == xo.shape[0]
    flips = 0
    for i, d in enumerate(_device_feature(ctx, s)):
        a = _predict_feature(oracle, cam8, x, P, i)
        _assert_feature_bits(d, a, (s, i))
        if n_select >= xo.shape[0]:
            y = x[13 + 3 * i:16 + 3 * i]
            code = oracle.visibility_test(cam8, x[:7], y, xo[i], a[0])
            if (fg["select_rank"][i] >= 0) != (code == 0):
                angle = mc.gates(x[:7], y, xo[i])[1]
                assert code & ~8 == 0 and abs(angle - mc.ANGLE_MAX) < ANGLE_EXACT_MARGIN, (s, i, code, angle)
                flips += 1
    if flips == 0:
        o = _oracle_slam(oracle, cam8, x, P, xo, n_select)
        assert nv == o.select(), s
        assert (fg["select_rank"] == o.features()["select_rank"]).all(), s
    assert (fg["select_rank"] >= 0).sum() == min(n_select, nv) or flips
    return flips


@pytest.mark.gpu
def test_viewpoint_gates_and_selection_many_features(oracle):
    """24 streams of up to 128 features at general poses in one context of capacity 128 (so every per-stream offset
    is used), once selecting up to 128 (every visible feature) and once 7 (fewer than the visible count)."""
    streams = mc.viewpoint_streams()
    flips = {}
    for n_select in (128, 7):
        ctx = sl2.Context(_cfg(mc.CAMS[0], 128, n_select=n_select, streams=len(streams)))
        for s, st in enumerate(streams):
            _load(ctx, s, st["x"], st["P"], st["xp_org"])
        for s, st in enumerate(streams):
            if n_select == 128:
                flips[s] = _compare_stream(oracle, ctx, s, st, n_select)
                assert flips[s] == 0 or st["probe"], s
            elif flips[s] == 0:                  # a flipped angle gate also moves the ranks
                _compare_stream(oracle, ctx, s, st, n_select)
        ctx.close()
    probes = sum(abs(mc.gates(st["x"][:7], st["x"][13 + 3 * i:16 + 3 * i], xo)[1] - mc.ANGLE_MAX) < ANGLE_EXACT_MARGIN
                 for st in streams for i, xo in enumerate(st["xp_org"]))
    print("\nviewpoint streams: %d features; %d of the %d view angles closer than %.0e to 45 degrees flip"
          % (sum(len(st["xp_org"]) for st in streams), sum(flips.values()), probes, ANGLE_EXACT_MARGIN))
    assert sum(flips.values()) <= 2


def _drop(st, i):
    nf = st["xp_org"].shape[0]
    keep = np.r_[0:13, [13 + 3 * f + c for f in range(nf) if f != i for c in range(3)]]
    return dict(st, x=st["x"][keep], P=st["P"][np.ix_(keep, keep)], xp_org=np.delete(st["xp_org"], i, axis=0))


@pytest.mark.gpu
def test_xp_org_moves_with_deleted_and_appended_features(oracle):
    """sl2_delete_feature from the middle, the first and the last slot and sl2_append_feature with a distinct xp_org
    (one failing the angle gate, one passing), on three streams of a full context: after every change each stream's
    measurement prediction and selection equal those of a fresh oracle Slam of the surviving map."""
    streams = mc.viewpoint_streams()
    ctx = sl2.Context(_cfg(mc.CAMS[0], 128, streams=len(streams)))
    for s, st in enumerate(streams):
        _load(ctx, s, st["x"], st["P"], st["xp_org"])
    rng = np.random.default_rng(4242)
    B = ctx.cfg.boxsize
    for s in (5, 11, 23):
        st = streams[s]
        for where in ("middle", "first", "last"):
            nf = st["xp_org"].shape[0]
            i = {"middle": nf // 2, "first": 0, "last": nf - 1}[where]
            ctx.delete_feature(s, i)
            st = _drop(st, i)
            _compare_stream(oracle, ctx, s, st, 128)
        for angle in (1.2, 0.3):
            x, P = st["x"], st["P"]
            n = x.size
            j = int(rng.integers(0, st["xp_org"].shape[0]))
            b = slice(13 + 3 * j, 16 + 3 * j)
            xo = mc.place_xp_org(rng, x[:13], x[b], 1.1, angle)
            Pcol = np.vstack([P[:, b], P[b, b]])
            assert ctx.append_feature(s, x[b], xo, np.zeros((B, B), np.uint8), Pcol) == st["xp_org"].shape[0]
            P2 = np.zeros((n + 3, n + 3))
            P2[:n, :n], P2[:, n:], P2[n:, :n] = P, Pcol, Pcol[:n].T
            st = dict(st, x=np.concatenate([x, x[b]]), P=P2, xp_org=np.vstack([st["xp_org"], xo]))
            _compare_stream(oracle, ctx, s, st, 128)
        streams[s] = st
    for s, st in enumerate(streams):                  # the other streams are untouched
        if not st["probe"]:
            _compare_stream(oracle, ctx, s, st, 128)
    ctx.close()


def _gated_scene(stream_id, bad=(), gated=(), override=True, n_frames=12):
    """C2 scene whose features each have their own xp_org: the `gated` ones fail the distance-ratio or angle gate
    (never selected), the others pass with a distinct viewpoint; the `bad` templates are random bytes (culled at the
    10th step)."""
    sc = synth.make_scene("C2", stream_id=stream_id, n_frames=n_frames, n_features=30, override=override)
    rng = np.random.default_rng(500 + stream_id)
    xo = np.zeros_like(sc.xp_org)
    for i in range(sc.n_features):
        y = sc.x0[13 + 3 * i:16 + 3 * i]
        if i in gated:
            ratio, angle = (3.0, 0.2) if i % 2 else (1.0, 1.1)
        else:
            ratio, angle = rng.uniform(0.7, 1.4), rng.uniform(0.0, 0.5)
        xo[i] = mc.place_xp_org(rng, sc.x0[:13], y, ratio, angle)
    sc.xp_org = xo
    patches = sc.patches.copy()
    for i in bad:
        patches[i] = rng.integers(0, 256, patches[i].shape, dtype=np.uint8)
    sc.patches = patches
    return sc


@pytest.mark.gpu
def test_fused_step_culls_compact_xp_org(oracle):
    """Bad templates interleaved with gate-failing xp_org: the cull at the 10th step must move every later feature's
    xp_org with it, or a gated feature inherits a passing viewpoint (and the reverse)."""
    scenes = [_gated_scene(0, bad=(2, 9, 16), gated=(3, 5, 10, 17, 25)),
              _gated_scene(1, bad=(0, 1, 20), gated=(2, 4, 21, 29), override=False),
              _gated_scene(2, bad=(14, 28), gated=(15, 29))]
    ctx = ctx_from_scenes(scenes)
    oracles = [oracle_slam_from_scene(oracle, sc) for sc in scenes]
    for t in range(12):
        step_frames(ctx, np.stack([sc.frames[t] for sc in scenes]))
        check_streams_against_oracle(ctx, oracles, range(len(scenes)), lambda s: scenes[s], t)
    assert [ctx.num_features(s) for s in range(3)] == [27, 27, 28]
    for s in range(3):
        assert ((ctx.features(s)["flags"] & 1) == 0).sum() >= 2        # gated features stay unselected
    ctx.close()


# ---- GPU: a fused run in a rigidly moved world ----------------------------------------------------------------------
@pytest.mark.gpu
def test_rotated_world_fused_run(oracle):
    """C2-sized streams in rigidly moved worlds (one near 180 degrees), general omega in some, bad templates, with
    fixed and with EKF ellipses: every stream against the oracle on every step, and with fixed windows against the
    unmoved run on the GPU while the run is equivariant (EQUIVARIANT_STEPS): selection, flags, match positions and
    counters identical, h within 1e-9 px, S within 1e-9 relative, x and P mapped back within RTOL_TEST."""
    def base(sid, override, omega):
        sc = synth.make_scene("C2", stream_id=sid, n_frames=12, n_features=24, override=override)
        if omega:
            sc.x0[10:13] = GENERAL_OMEGA
        patches = sc.patches.copy()
        patches[[3, 17]] = np.random.default_rng(sid).integers(0, 256, patches[[3, 17]].shape, dtype=np.uint8)
        sc.patches = patches
        return _tangent_prior(oracle, sc)

    for override in (True, False):
        b0, b1 = base(10, override, True), base(11, override, False)
        scenes = [b0, rigid_transform_scene(b0, *TRANSFORMS[0]), rigid_transform_scene(b0, *TRANSFORMS[1]),
                  b1, rigid_transform_scene(b1, *TRANSFORMS[2]), rigid_transform_scene(b1, *TRANSFORMS[0])]
        pairs = [(0, 1), (0, 2), (3, 4), (3, 5)]
        ctx = ctx_from_scenes(scenes)
        oracles = [oracle_slam_from_scene(oracle, sc) for sc in scenes]
        worst, late, late_discrete = [0.0, 0.0, 0.0], [0.0, 0.0, 0.0], 0
        for t in range(12):
            step_frames(ctx, np.stack([sc.frames[t] for sc in scenes]))
            check_streams_against_oracle(ctx, oracles, range(len(scenes)), lambda s: scenes[s], t)
            if not override:
                continue
            for a, b in pairs:
                fa, fb = ctx.features(a), ctx.features(b)
                same = all((fa[k] == fb[k]).all() for k in ("select_rank", "flags", "z", "attempted", "successful"))
                assert same or t >= EQUIVARIANT_STEPS, (t, a, b)
                late_discrete += not same
                eh = np.abs(fa["h"] - fb["h"]).max()
                eS = (np.abs(fa["S"] - fb["S"]).max(axis=1) / np.abs(fa["S"]).max(axis=1)).max()
                xb, Pb = untransform_state(*ctx.get_state(b), *scenes[b].meta["rigid"])
                es = max(state_err(xb, Pb, *ctx.get_state(a)))
                if t < EQUIVARIANT_STEPS:
                    assert eh <= 1e-9 and eS <= 1e-9 and es <= RTOL_TEST, (t, a, b, eh, eS, es)
                    worst = [max(worst[0], eh), max(worst[1], eS), max(worst[2], es)]
                else:
                    late = [max(late[0], eh), max(late[1], eS), max(late[2], es)]
        assert all(ctx.num_features(s) == 22 for s in range(len(scenes)))
        ctx.close()
        if override:
            print("\nmoved vs unmoved world on the GPU, first step: h %.2e px, S %.2e relative, state %.2e; "
                  "later (|q| != 1): h %.2e px, S %.2e, state %.2e, %d of %d stream-steps with other selections, "
                  "flags or matches" % tuple(worst + late + [late_discrete, len(pairs) * (12 - EQUIVARIANT_STEPS)]))
