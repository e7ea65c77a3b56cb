"""Pins the oracle's restatement to the REFERENCE's own source: golden vectors under tests/golden/ were produced by
oracle/_ref/libsl2ref.so = the original scenelib2/improc/{improc,search_multiple_overlapping_ellipses}.cpp compiled
unmodified (see tests/golden/make_golden.py), and the `reference` fixture replays what oracle/_ref returned for the
inputs each test builds (see tests/ref_golden.py)."""
import os

import numpy as np
import pytest

from model_cases import measurement_cases, motion_cases, particle_cases

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_a1_matches_reference_golden(oracle):
    k = np.load(os.path.join(G, "a1_ref_kat.npz"))
    assert len(k["B"]) == 48
    for B, patch, image, xy, out in zip(k["B"], k["patch"], k["image"], k["xy"], k["out"]):
        c, s0, s1 = oracle.correlate2_warning(patch[:B, :B], image, xy[0], xy[1])
        # bit-exact, NaN-safe
        assert np.array([c, s0, s1]).tobytes() == out.tobytes()
    # the degenerate branches (improc.cpp:117-125) are present in the vectors
    assert (k["out"][:, 1] == 0).any() and (k["out"][:, 2] == 0).any()
    assert ((k["out"][:, 1] == 0) & (k["out"][:, 2] == 0) & (k["out"][:, 0] == 0)).any()


def test_a11_matches_reference_golden(oracle):
    k = np.load(os.path.join(G, "a11_ref_kat.npz"))
    ru, rv, rf, _ = oracle.smoe_search(k["image"], k["patch"], k["puinv3"], k["centres"])
    assert (ru == k["res_u"]).all() and (rv == k["res_v"]).all() and (rf == k["res_flag"]).all()
    assert rf.any() and not rf.all()


def test_a1_live_reference_random(oracle, reference):
    rng = np.random.default_rng(7)
    for B in (11, 15, 9):
        img = rng.integers(0, 256, (40, 50), dtype=np.uint8)
        for _ in range(200):
            patch = rng.integers(0, 256, (B, B), dtype=np.uint8)
            x1, y1 = int(rng.integers(0, 50 - B)), int(rng.integers(0, 40 - B))
            a = oracle.correlate2_warning(patch, img, x1, y1)
            b = reference.call("correlate2_warning", patch, img, x1, y1)
            assert np.array(a).tobytes() == np.array(b).tobytes()


def test_a11_live_reference_random(oracle, reference):
    from scenelib2_b200 import synth
    rng = np.random.default_rng(11)
    img = synth.make_texture(rng, 96, 128)
    img[20:50, 30:70] = 90
    for B in (11, 15):
        patch = img[60:60 + B, 80:80 + B].copy()
        K = 20
        centres = np.column_stack([rng.uniform(0, 128, K), rng.uniform(0, 96, K)])
        centres[:4] = [[80 + B // 2 + 0.4, 60 + B // 2 + 0.6]] * 4
        sx, sy = rng.uniform(1.5, 6, K), rng.uniform(1.5, 6, K)
        rho = rng.uniform(-0.8, 0.8, K)
        pu = []
        for a, b, r in zip(sx, sy, rho):
            Si = np.linalg.inv(np.array([[a * a, r * a * b], [r * a * b, b * b]]))
            pu.append([Si[0, 0], Si[0, 1], Si[1, 1]])
        pu = np.array(pu)
        a = oracle.smoe_search(img, patch, pu, centres)
        b = reference.call("smoe_search", img, patch, pu, centres)
        for x, y in zip(a[:3], b[:3]):
            assert (x == y).all()


def test_a2_equals_a11_where_they_coincide(oracle):
    """A2 (monoslam.cpp:401-477) and A11 share the scan; with integer+0.0 centres (rounding ==
    truncation), image sigma >= 10 everywhere and one ellipse they must agree exactly."""
    from scenelib2_b200 import synth
    rng = np.random.default_rng(5)
    img = synth.make_texture(rng, 100, 140)
    B = 11
    for _ in range(10):
        cx, cy = int(rng.integers(10, 130)), int(rng.integers(10, 90))
        patch = img[cy - 5:cy + 6, cx - 5:cx + 6].copy()
        c = np.array([[cx + int(rng.integers(-4, 5)), cy + int(rng.integers(-4, 5))]], float)
        a, b, r = rng.uniform(2, 7), rng.uniform(2, 7), rng.uniform(-0.7, 0.7)
        Si = np.linalg.inv(np.array([[a * a, r * a * b], [r * a * b, b * b]]))
        pu = np.array([[Si[0, 0], Si[0, 1], Si[1, 1]]])
        u, v, f, best = oracle.elliptical_search(img, patch[None], c, pu)
        ru, rv, rf, rbest = oracle.smoe_search(img, patch, pu, c)
        assert (u[0], v[0], f[0]) == (ru[0], rv[0], rf[0])
        assert best[0] == rbest[0]


# ---- closed-form models: the reference's OWN motion_model.cpp / camera.cpp / feature_model.cpp /
# full_feature_model.cpp / support/math_util.cpp, compiled unmodified against oracle/stubs_arith (a minimal
# matrix class with plain-loop arithmetic, NOT Eigen), vs the oracle's restatement.  Pins every formula
# (Jacobians, Q, projection + distortion, R_i, S_i, visibility); Eigen's summation order stays unpinned.

def test_motion_model_matches_reference_source(oracle, reference):
    worst = 0.0
    for xv, dt, u in motion_cases():
        a = oracle.motion(xv, dt, u)
        b = reference.call("motion", xv, dt, u)
        for x, y in zip(a, b):
            assert np.isfinite(y).all()
            worst = max(worst, np.abs(x - y).max() / max(1.0, np.abs(y).max()))
        J = oracle.dxvnorm_by_dxv(xv)
        Jr, xn = reference.call("dxvnorm_by_dxv", xv)
        assert (J == Jr).all()                               # scalar formulas only: bit-exact
        assert (xn == xv).all()                              # quirk Q1: xv comes back un-normalised
    assert worst < 1e-15, worst


def test_measurement_model_matches_reference_source(oracle, reference):
    worst = 0.0
    flags_seen = set()
    for k, (cam8, xv, y, P, xp_org) in enumerate(measurement_cases()):
        Pxx, Pxy, Pyy = P[:13, :13], P[:13, 13:], P[13:, 13:]
        a = oracle.predict_feature(cam8, xv, y, Pxx, Pxy, Pyy)
        b = reference.call("predict_feature", cam8, xv, y, Pxx, Pxy, Pyy)
        for x, r in zip(a, b):
            if np.isfinite(r).all():
                worst = max(worst, np.abs(x - r).max() / max(1.0, np.abs(r).max()))
            else:
                assert not np.isfinite(x).all()
        h = a[0] if np.isfinite(a[0]).all() else np.array([100.0, 100.0])
        va = oracle.visibility_test(cam8, xv[:7], y, xp_org, h)
        vb = reference.call("visibility_test", cam8, xv[:7], y, xp_org, h)
        assert va == vb, (k, va, vb)
        flags_seen.add(vb)
    assert worst < 1e-13, worst
    assert 0 in flags_seen and len(flags_seen) >= 5          # visible and several distinct failure codes


def test_particle_prediction_matches_reference_source(oracle, reference):
    """N2 prediction (monoslam.cpp:1347-1400): the oracle's PartFeatureModel::predict_particle against the
    reference's own part_feature_model.cpp / feature_model.cpp / feature_init_info.cpp (compiled unmodified
    against oracle/stubs_arith): h, S, S^-1, det S per depth particle."""
    worst = 0.0
    for cam8, xv, ypi, P, lam in particle_cases():
        a = oracle.predict_particles(cam8, xv, ypi, lam, P[:13, :13], P[:13, 13:], P[13:, 13:])
        b = reference.call("predict_particles", cam8, xv, ypi, lam, P[:13, :13], P[:13, 13:], P[13:, 13:])
        for x, r in zip(a, b):
            assert np.isfinite(r).all()
            worst = max(worst, np.abs(x - r).max() / max(1.0, np.abs(r).max()))
    assert worst < 1e-13, worst


def test_sinv_matches_reference_source(oracle, reference):
    """Particle::set_S (the reference's own feature_init_info.cpp:55-63, compiled against oracle/stubs_arith)
    runs the same LLT -> matrixL -> inverse -> L^-T L^-1 sequence as MonoSLAM::measure_feature
    (monoslam.cpp:371-374), i.e. the oracle's S -> PuInv (A3).  (The particle bookkeeping of that file is
    checked bit-exactly in test_particle_cycle_matches_reference_source.)"""
    rng = np.random.default_rng(33)
    for _ in range(300):
        a, b = rng.uniform(1, 400, 2)
        r = rng.uniform(-0.95, 0.95)
        S = np.array([[a, r * np.sqrt(a * b)], [r * np.sqrt(a * b), b]])
        Sinv_ref, det_ref = reference.call("particle_set_S_ref", S, live=oracle.particle_set_S_ref)
        pu = oracle.puinv_from_S(S)
        ref3 = np.array([Sinv_ref[0, 0], Sinv_ref[0, 1], Sinv_ref[1, 1]])
        np.testing.assert_allclose(pu, ref3, rtol=4e-15, atol=0)
        assert Sinv_ref[0, 1] == Sinv_ref[1, 0]
        np.testing.assert_allclose(det_ref, a * b * (1 - r * r), rtol=1e-12)


# ---- the whole tracking step: the reference's OWN monoslam.cpp / kalman.cpp / feature.cpp (+ models, improc)
# compiled unmodified against oracle/stubs_arith and driven through MonoSLAM::Init / AddNewKnownFeature /
# fill_* / GoOneStep (oracle/ref_slam_shim.cpp), vs the oracle.  Integer results must be identical; state and
# covariance agree up to summation order (the stand-in matrix class is not Eigen).

def _compare_step(r, o, t, tol):
    fr, fo = r.features(), o.features()
    assert r.num_features == o.num_features and r.n == o.n
    assert (fr["label"] == fo["label"]).all()
    assert (fr["select_rank"] == fo["select_rank"]).all(), t
    assert ((fr["flags"] & 1) == (fo["flags"] & 1)).all(), t
    seen = fo["attempted"] > 0      # the reference leaves the success flag uninitialised until first measured
    assert ((fr["flags"] & 2)[seen] == (fo["flags"] & 2)[seen]).all(), t
    ok = (fo["flags"] & 2) > 0
    assert (fr["z"][ok] == fo["z"][ok]).all(), t                       # bit-exact match positions
    assert (fr["attempted"] == fo["attempted"]).all() and (fr["successful"] == fo["successful"]).all()
    sel = fo["select_rank"] >= 0
    np.testing.assert_allclose(fr["h"][sel], fo["h"][sel], rtol=tol, atol=tol)
    np.testing.assert_allclose(fr["S"][sel], fo["S"][sel], rtol=tol, atol=tol)
    xr, Pr = r.get_state()
    xo, Po = o.get_state()
    d = np.sqrt(np.abs(np.diag(Po))) + 1e-300
    assert np.abs(xr - xo).max() <= tol * max(1.0, np.abs(xo).max())
    stored = np.isfinite(Pr)                                           # the stored entries of the reference's P
    assert (np.abs(Pr - Po) <= tol * d[:, None] * d[None, :])[stored].all()
    assert r.symmetric


def test_whole_step_matches_reference_source(oracle, reference, tmp_path):
    from scenelib2_b200 import synth
    from test_oracle_slam import make_oracle_slam
    kp = np.load(os.path.join(G, "known_patches.npy"))
    # C1: 20 features, 10 selected per frame by trace(S), ellipses from the EKF's own S_i
    sc = synth.make_scene("C1", n_frames=12, known_patches=kp)
    r, o = reference.slam(sc, str(tmp_path / "c1")), make_oracle_slam(oracle, sc)
    xr, Pr = r.get_state()
    xo, Po = o.get_state()
    assert (xr == xo).all() and (Pr == Po)[np.isfinite(Pr)].all()   # Init + AddNewKnownFeature + fill_* round trip
    for t in range(12):
        r.step(sc.frames[t])
        o.step(sc.frames[t])
        _compare_step(r, o, t, 1e-12)
    # C2-like without the benchmark's ellipse override: every feature selected (m = 2N), bigger update
    sc = synth.make_scene("C2", n_frames=4, n_features=24, override=False)
    r, o = reference.slam(sc, str(tmp_path / "c2")), make_oracle_slam(oracle, sc)
    for t in range(4):
        r.step(sc.frames[t])
        o.step(sc.frames[t])
        _compare_step(r, o, t, 1e-11)
    assert (o.features()["select_rank"] >= 0).sum() == 24


def test_bad_feature_deletion_matches_reference_source(oracle, reference, tmp_path):
    """delete_bad_features / delete_feature (monoslam.cpp:644-703, 770-812): a template that never matches is
    culled after 10 attempts; the compaction of state, covariance blocks and lists is the reference's own."""
    from scenelib2_b200 import synth
    from test_oracle_slam import make_oracle_slam
    sc = synth.make_scene("C2", n_frames=2, n_features=12, override=False)
    bad = sc.patches.copy()
    bad[3] = np.random.default_rng(0).integers(0, 256, bad[3].shape, dtype=np.uint8)
    sc.patches = bad
    r, o = reference.slam(sc, str(tmp_path)), make_oracle_slam(oracle, sc)
    n0 = o.n
    for t in range(12):
        r.step(sc.frames[t % 2])
        o.step(sc.frames[t % 2])
        _compare_step(r, o, t, 1e-11)
    assert r.num_features == 11 and r.n == n0 - 3


def test_elliptical_search_and_detector_match_reference_source(oracle, reference):
    """A2 / A3 / N3 one by one against the reference's own monoslam.cpp: MonoSLAM::elliptical_search (rotated and
    border-clamped ellipses, plateaus, 11x11 and 15x15), measure_feature (S -> PuInv -> search) and
    find_best_patch_inside_region (positions and FP64 eigenvalue bits)."""
    from scenelib2_b200 import synth
    rng = np.random.default_rng(41)
    img = synth.make_texture(rng, 120, 160)
    img[30:60, 40:90] = 128                                   # plateau: low sigma, ties
    n_found = 0
    for B in (11, 15):
        h = (B - 1) // 2
        for k in range(120):
            cu, cv = int(rng.integers(h, 160 - h)), int(rng.integers(h, 120 - h))
            patch = img[cv - h:cv + h + 1, cu - h:cu + h + 1].copy()
            if k % 4 == 0:
                patch = rng.integers(0, 256, (B, B), dtype=np.uint8)      # no good match anywhere
            a, b = rng.uniform(2, 14, 2)
            th = rng.uniform(0, np.pi)
            R = np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]])
            Si = np.linalg.inv(R @ np.diag([a * a / 9, b * b / 9]) @ R.T)
            pu = np.array([Si[0, 0], Si[0, 1], Si[1, 1]])
            centre = np.array([cu + rng.uniform(-4, 4), cv + rng.uniform(-4, 4)])
            if k % 7 == 0:
                centre = np.array([rng.choice([1.5, 158.2]), rng.choice([2.4, 117.9])])   # clamped at a corner
            ok, ru, rv = reference.call("elliptical_search_ref", img, patch, centre, pu, live=oracle.elliptical_search_ref)
            ou, ov, of, _ = oracle.elliptical_search(img, patch[None], centre[None], pu[None])
            assert bool(of[0]) == bool(ok), (B, k)
            if ok:
                assert (ou[0], ov[0]) == (ru, rv), (B, k)
                n_found += 1
    assert n_found > 60
    for k in range(100):                                       # A3: S -> PuInv -> search, 11x11
        cu, cv = int(rng.integers(10, 150)), int(rng.integers(10, 110))
        patch = img[cv - 5:cv + 6, cu - 5:cu + 6].copy()
        a, b = rng.uniform(4, 60, 2)
        r = rng.uniform(-0.8, 0.8)
        S = np.array([[a, r * np.sqrt(a * b)], [r * np.sqrt(a * b), b]])
        hh = np.array([cu + rng.uniform(-3, 3), cv + rng.uniform(-3, 3)])
        ok, z = reference.call("measure_feature_ref", img, patch, hh, S, live=oracle.measure_feature_ref)
        pu = oracle.puinv_from_S(S)
        ou, ov, of, _ = oracle.elliptical_search(img, patch[None], hh[None], pu[None])
        assert bool(of[0]) == bool(ok), k
        if ok:
            assert (z == [ou[0], ov[0]]).all(), k
    regions = np.array([[40, 30, 120, 90], [-5, -7, 60, 40], [100, 70, 400, 300], [0, 0, 160, 120],
                        [50, 50, 50, 80], [3, 3, 40, 30], [90, 20, 91, 21], [10, 10, 30, 25]], np.int32)
    for B in (11, 15):
        for reg in regions:
            a = oracle.find_best_patch(img, B, reg, ubest=-7, vbest=-9)
            b = reference.call("find_best_patch", img, B, reg, ubest=-7, vbest=-9)
            assert a[:2] == b[:2] and np.float64(a[2]).tobytes() == np.float64(b[2]).tobytes(), (B, reg)


def test_particle_cycle_matches_reference_source(oracle, reference, tmp_path):
    """N2 end to end on the reference's own code: InitialiseFeature creates a partially-initialised feature with
    100 depth particles; after the camera has moved, predict_partially_initialised_feature_measurements
    (part_feature_model.cpp), measure_feature_with_multiple_priors (SMOE) and
    update_partially_initialised_feature_probabilities run as in MatchPartiallyInitialisedFeatures
    (monoslam.cpp:1299-1340).  Fed with the same particle inputs, the oracle's SMOE search and particle update
    give identical matches, survivors, probabilities (bit-exact), mean and variance."""
    from scenelib2_b200 import synth
    kp = np.load(os.path.join(G, "known_patches.npy"))
    sc = synth.make_scene("C1", n_frames=6, known_patches=kp)
    cycles = 0
    for (u, v, dx) in ((150, 110, (0.03, -0.01, 0.0)), (90, 70, (-0.02, 0.02, 0.01)), (200, 150, (0.0, 0.04, 0.0))):
        r = reference.slam(sc, str(tmp_path / ("p%d_%d" % (u, v))))
        r.init_partial_feature(sc.frames[0], u, v)
        assert r.num_features == sc.n_features + 1 and r.n == 13 + 3 * sc.n_features + 6
        assert r.particle_cycle(sc.frames[0]) is None          # no match attempt right after initialisation
        patch = sc.frames[0][v - 5:v + 6, u - 5:u + 6]
        for t in (1, 2, 3):
            x, P = r.get_state()
            x[:3] += dx                                        # the camera moves: the depth line spreads out
            r.set_state(x, P)
            c = r.particle_cycle(sc.frames[t])
            if c is None:
                break
            ou, ov, of, _ = oracle.smoe_search(sc.frames[t], patch, c["sinv3"], c["h"])
            assert (of == c["found"]).all()
            assert (ou[of > 0] == c["z"][of > 0, 0]).all() and (ov[of > 0] == c["z"][of > 0, 1]).all()
            o = oracle.particle_update(c["h"], c["sinv3"], c["detS"], c["lam"], c["z"], c["found"], 0.05,
                                       c["prob_before"])
            assert o[0] == c["K_after"] and (o[2] == c["keep"]).all()
            kk = c["keep"] > 0
            assert o[1][kk].tobytes() == c["prob_after"][kk].tobytes()
            assert o[3][kk].tobytes() == c["cum"][kk].tobytes()
            assert o[4].tobytes() == c["mean_var"].tobytes()
            cycles += 1
            if c["K_after"] == 0:
                break
    assert cycles >= 4


def test_c4_size_step_matches_reference_source(oracle, reference, tmp_path):
    """Full-size update (n = 313, all 100 features measured, m = 200; ellipses from the EKF's own S_i since the
    reference has no fixed-ellipse switch): Kalman::KalmanFilterUpdate as written (kalman.cpp:72-119) with its
    gather / scatter, on the reference's own code vs the oracle."""
    from scenelib2_b200 import synth
    from test_oracle_slam import make_oracle_slam
    sc = synth.make_scene("C4", n_frames=3, override=False)
    r, o = reference.slam(sc, str(tmp_path)), make_oracle_slam(oracle, sc)
    for t in range(3):
        r.step(sc.frames[t])
        o.step(sc.frames[t])
        _compare_step(r, o, t, 1e-11)
    f = o.features()
    assert ((f["flags"] & 2) > 0).sum() == 100 and o.n == 313
