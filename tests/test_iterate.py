"""The iterated EKF update (sl2_set_stream_iterated) on the CPU: the op-for-op restatement of iterate_kernel
(tests/iterate_ref.py) against the update from its definition (tests/iterate_truth.py), the decision rule at its knife
edges, invalid relinearisations, known features, what the iteration buys on nonlinear priors, broken copies of the
restatement, and the struct's layout."""
import ctypes
import math

import mpmath
import numpy as np
import pytest

import iterate_ref as ref
import iterate_truth as tr
from rescue_truth import Ext, Mp
from test_abi import AbiCase, _c_layout
import scenelib2_b200.lib as mirror

U = 2.0 ** -53
CAM8 = np.array([320.0, 240.0, 195.0, 195.0, 162.0, 125.0, 9e-6, 1.0])


def nonlinear_case(seed, K=4, depth_sigma=0.4, cam_sigma=0.03, qnorm=1.0, depth=(0.5, 1.2), known=()):
    """A camera at the origin looking along +z and K near features whose covariance is a converted depth ray: depth
    sigma depth_sigma x depth along the ray, 1 % of the depth across it; the camera position uncertain across the view
    by cam_sigma.  Features in `known` have zero rows and columns (a known feature).  The true state differs from the
    estimate by one sigma in depth; z = h(true) + 0.3 px noise.  -> (x0, P0, feats, z, Rvar)."""
    rng = np.random.default_rng(seed)
    n = 13 + 3 * K
    x0 = np.zeros(n)
    x0[3] = qnorm
    x0[7:13] = rng.normal(0.0, 1e-3, 6)
    P0 = np.zeros((n, n))
    P0[:13, :13] = np.diag([cam_sigma ** 2, cam_sigma ** 2, 1e-6, 1e-8, 1e-8, 1e-8, 1e-8] + [1e-4] * 6)
    xt = x0.copy()
    for k in range(K):
        pos = 13 + 3 * k
        d = rng.uniform(*depth)
        ray = np.array([rng.uniform(-0.5, 0.5), rng.uniform(-0.4, 0.4), 1.0])
        ray /= np.linalg.norm(ray)
        x0[pos:pos + 3] = d * ray
        if k in known:
            xt[pos:pos + 3] = x0[pos:pos + 3]
            continue
        sd, sl = depth_sigma * d, 0.01 * d
        P0[pos:pos + 3, pos:pos + 3] = sd ** 2 * np.outer(ray, ray) + sl ** 2 * (np.eye(3) - np.outer(ray, ray))
        xt[pos:pos + 3] = (d + rng.choice([-1.0, 1.0]) * 0.8 * sd) * ray
    xt[:2] += rng.normal(0.0, cam_sigma, 2)
    feats = list(range(K))
    h, _, _, _ = ref.lin0(CAM8, xt, feats)
    z = h + rng.normal(0.0, 0.3, h.shape)
    Rvar = [1.0] * K
    return x0, P0, feats, z, Rvar


def _band(P0, feats, L, z, Rvar, x0):
    """|x_1 - truth| bound per entry from the operation count: each entry's chain is the two panel solves (at most m +
    16 operations per row of t each) and the m-term product plus the add, every one rounding with relative error u;
    the solve amplifies by cond(S).  8 (2 m + 34) u cond(S) (|x0_j| + sum_r |(H P0)_rj t_r|)."""
    HP, S, U_, W, nu = ref.factor(P0, feats, L, z, Rvar)
    t = np.linalg.solve(S, nu)
    m = len(nu)
    return 8 * (2 * m + 34) * U * np.linalg.cond(S) * (np.abs(x0) + np.abs(HP.T) @ np.abs(t))


@pytest.mark.parametrize("seed,K,qn", [(1, 2, 1.0), (2, 5, 1.0), (3, 9, 1.013), (4, 12, 0.985)])
def test_restatement_within_band_of_truth(seed, K, qn):
    x0, P0, feats, z, Rvar = nonlinear_case(seed, K=K, qnorm=qn)
    L0 = ref.lin0(CAM8, x0, feats)[:3]
    r = ref.iterated(CAM8, x0, P0, feats, z, Rvar, 3, 0.0, L0)
    t = tr.iterated_truth(Ext, CAM8, x0, P0, feats, z, Rvar, 3, 0.0, L0)
    assert r["status"] == t["status"] == 2 and r["iterations"] == t["iterations"] == 3
    band = _band(P0, feats, L0, z, Rvar, x0)
    err = np.abs(r["xs"][0] - np.asarray(t["xs"][0], np.float64))
    assert (err <= band).all(), (err / band).max()
    # the relinearisation at the restatement's own x_1 against the definition's model at the same point: the model's
    # chain is about 200 operations, each rounding with relative error u, on the scale of the tables (|H| ~ fku / z2)
    ok, L1 = ref.relinearise(CAM8, x0, r["xs"][0], feats)
    assert ok
    for a, b in zip(L1, _truth_tables_at(x0, r["xs"][0], feats)):
        b = np.asarray(b, np.float64)
        assert np.abs(a - b).max() <= 400 * U * np.abs(b).max(), np.abs(a - b).max() / np.abs(b).max()


def _truth_tables_at(x0, xn, feats):
    from rescue_truth import model
    hs, xs, ys = [], [], []
    x0a, xa = Ext.conv(x0), Ext.conv(xn)
    for f in feats:
        pos = 13 + 3 * f
        h, Hxp, Hy, _, _ = model(Ext, CAM8, xa[:7], xa[pos:pos + 3])
        hs.append([h[r] + sum(Hxp[r][c] * (x0a[c] - xa[c]) for c in range(7)) +
                   sum(Hy[r][c] * (x0a[pos + c] - xa[pos + c]) for c in range(3)) for r in range(2)])
        xs.append(Hxp), ys.append(Hy)
    return np.array(hs), np.array(xs), np.array(ys)


def test_truth_agrees_with_50_digits():
    x0, P0, feats, z, Rvar = nonlinear_case(7, K=1)
    L0 = ref.lin0(CAM8, x0, feats)[:3]
    e = tr.iterated_truth(Ext, CAM8, x0, P0, feats, z, Rvar, 2, 0.0, L0)
    with mpmath.workdps(50):
        m = tr.iterated_truth(Mp(), CAM8, x0, P0, feats, z, Rvar, 2, 0.0, L0)
        for xe, xm in zip(e["xs"], m["xs"]):
            for j in range(len(x0)):
                s = max(abs(float(xm[j])), math.sqrt(P0[j, j]))
                assert abs(float(xe[j]) - float(xm[j])) <= 2e-16 * s, j


def test_zero_iterations_is_the_plain_update():
    x0, P0, feats, z, Rvar = nonlinear_case(5)
    L0 = ref.lin0(CAM8, x0, feats)[:3]
    r = ref.iterated(CAM8, x0, P0, feats, z, Rvar, 0, 0.0, L0)
    assert r["status"] == 0 and r["iterations"] == 0 and not r["xs"]
    assert all(a is b for a, b in zip(r["L"], L0))


def test_decision_at_the_knife_edge():
    x0, P0, feats, z, Rvar = nonlinear_case(6)
    L0 = ref.lin0(CAM8, x0, feats)[:3]
    d0 = ref.iterated(CAM8, x0, P0, feats, z, Rvar, 1, 0.0, L0)["delta"]
    assert d0 > 0
    at = ref.iterated(CAM8, x0, P0, feats, z, Rvar, 2, d0, L0)
    assert at["status"] == 1 and at["iterations"] == 0 and at["L"][0] is L0[0]
    below = d0
    for _ in range(3):
        below = np.nextafter(below, 0.0)
    on = ref.iterated(CAM8, x0, P0, feats, z, Rvar, 1, below, L0)
    assert on["status"] == 2 and on["iterations"] == 1
    # the truth makes the same decisions away from the edge
    t = tr.iterated_truth(Ext, CAM8, x0, P0, feats, z, Rvar, 1, d0 * 0.5, L0)
    assert t["status"] == 2


def test_invalid_relinearisation_keeps_the_last_linearisation():
    """A feature one unit off axis at depth 1 with a large lateral prior and a match 500 px away: the linear step
    moves it behind the camera, so pass 0's relinearisation is invalid and the final update reads L_0."""
    x0, P0, feats, z, Rvar = nonlinear_case(8, K=2)
    pos = 13
    x0[pos:pos + 3] = [1.0, 0.0, 1.0]
    P0[pos:pos + 3, :] = 0.0
    P0[:, pos:pos + 3] = 0.0
    P0[pos:pos + 3, pos:pos + 3] = np.eye(3) * 4.0
    L0 = ref.lin0(CAM8, x0, feats)[:3]
    z = L0[0].copy()
    z[0, 0] -= 500.0
    r = ref.iterated(CAM8, x0, P0, feats, z, Rvar, 3, 0.0, L0)
    t = tr.iterated_truth(Ext, CAM8, x0, P0, feats, z, Rvar, 3, 0.0, L0)
    assert r["status"] == t["status"] == 3 and r["iterations"] == t["iterations"] == 0
    assert r["xs"][0][pos + 2] < 0
    assert all(a is b for a, b in zip(r["L"], L0))


def test_known_features_are_skipped_in_the_step():
    x0, P0, feats, z, Rvar = nonlinear_case(9, K=4, known=(1, 3))
    assert (np.diag(P0)[13 + 3:13 + 6] == 0).all()
    L0 = ref.lin0(CAM8, x0, feats)[:3]
    r = ref.iterated(CAM8, x0, P0, feats, z, Rvar, 1, 0.0, L0)
    d = np.diag(P0)
    on = d > 0
    assert math.isfinite(r["delta"])
    assert r["delta"] == np.max(np.abs(r["xs"][0] - x0)[on] / np.sqrt(d[on]))


# Capability on constructed nonlinear priors (depth sigma 30-50 % along the ray, lateral camera sigma 3 cm): J at the
# converged iterate against J at the plain EKF update's state.  From the truth (np.longdouble) on these seeds: J(IEKF) /
# J(EKF) was 0.056 - 0.255 (J(EKF) 12 - 76), the iteration converged in 6 - 7 relinearisations at tol = 1e-6, and the
# converged iterate was within 6.5e-8 prior sigmas of the Gauss-Newton minimiser.
J_RATIO_MAX = 0.5
GN_DIST_MAX = 1e-6
@pytest.mark.parametrize("seed,ds", [(11, 0.3), (12, 0.4), (13, 0.5), (14, 0.45)])
def test_iteration_lowers_the_posterior_cost(seed, ds):
    x0, P0, feats, z, Rvar = nonlinear_case(seed, K=6, depth_sigma=ds, depth=(0.4, 0.9))
    L0 = ref.lin0(CAM8, x0, feats)[:3]
    r = ref.iterated(CAM8, x0, P0, feats, z, Rvar, 8, 1e-6, L0)
    assert r["status"] == 1
    x_ekf = tr.iterated_truth(Ext, CAM8, x0, P0, feats, z, Rvar, 1, 0.0, L0)["xs"][0]
    x_iekf = r["xs"][-1]
    J_ekf = tr.cost(CAM8, x0, P0, feats, z, Rvar, np.asarray(x_ekf, np.float64))
    J_iekf = tr.cost(CAM8, x0, P0, feats, z, Rvar, x_iekf)
    assert J_iekf < J_ekf * J_RATIO_MAX, (float(J_iekf), float(J_ekf))
    xs = np.asarray(tr.gauss_newton(CAM8, x0, P0, feats, z, Rvar, L0), np.float64)
    d = np.diag(P0)
    assert (np.abs(x_iekf - xs) / np.sqrt(d)).max() <= GN_DIST_MAX


# ---- broken copies of the restatement, each caught by a named check ----------------------------------------------------
def _checks(case):
    """name -> bool for the checks the restatement passes: x_2 and the tables at x_1 against the truth (non-unit q),
    and the iteration count."""
    x0, P0, feats, z, Rvar = case
    L0 = ref.lin0(CAM8, x0, feats)[:3]
    r = ref.iterated(CAM8, x0, P0, feats, z, Rvar, 2, 0.0, L0)
    t = tr.iterated_truth(Ext, CAM8, x0, P0, feats, z, Rvar, 2, 0.0, L0)
    sig = np.sqrt(np.diag(P0))
    x2 = np.abs(r["xs"][1] - np.asarray(t["xs"][1], np.float64)) / np.maximum(sig, 1e-300)
    _, L1 = ref.relinearise(CAM8, x0, r["xs"][0], feats)
    tt = _truth_tables_at(x0, r["xs"][0], feats)
    tab = max(np.abs(a - np.asarray(b, np.float64)).max() for a, b in zip(L1, tt))
    return {"x2_matches_truth": x2.max() <= 1e-8, "tables_match_truth": tab <= 1e-8,
            "iterations_match_truth": r["iterations"] == t["iterations"] == 2 and r["status"] == t["status"]}


BROKEN = {
    "no_correction_term": ("correction", lambda h, Hxp, Hy, dx, dy: np.array(h, np.float64), "x2_matches_truth"),
    "posterior_prior": ("pass_prior", lambda P0, Pa: Pa, "x2_matches_truth"),
    "renormalised_q": ("model_pose", lambda xn: np.concatenate([xn[:3], xn[3:7] / np.linalg.norm(xn[3:7])]),
                       "tables_match_truth"),
    "count_off_by_one": ("count_after", lambda i: i, "iterations_match_truth"),
}


def test_restatement_passes_the_named_checks():
    assert all(_checks(nonlinear_case(21, K=5, qnorm=1.02)).values())


@pytest.mark.parametrize("name", sorted(BROKEN))
def test_broken_copy_is_caught(monkeypatch, name):
    attr, fn, check = BROKEN[name]
    monkeypatch.setattr(ref, attr, fn)
    assert not _checks(nonlinear_case(21, K=5, qnorm=1.02))[check]


def test_struct_matches_header(tmp_path):
    case = AbiCase("sl2_stream_iterated", mirror.Sl2StreamIterated, ("max_iterations", "reserved", "tol"), size=16,
                   consts={"SL2_MAX_ITERATIONS": (mirror.SL2_MAX_ITERATIONS, 8)})
    out = _c_layout(tmp_path, case)
    assert out["SL2_MAX_ITERATIONS"] == (8,) and out["sizeof"] == (16,)
    for f, t in mirror.Sl2StreamIterated._fields_:
        assert out[f] == (getattr(mirror.Sl2StreamIterated, f).offset, ctypes.sizeof(t)), f
