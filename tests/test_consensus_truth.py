"""The two restatements of the match consensus (consensus_ref.restated in Python floats, consensus_oracle.consensus in
C++ on the oracle) against the consensus from its definition in extended precision (consensus_truth): squared
distances within a bound set from what is measured, and masks, supports and winners equal wherever no decision lies
inside that bound of fl(tau tau).  The cases are those of test_consensus.py and ones that tell a right algebra from a
wrong one: strongly correlated maps, |q| != 1, both distorted cameras, ill-conditioned S, innovations of tens of
pixels, points near depth 0 on both sides and an asymmetric P.  Deliberately broken copies of the restatement must
fail the same checks."""
import functools

import numpy as np
import pytest

import consensus_oracle as co
import consensus_ref
from camera_ref import quat_to_R
from consensus_truth import EPS, consensus_truth, s_consistency
from oracle import pyoracle as po
from scenelib2_b200 import synth
from test_consensus import _cluster_case, behind_camera_case, make_case

C1 = synth.camera_params(320, 240)   # kd1 = 9e-6
C3 = synth.camera_params(640, 480)   # kd1 = 2.25e-6
KEYS = ("cam8", "x", "P", "pos", "z", "h", "S", "dh_dxp", "dh_dy")
# |d2_restated - d2_truth| <= D2_BOUND max(1, d2_truth).  Worst measured over every case below (x86-64): 4.1e-12, on
# the ill-conditioned S of R blocks with 1 - |rho| = 1e-6 (the well-conditioned cases stay below 1.3e-13); the bound
# leaves a factor of 25 (test_distances_within_bound prints the worst).
D2_BOUND = 1e-10
# a point in front of or behind the camera is a decision too: |depth| below this is inside the band
DEPTH_BAND = 1e-12


# ---- cases ---------------------------------------------------------------------------------------------------------
def _args(case):
    return [case[k] for k in KEYS]


def _repredicted(case):
    """h, S and the Jacobians predicted again from the case's x and P (after a constructor changed them), z kept."""
    x, P, cam8 = case["x"], case["P"], case["cam8"]
    for j, p in enumerate(case["pos"]):
        h, dxv, dy, _, S = po.predict_feature(cam8, x[:13], x[p:p + 3], P[:13, :13], P[:13, p:p + 3],
                                              P[p:p + 3, p:p + 3])
        case["h"][j], case["S"][j], case["dh_dxp"][j], case["dh_dy"][j] = h, S, dxv[:, :7], dy
    return case


def _correlated_case(rng, k, cam8=C1):
    """A map initialised from one camera pose: every feature carries that pose's uncertainty (position 5 cm, attitude
    0.03 rad) plus its own depth along its ray, so P[y_j, y_i] is as large as P[y_i, y_i]; the current camera is
    known well relative to the map (5 mm, 0.003 rad).  Some matches are off by (6, -4) px."""
    nf = k + 2
    n = 13 + 3 * nf
    xv = np.concatenate([rng.normal(0.0, 0.05, 3), [1.0, 0.0, 0.0, 0.0], rng.normal(0.0, 0.02, 6)])
    q = rng.normal(0.0, 0.04, 3)
    xv[3:7] = np.array([1.0, *q]) / np.sqrt(1.0 + q @ q)
    R = np.array(quat_to_R(*xv[3:7]))
    d = rng.uniform(0.6, 1.6, nf)
    cpts = np.stack([rng.uniform(-0.35, 0.35, nf) * d, rng.uniform(-0.25, 0.25, nf) * d, d], axis=1)
    wpts = cpts @ R.T                     # y - r in the world
    cols = 12 + nf                        # map pose (6), camera relative to it (6), one depth per feature
    G = np.zeros((n, cols))
    w, x, y, z = xv[3:7]
    dq = 0.5 * np.array([[-x, -y, -z], [w, -z, y], [z, w, -x], [-y, x, w]])   # d q / d theta (body increment)
    for c0 in (0, 6):
        G[0:3, c0:c0 + 3] = np.eye(3)
        G[3:7, c0 + 3:c0 + 6] = dq
    for f in range(nf):
        p = 13 + 3 * f
        v = wpts[f]
        G[p:p + 3, 0:3] = np.eye(3)
        G[p:p + 3, 3:6] = -np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])
        G[p:p + 3, 12 + f] = v / np.linalg.norm(v)
    sig = np.concatenate([np.full(3, 0.05), np.full(3, 0.03), np.full(3, 0.005), np.full(3, 0.003),
                          0.02 * d])
    P = (G * sig ** 2) @ G.T + 1e-8 * np.eye(n)
    P[7:13, 7:13] += np.eye(6) * 1e-4
    P = 0.5 * (P + P.T)
    return make_case(rng, k, nf=nf, P=P, camera_pts=cpts, xv=xv, cam8=cam8,
                     outliers=rng.permutation(k)[:k // 4], offset=(6.0, -4.0))


def _non_unit_q_case(rng, k, scale):
    xv = np.concatenate([rng.normal(0.0, 0.05, 3), [1.0, 0.0, 0.0, 0.0], rng.normal(0.0, 0.02, 6)])
    q = np.array([1.0, *rng.normal(0.0, 0.08, 3)])
    xv[3:7] = scale * q / np.linalg.norm(q)
    return make_case(rng, k, xv=xv, outliers=[1], offset=(5.0, 3.0))


def _rho_case(rng, k, one_minus_rho):
    """Ill-conditioned S_i = H_i P H_i^T + R_i from R blocks var [[1, rho], [rho, 1]], |rho| = 1 - one_minus_rho,
    on a small P (sigmas / 300) so that R dominates.  Returns the case and its R blocks."""
    n = 13 + 3 * (k + 3)
    P = synth.make_prior_covariance(rng, n, sig_y=0.01) / 300.0 ** 2
    case = make_case(rng, k, P=P)
    R = np.zeros((k, 2, 2))
    for j in range(k):
        rho = (1.0 - one_minus_rho) * rng.choice([-1.0, 1.0])
        var = rng.uniform(1.0, 4.0)
        R[j] = var * np.array([[1.0, rho], [rho, 1.0]])
        H = np.zeros((2, n))
        H[:, :7], H[:, case["pos"][j]:case["pos"][j] + 3] = case["dh_dxp"][j], case["dh_dy"][j]
        S = H @ P @ H.T + R[j]
        case["S"][j] = 0.5 * (S + S.T)
    return case, R


def _stretched_case(rng, k, lam):
    """Camera uncertainty stretched along one direction of (r, q): P[0:7, 0:7] += lam v v^T (|v| = 1).  S_i is then
    nearly rank one."""
    n = 13 + 3 * (k + 3)
    P = synth.make_prior_covariance(rng, n, sig_y=0.01)
    v = rng.normal(0.0, 1.0, 7)
    v[3:7] *= 0.3
    v /= np.linalg.norm(v)
    P[:7, :7] += lam * np.outer(v, v)
    return make_case(rng, k, P=P, outliers=[0, 3], offset=(7.0, 7.0))


def _large_innovation_case(rng, k, cam8=C1):
    """The camera moved: every z off its prediction by a common (22, -17) px, a third off by a further (-30, 12)."""
    case = make_case(rng, k, cam8=cam8)
    case["z"] = case["z"] + [22.0, -17.0]
    case["z"][rng.permutation(k)[:k // 3]] += [-30.0, 12.0]
    return case


def _near_depth_zero_case(rng, k):
    """Points a few mm in front of and behind the camera (camera-frame depth +-2..20 mm, lateral offset in proportion
    so that they project into the image) with 1 cm feature sigmas: hypotheses move them across depth 0."""
    d = rng.uniform(0.002, 0.02, k + 3) * np.where(np.arange(k + 3) % 2 == 0, 1.0, -1.0)
    pts = np.stack([rng.uniform(-0.35, 0.35, k + 3) * d, rng.uniform(-0.25, 0.25, k + 3) * d, d], axis=1)
    pts[::3] *= 50.0   # and some ordinary points 10 cm .. 1 m away
    return make_case(rng, k, camera_pts=pts)


def _asymmetric_case(rng, k):
    """P = P_sym + A with A antisymmetric (30 % of the natural scale sqrt(P_ii P_jj)); S from P_sym, so P[a, b] and
    P[b, a] differ while S is the one the algebra assumes."""
    case = make_case(rng, k, outliers=[2], offset=(6.0, -5.0))
    P = case["P"]
    s = np.sqrt(np.diag(P))
    A = rng.normal(0.0, 0.3, P.shape) * np.outer(s, s)
    case["P"] = P + 0.5 * (A - A.T)
    return case


@functools.lru_cache(maxsize=None)
def cases():
    """[(name, case, tau, R blocks or None)]"""
    out = []
    rng = np.random.default_rng(101)
    for t in range(24):   # test_consensus's random cases, on both distorted cameras
        cam8 = C1 if t % 2 == 0 else C3
        k = int(rng.integers(2, 25))
        outl = rng.permutation(k)[:int(rng.integers(0, max(1, k // 3) + 1))]
        case = make_case(rng, k, outliers=outl, offset=rng.uniform(-15, 15, 2).round(), cam8=cam8)
        out.append(("random-%s-%d" % ("C1" if t % 2 == 0 else "C3", t), case, float(rng.choice([1.5, 2.0, 3.0, 5.0])),
                    None))
    rng = np.random.default_rng(102)
    out.append(("small-k2", make_case(rng, 2), 3.0, None))
    out.append(("small-k2-apart", make_case(rng, 2, outliers=[1], offset=(14.0, 9.0)), 2.0, None))
    for k in (3, 8, 20):
        out.append(("agreeing-%d" % k, make_case(rng, k), 3.0, None))
    for k in (4, 6, 10):
        out.append(("clusters-%d" % k, _cluster_case(rng, k), 2.5, None))
    out.append(("behind-camera", _repredicted(behind_camera_case(rng)), 1000.0, None))
    out.append(("knife-edge-case", make_case(rng, 8, outliers=[5], offset=(4.0, 3.0)), 3.0, None))
    for k, cam8 in ((6, C1), (12, C3), (20, C1)):
        out.append(("correlated-%d" % k, _correlated_case(rng, k, cam8), 2.5, None))
    for scale in (0.97, 1.03, 1.2):
        out.append(("q-norm-%.2f" % scale, _non_unit_q_case(rng, 10, scale), 3.0, None))
    for e in (3, 6, 9):
        case, R = _rho_case(rng, 8, 10.0 ** -e)
        out.append(("rho-1e-%d" % e, case, 3.0, R))
    for lam in (1e-2, 1.0):
        out.append(("stretched-%g" % lam, _stretched_case(rng, 10, lam), 3.0, None))
    out.append(("innovation-C1", _large_innovation_case(rng, 12, C1), 4.0, None))
    out.append(("innovation-C3", _large_innovation_case(rng, 12, C3), 4.0, None))
    out.append(("near-depth-0", _near_depth_zero_case(rng, 12), 3.0, None))
    out.append(("near-depth-0-wide", _near_depth_zero_case(rng, 12), 1000.0, None))
    out.append(("asymmetric-P", _asymmetric_case(rng, 10), 3.0, None))
    return out


@functools.lru_cache(maxsize=None)
def truths(prec="ld"):
    return [consensus_truth(*_args(c), tau, prec=prec) for _, c, tau, _ in cases()]


# ---- the checks ----------------------------------------------------------------------------------------------------
def compare(case, tau, tr, restate=consensus_ref.restated):
    """-> (failures, worst relative d2 error, inside the band).  failures holds ("distance", ...) and ("decision", ...)
    entries; no decision is compared where one that matters lies inside the band."""
    keep, sup, win, d2 = restate(*_args(case), tau)
    fail = []
    front = ~np.isnan(tr.d2)
    depth_ok = np.abs(tr.depth) > DEPTH_BAND * (1.0 + np.abs(tr.depth).max())
    if ((np.isnan(d2) != ~front) & depth_ok).any():
        fail.append(("distance", "a point's side of the camera differs"))
    both = front & ~np.isnan(d2)
    err = np.abs(d2[both] - tr.d2[both]) / np.maximum(1.0, tr.d2[both])
    worst = float(err.max()) if err.size else 0.0
    if worst > D2_BOUND:
        fail.append(("distance", "d2 off by %.3e relative" % worst))
    band = tr.margin <= D2_BOUND * max(1.0, tau * tau) or not depth_ok.all()
    if not band:
        if not ((d2 <= tau * tau) == tr.inlier).all():
            fail.append(("decision", "inlier masks differ"))
        if not ((sup == tr.support).all() and win == tr.winner and (keep == tr.keep).all()):
            fail.append(("decision", "support %s / %s, winner %d / %d" % (sup, tr.support, win, tr.winner)))
    return fail, worst, band


def test_longdouble_truth_agrees_with_mpmath():
    """The mpmath truth (50 digits) is the definition; the longdouble one, which the other checks and the GPU tests use,
    must give the same decisions and d2 to far inside D2_BOUND."""
    worst = 0.0
    picked = [i for i, (name, c, _, _) in enumerate(cases()) if len(c["pos"]) <= 12]
    assert len(picked) >= 20
    for i in picked:
        tm, tl = consensus_truth(*_args(cases()[i][1]), cases()[i][2], prec="mp"), truths()[i]
        assert (np.isnan(tm.d2) == np.isnan(tl.d2)).all()
        f = ~np.isnan(tm.d2)
        e = np.abs(tm.d2[f] - tl.d2[f]) / np.maximum(1.0, tm.d2[f])
        worst = max(worst, float(e.max()) if e.size else 0.0)
        assert (tm.inlier == tl.inlier).all() and tm.winner == tl.winner and (tm.keep == tl.keep).all()
    print("longdouble vs mpmath truth over %d cases: worst relative d2 difference %.3e" % (len(picked), worst))
    assert worst <= D2_BOUND * 1e-3


def test_s_is_the_one_the_algebra_assumes():
    """S_i = H_i P H_i^T + R_i (R_i = Camera::MeasurementNoise of h_i, or the designed blocks) to FP64 rounding: the
    S the consensus is handed is the S its one-point update assumes."""
    worst = 0.0
    for name, c, _, R in cases():
        if len(c["pos"]):
            e = s_consistency(c["cam8"], c["P"], c["pos"], c["h"], c["S"], c["dh_dxp"], c["dh_dy"], R)
            worst = max(worst, e)
            assert e <= 64 * EPS, (name, e)
    print("worst |S - (H P H^T + R)| / (|H| |P| |H|^T + |R|): %.3e = %.1f eps" % (worst, worst / EPS))


def test_distances_within_bound():
    worst, nearest, diag = 0.0, np.inf, 0.0
    for (name, c, tau, _), tr in zip(cases(), truths()):
        fail, w, _ = compare(c, tau, tr)
        assert not [f for f in fail if f[0] == "distance"], (name, fail)
        worst = max(worst, w)
        nearest = min(nearest, tr.margin)
        _, _, _, d2 = consensus_ref.restated(*_args(c), tau)
        dd, td = np.diag(d2), np.diag(tr.d2)
        f = ~np.isnan(td)
        if f.any():
            diag = max(diag, float((np.abs(dd[f] - td[f]) / np.maximum(1.0, td[f])).max()))
    print("worst |d2_restated - d2_truth| / max(1, d2_truth) over %d cases: %.3e (i = j pairs: %.3e); bound %.0e; "
          "nearest d2 to fl(tau^2): %.3e px^2" % (len(cases()), worst, diag, D2_BOUND, nearest))


@pytest.mark.parametrize("which", ["restated", "oracle"])
def test_decisions_equal_the_truth(which):
    def oracle(*a):
        keep, sup, win = co.consensus(*a)
        _, _, _, d2 = consensus_ref.restated(*a)   # the oracle's d2 is not exposed: its decisions are compared
        return keep, sup, win, d2
    restate = consensus_ref.restated if which == "restated" else oracle
    inside = []
    rejected = 0
    for (name, c, tau, _), tr in zip(cases(), truths()):
        fail, _, band = compare(c, tau, tr, restate)
        assert not [f for f in fail if f[0] == "decision"], (name, fail)
        if band:
            inside.append(name)
            print("inside the band, decisions not compared: %s (margin %.3e px^2, depth margin %.3e)"
                  % (name, tr.margin, tr.depth_margin))
        rejected += int((~tr.keep).sum())
    assert len(inside) <= 2 and rejected > 0, inside


# ---- the checks can see ----------------------------------------------------------------------------------------------
class _P:
    """A view of P for a broken restatement: `drop` zeroes P[y_j, y_i] (both indices in the map), `transpose` reads
    P[c, r] for P[r, c]."""

    def __init__(self, P, how):
        self.P, self.how = P, how

    def __getitem__(self, rc):
        r, c = rc
        if self.how == "drop" and r >= 13 and c >= 13:
            return 0.0
        return self.P[c, r] if self.how == "transpose" else self.P[r, c]


MUTATIONS = ["drop-Pyy-b", "P-transposed", "S-for-Sinv", "normalised-q", "kd1-zero"]


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_mutations_are_caught(mutation, monkeypatch):
    """Each broken copy of the restatement fails the distance or decision checks on at least one case."""
    reproj = consensus_ref.reprojection_d2

    def restate(cam8, x, P, *rest):
        if mutation == "drop-Pyy-b":
            P = _P(P, "drop")
        elif mutation == "P-transposed":
            P = _P(P, "transpose")
        return consensus_ref.restated(cam8, x, P, *rest)

    if mutation == "S-for-Sinv":
        monkeypatch.setattr(consensus_ref, "_sinv", lambda S: (float(S[0, 0]), float(S[1, 0]), float(S[1, 1])))
    elif mutation == "normalised-q":
        def normalised(cam8, xp, y, z):
            xp = np.array(xp, np.float64)
            xp[3:7] /= np.linalg.norm(xp[3:7])
            return reproj(cam8, xp, y, z)
        monkeypatch.setattr(consensus_ref, "reprojection_d2", normalised)
    elif mutation == "kd1-zero":
        monkeypatch.setattr(consensus_ref, "reprojection_d2",
                            lambda cam8, xp, y, z: reproj(np.concatenate([cam8[:6], [0.0], cam8[7:]]), xp, y, z))
    caught = {}
    for (name, c, tau, _), tr in zip(cases(), truths()):
        for kind in sorted({f[0] for f in compare(c, tau, tr, restate)[0]}):
            caught.setdefault(kind, []).append(name)
    print("%s: %s" % (mutation, {k: "%d cases, first %s" % (len(v), v[0]) for k, v in caught.items()}))
    assert caught
