"""The mutual-information selection's rule (include/sl2b200.h, sl2_set_stream_selection) on the CPU: the NumPy
restatement (tests/selection_ref.py) against an extended-precision truth that recomputes every conditional q from
scratch, and against constructed cases whose answer is known exactly: no correlation, a duplicate feature, the
threshold's knife edge and degenerate innovation covariances."""
import math

import mpmath
import numpy as np
import pytest

import selection_ref as sr
from scenelib2_b200 import synth

NXV = 13
# |q_restated - q_true| <= Q_RTOL q_true at every decision of the random cases below: the restatement starts from the
# rounded S_i and accumulates O(10 r) rounding errors per pick, each amplified by at most the condition of the picked
# block (< 1e2 here).  The worst seen over the cases is 6e-15; it is printed.
Q_RTOL = 1e-12


def problem(seed, nf, camera_share=0.9):
    """A map of nf features whose innovations share a camera-pose term: P from synth's prior (dense, SPD) with the
    camera block scaled up, Jacobians drawn at pixel scale, R growing away from the image centre as
    measurement_noise does.  Returns P, S (nf, 4) column-major as the prediction stores it, A, B, R."""
    rng = np.random.default_rng(seed)
    n = NXV + 3 * nf
    P = synth.make_prior_covariance(rng, n, sig_r=0.02 * camera_share + 0.002, sig_y=0.01)
    A = rng.standard_normal((nf, 2, 7)) * 300.0
    B = rng.standard_normal((nf, 2, 3)) * 300.0
    R = (1.0 + rng.uniform(0, 1, nf)) ** 2
    S = np.zeros((nf, 4))
    for j in range(nf):
        H = np.zeros((2, n))
        H[:, :7] = A[j]
        H[:, NXV + 3 * j:NXV + 3 * j + 3] = B[j]
        Sj = H @ P @ H.T + R[j] * np.eye(2)
        S[j] = [Sj[0, 0], Sj[1, 0], Sj[1, 0], Sj[1, 1]]
    return P, S, A, B, R


class Truth:
    """det(C_j | picked) / R_j^2 at 50 digits: the Schur complement of the picked features' block in
    S = H P H^T + R, from the float inputs taken as exact."""

    def __init__(self, P, A, B, R):
        mpmath.mp.dps = 50
        self.n, self.A, self.B, self.R = P.shape[0], A, B, R
        self.P = mpmath.matrix(P.tolist())
        self.HP, self.blk = {}, {}

    def H(self, f):
        h = mpmath.zeros(2, self.n)
        for a in range(2):
            for k in range(7):
                h[a, k] = mpmath.mpf(float(self.A[f, a, k]))
            for k in range(3):
                h[a, NXV + 3 * f + k] = mpmath.mpf(float(self.B[f, a, k]))
        return h

    def block(self, f, g):
        if (f, g) not in self.blk:
            if f not in self.HP:
                self.HP[f] = self.H(f) * self.P
            b = self.HP[f] * self.H(g).T
            if f == g:
                for a in range(2):
                    b[a, a] += mpmath.mpf(float(self.R[f]))
            self.blk[(f, g)] = b
        return self.blk[(f, g)]

    def q(self, picked, j):
        k = 2 * len(picked)
        Sjj = self.block(j, j).copy()
        if k:
            Spp, Spj = mpmath.zeros(k, k), mpmath.zeros(k, 2)
            for x, f in enumerate(picked):
                for y, g in enumerate(picked):
                    b = self.block(f, g)
                    for a in range(2):
                        for c in range(2):
                            Spp[2 * x + a, 2 * y + c] = b[a, c]
                b = self.block(f, j)
                for a in range(2):
                    for c in range(2):
                        Spj[2 * x + a, c] = b[a, c]
            X = mpmath.zeros(k, 2)
            for c in range(2):
                col = mpmath.lu_solve(Spp, mpmath.matrix([Spj[x, c] for x in range(k)]))
                for x in range(k):
                    X[x, c] = col[x]
            Sjj = Sjj - Spj.T * X
        det = Sjj[0, 0] * Sjj[1, 1] - Sjj[0, 1] * Sjj[1, 0]
        return det / mpmath.mpf(float(self.R[j])) ** 2


@pytest.mark.parametrize("seed,nf,n_select,min_bits", [(1, 12, 6, 0.0), (2, 16, 8, 0.5), (3, 10, 10, 0.0),
                                                        (4, 14, 5, 1.5)])
def test_restatement_against_extended_precision(seed, nf, n_select, min_bits):
    P, S, A, B, R = problem(seed, nf)
    feats = np.arange(nf)
    rho = np.argsort(np.argsort(-(S[:, 0] + S[:, 3]), kind="stable"), kind="stable")
    t = 2.0 ** (2 * min_bits)
    picks, info = sr.information_select(P, feats, rho, S, A, B, R, n_select, t)
    truth = Truth(P, A, B, R)
    worst = 0.0
    for r, d in enumerate(info):
        before = picks[:r]
        qt = {}
        for j in range(nf):
            if j in before:
                continue
            q_true = truth.q(before, j)
            err = abs(mpmath.mpf(float(d["qall"][j])) - q_true) / q_true
            worst = max(worst, float(err))
            assert err <= Q_RTOL, (r, j, float(err))
            qt[j] = q_true
        # where the restatement's winning margin exceeds the bound, the truth decides the same
        ok = [j for j in qt if qt[j] > t]
        if not d["stop"]:
            win, second = d["q"], d["second"]
            if not np.isfinite(second) or (win - second) > 4 * Q_RTOL * win:
                assert max(ok, key=lambda j: (qt[j], -rho[j])) == picks[r]
        elif all(abs(float(qt[j]) - t) > 4 * Q_RTOL * t for j in qt):
            assert not ok
    print("seed", seed, "worst relative q error", worst, "margins", sr.margins(info, t))
    assert len(picks) <= n_select


def iso_problem(p, R, b=1.0):
    """No correlation: P_xx = 0, P_xy = 0, P_yy = diag(p_j I3); B_j = b [I2 | 0]; S_j = (p_j b b + R) I exactly."""
    nf = len(p)
    n = NXV + 3 * nf
    P = np.zeros((n, n))
    for j in range(nf):
        for k in range(3):
            P[NXV + 3 * j + k, NXV + 3 * j + k] = p[j]
    A = np.ones((nf, 2, 7)) * 7.0  # multiplies zeros only
    B = np.zeros((nf, 2, 3))
    B[:, 0, 0] = b
    B[:, 1, 1] = b
    Rv = np.full(nf, R)
    s = np.array(p) * b * b + R
    S = np.stack([s, np.zeros(nf), np.zeros(nf), s], axis=1)
    return P, S, A, B, Rv


@pytest.mark.parametrize("n_select", [1, 2, 5, 12])
def test_without_correlation_the_information_order_is_the_trace_order(n_select):
    p = [3.0, 5.0, 5.0, 1.0, 8.0, 5.0, 0.5, 8.0, 2.0, 2.0, 9.0, 0.25]  # ties included
    P, S, A, B, R = iso_problem(p, R=2.0, b=4.0)
    feats, rho = sr.trace_candidates(S, np.ones(len(p), bool))
    picks, info = sr.information_select(P, feats, rho, S, A, B, R, n_select, 1.0)
    trace_sel = list(feats[np.argsort(rho)][:n_select])
    assert picks == trace_sel
    # no pick changes another candidate's C: every q is the unconditioned det(S_i) / R_i^2
    for d in info:
        live = ~np.isnan(d["qall"])
        assert (d["qall"][live] == ((S[:, 0] * S[:, 3]) / (R * R))[live]).all()


def test_a_duplicate_is_never_the_next_pick_after_its_twin():
    P, S, A, B, R = problem(7, 10, camera_share=0.3)
    # feature 1 duplicates feature 0: the same y, Jacobians and noise, and the largest innovation of all
    n = P.shape[0]
    y0, y1 = slice(NXV, NXV + 3), slice(NXV + 3, NXV + 6)
    P[y0, y0] *= 25.0
    P[y0, :NXV] *= 5.0
    P[:NXV, y0] *= 5.0
    P[NXV + 6:, y0] *= 5.0
    P[y0, NXV + 6:] *= 5.0
    P[y1, :] = P[y0, :]
    P[:, y1] = P[:, y0]
    A[1], B[1], R[1] = A[0], B[0], R[0]
    for j in range(10):
        H = np.zeros((2, n))
        H[:, :7] = A[j]
        H[:, NXV + 3 * j:NXV + 3 * j + 3] = B[j]
        Sj = H @ P @ H.T + R[j] * np.eye(2)
        S[j] = [Sj[0, 0], Sj[1, 0], Sj[1, 0], Sj[1, 1]]
    feats = np.arange(10)
    rho = np.argsort(np.argsort(-(S[:, 0] + S[:, 3]), kind="stable"), kind="stable")
    picks, info = sr.information_select(P, feats, rho, S, A, B, R, 10, 1.0)
    first = picks.index(0) if picks.index(0) < picks.index(1) else picks.index(1)
    assert set(picks[:1]) <= {0, 1} and first == 0  # the twins carry the most information
    assert picks[1] not in (0, 1)
    twin = 1 if picks[0] == 0 else 0
    # conditioned on its twin, the duplicate's innovation is its own noise plus the twin's: R (I + M (M + R)^-1) with
    # M = H P H^T, eigenvalues in [R, 2R), so q < 4 (< 1 bit), below every independent candidate here
    assert 1.0 <= info[1]["qall"][twin] < 4.0
    assert info[1]["q"] > 4.0


@pytest.mark.parametrize("min_bits", [0.0, 0.5, 1.0, 1.5])
def test_knife_edge_of_the_threshold(min_bits):
    t = 2.0 ** (2 * min_bits)
    assert t == math.ldexp(1.0, int(2 * min_bits))  # exact for 2 min_bits an integer
    # C = diag(c, c) with c c = t R^2 exactly, R = 1: one candidate at t, one a double above, one below
    c = math.sqrt(t) if min_bits in (0.0, 1.0) else None
    R = 1.0
    rows = []
    if c is not None:
        rows = [(c, c), (c, np.nextafter(c, 9.0)), (np.nextafter(c, 0.0), c)]
    else:  # t = 2 or 8: C00 = 1 or 2, C11 = 2 or 4
        a = 1.0 if min_bits == 0.5 else 2.0
        rows = [(a, t / a), (a, np.nextafter(t / a, 99.0)), (a, np.nextafter(t / a, 0.0))]
    S = np.array([[c0, 0.0, 0.0, c1] for c0, c1 in rows])
    nf = len(rows)
    P = np.zeros((NXV + 3 * nf, NXV + 3 * nf))
    A, B, Rv = np.zeros((nf, 2, 7)), np.zeros((nf, 2, 3)), np.full(nf, R)
    q = (S[:, 0] * S[:, 3]) / (Rv * Rv)
    assert q[0] == t and q[1] == np.nextafter(t, 99.0) and q[2] < t
    picks, info = sr.information_select(P, np.arange(nf), np.arange(nf), S, A, B, Rv, 3, t)
    assert picks == [1]
    assert info[-1]["stop"]


def test_degenerate_C_is_never_picked():
    nf = 5
    S = np.array([[np.nan, 0.0, 0.0, 50.0], [0.0, 0.0, 0.0, 50.0], [-1.0, 0.0, 0.0, -50.0], [4.0, 0.0, 0.0, 4.0],
                  [9.0, np.nan, np.nan, 9.0]])
    P = np.zeros((NXV + 3 * nf, NXV + 3 * nf))
    A, B, R = np.zeros((nf, 2, 7)), np.zeros((nf, 2, 3)), np.ones(nf)
    picks, info = sr.information_select(P, np.arange(nf), np.arange(nf), S, A, B, R, 5, 1.0)
    assert picks == [3]


def test_trace_candidates_cut_at_the_first_zero_trace():
    S = np.array([[1.0, 0, 0, 1.0], [0.0, 0, 0, 0.0], [3.0, 0, 0, 0.0], [1.0, 0, 0, 1.0], [5.0, 0, 0, 5.0]])
    feats, rho = sr.trace_candidates(S, np.array([True, True, True, False, True]))
    assert feats.tolist() == [0, 2, 4] and rho.tolist() == [2, 1, 0]
