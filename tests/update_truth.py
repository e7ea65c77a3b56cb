"""An extended-precision Kalman update to hold the EKF update (update.cu) to, an FP64 Cholesky update as the yardstick
of what a backward-stable FP64 update achieves, and measurement sets whose innovation covariance S has a designed
condition number.

The device update is  S = H P H^T + R = U^T U,  Y = U^-T [H P | nu],  P -= Y^T Y,  x += Y^T w,  then upd_finish:
P <- J P J^T with J = dxvnorm_by_dxv of the new x, and P <- (P + P^T) / 2 (x stays un-normalised, quirk Q1).
truth_update runs that sequence in np.longdouble (64-bit mantissa) on exactly the FP64 arrays the device receives;
chol64_update runs it in FP64 with LAPACK.  oracle_update is the CPU oracle (kalman.cpp as written: explicit S^-1,
then P - K S K^T), which stops being a reference once S is poorly conditioned.

H is never dense here: a measurement row has 13 dense columns (dh/dxv) and 3 structural ones (dh/dy of its feature),
like the rows of sl2_ekf_update.  Helpers in this file use NumPy, SciPy, mpmath and the oracle only."""
import collections
import math

import mpmath
import numpy as np
import scipy.linalg as sla

from oracle import pyoracle as oracle

LD = np.longdouble
EPS = float(np.finfo(np.float64).eps)
EPS_LD = float(np.finfo(LD).eps)
MECHANISMS = ("A", "B", "C", "D")
# mechanism A builds this target with Pyy exactly 0 (known features); every other target with a tiny Pyy
A_ZERO_PYY_COND = 1e6
RHO_MAX = 1.0 - 1e-9      # mechanism D: largest |correlation| inside an R block

Update = collections.namedtuple("Update", "x P cond nis logdet")
Case = collections.namedtuple("Case", "x P feats Hxv Hy R nu mechanism target")


# ---- the update in any precision ------------------------------------------------------------------------------------
def _cols(feats):
    """(m, 3) state columns of each measurement row's dh/dy block."""
    return 13 + 3 * np.repeat(np.asarray(feats, np.int64), 2)[:, None] + np.arange(3)


def _rfull(R, dtype):
    K = len(R)
    out = np.zeros((2 * K, 2 * K), dtype)
    for k in range(K):
        out[2 * k:2 * k + 2, 2 * k:2 * k + 2] = np.asarray(R[k], dtype)
    return out


def form_hp_s(P, feats, Hxv, Hy, R):
    """H P (m x n) and S = (H P) H^T + R (full 2x2 R blocks) in P's dtype, from H's structure."""
    dt = P.dtype
    Hx, Hc, cols = np.asarray(Hxv, dt), np.asarray(Hy, dt), _cols(feats)
    HP = Hx @ P[:13, :] + np.einsum("ic,icj->ij", Hc, P[cols, :])
    S = HP[:, :13] @ Hx.T + np.einsum("jc,ijc->ij", Hc, HP[:, cols]) + _rfull(R, dt)
    return HP, S


def _chol_upper(A):
    """Upper Cholesky factor (U^T U = A) in A's dtype; LinAlgError on a non-positive pivot."""
    m = A.shape[0]
    U = np.zeros_like(A)
    for k in range(m):
        r = A[k, k:] - U[:k, k] @ U[:k, k:]
        if not r[0] > 0:
            raise np.linalg.LinAlgError("pivot %d of S is not positive" % k)
        d = np.sqrt(r[0])
        U[k, k] = d
        U[k, k + 1:] = r[1:] / d
    return U


def _forward(U, B):
    """U^-T B (forward substitution) in the common dtype."""
    Y = np.zeros_like(B)
    for k in range(U.shape[0]):
        Y[k] = (B[k] - U[:k, k] @ Y[:k]) / U[k, k]
    return Y


def _cond(S, U):
    """2-norm condition number of S = U^T U: largest eigenvalue of S times largest of S^-1 = Z^T Z, Z = U^-T (both
    formed in U's precision, their largest eigenvalues taken after rounding to FP64: accurate to a few ulps)."""
    Z = _forward(U, np.eye(U.shape[0], dtype=U.dtype))
    lmax = np.linalg.eigvalsh(np.asarray(S, np.float64))[-1]
    lmax_inv = np.linalg.eigvalsh(np.asarray(Z.T @ Z, np.float64))[-1]
    return float(lmax * lmax_inv)


def kalman_ld(x, P, feats, Hxv, Hy, R, nu):
    """The Kalman update before upd_finish, in np.longdouble: (x+, P+, cond(S), NIS, log det S)."""
    xl, Pl = np.asarray(x, LD), np.asarray(P, LD)
    HP, S = form_hp_s(Pl, feats, Hxv, Hy, R)
    U = _chol_upper(S)
    Y = _forward(U, np.concatenate([HP, np.asarray(nu, LD)[:, None]], axis=1))
    Yp, w = Y[:, :-1], Y[:, -1]
    return Update(xl + Yp.T @ w, Pl - Yp.T @ Yp, _cond(S, U), float(w @ w), float(2 * np.log(np.diag(U)).sum()))


def finish(x, P):
    """upd_finish's normalisation and symmetrisation in P's dtype: J = dxvnorm_by_dxv of x rounded to FP64,
    P <- J P J^T, P <- (P + P^T) / 2; x is left as it is (quirk Q1)."""
    J = np.asarray(oracle.dxvnorm_by_dxv(np.asarray(x[:13], np.float64)), P.dtype)
    P = P.copy()
    P[:13, :] = J @ P[:13, :]
    P[:, :13] = P[:, :13] @ J.T
    return (P + P.T) / 2


def truth_update(x, P, feats, Hxv, Hy, R, nu):
    """The update and upd_finish in np.longdouble on the FP64 inputs; x and P rounded to FP64, cond(S), NIS, log det S."""
    k = kalman_ld(x, P, feats, Hxv, Hy, R, nu)
    xf = np.asarray(k.x, np.float64)
    return Update(xf, np.asarray(finish(xf, k.P), np.float64), k.cond, k.nis, k.logdet)


def chol64_update(x, P, feats, Hxv, Hy, R, nu):
    """The same sequence in plain FP64 with LAPACK (cho_factor / solve_triangular): the yardstick."""
    x, P = np.asarray(x, np.float64), np.asarray(P, np.float64)
    HP, S = form_hp_s(P, feats, Hxv, Hy, R)
    U = sla.cho_factor(S, lower=False)[0]
    U = np.triu(U)
    Y = sla.solve_triangular(U, np.concatenate([HP, np.asarray(nu, np.float64)[:, None]], axis=1), trans="T")
    Yp, w = Y[:, :-1], Y[:, -1]
    xn = x + Yp.T @ w
    return Update(xn, finish(xn, P - Yp.T @ Yp), float(np.linalg.cond(S)), float(w @ w),
                  float(2 * np.log(np.diag(U)).sum()))


def dense_rows(n, feats, Hxv, Hy, R):
    """The dense H (m x n) and R (m x m) of kalman.cpp."""
    m = len(Hxv)
    H = np.zeros((m, n))
    H[:, :13] = Hxv
    np.put_along_axis(H, _cols(feats), np.asarray(Hy, np.float64), axis=1)
    return H, _rfull(R, np.float64)


def oracle_update(x, P, feats, Hxv, Hy, R, nu):
    """The CPU oracle's update (explicit S^-1), normalised and symmetrised like upd_finish: (x, P)."""
    H, Rf = dense_rows(len(x), feats, Hxv, Hy, R)
    xo, Po = oracle.kalman_update_dense(x, P, H, Rf, nu)
    return xo, finish(xo, np.asarray(Po, np.float64))


def update_err(xg, Pg, xt, Pt):
    """(state error, covariance error) of (xg, Pg) against the truth (xt, Pt): |dP_ij| / sqrt(Pt_ii Pt_jj) and
    |dx_i| / max(|xt_i|, sigma_i) (gpu_util.state_err's measure).  An entry whose truth scale is exactly 0 has to match
    exactly: it counts as 0 when it does and as inf when it does not."""
    xg, Pg, xt, Pt = (np.asarray(a, np.float64) for a in (xg, Pg, xt, Pt))
    d = np.sqrt(np.abs(np.diag(Pt)))

    def rel(diff, scale):
        with np.errstate(divide="ignore", invalid="ignore"):
            e = np.where(scale > 0, diff / np.where(scale > 0, scale, 1.0), np.where(diff == 0, 0.0, np.inf))
        return float(e.max()) if e.size else 0.0

    return rel(np.abs(xg - xt), np.maximum(np.abs(xt), d)), rel(np.abs(Pg - Pt), d[:, None] * d[None, :])


# ---- the same update at 50 digits (small cases: checks the longdouble truth itself) ---------------------------------
def kalman_mp(x, P, feats, Hxv, Hy, R, nu, dps=50):
    """kalman_ld's sequence in mpmath at `dps` digits on the same FP64 inputs: (x+, P+) as mpmath matrices."""
    with mpmath.workdps(dps):
        n, m = len(x), len(nu)
        H, Rf = dense_rows(n, feats, Hxv, Hy, R)
        nz = [np.nonzero(H[i])[0] for i in range(m)]
        Pm = mpmath.matrix(P.tolist())
        HP = mpmath.matrix(m, n)
        for i in range(m):
            for j in range(n):
                HP[i, j] = mpmath.fsum(mpmath.mpf(H[i, k]) * Pm[k, j] for k in nz[i])
        S = mpmath.matrix(m, m)
        for i in range(m):
            for j in range(m):
                S[i, j] = mpmath.fsum(HP[i, k] * mpmath.mpf(H[j, k]) for k in nz[j]) + mpmath.mpf(Rf[i, j])
        L = mpmath.cholesky(S)                       # lower, L L^T = S
        B = mpmath.matrix(m, n + 1)
        for i in range(m):
            for j in range(n):
                B[i, j] = HP[i, j]
            B[i, n] = mpmath.mpf(nu[i])
        Y = _mp_forward(L, B)
        xo = mpmath.matrix([mpmath.mpf(v) for v in x])
        Po = Pm.copy()
        for i in range(n):
            xo[i] += mpmath.fsum(Y[k, i] * Y[k, n] for k in range(m))
            for j in range(n):
                Po[i, j] -= mpmath.fsum(Y[k, i] * Y[k, j] for k in range(m))
        return xo, Po


def finish_mp(x, Po, dps=50):
    """finish() at `dps` digits on an mpmath P: J = dxvnorm_by_dxv of x (FP64), P <- J P J^T, P <- (P + P^T) / 2."""
    with mpmath.workdps(dps):
        J = mpmath.matrix(np.asarray(oracle.dxvnorm_by_dxv(np.asarray(x[:13], np.float64)), np.float64).tolist())
        n = Po.rows
        T = Po.copy()
        for i in range(13):
            for j in range(n):
                T[i, j] = mpmath.fsum(J[i, k] * Po[k, j] for k in range(13))
        Q = T.copy()
        for i in range(n):
            for j in range(13):
                Q[i, j] = mpmath.fsum(T[i, k] * J[j, k] for k in range(13))
        return (Q + Q.T) / 2


def _mp_forward(L, B):
    m, c = B.rows, B.cols
    Y = mpmath.matrix(m, c)
    for i in range(m):
        for j in range(c):
            Y[i, j] = (B[i, j] - mpmath.fsum(L[i, k] * Y[k, j] for k in range(i))) / L[i, i]
    return Y


def _mpf(v):
    """An np.longdouble as an mpmath number, exactly (its 64-bit mantissa is the sum of two doubles)."""
    hi = float(v)
    return mpmath.mpf(hi) + mpmath.mpf(float(LD(v) - LD(hi)))


def mp_err(k, xo, Po, dps=50):
    """update_err's measure of the longdouble update k against the mpmath one, evaluated at mpmath precision."""
    with mpmath.workdps(dps):
        return _mp_err(k, xo, Po)


def _mp_err(k, xo, Po):
    n = len(k.x)
    d = [mpmath.sqrt(abs(Po[i, i])) for i in range(n)]
    eP = mpmath.mpf(0)
    for i in range(n):
        for j in range(n):
            s = d[i] * d[j]
            diff = abs(_mpf(k.P[i, j]) - Po[i, j])
            eP = max(eP, diff / s if s > 0 else (0 if diff == 0 else mpmath.inf))
    ex = max(abs(_mpf(k.x[i]) - xo[i]) / max(abs(xo[i]), d[i]) for i in range(n))
    return float(ex), float(eP)


# ---- measurement sets with a designed cond(S) -----------------------------------------------------------------------
def _state(rng, nf):
    """A camera near the origin with a quaternion off unit length by ~1e-3 (as an update leaves it) and nf features
    a few metres in front of it."""
    x = np.zeros(13 + 3 * nf)
    x[0:3] = rng.normal(0, 0.3, 3)
    q = rng.normal(0, 0.3, 4)
    q[0] += 1.0
    x[3:7] = q / np.linalg.norm(q) * (1.0 + 1e-3 * rng.standard_normal())
    x[7:13] = rng.normal(0, 0.5, 6)
    x[13:] = (rng.normal(0, 1, (nf, 3)) + [0.0, 0.0, 3.0]).ravel()
    return x


def _factor(rng, n, sigma=1e-3):
    """M (n x 2n) with P = M M^T a well-conditioned covariance, standard deviations around `sigma`."""
    s = sigma * np.exp(rng.uniform(-0.5, 0.5, n))
    return s[:, None] * rng.standard_normal((n, 2 * n)) / math.sqrt(2 * n)


def _rows(rng, K):
    """Measurement rows like the staged API's: 13 dense dh/dxv columns (the dh/dxp ones large), 3 dh/dy columns."""
    Hxv = rng.standard_normal((2 * K, 13)) * 60
    Hxv[:, 7:] /= 3
    return Hxv, rng.standard_normal((2 * K, 3)) * 300


def _sym(P):
    return (P + P.T) / 2


def _cond64(S):
    e = np.linalg.eigvalsh(S)
    return e[-1] / e[0] if e[0] > 0 else np.inf


def _tune(cond_of, target, lo, hi, iters=80):
    """p in [lo, hi] with cond_of(p) within 5% of target (cond_of increasing in p), by bisection."""
    for _ in range(iters):
        p = 0.5 * (lo + hi)
        c = cond_of(p)
        if abs(math.log(c / target)) < 0.05:
            return p
        lo, hi = (p, hi) if c < target else (lo, p)
    raise AssertionError("cond(S) = %g not reachable near %g (p in [%g, %g])" % (c, target, lo, hi))


def _idx(feats):
    return np.r_[np.arange(13), _cols(feats)[::2].ravel()]


def _compact(P_or_idx_block, feats, Hxv, Hy, R):
    """S from the rows / columns of P the measurements touch (P_or_idx_block = P[idx, idx], idx = _idx(feats))."""
    K = len(feats)
    return form_hp_s(P_or_idx_block, np.arange(K), Hxv, Hy, R)[1]


def inflate_camera(rng, P, feats, Hxv, Hy, R, target_cond, F=None):
    """P with s v v^T added to its camera block (v a random unit direction; with F, F v, as a prediction by F carries
    it) and s such that S = H P H^T + R of the rows has condition number target_cond: a camera whose uncertainty has
    grown along one direction, after a long prediction or a lost track."""
    v = rng.standard_normal(13)
    v /= np.linalg.norm(v)
    if F is not None:
        v = F @ v
    idx = _idx(feats)
    S0 = _compact(P[np.ix_(idx, idx)], feats, Hxv, Hy, R)
    g = np.asarray(Hxv) @ v
    p = _tune(lambda p: _cond64(S0 + 10 ** p * np.outer(g, g)), target_cond, -8, 24)
    P = P.copy()
    P[:13, :13] += 10 ** p * np.outer(v, v)
    return _sym(P)


def conditioned_case(rng, nf, K, mechanism, target_cond):
    """x, P and sl2_ekf_update rows of K measured features of an nf-feature map (measurement order shuffled against
    the feature order) whose S = H P H^T + R has condition number target_cond, reached by one mechanism:
      A  known features (Pxy = 0, Pyy tiny, exactly 0 at A_ZERO_PYY_COND), R = 1 px^2, and a camera whose
         uncertainty has grown along one direction: Pxx = A0 + s v v^T, s raised until cond(S) reaches the target;
      B  near-duplicate features: consecutive measured features in pairs at almost the same y with identical H rows
         and Pyy blocks correlated to 1 - delta (an odd one out has its two rows nearly coincide), R = delta a I
         with a the rows' typical H P H^T; cond(S) ~ 1 / delta;
      C  badly scaled but well-conditioned: every row of H, its R and nu scaled by t_i, log t_i evenly spread, so that
         S = T S0 T has its pivots spread over the decades of the target while T^-1 S T^-1 stays well conditioned;
      D  near-singular R blocks: R_k = [[a^2, rho a b], [rho a b, b^2]] with 1 - |rho| >= 1 - RHO_MAX and, past what
         rho alone reaches, a / b > 1; H scaled so that H P H^T is of the size of R's small eigenvalue.
    nu ~ N(0, S).  The case's FP64 S is checked to factor (LAPACK): every case is positive definite in FP64."""
    assert mechanism in MECHANISMS and 1 <= K <= nf
    n, m = 13 + 3 * nf, 2 * K
    x = _state(rng, nf)
    feats = rng.permutation(nf)[:K].astype(np.int32)
    idx = _idx(feats)
    M = _factor(rng, n)
    Hxv, Hy = _rows(rng, K)
    R = np.tile(np.eye(2), (K, 1, 1))
    if mechanism == "A":
        P = _sym(M @ M.T)
        P[:13, :13] *= 1e-4
        P[:13, 13:] = P[13:, :13] = 0.0
        P[13:, 13:] *= 0.0 if target_cond == A_ZERO_PYY_COND else 1e-8
        P = inflate_camera(rng, P, feats, Hxv, Hy, R, target_cond)
    elif mechanism == "B":
        pairs = [(feats[i], feats[i + 1]) for i in range(0, K - 1, 2)]
        solo = K % 2 == 1
        for a, b in pairs:                              # same point: same H rows, y a micrometre apart
            ra, rb = 2 * list(feats).index(a), 2 * list(feats).index(b)
            Hxv[rb:rb + 2], Hy[rb:rb + 2] = Hxv[ra:ra + 2], Hy[ra:ra + 2]
            x[13 + 3 * b:16 + 3 * b] = x[13 + 3 * a:16 + 3 * a] + 1e-6 * rng.standard_normal(3)
        # P = M' M'^T with the rows of a pair's second feature b = (1 - delta) (rows of a) + sqrt(2 delta - delta^2)
        # (fresh noise of covariance Pyy_a in columns of its own): Pyy_b = Pyy_a, Pyy_ab = (1 - delta) Pyy_a
        q = M.shape[1]
        Mx = np.concatenate([M, np.zeros((n, 3 * len(pairs)))], axis=1)
        second = []
        for i, (a, b) in enumerate(pairs):
            Ma = M[13 + 3 * a:16 + 3 * a]
            second.append((b, Ma, i, np.linalg.cholesky(Ma @ Ma.T)))
        dH = rng.standard_normal(16)

        def build(p, full):
            d = 10.0 ** -p
            rows, sub = (np.arange(n), idx) if full else (idx, np.arange(len(idx)))
            Mb = Mx[rows].copy()
            pos = {r: k for k, r in enumerate(rows)}
            for b, Ma, i, La in second:
                for c in range(3):
                    k = pos[13 + 3 * b + c]
                    Mb[k, :q] = (1 - d) * Ma[c]
                    Mb[k, q + 3 * i:q + 3 * i + 3] = math.sqrt(2 * d - d * d) * La[c]
            H1, H2 = Hxv.copy(), Hy.copy()
            if solo:                                    # the odd feature out: its second row ~ its first
                H1[m - 1] = H1[m - 2] + math.sqrt(d) * 60 * dH[:13]
                H2[m - 1] = H2[m - 2] + math.sqrt(d) * 300 * dH[13:]
            Pb = _sym(Mb @ Mb.T)
            S = _compact(Pb[np.ix_(sub, sub)], feats, H1, H2, 0 * R)
            return Pb, H1, H2, np.tile(d * float(np.mean(np.diag(S))) * np.eye(2), (K, 1, 1)), S

        def cond_of(p):
            _, _, _, Rb, S = build(p, False)
            return _cond64(S + _rfull(Rb, np.float64))

        p = _tune(cond_of, target_cond, 0, 16)
        P, Hxv, Hy, R, _ = build(p, True)
    elif mechanism == "C":
        P = _sym(M @ M.T)
        u = rng.permutation(np.linspace(-0.5, 0.5, m))
        S0 = _compact(P[np.ix_(idx, idx)], feats, Hxv, Hy, R)
        p = _tune(lambda p: _cond64(S0 * np.outer(10 ** (p * u), 10 ** (p * u))), target_cond, 0, 16)
        t = 10 ** (p * u)
        Hxv, Hy = Hxv * t[:, None], Hy * t[:, None]
        R = np.array([np.diag(t[2 * k:2 * k + 2] ** 2) for k in range(K)])
    else:
        P = _sym(M @ M.T)
        sign = rng.choice([-1.0, 1.0], K)
        scale = np.exp(rng.uniform(-0.3, 0.3, K))
        swap = rng.random(K) < 0.5
        S0 = _compact(P[np.ix_(idx, idx)], feats, Hxv, Hy, 0 * R)
        h0 = float(np.mean(np.diag(S0)))

        def blocks(p):
            d = max(1.0 - RHO_MAX, 10.0 ** -p)
            kap = max(1.0, 10.0 ** p * d)
            out = np.zeros((K, 2, 2))
            for k in range(K):
                a2, b2 = scale[k] * kap, scale[k]
                if swap[k]:
                    a2, b2 = b2, a2
                rab = sign[k] * (1 - d) * math.sqrt(a2 * b2)
                out[k] = [[a2, rab], [rab, b2]]
            lmin = min(np.linalg.eigvalsh(b)[0] for b in out)
            return out, lmin / h0

        def cond_of(p):
            Rb, eta2 = blocks(p)
            return _cond64(eta2 * S0 + _rfull(Rb, np.float64))

        p = _tune(cond_of, target_cond, 0, 16)
        R, eta2 = blocks(p)
        Hxv, Hy = Hxv * math.sqrt(eta2), Hy * math.sqrt(eta2)
    P = _sym(np.asarray(P, np.float64))
    _, S = form_hp_s(P, feats, Hxv, Hy, R)
    U = sla.cho_factor(S, lower=False)[0]              # positive definite in FP64, or this raises
    nu = np.triu(U).T @ rng.standard_normal(m)
    return Case(x, P, feats, np.ascontiguousarray(Hxv), np.ascontiguousarray(Hy), np.ascontiguousarray(R), nu,
                mechanism, target_cond)


def rows_of(case):
    """The sl2_ekf_update arguments of a case: feat_index, H_xv, H_y, R, nu."""
    return case.feats, case.Hxv, case.Hy, case.R, case.nu


def fresh_nu(rng, P, feats, Hxv, Hy, R):
    """An innovation drawn from N(0, S) of the rows."""
    _, S = form_hp_s(np.asarray(P, np.float64), feats, Hxv, Hy, R)
    return np.triu(sla.cho_factor(S, lower=False)[0]).T @ rng.standard_normal(len(Hxv))


# ---- the sweep: (capacity, nf, K) x mechanism x cond(S) ---------------------------------------------------------------
# m = 2 K covers m mod 16 = 0, 2, 8 and 14 (the ragged last 16-row panel of upd_chol / upd_solve)
SWEEP_SHAPES = [(128, 1, 1), (128, 9, 9), (128, 24, 24), (128, 50, 17), (128, 36, 20), (128, 80, 63), (128, 97, 97),
                (128, 128, 128), (256, 256, 128)]
SWEEP_CONDS = (1e2, 1e4, 1e6, 1e8, 1e10, 1e12)


def case_rng(nf, K, mechanism, target_cond):
    return np.random.default_rng([nf, K, MECHANISMS.index(mechanism), int(round(math.log10(target_cond)))])


def sweep_case(nf, K, mechanism, target_cond):
    return conditioned_case(case_rng(nf, K, mechanism, target_cond), nf, K, mechanism, target_cond)


# ---- the rows of a tracking step -------------------------------------------------------------------------------------
def slam_rows(slam, cam8):
    """The update's inputs (x, P, feats, Hxv, Hy, R, nu) of an oracle Slam after predict(), select() and
    measure(frame): the found features in selection order, their rows from the measurement model at the predicted
    state (dh/dxv = [dh/dxp | 0], R = var I) and nu = z - h."""
    x, P = slam.get_state()
    f = slam.features()
    meas = [i for i in np.argsort(f["select_rank"], kind="stable") if f["select_rank"][i] >= 0 and f["flags"][i] & 2]
    K = len(meas)
    Hxv, Hy, R, nu = np.zeros((2 * K, 13)), np.zeros((2 * K, 3)), np.zeros((K, 2, 2)), np.zeros(2 * K)
    for k, i in enumerate(meas):
        c = slice(13 + 3 * i, 16 + 3 * i)
        h, dxv, dy, Ri, _ = oracle.predict_feature(cam8, x[:13], x[c], P[:13, :13], P[:13, c], P[c, c])
        Hxv[2 * k:2 * k + 2], Hy[2 * k:2 * k + 2], R[k] = dxv, dy, Ri
        nu[2 * k:2 * k + 2] = f["z"][i] - h
    return x, P, np.array(meas, np.int32), Hxv, Hy, R, nu
