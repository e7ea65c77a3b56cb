"""The iterated EKF update (include/sl2b200.h, sl2_set_stream_iterated; csrc/iterate.cu iterate_kernel) restated in
IEEE doubles, op for op in the kernel's order: the panel solves t = S^-1 nu, x_{i+1} = x0 + (H P0)^T t, the step
delta_i, the decision and the relinearisation with the prediction's model (rescue_ref.predict restates predict_feature;
its S part is not used here).  NumPy's elementwise float64 operations are correctly rounded and never fused, so a
vector operation over j is the kernel's per-thread operation for every j.

The factor half of a pass (upd_hp, upd_chol: G = [S | H P | nu], U, W_pp = U_pp^-T) runs on the tensor cores on the
device and is not restated: factor() forms the same quantities in FP64 with NumPy.  The module-level hooks
(pass_prior, correction, model_pose, count_after) are the places the broken copies of tests/test_iterate.py change."""
import math

import numpy as np

import rescue_ref
from update_truth import _chol_upper


def lin0(cam8, x, feats):
    """L_0: the prediction's h (K, 2), dh/dxp (K, 2, 7), dh/dy (K, 2, 3) and depth of the features at x."""
    hs, xs, ys, ds = [], [], [], []
    Pz = np.zeros((len(x), len(x)))
    for f in feats:
        pos = 13 + 3 * f
        pr = rescue_ref.predict(cam8, x[:7], x[pos:pos + 3], Pz, pos)
        hs.append(pr["h"]), xs.append(pr["dxp"]), ys.append(pr["dy"]), ds.append(pr["depth"])
    return np.array(hs), np.array(xs), np.array(ys), np.array(ds)


def dense_h(n, feats, Hxp, Hy):
    """The dense H (2K x n) of the rows."""
    H = np.zeros((2 * len(feats), n))
    for k, f in enumerate(feats):
        H[2 * k:2 * k + 2, :7] = Hxp[k]
        H[2 * k:2 * k + 2, 13 + 3 * f:16 + 3 * f] = Hy[k]
    return H


def factor(P, feats, L, z, Rvar):
    """What upd_hp and upd_chol leave for a pass at L = (h, Hxp, Hy): H P (m x n), U, the panel inverses W_pp
    (16 x 16 each, lower triangular, zero past a ragged panel), nu = z - h (FP64, upd_hp's subtraction)."""
    h, Hxp, Hy = L
    H = dense_h(P.shape[0], feats, Hxp, Hy)
    HP = H @ P
    S = HP @ H.T + np.diag(np.repeat(np.asarray(Rvar, np.float64), 2))
    U = _chol_upper(S)
    m = S.shape[0]
    W = []
    for p0 in range(0, m, 16):
        nb = min(16, m - p0)
        Wp = np.zeros((16, 16))
        Wp[:nb, :nb] = np.tril(np.linalg.inv(U[p0:p0 + nb, p0:p0 + nb]).T)
        W.append(Wp)
    nu = (np.asarray(z, np.float64) - h).reshape(-1)
    return HP, S, U, W, nu


def solve_panels(U, W, nu):
    """t = S^-1 nu as iterate_kernel forms it from U and the W_pp."""
    m = len(nu)
    v = [float(a) for a in nu]
    npan = (m + 15) // 16
    for p in range(npan):
        p0, nb = 16 * p, min(16, m - 16 * p)
        Wp = W[p]
        w = []
        for a in range(nb):
            acc = float(Wp[a, 0]) * v[p0]
            for b in range(1, nb):
                acc = acc + float(Wp[a, b]) * v[p0 + b]
            w.append(acc)
        v[p0:p0 + nb] = w
        for j in range(p0 + nb, m):
            r = v[j]
            for a in range(nb):
                r = r - float(U[p0 + a, j]) * v[p0 + a]
            v[j] = r
    for p in reversed(range(npan)):
        p0, nb = 16 * p, min(16, m - 16 * p)
        Wp = W[p]
        t = []
        for a in range(nb):
            acc = float(Wp[0, a]) * v[p0]
            for b in range(1, nb):
                acc = acc + float(Wp[b, a]) * v[p0 + b]
            t.append(acc)
        v[p0:p0 + nb] = t
        for j in range(p0):
            r = v[j]
            for a in range(nb):
                r = r - float(U[j, p0 + a]) * v[p0 + a]
            v[j] = r
    return np.array(v)


def x_next(x0, HP, t):
    acc = HP[0] * t[0]
    for r in range(1, len(t)):
        acc = acc + HP[r] * t[r]
    return x0 + acc


def step_delta(xn, xo, P0):
    if not np.isfinite(xn).all():
        return math.nan
    d = np.diag(P0)
    on = d > 0
    return float(np.max(np.abs(xn - xo)[on] / np.sqrt(d[on]), initial=0.0))


# ---- hooks (the broken copies replace these) -------------------------------------------------------------------------
def pass_prior(P0, P_after):
    """The covariance every pass forms S and H P from: P0."""
    return P0


def correction(h, Hxp, Hy, dx, dy):
    """h_eff = h + (Hxp dx + Hy dy), the products summed left to right from the first."""
    out = np.empty(2)
    for r in range(2):
        acc = Hxp[r, 0] * dx[0]
        for c in range(1, 7):
            acc = acc + Hxp[r, c] * dx[c]
        for c in range(3):
            acc = acc + Hy[r, c] * dy[c]
        out[r] = h[r] + acc
    return out


def model_pose(xn):
    """The pose the model reads: x_{i+1}[0:7], q as it is (quirk Q1)."""
    return xn[:7]


def count_after(i):
    """iterations after a successful relinearisation in pass i."""
    return i + 1


def relinearise(cam8, x0, xn, feats):
    """(valid, (h_eff, Hxp, Hy)) of the rows at x_{i+1}."""
    hs, xs, ys = [], [], []
    ok = bool(np.isfinite(xn).all())
    Pz = np.zeros((len(xn), len(xn)))
    xp = model_pose(xn)
    dx = x0[:7] - xn[:7]
    for f in feats:
        pos = 13 + 3 * f
        pr = rescue_ref.predict(cam8, xp, xn[pos:pos + 3], Pz, pos)
        he = correction(pr["h"], pr["dxp"], pr["dy"], dx, x0[pos:pos + 3] - xn[pos:pos + 3])
        ok = ok and pr["depth"] > 0 and np.isfinite(he).all() and np.isfinite(pr["dxp"]).all() and \
            np.isfinite(pr["dy"]).all()
        hs.append(he), xs.append(pr["dxp"]), ys.append(pr["dy"])
    return ok, (np.array(hs), np.array(xs), np.array(ys))


def iterated(cam8, x0, P0, feats, z, Rvar, N, tol, L0=None):
    """The iteration of one stream from x0, P0 with the rows feats (rank order), matches z (K, 2) and R = Rvar I:
    -> dict(L = the final update's (h, Hxp, Hy), iterations, status, delta (last), xs = [x_1, x_2, ...])."""
    x0, P0 = np.asarray(x0, np.float64), np.asarray(P0, np.float64)
    L = L0 if L0 is not None else lin0(cam8, x0, feats)[:3]
    out = dict(iterations=0, status=0, delta=0.0, xs=[])
    if N == 0 or len(feats) == 0:
        return dict(out, L=L)
    xi, P_after = x0, P0
    for i in range(N):
        HP, S, U, W, nu = factor(pass_prior(P0, P_after), feats, L, z, Rvar)
        t = solve_panels(U, W, nu)
        xn = x_next(x0, HP, t)
        P_after = P0 - HP.T @ np.linalg.solve(S, HP)
        out["xs"].append(xn)
        d = step_delta(xn, xi, P0)
        out["delta"] = d
        if d <= tol:
            out["status"] = 1
            return dict(out, L=L)
        ok, Ln = relinearise(cam8, x0, xn, feats)
        if not ok:
            out["status"] = 3
            return dict(out, L=L)
        L, xi = Ln, xn
        out["iterations"] = count_after(i)
    out["status"] = 2
    return dict(out, L=L)
