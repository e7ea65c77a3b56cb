"""The iterated EKF update from its definition (include/sl2b200.h, sl2_set_stream_iterated), in extended precision
(np.longdouble; the same code in mpmath at 50 digits checks it), reusing none of the device's operation order:

  pass i      H_i dense from L_i, S_i = H_i P0 H_i^T + R, t = S_i^-1 nu_i (Cholesky), x_{i+1} = x0 + (H_i P0)^T t
  step        delta_i = max over P0_jj > 0 of |x_{i+1,j} - x_{i,j}| / sqrt(P0_jj)
  relinearise the model (rescue_truth.model) at x_{i+1}; h_eff = h + Hxp (x0[0:7] - x_{i+1}[0:7]) + Hy (y0 - y_{i+1})

final_truth() is the final update from x0, P0 at a linearisation (update_truth.truth_update).  gauss_newton() runs the
iteration until the step stops changing in extended precision: the minimiser of the posterior cost
J(x) = |x - x0|^2_{P0^-1} + sum_k |z_k - h_k(x)|^2 / var_k, which cost() evaluates (Bell & Cathey, IEEE TAC 1993)."""
import numpy as np

import update_truth as ut
from rescue_truth import Ext, _chol_solve, model


def _dense(ar, n, feats, Hxp, Hy):
    H = ar.conv(np.zeros((2 * len(feats), n)))
    for k, f in enumerate(feats):
        for r in range(2):
            for c in range(7):
                H[2 * k + r, c] = Hxp[k][r][c]
            for c in range(3):
                H[2 * k + r, 13 + 3 * f + c] = Hy[k][r][c]
    return H


def iterated_truth(ar, cam8, x0, P0, feats, z, Rvar, N, tol, L0):
    """L0 = the prediction's (h, Hxp, Hy) as FP64 arrays (the device's and the restatement's input).  -> dict(L (final,
    in ar), iterations, status, deltas, xs)."""
    x0a, P0a = ar.conv(x0), ar.conv(P0)
    n = len(x0a)
    L = tuple(ar.conv(a) for a in L0)
    za, Ra = ar.conv(z), ar.conv(np.repeat(np.asarray(Rvar, np.float64), 2))
    out = dict(iterations=0, status=0, deltas=[], xs=[])
    if N == 0 or len(feats) == 0:
        return dict(out, L=L)
    xi = x0a
    for i in range(N):
        h, Hxp, Hy = L
        H = _dense(ar, n, feats, Hxp, Hy)
        HP = H.dot(P0a)
        S = HP.dot(H.T)
        for r in range(len(Ra)):
            S[r, r] = S[r, r] + Ra[r]
        nu = za.reshape(-1) - np.asarray(h).reshape(-1)
        t = _chol_solve(ar, S, nu)
        xn = x0a + HP.T.dot(t)
        out["xs"].append(xn)
        d = max((abs(xn[j] - xi[j]) / ar.sqrt(P0a[j, j]) for j in range(n) if P0a[j, j] > 0), default=0 * xn[0])
        out["deltas"].append(d)
        if d <= tol:
            out["status"] = 1
            return dict(out, L=L)
        hs, xs, ys, ok = [], [], [], True
        for f in feats:
            pos = 13 + 3 * f
            hm, Hxpm, Hym, _, depth = model(ar, cam8, xn[:7], xn[pos:pos + 3])
            ok = ok and depth > 0
            dx = [x0a[c] - xn[c] for c in range(7)]
            dy = [x0a[pos + c] - xn[pos + c] for c in range(3)]
            hs.append([hm[r] + sum(Hxpm[r][c] * dx[c] for c in range(7)) + sum(Hym[r][c] * dy[c] for c in range(3))
                       for r in range(2)])
            xs.append(Hxpm), ys.append(Hym)
        if not ok:
            out["status"] = 3
            return dict(out, L=L)
        L = (np.array(hs), np.array(xs), np.array(ys))
        xi = xn
        out["iterations"] = i + 1
    out["status"] = 2
    return dict(out, L=L)


def final_truth(x0, P0, feats, L, z, Rvar):
    """The final update at L from x0, P0 (with upd_finish), in np.longdouble on the FP64-rounded tables."""
    h, Hxp, Hy = (np.asarray(np.asarray(a, np.longdouble), np.float64) for a in L)
    K = len(feats)
    Hxv = np.zeros((2 * K, 13))
    Hxv[:, :7] = Hxp.reshape(2 * K, 7)
    R = [np.eye(2) * v for v in Rvar]
    nu = (np.asarray(z, np.float64) - h).reshape(-1)
    return ut.truth_update(x0, P0, feats, Hxv, Hy.reshape(2 * K, 3), R, nu)


def gauss_newton(cam8, x0, P0, feats, z, Rvar, L0, steps=40):
    """The minimiser of J (np.longdouble): the iteration run until its step is below 1e-17 prior sigmas."""
    r = iterated_truth(Ext, cam8, x0, P0, feats, z, Rvar, steps, 1e-17, L0)
    assert r["status"] == 1, r["status"]
    return r["xs"][-1]


def cost(cam8, x0, P0, feats, z, Rvar, x):
    """J(x) in np.longdouble."""
    x0a, P0a, xa = Ext.conv(x0), Ext.conv(P0), Ext.conv(x)
    e = xa - x0a
    J = e.dot(_chol_solve(Ext, P0a, e))
    for k, f in enumerate(feats):
        pos = 13 + 3 * f
        h = model(Ext, cam8, xa[:7], xa[pos:pos + 3])[0]
        J = J + sum((Ext.conv(z[k][r]) - h[r]) ** 2 for r in range(2)) / Ext.conv(Rvar[k])
    return J
