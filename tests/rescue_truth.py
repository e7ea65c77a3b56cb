"""The consensus rescue's gate from its definition, in extended precision (np.longdouble; the same code in mpmath at 50
digits checks it): none of the device's operation order is reused.

  update 1    the dense Kalman update of the prior x, P with the inliers: H_i = the model's Jacobian at x, R_i =
              var_i I, nu_i = z_i - h_i(x); S = H P H^T + R, K = P H^T S^-1, x' = x + K nu, P' = P - K S K^T, then the
              update's normalisation P' <- J P' J^T (J = the reference's dqnorm/dq, quirk Q2 of csrc/update.cu) and
              symmetrisation of P'.
  gate        for every rejected j: h_j(x'), S'_j = H_j(x') P' H_j(x')^T + R_j(x'), q_j = nu'^T S'_j^-1 nu' with
              nu' = z_j - h_j(x'); rescued iff the camera-frame depth at x' is > 0 and q_j <= chi2.

The model (camera.cpp, full_feature_model.cpp, feature_model.cpp): z = RRW (y - r) with RRW the rotation of q^-1;
(uc, vc) = (-fku z0 / z2, -fkv z1 / z2), f = sqrt(1 + 2 kd1 (uc^2 + vc^2)), h = (uc / f + u0, vc / f + v0);
var = (sd (1 + |h - c| / |c|))^2 with c = (u0, v0); dz/dq = d(R(qbar) a)/dqbar diag(1, -1, -1, -1) at qbar = q^-1.

q_band(...) bounds how far a double-precision evaluation of the same q can be from the truth, from the operation
count: the longest chain of the double computation (update 1: n m1 + m1^3 products and sums; the prediction and S'
about 200 operations) times the unit roundoff u = 2^-53, amplified by the condition number of S of update 1 (the
solve), on the scale max(q, 1)."""
import numpy as np

U = 2.0 ** -53


class F64:
    """double arithmetic: the same definition evaluated the way a double-precision filter would"""
    T = np.float64

    @staticmethod
    def sqrt(v):
        return np.sqrt(np.float64(v))

    @staticmethod
    def conv(a):
        return np.asarray(a, dtype=np.float64)


class Ext:
    """np.longdouble arithmetic"""
    T = np.longdouble

    @staticmethod
    def sqrt(v):
        return np.sqrt(np.longdouble(v))

    @staticmethod
    def conv(a):
        return np.asarray(a, dtype=np.longdouble)


class Mp:
    """mpmath at the caller's working precision (mpmath.workdps(50))"""
    T = object

    def __init__(self):
        import mpmath
        self.mp = mpmath.mp

    def sqrt(self, v):
        return self.mp.sqrt(v)

    def conv(self, a):
        a = np.asarray(a, dtype=np.float64)
        out = np.empty(a.shape, dtype=object)
        for idx in np.ndindex(a.shape):
            out[idx] = self.mp.mpf(float(a[idx]))
        return out


def model(ar, cam8, xp, y):
    """h (2,), H_xp (2, 7), H_y (2, 3), var, depth of the map point y seen from the pose xp (7)."""
    cam = ar.conv(np.asarray(cam8, np.float64))
    fku, fkv, u0, v0, kd1, sd = (cam[i] for i in range(2, 8))
    w, qx, qy, qz = xp[3], xp[4], xp[5], xp[6]
    n2 = w * w + qx * qx + qy * qy + qz * qz
    qi = (w / n2, -qx / n2, -qy / n2, -qz / n2)
    a, b, c, d = qi
    R = [[1 - 2 * (c * c + d * d), 2 * (b * c - a * d), 2 * (b * d + a * c)],
         [2 * (b * c + a * d), 1 - 2 * (b * b + d * d), 2 * (c * d - a * b)],
         [2 * (b * d - a * c), 2 * (c * d + a * b), 1 - 2 * (b * b + c * c)]]
    dv = [y[i] - xp[i] for i in range(3)]
    zc = [sum(R[i][k] * dv[k] for k in range(3)) for i in range(3)]
    # d(R(qbar) a)/dqbar, columns w, x, y, z (feature_model.cpp:187-238), then diag(1, -1, -1, -1)
    m0 = [[a, -d, c], [d, a, -b], [-c, b, a]]
    mx = [[b, c, d], [c, -b, -a], [d, a, -b]]
    my = [[-c, b, a], [b, c, d], [-a, d, -c]]
    mz = [[-d, -a, b], [a, -d, c], [b, c, d]]
    dzq = [[2 * sum(m[i][k] * dv[k] for k in range(3)) * sg for m, sg in ((m0, 1), (mx, -1), (my, -1), (mz, -1))]
           for i in range(3)]
    dz_dxp = [[-R[i][j] for j in range(3)] + dzq[i] for i in range(3)]
    uc, vc = -fku * zc[0] / zc[2], -fkv * zc[1] / zc[2]
    r2 = uc * uc + vc * vc
    f = ar.sqrt(1 + 2 * kd1 * r2)
    h = [uc / f + u0, vc / f + v0]
    du = [[-fku / zc[2], 0 * fku, fku * zc[0] / (zc[2] * zc[2])], [0 * fkv, -fkv / zc[2], fkv * zc[1] / (zc[2] * zc[2])]]
    f3 = f * f * f
    dh = [[1 / f - 2 * kd1 * uc * uc / f3, -2 * kd1 * uc * vc / f3], [-2 * kd1 * vc * uc / f3, 1 / f - 2 * kd1 * vc * vc / f3]]
    J = [[sum(dh[i][k] * du[k][j] for k in range(2)) for j in range(3)] for i in range(2)]
    Hxp = [[sum(J[i][k] * dz_dxp[k][j] for k in range(3)) for j in range(7)] for i in range(2)]
    Hy = [[sum(J[i][k] * R[k][j] for k in range(3)) for j in range(3)] for i in range(2)]
    ex, ey = h[0] - u0, h[1] - v0
    ratio = ar.sqrt(ex * ex + ey * ey) / ar.sqrt(u0 * u0 + v0 * v0)
    var = (sd * (1 + ratio)) ** 2
    return h, Hxp, Hy, var, zc[2]


def _chol_solve(ar, S, B):
    """S^-1 B for a symmetric positive definite S (Cholesky, in the arithmetic of ar)."""
    m = S.shape[0]
    L = np.zeros_like(S)
    for j in range(m):
        s = S[j, j] - sum(L[j, k] * L[j, k] for k in range(j))
        L[j, j] = ar.sqrt(s)
        for i in range(j + 1, m):
            L[i, j] = (S[i, j] - sum(L[i, k] * L[j, k] for k in range(j))) / L[j, j]
    Y = B.copy()
    for i in range(m):
        Y[i] = (Y[i] - sum(L[i, k] * Y[k] for k in range(i))) / L[i, i]
    for i in reversed(range(m)):
        Y[i] = (Y[i] - sum(L[k, i] * Y[k] for k in range(i + 1, m))) / L[i, i]
    return Y


def _rows(ar, cam8, x, feats):
    """H (2k, n), R diag (2k,), h (2k,), depth (k,) of the features at state positions 13 + 3 i."""
    n = x.shape[0]
    k = len(feats)
    H = ar.conv(np.zeros((2 * k, n)))
    Rd, hs, dep = [], [], []
    for a, i in enumerate(feats):
        p = 13 + 3 * int(i)
        h, Hxp, Hy, var, depth = model(ar, cam8, x[0:7], x[p:p + 3])
        for r in range(2):
            for c in range(7):
                H[2 * a + r, c] = Hxp[r][c]
            for c in range(3):
                H[2 * a + r, p + c] = Hy[r][c]
        Rd += [var, var]
        hs += h
        dep.append(depth)
    return H, Rd, hs, dep


def update_1(ar, cam8, x, P, inl, z_inl):
    """x', P' and S of the dense update of x, P with the inliers (feature indices inl, matches z_inl (k, 2))."""
    x, P = ar.conv(x), ar.conv(P)
    if len(inl) == 0:
        return x, P, None
    H, Rd, h, _ = _rows(ar, cam8, x, inl)
    z = ar.conv(np.asarray(z_inl, np.float64).reshape(-1))
    nu = z - np.array(h, dtype=z.dtype)
    PHt = P.dot(H.T)
    S = H.dot(PHt)
    for i in range(S.shape[0]):
        S[i, i] = S[i, i] + Rd[i]
    W = _chol_solve(ar, S, PHt.T).T          # K = P H^T S^-1
    x1 = x + W.dot(nu)
    P1 = P - W.dot(PHt.T)                    # P - K S K^T = P - K H P
    q = x1[3:7]
    qq = sum(v * v for v in q)
    J = ar.conv(np.eye(4))
    for i in range(4):                       # motion_model.cpp:371-380, quirk Q2
        for j in range(4):
            J[i, j] = (1 - q[i] * q[i] / (qq * qq)) / qq if i == j else -q[i] * q[j] / (qq * qq * qq)
    P1[3:7, :] = J.dot(P1[3:7, :])
    P1[:, 3:7] = P1[:, 3:7].dot(J.T)
    P1 = (P1 + P1.T) / 2
    return x1, P1, S


def gate_at(ar, cam8, x1, P1, rej, z_rej, chi2):
    """q_j and the decisions of the rejected features rej at the updated x1, P1."""
    q, ok = [], []
    for a, i in enumerate(rej):
        H, Rd, h, dep = _rows(ar, cam8, x1, [i])
        S = H.dot(P1).dot(H.T)
        S[0, 0] = S[0, 0] + Rd[0]
        S[1, 1] = S[1, 1] + Rd[1]
        nu = ar.conv(np.asarray(z_rej[a], np.float64)) - np.array(h, dtype=x1.dtype)
        qj = nu.dot(_chol_solve(ar, S, nu.reshape(2, 1)).reshape(2))
        q.append(qj)
        ok.append(bool(dep[0] > 0 and qj <= chi2))
    return q, np.array(ok, bool)


def truth(cam8, x, P, inl, z_inl, rej, z_rej, chi2, ar=Ext):
    """-> q (k,) in the arithmetic of ar, decisions (k,) bool, cond(S of update 1)."""
    x1, P1, S = update_1(ar, cam8, x, P, inl, z_inl)
    q, ok = gate_at(ar, cam8, x1, P1, rej, z_rej, chi2)
    cond = 1.0 if S is None else float(np.linalg.cond(np.asarray(S, dtype=np.float64)))
    return q, ok, cond


def q_band(q, n, m1, cond):
    """How far a double-precision q may lie from the truth (module docstring)."""
    N = n * m1 + m1 ** 3 + 200
    return max(abs(float(q)), 1.0) * N * U * max(cond, 1.0)
