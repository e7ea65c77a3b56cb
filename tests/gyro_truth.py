"""The gyroscope update from its definition, in extended precision (np.longdouble, 64-bit significand): the measurement
z = H x + b + noise(C) with the dense 3 x n H = R_gc [0 | I3 at columns 10..12 | 0], the gyro-frame innovation
nu = z - b - H x, S = H P H^T + C, its exact inverse (adjugate over determinant), K = P H^T S^-1, x' = x + K nu,
P' = P - K S K^T and NIS = nu^T S^-1 nu.  It shares no code and no operation order with csrc/gyro.cu or
tests/gyro_ref.py, which work in the camera frame with a Cholesky factor.  `mp_update` is the same definition at 50
digits (mpmath), used once to check this one."""
import numpy as np

LD = np.longdouble


def _inv3(S):
    a = S
    adj = np.empty((3, 3), dtype=a.dtype)
    adj[0, 0] = a[1, 1] * a[2, 2] - a[1, 2] * a[2, 1]
    adj[0, 1] = a[0, 2] * a[2, 1] - a[0, 1] * a[2, 2]
    adj[0, 2] = a[0, 1] * a[1, 2] - a[0, 2] * a[1, 1]
    adj[1, 0] = a[1, 2] * a[2, 0] - a[1, 0] * a[2, 2]
    adj[1, 1] = a[0, 0] * a[2, 2] - a[0, 2] * a[2, 0]
    adj[1, 2] = a[0, 2] * a[1, 0] - a[0, 0] * a[1, 2]
    adj[2, 0] = a[1, 0] * a[2, 1] - a[1, 1] * a[2, 0]
    adj[2, 1] = a[0, 1] * a[2, 0] - a[0, 0] * a[2, 1]
    adj[2, 2] = a[0, 0] * a[1, 1] - a[0, 1] * a[1, 0]
    det = a[0, 0] * adj[0, 0] + a[0, 1] * adj[1, 0] + a[0, 2] * adj[2, 0]
    return adj / det


def update(x, P, R, bias, cov, z):
    """-> (x', P', NIS, S, D) in longdouble; D = diag(K S K^T), the scale of the correction."""
    x = np.asarray(x, np.float64).astype(LD)
    P = np.asarray(P, np.float64).astype(LD)
    n = x.size
    H = np.zeros((3, n), LD)
    H[:, 10:13] = np.asarray(R, np.float64).reshape(3, 3).astype(LD)
    C = np.asarray(cov, np.float64).reshape(3, 3).astype(LD)
    nu = np.asarray(z, np.float64).astype(LD) - np.asarray(bias, np.float64).astype(LD) - H @ x
    PHt = P @ H.T
    S = H @ PHt + C
    Si = _inv3(S)
    K = PHt @ Si
    KSK = K @ S @ K.T
    return x + K @ nu, P - KSK, nu @ Si @ nu, S, np.diag(KSK).copy()


def mp_update(x, P, R, bias, cov, z, dps=50):
    """The same definition at `dps` digits: -> (x', P', NIS) as mpmath matrices."""
    import mpmath as mp
    mp.mp.dps = dps
    n = len(x)
    X = mp.matrix([mp.mpf(float(v)) for v in x])
    Pm = mp.matrix(n, n)
    for i in range(n):
        for j in range(n):
            Pm[i, j] = mp.mpf(float(P[i, j]))
    H = mp.matrix(3, n)
    Rn = np.asarray(R, np.float64).reshape(3, 3)
    for i in range(3):
        for j in range(3):
            H[i, 10 + j] = mp.mpf(float(Rn[i, j]))
    Cm = mp.matrix([[mp.mpf(float(v)) for v in row] for row in np.asarray(cov, np.float64).reshape(3, 3)])
    nu = mp.matrix([mp.mpf(float(z[i])) - mp.mpf(float(bias[i])) for i in range(3)]) - H * X
    PHt = Pm * H.T
    S = H * PHt + Cm
    Si = S ** -1
    K = PHt * Si
    return X + K * nu, Pm - K * S * K.T, (nu.T * Si * nu)[0, 0]


def errors(x_got, P_got, nis_got, truth):
    """Scaled errors of a result (float64 or longdouble) against the truth: x entry r against |x'_r| + sqrt(D_r NIS),
    P entry (i, j) against |P'_ij| + sqrt(D_i D_j), NIS relative.  -> (ex, eP, enis)"""
    xt, Pt, qt, _, D = truth
    D = np.maximum(D.astype(np.float64), 0.0)
    q = float(qt)
    sx = np.abs(xt.astype(np.float64)) + np.sqrt(D * q) + 1e-300
    sP = np.abs(Pt.astype(np.float64)) + np.sqrt(D[:, None] * D[None, :]) + 1e-300
    ex = float((np.abs((np.asarray(x_got).astype(LD) - xt).astype(np.float64)) / sx).max())
    eP = float((np.abs((np.asarray(P_got).astype(LD) - Pt).astype(np.float64)) / sP).max())
    enis = abs(float(LD(nis_got) - qt)) / max(q, 1e-300)
    return ex, eP, enis


# The restatement's longest chain of dependent rounded operations is about 30 (zc, S, the factor, w, W, the product and
# the subtraction).  Its error is bounded by twice that count times u times the amplification of the inputs' rounding:
# cond(S) through the factor, and |zc| / |nu| through the innovation's cancellation (z close to R_gc omega + b).  The
# worst seen over tests/test_gyro.py's cases is 48 u cond(S), at cond(S) = 1e12.
OPS = 64


def kappa_nu(x, R, b, z):
    nu = np.asarray(z) - np.asarray(b) - np.asarray(R) @ np.asarray(x)[10:13]
    return (np.linalg.norm(z) + np.linalg.norm(b) + np.linalg.norm(np.asarray(x)[10:13])) / np.linalg.norm(nu)


def bound(truth, x, R, b, z):
    """The bound of a float64 result's gt.errors against the truth: OPS u (cond(S) + |zc| / |nu|)."""
    return OPS * float(np.finfo(np.float64).eps) * (cond(truth[3]) + kappa_nu(x, R, b, z))


def cond(S):
    ev = np.linalg.eigvalsh(np.asarray(S, np.float64))
    return float(ev.max() / ev.min())
