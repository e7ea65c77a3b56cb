"""The accelerometer's motion prediction from its definition, in extended precision (np.longdouble, 64-bit significand):
a = R(q) R_ac^T (f - b) + g with R(q) v = v + 2 w (u x v) + 2 (u (u . v) - |u|^2 v) for q = (w, u) (the same matrix
as Eigen's toRotationMatrix, also for |q| != 1); D = d(Rh(q) f_c)/dq, differentiated by hand from the homogeneous form
Rh(q) v = (w^2 - |u|^2) v + 2 (u . v) u + 2 w (u x v) = R(q) v + (|q|^2 - 1) v that the reference's dR_by_dq matrices
differentiate (equal to d(R(q) f_c)/dq along directions tangent to |q| = 1); F the reference's F with the two blocks, Pnn's linear block dt^2 (R(q) R_ac^T C R_ac R(q)^T + sd_a^2 I), and P' = F P F^T + Gn Pnn Gn^T
as matrix products.  It shares no code and no operation order with csrc/ekf.cu or tests/accel_ref.py.  The reference
model's own parts (q', F and Gn of the reference prediction) are inputs, as for the restatement.  `mp_predict` is the
same definition at 50 digits (mpmath), used once to check this one."""
import numpy as np

LD = np.longdouble


def _rot_times(q, v):
    w, u = q[0], q[1:4]
    return v + 2 * w * np.cross(u, v) + 2 * (u * (u @ v) - (u @ u) * v)


def _d_rot_times(q, v):
    """d(Rh(q) v)/dq, columns (w, x, y, z)."""
    w, u = q[0], q[1:4]
    D = np.zeros((3, 4), dtype=v.dtype)
    D[:, 0] = 2 * w * v + 2 * np.cross(u, v)
    for k in range(3):
        e = np.zeros(3, dtype=v.dtype)
        e[k] = 1
        D[:, 1 + k] = -2 * u[k] * v + 2 * (v[k] * u + (u @ v) * e) + 2 * w * np.cross(e, v)
    return D


def parts(x13, dt, setting, f, dtype=LD):
    """-> (a, D, Lin) of the definition in `dtype`."""
    q = np.asarray(x13[3:7], np.float64).astype(dtype)
    Rac = np.asarray(setting["R_ac"], np.float64).reshape(3, 3).astype(dtype)
    C = np.asarray(setting["cov"], np.float64).reshape(3, 3).astype(dtype)
    fc = Rac.T @ (np.asarray(f, np.float64).astype(dtype) - np.asarray(setting["bias"], np.float64).astype(dtype))
    a = _rot_times(q, fc) + np.asarray(setting["gravity"], np.float64).astype(dtype)
    D = _d_rot_times(q, fc)
    Rq = np.stack([_rot_times(q, e) for e in np.eye(3, dtype=dtype)], 1)
    sd = dtype(float(setting["sd_a"]))
    dtl = dtype(float(dt))
    Lin = dtl * dtl * (Rq @ (Rac.T @ C @ Rac) @ Rq.T + sd * sd * np.eye(3, dtype=dtype))
    return a, D, Lin


def predict(x, P, dt, setting, f, skeleton):
    """-> (x', P', Q, a, F) in longdouble."""
    fv, F0, Gn = skeleton
    x = np.asarray(x, np.float64).astype(LD)
    P = np.asarray(P, np.float64).astype(LD)
    n = x.size
    dtl = LD(float(dt))
    a, D, Lin = parts(x[:13], dt, setting, f)
    Fx = np.asarray(F0, np.float64).astype(LD)
    Fx[0:3, 3:7] = dtl * dtl / 2 * D
    Fx[7:10, 3:7] = dtl * D
    F = np.eye(n, dtype=LD)
    F[:13, :13] = Fx
    Pnn = np.zeros((6, 6), LD)
    Pnn[:3, :3] = Lin
    Pnn[3:, 3:] = 36 * dtl * dtl * np.eye(3, dtype=LD)
    G = np.asarray(Gn, np.float64).astype(LD)
    Q = G @ Pnn @ G.T
    Pn = F @ P @ F.T
    Pn[:13, :13] += Q
    xn = x.copy()
    xn[:3] = x[:3] + x[7:10] * dtl + a * dtl * dtl / 2
    xn[3:7] = np.asarray(fv[3:7], np.float64).astype(LD)
    xn[7:10] = x[7:10] + a * dtl
    return xn, Pn, Q, a, F


def mp_predict(x, P, dt, setting, f, skeleton, dps=50):
    """The same definition at `dps` digits: -> (x', P') as mpmath matrices."""
    import mpmath as mp
    mp.mp.dps = dps
    fv, F0, Gn = skeleton
    n = len(x)
    M = lambda A: mp.matrix([[mp.mpf(float(v)) for v in row] for row in np.asarray(A, np.float64)])  # noqa: E731
    V = lambda v: mp.matrix([mp.mpf(float(t)) for t in np.asarray(v, np.float64).ravel()])  # noqa: E731
    w, u = mp.mpf(float(x[3])), V(x[4:7])
    cross = lambda p, r: mp.matrix([p[1] * r[2] - p[2] * r[1], p[2] * r[0] - p[0] * r[2],  # noqa: E731
                                    p[0] * r[1] - p[1] * r[0]])
    dot = lambda p, r: p[0] * r[0] + p[1] * r[1] + p[2] * r[2]  # noqa: E731
    rot = lambda v: v + 2 * w * cross(u, v) + 2 * (u * dot(u, v) - dot(u, u) * v)  # noqa: E731
    Rac = M(np.asarray(setting["R_ac"]).reshape(3, 3))
    fc = Rac.T * (V(f) - V(setting["bias"]))
    a = rot(fc) + V(setting["gravity"])
    D = mp.matrix(3, 4)
    D[:, 0] = 2 * w * fc + 2 * cross(u, fc)
    for k in range(3):
        e = V([1.0 if i == k else 0.0 for i in range(3)])
        col = -2 * u[k] * fc + 2 * (fc[k] * u + dot(u, fc) * e) + 2 * w * cross(e, fc)
        for i in range(3):
            D[i, 1 + k] = col[i]
    Rq = mp.matrix(3, 3)
    for j in range(3):
        c = rot(V([1.0 if i == j else 0.0 for i in range(3)]))
        for i in range(3):
            Rq[i, j] = c[i]
    dtm = mp.mpf(float(dt))
    sd = mp.mpf(float(setting["sd_a"]))
    Lin = dtm * dtm * (Rq * (Rac.T * M(np.asarray(setting["cov"]).reshape(3, 3)) * Rac) * Rq.T + sd * sd * mp.eye(3))
    F = mp.eye(n)
    F0m = M(F0)
    for i in range(13):
        for j in range(13):
            F[i, j] = F0m[i, j]
    for i in range(3):
        for j in range(4):
            F[i, 3 + j] = dtm * dtm / 2 * D[i, j]
            F[7 + i, 3 + j] = dtm * D[i, j]
    Pnn = mp.zeros(6, 6)
    for i in range(3):
        for j in range(3):
            Pnn[i, j] = Lin[i, j]
        Pnn[3 + i, 3 + i] = 36 * dtm * dtm
    G = M(Gn)
    Q = G * Pnn * G.T
    Pn = F * M(P) * F.T
    for i in range(13):
        for j in range(13):
            Pn[i, j] += Q[i, j]
    xn = V(x)
    for i in range(4):
        xn[3 + i] = mp.mpf(float(fv[3 + i]))
    for i in range(3):
        xn[i] = xn[i] + xn[7 + i] * dtm + a[i] * dtm * dtm / 2
        xn[7 + i] = xn[7 + i] + a[i] * dtm
    return xn, Pn


# The restatement's longest chain of dependent rounded operations per entry of P' is a 13-term sum of 13-term sums plus
# the few operations of F's new blocks and of Q's linear block: under 40.  Each entry's error is then bounded by a
# multiple of u (|F| |P| |F|^T + |Q|) at that entry, and each state entry's by a multiple of u times the sum of the
# magnitudes of its terms (the rounding of f - b against |f| + |b| carried through |R(q)|).
OPS = 64


def scales(x, P, dt, setting, f, truth):
    """(scale of x' (n), scale of P' (n x n)) of the bound, in float64."""
    xn, Pn, Q, a, F = truth
    Fa = np.abs(F.astype(np.float64))
    SP = Fa @ np.abs(np.asarray(P, np.float64)) @ Fa.T
    SP[:13, :13] += np.abs(Q.astype(np.float64))
    qn = float(np.linalg.norm(np.asarray(x[3:7], np.float64)))
    fa = (np.abs(np.asarray(setting["R_ac"])).T @ (np.abs(np.asarray(f)) + np.abs(np.asarray(setting["bias"]))))
    amag = np.full(3, max(qn * qn, 1.0) * 3 * float(fa.max())) + np.abs(np.asarray(setting["gravity"]))
    x = np.asarray(x, np.float64)
    sx = np.abs(x).copy()
    sx[:3] += np.abs(x[7:10]) * dt + amag * dt * dt
    sx[7:10] += amag * dt
    sx[3:7] = np.abs(xn[3:7].astype(np.float64))
    return sx, SP


def errors(x_got, P_got, x, P, dt, setting, f, truth):
    """(max |x - x'| / scale, max |P - P'| / scale) of a float64 result against the truth, in units of u."""
    u = float(np.finfo(np.float64).eps)
    sx, SP = scales(x, P, dt, setting, f, truth)
    ex = np.abs((np.asarray(x_got).astype(LD) - truth[0]).astype(np.float64)) / (sx + 1e-300)
    eP = np.abs((np.asarray(P_got).astype(LD) - truth[1]).astype(np.float64)) / (SP + 1e-300)
    return float(ex.max()) / u, float(eP.max()) / u
