"""The accelerometer's motion prediction restated op for op (include/sl2b200.h, sl2_set_stream_accel; csrc/ekf.cu:
accel_model, motion_model and predict_kernel): Python floats for the 3 x 3 and 13 x 13 parts and NumPy elementwise
float64 operations for the 13 x 3N panel, each one correctly rounded and never fused, in the kernel's order.

The reference model's own parts (q' and the sin / cos terms of F and Gn) come in as a `skeleton` (fv, F, Gn) of the
reference prediction of the same x13 and dt with u = 0: `reference_skeleton` restates them with the host's sin and cos
for the CPU tests, and the GPU tests read the device's own (test_gpu_accel.py), whose sin and cos need not round like
the host's.  x and P are the stream's state of size n (P column-major as sl2_get_state returns it)."""
import math

import numpy as np

from camera_ref import quat_to_R
from gyro_ref import rc_of


# ---- the reference's motion model (motion_model.cpp:84-217 via ekf.cu motion_model) ---------------------------------
def _quat_mul(a, b):
    aw, ax, ay, az = a
    bw, bx, by, bz = b
    return (((aw * bw - ax * bx) - ay * by) - az * bz, ((aw * bx + ax * bw) + ay * bz) - az * by,
            ((aw * by + ay * bw) + az * bx) - ax * bz, ((aw * bz + az * bw) + ax * by) - ay * bx)


def _dqomegadt_by_domega(om, dt):
    omega = math.sqrt((om[0] * om[0] + om[1] * om[1]) + om[2] * om[2])
    s, c = math.sin((omega * dt) / 2.0), math.cos((omega * dt) / 2.0)
    oo = omega * omega
    d0 = lambda a: (((-dt) / 2.0) * (a / omega)) * s  # noqa: E731
    dAA = lambda a: (((dt / 2.0) * a) * a) / oo * c + ((1.0 / omega) * (1.0 - (a * a) / oo)) * s  # noqa: E731
    dAB = lambda a, b: ((a * b) / oo) * ((dt / 2.0) * c - (1.0 / omega) * s)  # noqa: E731
    return [[d0(om[0]), d0(om[1]), d0(om[2])],
            [dAA(om[0]), dAB(om[0], om[1]), dAB(om[0], om[2])],
            [dAB(om[1], om[0]), dAA(om[1]), dAB(om[1], om[2])],
            [dAB(om[2], om[0]), dAB(om[2], om[1]), dAA(om[2])]]


def reference_skeleton(x13, dt, u=None):
    """-> (fv (13), F (13 x 13), Gn (13 x 6)) of the reference prediction with the control u (None: 0)."""
    x = [float(v) for v in x13[:13]]
    q = x[3:7]
    om = x[10:13]
    av = [om[i] * dt for i in range(3)]
    angle = math.sqrt((av[0] * av[0] + av[1] * av[1]) + av[2] * av[2])
    if angle > 0.0:
        s = math.sin(angle / 2.0) / angle
        qwt = (math.cos(angle / 2.0), s * av[0], s * av[1], s * av[2])
    else:
        qwt = (1.0, 0.0, 0.0, 0.0)
    qn = _quat_mul(q, qwt)
    u = [0.0] * 3 if u is None else [float(v) for v in u]
    fv = np.array([x[i] + x[7 + i] * dt for i in range(3)] + list(qn) + [x[7 + i] + u[i] * dt for i in range(3)]
                  + om)
    F = np.eye(13)
    Gn = np.zeros((13, 6))
    for i in range(3):
        F[i, 7 + i] = 1.0 * dt
    w, qx, qy, qz = qwt
    F[3:7, 3:7] = [[w, -qx, -qy, -qz], [qx, w, qz, -qy], [qy, -qz, w, qx], [qz, qy, -qx, w]]  # dq3_by_dq2(qwt)
    w, qx, qy, qz = q
    t44 = [[w, -qx, -qy, -qz], [qx, w, -qz, qy], [qy, qz, w, -qx], [qz, -qy, qx, w]]  # dq3_by_dq1(qold)
    m43 = _dqomegadt_by_domega(om, dt)
    for i in range(4):
        for j in range(3):
            a = 0.0
            for k in range(4):
                a = a + t44[i][k] * m43[k][j]
            F[3 + i, 10 + j] = Gn[3 + i, 3 + j] = a
    for i in range(3):
        Gn[7 + i, i] = 1.0
        Gn[10 + i, 3 + i] = 1.0
        Gn[i, i] = 1.0 * dt
    return fv, F, Gn


# ---- the accelerometer (accel_model) --------------------------------------------------------------------------------
def dRq_times_a_by_dq(q, a):
    """d(R(q) a)/dq (3 x 4, columns w, x, y, z), sl2_model.cuh's sums."""
    w2, x2, y2, z2 = (2.0 * float(v) for v in q)
    m0 = [w2, -z2, y2, z2, w2, -x2, -y2, x2, w2]
    mx = [x2, y2, z2, y2, -x2, -w2, z2, w2, -x2]
    my = [-y2, x2, w2, x2, y2, z2, -w2, z2, -y2]
    mz = [-z2, -w2, x2, w2, -z2, y2, x2, y2, z2]
    D = [[0.0] * 4 for _ in range(3)]
    for i in range(3):
        for c, m in enumerate((m0, mx, my, mz)):
            s = 0.0
            for k in range(3):
                s = s + m[i * 3 + k] * a[k]
            D[i][c] = s
    return D


def accel_model(x13, dt, R_ac, bias, Rc, gravity, sd2, f, transpose_R=False, flip_gravity=False, dqbar=False):
    """-> (status, a, D, L): status 1 applied, 2 skipped (a, D or L not finite).  The keyword arguments make the
    broken copies the tests must catch."""
    R = np.asarray(R_ac, np.float64).reshape(3, 3)
    R = R.T if transpose_R else R
    R = [[float(v) for v in row] for row in R]
    g = [(-1.0 if flip_gravity else 1.0) * float(v) for v in gravity]
    d = [float(f[k]) - float(bias[k]) for k in range(3)]
    fc = [(R[0][i] * d[0] + R[1][i] * d[1]) + R[2][i] * d[2] for i in range(3)]
    q = [float(v) for v in x13[3:7]]
    Rq = quat_to_R(*q)
    a = []
    for i in range(3):
        s = 0.0
        for k in range(3):
            s = s + Rq[i][k] * fc[k]
        a.append(s + g[i])
    D = dRq_times_a_by_dq(q, fc)
    if dqbar:
        D = [[row[0], -row[1], -row[2], -row[3]] for row in D]
    M = [[0.0] * 3 for _ in range(3)]
    for i in range(3):
        for j in range(3):
            t = 0.0
            for m in range(3):
                t = t + Rq[i][m] * Rc[m][j]
            M[i][j] = t
    L = [[0.0] * 3 for _ in range(3)]
    for i in range(3):
        for j in range(i, 3):
            t = 0.0
            for m in range(3):
                t = t + M[i][m] * Rq[j][m]
            if i == j:
                t = t + sd2
            L[i][j] = L[j][i] = (t * dt) * dt
    ok = all(math.isfinite(v) for v in a + sum(D, []) + sum(L, []))
    return (1 if ok else 2), a, D, L


# ---- predict_kernel's passes ----------------------------------------------------------------------------------------
def covariance_passes(P, F, Gn, dt, L=None):
    """P' of predict_kernel: Q, TT = F Pxx, Pxx' = TT F^T + Q, the panel F Pxy mirrored.  L: the linear block of Pnn
    of an applied sample, or None: the reference's diagonal."""
    P = np.array(P, np.float64)
    n = P.shape[0]
    lin = ((4.0 * 4.0) * dt) * dt
    ang = ((6.0 * 6.0) * dt) * dt
    F = [[float(v) for v in row] for row in F]
    G = [[float(v) for v in row] for row in Gn]
    Pxx = [[float(P[i, j]) for j in range(13)] for i in range(13)]
    Q = [[0.0] * 13 for _ in range(13)]
    TT = [[0.0] * 13 for _ in range(13)]
    for i in range(13):
        for j in range(13):
            q = 0.0
            for k in range(6):
                if L is not None and k < 3:
                    gp = ((0.0 + G[i][0] * L[0][k]) + G[i][1] * L[1][k]) + G[i][2] * L[2][k]
                else:
                    gp = 0.0 + G[i][k] * (lin if k < 3 else ang)
                q = q + gp * G[j][k]
            t = 0.0
            for k in range(13):
                t = t + F[i][k] * Pxx[k][j]
            Q[i][j], TT[i][j] = q, t
    out = np.array(P)
    for i in range(13):
        for j in range(13):
            a = 0.0
            for k in range(13):
                a = a + TT[i][k] * F[j][k]
            out[i, j] = a + Q[i][j]
    if n > 13:
        col = P[:13, 13:]
        acc = np.zeros((13, n - 13))
        Fa = np.array(F)
        for k in range(13):
            acc = acc + Fa[:, k:k + 1] * col[k:k + 1, :]
        out[:13, 13:] = acc
        out[13:, :13] = acc.T
    return out, np.array(Q)


def predict(x, P, dt, setting, f, skeleton=None, drop_half=False, **broken):
    """The whole prediction of one step of an on stream with the sample f (None: no sample): -> (x', P', a, status).
    setting: dict(R_ac, bias, cov, gravity, sd_a).  skeleton: the reference's (fv, F, Gn) of x[:13] and dt (None:
    reference_skeleton).  drop_half and the keyword arguments of accel_model make broken copies."""
    x = np.array(x, np.float64)
    fv, F, Gn = reference_skeleton(x[:13], dt) if skeleton is None else skeleton
    status, a, D, L = 0, [0.0] * 3, None, None
    if f is not None:
        Rc = rc_of(setting["R_ac"], setting["cov"])
        sd = float(setting["sd_a"])
        status, a, D, L = accel_model(x[:13], dt, setting["R_ac"], setting["bias"], Rc, setting["gravity"], sd * sd, f,
                                      **broken)
    if status != 1:
        Pn, _ = covariance_passes(P, F, Gn, dt)
        xn = x.copy()
        xn[:13] = fv
        return xn, Pn, [0.0] * 3, status
    F = np.array(F)
    fv = np.array(fv)
    h = (0.5 * dt) * dt
    for i in range(3):
        r = float(x[i]) + float(x[7 + i]) * dt
        fv[i] = r if drop_half else r + a[i] * h
        fv[7 + i] = float(x[7 + i]) + a[i] * dt
        for j in range(4):
            F[i, 3 + j] = h * D[i][j]
            F[7 + i, 3 + j] = dt * D[i][j]
    Pn, _ = covariance_passes(P, F, Gn, dt, L)
    xn = x.copy()
    xn[:13] = fv
    return xn, Pn, a, status
