"""The consensus rescue's gate (include/sl2b200.h, sl2_set_stream_rescue; csrc/rescue.cu rescue_kernel) restated in
Python floats, independently of the oracle: predict_feature (csrc/sl2_model.cuh: zeroedyi, project, measurement_noise,
func_Si<3>) and the gate, one IEEE double operation at a time in the device's order (Python's float operations and
math.sqrt are correctly rounded and never fused)."""
import math

import numpy as np

from consensus_ref import _sinv


def _sum(terms):
    s = 0.0
    for t in terms:
        s = s + t
    return s


def _qinv(xp):
    w, x, y, z = (float(v) for v in xp[3:7])
    n2 = w * w + x * x + y * y + z * z
    if n2 > 0.0:
        return w / n2, (-x) / n2, (-y) / n2, (-z) / n2
    return 0.0, 0.0, 0.0, 0.0


def _quat_to_R(w, x, y, z):
    tx, ty, tz = 2.0 * x, 2.0 * y, 2.0 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return [[1.0 - (tyy + tzz), txy - twz, txz + twy],
            [txy + twz, 1.0 - (txx + tzz), tyz - twx],
            [txz - twy, tyz + twx, 1.0 - (txx + tyy)]]


def predict(cam8, xv, y, P, pos):
    """predict_feature of the map point y (3,) at state position pos, camera state xv (>= 7), covariance P (n, n):
    -> dict(h (2,), dxp (2, 7), dy (2, 3), var, S (2, 2), depth)."""
    fku, fkv, u0, v0, kd1, sd = (float(v) for v in cam8[2:8])
    qi = _qinv(xv)
    R = _quat_to_R(*qi)
    d = [float(y[i]) - float(xv[i]) for i in range(3)]
    z = [_sum(R[i][k] * d[k] for k in range(3)) for i in range(3)]
    w2, x2, y2, z2 = (2.0 * v for v in qi)
    m0 = [w2, -z2, y2, z2, w2, -x2, -y2, x2, w2]
    mx = [x2, y2, z2, y2, -x2, -w2, z2, w2, -x2]
    my = [-y2, x2, w2, x2, y2, z2, -w2, z2, -y2]
    mz = [-z2, -w2, x2, w2, -z2, y2, x2, y2, z2]
    dz = [[R[i][j] * -1.0 for j in range(3)] + [0.0] * 4 for i in range(3)]
    for i in range(3):
        s = [_sum(m[i * 3 + k] * d[k] for k in range(3)) for m in (m0, mx, my, mz)]
        dz[i][3:7] = [s[0], -s[1], -s[2], -s[3]]
    # project (Camera::Project and ProjectionJacobian)
    uc = ((-fku) * z[0]) / z[2]
    vc = ((-fkv) * z[1]) / z[2]
    factor = math.sqrt(1.0 + (2.0 * kd1) * (uc * uc + vc * vc))
    h = [uc / factor + u0, vc / factor + v0]
    fku_yz, fkv_yz = fku / z[2], fkv / z[2]
    du = [[-fku_yz, 0.0, (fku_yz * z[0]) / z[2]], [0.0, -fkv_yz, (fkv_yz * z[1]) / z[2]]]
    dh = [[uc * uc, uc * vc], [vc * uc, vc * vc]]
    distor = 1.0 + (2.0 * kd1) * (dh[0][0] + dh[1][1])
    d12 = math.sqrt(distor)
    scale = ((-2.0) * kd1) / (d12 * distor)
    dh = [[v * scale for v in row] for row in dh]
    dh[0][0] = dh[0][0] + 1.0 / d12
    dh[1][1] = dh[1][1] + 1.0 / d12
    J = [[_sum(dh[i][k] * du[k][j] for k in range(2)) for j in range(3)] for i in range(2)]
    dxp = [[_sum(J[i][k] * dz[k][j] for k in range(3)) for j in range(7)] for i in range(2)]
    dy = [[_sum(J[i][k] * R[k][j] for k in range(3)) for j in range(3)] for i in range(2)]
    # measurement_noise
    ex, ey = h[0] - u0, h[1] - v0
    ratio = math.sqrt(ex * ex + ey * ey) / math.sqrt(u0 * u0 + v0 * v0)
    sd_use = sd * (1.0 + ratio)
    var = 1.0 * (sd_use * sd_use)
    # func_Si<3>
    Pf = lambda r, c: float(P[r, c])  # noqa: E731
    A = [[_sum(dxp[r][k] * Pf(k, j) for k in range(7)) for j in range(7)] for r in range(2)]
    Bm = [[_sum(dxp[r][k] * Pf(k, pos + j) for k in range(7)) for j in range(3)] for r in range(2)]
    Cm = [[_sum(dy[r][k] * Pf(pos + k, pos + j) for k in range(3)) for j in range(3)] for r in range(2)]
    S = np.zeros((2, 2))
    for r in range(2):
        for c in range(2):
            v = 0.0 + _sum(A[r][k] * dxp[c][k] for k in range(7))
            v = v + _sum(Bm[r][k] * dy[c][k] for k in range(3))
            v = v + _sum(Bm[c][k] * dy[r][k] for k in range(3))
            v = v + _sum(Cm[r][k] * dy[c][k] for k in range(3))
            S[r, c] = v + (var if r == c else 0.0)
    return dict(h=np.array(h), dxp=np.array(dxp), dy=np.array(dy), var=var, S=S, depth=z[2])


def q_of(z, h, S):
    """nu^T S^-1 nu with S^-1 = sinv_from_S(S), in the kernel's order (NaN when S is not positive definite)."""
    nu0, nu1 = float(z[0]) - float(h[0]), float(z[1]) - float(h[1])
    try:
        s00, s01, s11 = _sinv(S)
    except ValueError:  # math.sqrt of a negative: the device's sqrt gives NaN
        return math.nan
    w0, w1 = s00 * nu0 + s01 * nu1, s01 * nu0 + s11 * nu1
    return nu0 * w0 + nu1 * w1


def gate(cam8, x, P, pos, z, chi2):
    """The k rejected matches (positions pos (k,), z (k, 2)) seen from the updated x, P.
    -> rescued (k,) bool, q (k,), predictions (list of predict() dicts)."""
    preds = [predict(cam8, x, x[p:p + 3], P, int(p)) for p in pos]
    q = np.array([q_of(z[j], preds[j]["h"], preds[j]["S"]) for j in range(len(pos))])
    ok = np.array([preds[j]["depth"] > 0.0 and q[j] <= float(chi2) for j in range(len(pos))], bool)
    return ok, q, preds
