"""The match consensus (include/sl2b200.h, sl2_set_stream_consensus) restated in Python floats, independently of
the oracle: the operation order of csrc/ekf.cu consensus_kernel, one IEEE double operation at a time."""
import math

import numpy as np


def _quat_to_R(w, x, y, z):
    tx, ty, tz = 2.0 * x, 2.0 * y, 2.0 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return [[1.0 - (tyy + tzz), txy - twz, txz + twy],
            [txy + twz, 1.0 - (txx + tzz), tyz - twx],
            [txz - twy, tyz + twx, 1.0 - (txx + tyy)]]


def _rrw(xp):
    w, x, y, z = (float(v) for v in xp[3:7])
    n2 = w * w + x * x + y * y + z * z
    if n2 > 0.0:
        w, x, y, z = w / n2, (-x) / n2, (-y) / n2, (-z) / n2
    else:
        w = x = y = z = 0.0
    return _quat_to_R(w, x, y, z)


def _project(cam8, zc):
    fku, fkv, u0, v0, kd1 = (float(v) for v in cam8[2:7])
    uc = (-fku) * zc[0] / zc[2]
    vc = (-fkv) * zc[1] / zc[2]
    factor = math.sqrt(1.0 + 2.0 * kd1 * (uc * uc + vc * vc))
    return uc / factor + u0, vc / factor + v0


def _sinv(S):
    s00, s10, s11 = float(S[0, 0]), float(S[1, 0]), float(S[1, 1])
    l00 = math.sqrt(s00)
    l10 = s10 / l00
    l11 = math.sqrt(s11 - l10 * l10)
    x00, x11 = 1.0 / l00, 1.0 / l11
    x10 = (0.0 - l10 * x00) / l11
    return x00 * x00 + x10 * x10, x10 * x11, x11 * x11


def restated(cam8, x, P, pos, z, h, S, dxp, dy, tau):
    """-> keep, support, winner, d2 (k x k squared distances, NaN where the point is behind the camera)"""
    k = len(pos)
    tau2 = float(tau) * float(tau)
    a, b = [], []
    for j in range(k):
        nu0, nu1 = float(z[j, 0]) - float(h[j, 0]), float(z[j, 1]) - float(h[j, 1])
        s00, s01, s11 = _sinv(S[j])
        w0, w1 = s00 * nu0 + s01 * nu1, s01 * nu0 + s11 * nu1
        a.append([float(dxp[j, 0, c]) * w0 + float(dxp[j, 1, c]) * w1 for c in range(7)])
        b.append([float(dy[j, 0, c]) * w0 + float(dy[j, 1, c]) * w1 for c in range(3)])
    d2 = np.full((k, k), np.nan)
    support = np.zeros(k, np.int32)
    inl = np.zeros((k, k), bool)
    for i in range(k):
        xp = []
        for r in range(7):
            s = 0.0
            for c in range(7):
                s = s + float(P[r, c]) * a[i][c]
            for c in range(3):
                s = s + float(P[r, pos[i] + c]) * b[i][c]
            xp.append(float(x[r]) + s)
        R = _rrw(xp)
        for j in range(k):
            y = []
            for r in range(3):
                s = 0.0
                for c in range(7):
                    s = s + float(P[pos[j] + r, c]) * a[i][c]
                for c in range(3):
                    s = s + float(P[pos[j] + r, pos[i] + c]) * b[i][c]
                y.append(float(x[pos[j] + r]) + s)
            dd = [y[r] - xp[r] for r in range(3)]
            zc = []
            for r in range(3):
                s = 0.0
                for c in range(3):
                    s = s + R[r][c] * dd[c]
                zc.append(s)
            if zc[2] > 0.0:
                g = _project(cam8, zc)
                du, dv = float(z[j, 0]) - g[0], float(z[j, 1]) - g[1]
                d2[i, j] = du * du + dv * dv
                inl[i, j] = d2[i, j] <= tau2
        support[i] = int(inl[i].sum())
    win = int(np.argmax(support)) if k else -1
    if k == 0 or support[win] < 2:
        return np.ones(k, bool), support, -1, d2
    return inl[win].copy(), support, win, d2
