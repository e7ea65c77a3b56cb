"""The match consensus (include/sl2b200.h, sl2_set_stream_consensus) restated in Python floats, independently of
the oracle: the operation order of csrc/consensus.cu consensus_kernel, one IEEE double operation at a time; the camera
model is camera_ref's."""
import math

import numpy as np

from camera_ref import reprojection_d2


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
    for i in range(k):
        xp = []
        for r in range(7):
            s = 0.0
            for c in range(7):
                s = s + float(P[r, c]) * a[i][c]
            for c in range(3):
                s = s + float(P[r, pos[i] + c]) * b[i][c]
            xp.append(float(x[r]) + s)
        y = np.empty((k, 3))
        for j in range(k):
            for r in range(3):
                s = 0.0
                for c in range(7):
                    s = s + float(P[pos[j] + r, c]) * a[i][c]
                for c in range(3):
                    s = s + float(P[pos[j] + r, pos[i] + c]) * b[i][c]
                y[j, r] = float(x[pos[j] + r]) + s
        d2[i] = reprojection_d2(cam8, xp, y, z)
    inl = d2 <= tau2  # NaN: never
    support = inl.sum(axis=1).astype(np.int32)
    win = int(np.argmax(support)) if k else -1
    if k == 0 or support[win] < 2:
        return np.ones(k, bool), support, -1, d2
    return inl[win].copy(), support, win, d2
