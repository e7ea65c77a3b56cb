"""The match consensus (include/sl2b200.h, sl2_set_stream_consensus) from its definition, in extended precision: the
truth that tests/test_consensus_truth.py holds the restatements to and tests/test_gpu_consensus.py holds the device to.

It reads exactly what consensus_kernel reads (x, P, the matches' state positions, z, h, S, dh/dxp, dh/dy, the camera,
tau) and shares nothing with the kernel's factorisation or with camera_ref:
  hypothesis i:  the dense 2 x n H_i (columns 0..6 dh/dxp_i, 7..12 zero because the fused step's dh/dxv is
                 [dh/dxp | 0], pos_i..pos_i+2 dh/dy_i), K_i = P H_i^T S_i^-1 with the exact inverse of the given S_i
                 (its lower triangle, which is what the kernel reads), x'_i = x + K_i (z_i - h_i) over the whole state;
  match j of i:  the measurement model of the reference at (x'_i[0:7], x'_i[pos_j:pos_j+3]): zeroedyi
                 (full_feature_model.cpp: RRW = the rotation matrix of qRW = q^-1 = conj(q) / |q|^2, Eigen's formula,
                 which is not a rotation when |q| != 1; x is never renormalised, quirk Q1) and Camera::Project
                 (camera.cpp, radial distortion kd1); d2_ij = |z_j - h_j(x'_i)|^2, an inlier iff the camera-frame
                 depth is > 0 and d2_ij <= fl(tau tau), the threshold the device is handed;
  decision:      support, the winner (largest support, lowest rank on a tie, none below 2) and the kept matches.
Two precisions run the same code: mpmath at 50 digits (object arrays of mpf) and np.longdouble.  The first is the
definition; the second is fast enough for the GPU shapes and tests/test_consensus_truth.py shows the two agree."""
import collections

import mpmath
import numpy as np

DPS = 50
EPS = float(np.finfo(np.float64).eps)

Truth = collections.namedtuple("Truth", "d2 depth inlier support winner keep margin depth_margin")


class _Num:
    """Conversions and sqrt of one precision; FP64 inputs convert exactly in both."""

    def __init__(self, prec):
        self.prec = prec
        if prec == "mp":
            self.dtype = object
            self._mpf = np.vectorize(mpmath.mpf, otypes=[object])
            self._sqrt = np.vectorize(mpmath.sqrt, otypes=[object])
        elif prec == "ld":
            self.dtype = np.longdouble
        else:
            raise ValueError(prec)

    def __call__(self, a):
        a = np.asarray(a, np.float64)
        return self._mpf(a) if self.prec == "mp" else a.astype(np.longdouble)

    def zeros(self, shape):
        return self(np.zeros(shape))

    def sqrt(self, a):
        return self._sqrt(a) if self.prec == "mp" else np.sqrt(a)

    def f64(self, a):
        return np.asarray(np.asarray(a, dtype=self.dtype), np.float64) if self.prec == "mp" else np.asarray(a, np.float64)


def dense_h(n, pos, dh_dxp, dh_dy, num):
    """(k, 2, n) dense measurement Jacobians of the matches."""
    k = len(pos)
    H = num.zeros((k, 2, n))
    for i in range(k):
        H[i, :, 0:7] = num(dh_dxp[i])
        H[i, :, pos[i]:pos[i] + 3] = num(dh_dy[i])
    return H


def s_inverse(S, num):
    """(k, 2, 2) exact inverses of the symmetric S_i of lower triangle (S00, S10, S11)."""
    S = np.asarray(S, np.float64)
    s00, s10, s11 = num(S[:, 0, 0]), num(S[:, 1, 0]), num(S[:, 1, 1])
    det = s00 * s11 - s10 * s10
    out = num.zeros((len(S), 2, 2))
    out[:, 0, 0], out[:, 0, 1], out[:, 1, 0], out[:, 1, 1] = s11 / det, -s10 / det, -s10 / det, s00 / det
    return out


def rotation_rrw(q):
    """RRW of the camera quaternions q (..., 4) = (w, x, y, z): Eigen's toRotationMatrix of qRW = conj(q) / |q|^2
    (the zero quaternion for q = 0)."""
    w, x, y, z = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    n2 = w * w + x * x + y * y + z * z
    nz = n2 != 0
    n2 = np.where(nz, n2, 1)
    w, x, y, z = np.where(nz, w / n2, 0), np.where(nz, -x / n2, 0), np.where(nz, -y / n2, 0), np.where(nz, -z / n2, 0)
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                     np.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
                     np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], -2)


def project(cam8, zc, num):
    """Camera::Project of camera-frame points zc (..., 3) -> (..., 2); the point must not have depth 0."""
    fku, fkv, u0, v0, kd1 = (num(c) for c in cam8[2:7])
    uc = -fku * zc[..., 0] / zc[..., 2]
    vc = -fkv * zc[..., 1] / zc[..., 2]
    factor = num.sqrt(1 + 2 * kd1 * (uc * uc + vc * vc))
    return np.stack([uc / factor + u0, vc / factor + v0], -1)


def hypotheses(x, P, pos, z, h, S, dh_dxp, dh_dy, num):
    """(n, k) states x'_i = x + P H_i^T S_i^-1 nu_i, column i for hypothesis i."""
    n, k = len(x), len(pos)
    H = dense_h(n, pos, dh_dxp, dh_dy, num)
    Si = s_inverse(S, num)
    nu = num(z) - num(h)
    PHt = num(P) @ H.transpose(2, 0, 1).reshape(n, 2 * k)      # [P H_0^T | P H_1^T | ...]
    Knu = np.einsum("nkr,krc,kc->nk", PHt.reshape(n, k, 2), Si, nu)
    return num(x)[:, None] + Knu


def consensus_truth(cam8, x, P, pos, z, h, S, dh_dxp, dh_dy, tau, prec="mp"):
    """-> Truth: d2 (k x k, FP64 rounding of the exact value, NaN where the depth is not > 0), depth (k x k), the inlier
    mask, supports, winner, kept matches, margin = min |d2 - fl(tau tau)| over the pairs in front of the camera and
    depth_margin = min |depth| over every pair (decisions at which a rounding error could flip an answer)."""
    k = len(pos)
    num = _Num(prec)
    with mpmath.workdps(DPS):
        if k == 0:
            e = np.zeros((0, 0))
            return Truth(e, e, e.astype(bool), np.zeros(0, np.int32), -1, np.zeros(0, bool), np.inf, np.inf)
        t2 = float(tau) * float(tau)
        X = hypotheses(x, P, pos, z, h, S, dh_dxp, dh_dy, num)
        R = rotation_rrw(X[3:7].T)                                 # (k, 3, 3) per hypothesis
        idx = np.asarray(pos)[:, None] + np.arange(3)
        y = X[idx].transpose(2, 0, 1)                             # (i, j, 3): y'_j of hypothesis i
        d = y - X[0:3].T[:, None, :]
        zc = np.einsum("irc,ijc->ijr", R, d)
        depth = zc[..., 2]
        front = (depth > 0).astype(bool)
        zc = np.where(front[..., None], zc, 1)                    # nothing behind the camera is projected
        g = project(cam8, zc, num)
        du = num(z)[None, :, 0] - g[..., 0]
        dv = num(z)[None, :, 1] - g[..., 1]
        d2 = du * du + dv * dv
        inl = front & (d2 <= t2).astype(bool)
        gap = np.abs(d2 - t2)
        margin = float(num.f64(gap[front]).min()) if front.any() else np.inf
        d2f = np.where(front, num.f64(d2), np.nan)
        depth_f = num.f64(depth)
    support = inl.sum(axis=1).astype(np.int32)
    win = int(np.argmax(support))
    if support[win] < 2:
        win, keep = -1, np.ones(k, bool)
    else:
        keep = inl[win].copy()
    return Truth(d2f, depth_f, inl, support, win, keep, margin, float(np.abs(depth_f).min()))


def s_consistency(cam8, P, pos, h, S, dh_dxp, dh_dy, R=None):
    """The largest |S_i - (H_i P H_i^T + R_i)| over the matches, each relative to the same sum of absolute values
    (|H_i| |P| |H_i|^T + |R_i|): how far the S the kernel is handed is from the S its algebra assumes, in units of
    that sum.  R_i is Camera::MeasurementNoise of h_i (var I) unless given as (k, 2, 2).  P's antisymmetric part,
    if any, does not enter: H A H^T has a zero diagonal and only the lower triangle of S is read."""
    num = _Num("mp")
    with mpmath.workdps(DPS):
        n, k = P.shape[0], len(pos)
        H = dense_h(n, pos, dh_dxp, dh_dy, num)
        Pm = num(P)
        Pa = num(np.abs(P))
        if R is None:
            u0, v0, sd = (num(c) for c in cam8[[4, 5, 7]])
            hm = num(h)
            ratio = num.sqrt((hm[:, 0] - u0) ** 2 + (hm[:, 1] - v0) ** 2) / num.sqrt(u0 * u0 + v0 * v0)
            var = (sd * (1 + ratio)) ** 2
            Rm = num.zeros((k, 2, 2))
            Rm[:, 0, 0] = var
            Rm[:, 1, 1] = var
        else:
            Rm = num(R)
        worst = 0.0
        for i in range(k):
            Hi = H[i]
            HPH = Hi @ Pm @ Hi.T
            HPH = (HPH + HPH.T) / 2
            scale = np.abs(Hi) @ Pa @ np.abs(Hi).T + np.abs(Rm[i]) + 1e-300
            err = np.abs(num(S[i]) - (HPH + Rm[i])) / scale
            worst = max(worst, float(num.f64(err).max()))
    return worst
