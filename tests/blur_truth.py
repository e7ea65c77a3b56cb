"""The exposure blur (include/sl2b200.h, sl2_set_stream_blur) from its definition, in extended precision: the truth
that tests/test_blur.py holds the restatement (tests/blur_ref.py) to and tests/test_gpu_blur_truth.py holds the device
to.

It uses none of the device chain's operations (no unproject_point, no adjugate, no RRW^T):
  pose at s: r + v s and q (x) (cos(|w s| / 2), sin(|w s| / 2) w s / |w s|) in the working precision (x[0:7] for
             s = 0);
  source:    the pixel p = h0 + d, its ray solved as in tests/warp_truth.py (Newton on the distortion), cut with the
             plane nW . (X - y) = 0 through the exact inverse of the pose's RRW, projected into the reference camera
             (xo with centre ho when the warp is on, x[0:7] with centre h0 when it is off; the identity for the warp
             off and s = 0); valid: inside the reach, the ray's parameter > 0, zo[2] > 0;
  samples:   L = |src(s+) - src(s-)| at the centre pixel, K = min(32, max(1, ceil(L)));
  value:     the stated quadratic through the three sources at u_k = (k + 1/2) / K - 1/2, the exact bilinear values
             there (clamped to [0, B - 1]) and their mean; the byte is floor(v + 1/2).
Two precisions run the same code: mpmath at 50 digits and np.longdouble; tests/test_blur.py checks the second against
the first once.  A byte is decided when v lies farther than TOL_V from k + 1/2, and a case when L lies farther than
TOL_L from an integer: the FP64 chain's own error is many orders of magnitude below both at the tested sizes."""
import collections
import math

import mpmath
import numpy as np

from consensus_truth import DPS, _Num, project, rotation_rrw
from warp_truth import _floor, _inverse3, solve_ray

TOL_V = 1e-6
TOL_L = 1e-6
MAX_SAMPLES = 32

Truth = collections.namedtuple("Truth", ["v", "byte", "valid", "L", "K", "tie_gap", "src"])


def _trig(num):
    if num.prec == "mp":
        return mpmath.sin, mpmath.cos
    return np.sin, np.cos


def pose_at(x, s, num):
    """(r (3), q (4)) at time s, in the working precision."""
    x_ = num(np.asarray(x[:13], np.float64))
    if s == 0.0:
        return x_[0:3], x_[3:7]
    s_ = num(np.float64(s)) if num.prec == "mp" else np.longdouble(s)
    r = x_[0:3] + x_[7:10] * s_
    av = x_[10:13] * s_
    ang = num.sqrt(av[0] * av[0] + av[1] * av[1] + av[2] * av[2])
    sin, cos = _trig(num)
    if ang > 0:
        k = sin(ang / 2) / ang
        qw = [cos(ang / 2), k * av[0], k * av[1], k * av[2]]
    else:
        qw = [num(np.float64(1.0)), 0 * ang, 0 * ang, 0 * ang]
    a = x_[3:7]
    q = np.array([a[0] * qw[0] - a[1] * qw[1] - a[2] * qw[2] - a[3] * qw[3],
                  a[0] * qw[1] + a[1] * qw[0] + a[2] * qw[3] - a[3] * qw[2],
                  a[0] * qw[2] + a[2] * qw[0] + a[3] * qw[1] - a[1] * qw[3],
                  a[0] * qw[3] + a[3] * qw[0] + a[1] * qw[2] - a[2] * qw[1]], dtype=a.dtype)
    return r, q


def _sources(cam8, B, y_, nW, h0, ref, pose, ident, num, centre_only=False):
    half = (B - 1) // 2
    if centre_only:
        a = b = np.array([half])
    else:
        a, b = np.mgrid[0:B, 0:B]
    if ident:
        return np.stack([num(b.astype(np.float64)), num(a.astype(np.float64))], -1), np.ones(b.shape, bool)
    r, q = pose
    R = rotation_rrw(q)
    p = np.stack([h0[0] + num((b - half).astype(np.float64)), h0[1] + num((a - half).astype(np.float64))], -1)
    U, _, inside = solve_ray(cam8, p, num)
    zc = [-U[..., 0] / num(cam8[2]), -U[..., 1] / num(cam8[3]), num(np.ones(b.shape))]
    Minv = _inverse3(R, num)
    dW = [Minv[i, 0] * zc[0] + Minv[i, 1] * zc[1] + Minv[i, 2] * zc[2] for i in range(3)]
    numer = nW @ (y_ - r)
    den = nW[0] * dW[0] + nW[1] * dW[1] + nW[2] * dW[2]
    ok = inside & (numer * den > 0).astype(bool)
    lam = numer / np.where(ok, den, 1)
    X = np.stack([r[i] + lam * dW[i] for i in range(3)], -1)
    Rref, rref, cref = ref
    zo = np.einsum("ij,...j->...i", Rref, X - rref)
    ok = ok & (zo[..., 2] > 0).astype(bool)
    zs = np.where(ok[..., None], zo, num(np.array([0.0, 0.0, 1.0])))
    g = project(cam8, zs, num)
    return np.stack([g[..., 0] - cref[0] + half, g[..., 1] - cref[1] + half], -1), ok


def _bilinear(Tn, src, B, num):
    fl = _floor(num)
    sx = np.minimum(np.maximum(src[..., 0], 0), B - 1)
    sy = np.minimum(np.maximum(src[..., 1], 0), B - 1)
    x0 = np.minimum(num.f64(fl(sx)).astype(np.int64), B - 2)
    y0 = np.minimum(num.f64(fl(sy)).astype(np.int64), B - 2)
    fx, fy = sx - num(x0.astype(np.float64)), sy - num(y0.astype(np.float64))
    return ((1 - fy) * ((1 - fx) * Tn[y0, x0] + fx * Tn[y0, x0 + 1])
            + fy * ((1 - fx) * Tn[y0 + 1, x0] + fx * Tn[y0 + 1, x0 + 1]))


def plane_normal(y_, xo_, theta, num):
    """nW(theta) from its definition: nW0 = xo - y; E1 = camera o's x axis made orthogonal to nW0 and scaled to |nW0|;
    E2 = nW0 x E1 / |nW0|; nW0 + a E1 + b E2."""
    n0 = xo_[0:3] - y_
    if theta[0] == 0.0 and theta[1] == 0.0:
        return n0
    R0 = rotation_rrw(xo_[3:7])[0]
    nn = n0 @ n0
    q = R0 - (R0 @ n0) / nn * n0
    E1 = q * (num.sqrt(nn) / num.sqrt(q @ q))
    E2 = np.array([n0[1] * E1[2] - n0[2] * E1[1], n0[2] * E1[0] - n0[0] * E1[2], n0[0] * E1[1] - n0[1] * E1[0]],
                  dtype=n0.dtype) / num.sqrt(nn)
    a, b = (num(np.float64(v)) if num.prec == "mp" else np.longdouble(v) for v in theta)
    return n0 + a * E1 + b * E2


def blur_truth(cam8, T, y, xo, x, exposure, offset, warp, prec="ld", theta=(0.0, 0.0)):
    """-> Truth of one job: v (B, B) (None when a needed source is invalid), byte, valid, L, K, tie_gap, src (the
    three sources, FP64); theta: the feature's estimated tilt (normals on)."""
    num = _Num(prec)
    cam8 = np.asarray(cam8, np.float64)
    T = np.asarray(T, np.uint8)
    B = T.shape[0]
    with mpmath.workdps(DPS), np.errstate(invalid="ignore", divide="ignore"):
        y_, xo_ = num(np.asarray(y, np.float64)), num(np.asarray(xo, np.float64))
        x_ = num(np.asarray(x[:7], np.float64))
        R0 = rotation_rrw(x_[3:7])
        h0 = project(cam8, R0 @ (y_ - x_[0:3]), num)
        nW = plane_normal(y_, xo_, theta, num)
        if warp:
            Ro = rotation_rrw(xo_[3:7])
            ref = (Ro, xo_[0:3], project(cam8, Ro @ (y_ - xo_[0:3]), num))
        else:
            ref = (R0, x_[0:3], h0)
        hx = float(exposure) * 0.5
        ts = (float(offset) - hx, float(offset), float(offset) + hx)
        poses = [pose_at(x, s, num) for s in ts]
        ident = [(not warp) and s == 0.0 for s in ts]
        cs = [_sources(cam8, B, y_, nW, h0, ref, poses[k], ident[k], num, centre_only=True) for k in (0, 2)]
        d = cs[1][0][0] - cs[0][0][0]
        Lx = num.sqrt(d[0] * d[0] + d[1] * d[1])
        L = float(num.f64(Lx))
        ok = bool(cs[0][1][0] and cs[1][1][0]) and math.isfinite(L)
        K = int(min(MAX_SAMPLES, max(1, math.ceil(L)))) if ok else 1
        srcs = [_sources(cam8, B, y_, nW, h0, ref, poses[k], ident[k], num) for k in range(3)]
        need = [1] if K == 1 else [0, 1, 2]
        ok = ok and all(srcs[k][1].all() for k in need)
        src64 = np.stack([np.where(srcs[k][1][..., None], num.f64(srcs[k][0]), np.nan) for k in range(3)])
        if not ok:
            return Truth(None, None, False, L, K, None, src64)
        Tn = num(T.astype(np.float64))
        s0, s1, s2 = (srcs[k][0] for k in range(3))
        if K == 1:
            vv = _bilinear(Tn, s1, B, num)
        else:
            acc = 0
            for m in range(K):
                u = (num(np.float64(m)) + num(np.float64(0.5))) / K - num(np.float64(0.5))
                pt = s1 + u * (s2 - s0) + 2 * u * u * (s2 - 2 * s1 + s0)
                acc = acc + _bilinear(Tn, pt, B, num)
            vv = acc / K
        half = mpmath.mpf(1) / 2 if prec == "mp" else np.longdouble(0.5)
        fl = _floor(num)
        byte = num.f64(fl(vv + half)).astype(np.int64)
        tie = np.abs(vv - (fl(vv) + half))
        return Truth(num.f64(vv), byte, True, L, K, num.f64(tie), src64)


def decided(t):
    """(case decided, byte mask): L away from an integer, and v away from k + 1/2."""
    if not math.isfinite(t.L):
        return False, None
    case = abs(t.L - round(t.L)) > TOL_L or t.L < 1.0 - TOL_L
    if t.v is None:
        return case, None
    return case, t.tie_gap > TOL_V
