"""The planar patch warp (include/sl2b200.h, sl2_set_stream_warp) from its definition, in extended precision: the truth
that tests/test_warp_truth.py holds the restatement (tests/warp_ref.py) to and tests/test_gpu_warp_truth.py holds the
device to.

It states the header's geometry with the forward model of the prediction only, and with none of the device chain's
operations (no unproject_point, no RRW^T, no adjugate):
  centre:   h = Project(RRW(xp) (y - r)), ho = Project(RRW(xo) (y - xo[0:3])); RRW and Project are
            consensus_truth's rotation_rrw (Eigen's matrix of qRW = conj(q) / |q|^2, not a rotation when |q| != 1) and
            project (Camera::Project with radial distortion kd1);
  pixel:    output pixel (row a, column b): p = h + (b - HALF, a - HALF);
  ray:      the camera-frame direction z = (x, y, 1) with Project(z) = p, found by Newton's method on the distortion
            u / sqrt(1 + 2 kd1 |u|^2) = p - c (u = the undistorted image-centred point, c the principal point) and
            checked by its residual; the pixel is inside the model's reach when 1 - 2 kd1 |p - c|^2 > 0;
  plane:    X = r + lam RRW(xp)^-1 z, the exact inverse, with nW . (X - y) = 0, nW = xo[0:3] - y;
  source:   zo = RRW(xo) (X - xo[0:3]), src = Project(zo) - ho + (HALF, HALF);
  valid:    inside the reach, lam > 0 (finite), zo[2] > 0 (src is then finite);
  sample:   v = the exact bilinear value of the stored template at src clamped to [0, B - 1], x0 = min(floor(sx),
            B - 2) (y0 likewise); the byte is floor(v + 1/2).
Every output comes with the margins of the decisions it rests on and the conditioning terms that tests/warp_cases.py
builds its error bounds from.  Two precisions run the same code: mpmath at 50 digits and np.longdouble; the first is the
definition, tests/test_warp_truth.py shows that the second agrees with it."""
import collections

import mpmath
import numpy as np

from consensus_truth import DPS, _Num, project, rotation_rrw

Truth = collections.namedtuple("Truth", [
    "src", "v", "byte", "valid",            # (B, B, 2) src; (B, B) v, byte (-1 where invalid), validity
    "tie_gap",                              # |v - (floor(v) + 1/2)|: how far v is from a rounding tie
    "p", "X",                               # (B, B, 2) the pixels p, (B, B, 3) the plane points
    "m_reach", "m_lam", "m_zo",             # margins: 1 - 2 kd1 |p - c|^2; the signed product of the cosines of nW
                                            # with (y - r) and with the ray (lam > 0 iff > 0); zo[2] / |X - xo|
    "k_plane", "k_num", "Xr", "Xo", "zo2",  # |nW| |dW| / |nW . dW|, |nW| |y - r| / |nW . (y - r)|, |X - r|, |X - xo|,
                                            # zo[2]
    "lam",                                  # the depth of X seen from xp (RRW(xp) (X - r) = lam z)
    "rho_p", "rho_g", "g",                  # undistorted radius of p (the Newton solution) and of Project(zo); |Project(zo)|
    "h", "ho", "rho_h", "rho_ho",           # the centres and their undistorted radii
    "y_r", "z2", "y_xo", "zo2_y",           # |y - r|, depth of y from xp, |y - xo|, depth of y from xo
])


def _floor(num):
    return np.vectorize(mpmath.floor, otypes=[object]) if num.prec == "mp" else np.floor


def _norm(v, num):
    return num.sqrt(sum(c * c for c in v))


def _undistorted(cam8, zc, num):
    fku, fkv = num(cam8[2]), num(cam8[3])
    return num.sqrt((fku * zc[..., 0] / zc[..., 2]) ** 2 + (fkv * zc[..., 1] / zc[..., 2]) ** 2)


def _inverse3(M, num):
    """The exact inverse of the 3 x 3 M (cofactors over the determinant, in the working precision)."""
    C = num.zeros((3, 3))
    for i in range(3):
        for j in range(3):
            r = [k for k in range(3) if k != i]
            c = [k for k in range(3) if k != j]
            C[i, j] = (-1) ** (i + j) * (M[r[0], c[0]] * M[r[1], c[1]] - M[r[0], c[1]] * M[r[1], c[0]])
    det = sum(M[0, j] * C[0, j] for j in range(3))
    return C.T / det


def solve_ray(cam8, p, num, iters=200):
    """The undistorted image-centred points u (..., 2) with u / sqrt(1 + 2 kd1 |u|^2) = p - c, by Newton's method
    from u = p - c, for the pixels inside the model's reach (mask returned); zeros elsewhere.  Raises if a residual is
    not at the working precision."""
    u0, v0, kd1 = num(cam8[4]), num(cam8[5]), num(cam8[6])
    t = np.stack([p[..., 0] - u0, p[..., 1] - v0], -1)
    reach = 1 - 2 * kd1 * (t[..., 0] ** 2 + t[..., 1] ** 2)
    inside = (reach > 0).astype(bool)
    t = np.where(inside[..., None], t, 0)
    U = t.copy()
    tol = mpmath.mpf(10) ** (-(DPS - 8)) if num.prec == "mp" else 64 * np.finfo(np.longdouble).eps
    for _ in range(iters):
        s2 = U[..., 0] ** 2 + U[..., 1] ** 2
        F = num.sqrt(1 + 2 * kd1 * s2)
        g = U / F[..., None] - t
        c = 2 * kd1 / F ** 3
        j00, j01, j11 = 1 / F - c * U[..., 0] ** 2, -c * U[..., 0] * U[..., 1], 1 / F - c * U[..., 1] ** 2
        det = j00 * j11 - j01 * j01
        step = np.stack([(j11 * g[..., 0] - j01 * g[..., 1]) / det, (j00 * g[..., 1] - j01 * g[..., 0]) / det], -1)
        U = U - step
        size = np.abs(step).max() / (1 + np.abs(U).max())
        if size <= tol * 1e-3:
            break
    F = num.sqrt(1 + 2 * kd1 * (U[..., 0] ** 2 + U[..., 1] ** 2))
    res = np.abs(U / F[..., None] - t).max(axis=-1) / (1 + np.abs(t).max(axis=-1))
    if not (res <= tol).all():
        raise ArithmeticError("Newton's method did not reach the working precision: residual %s" % float(res.max()))
    return U, reach, inside


def warp_truth(cam8, B, y, xo, xp, T=None, prec="ld"):
    """-> Truth of the B x B warp of the feature y (3) first seen from xo (7) at the camera pose xp (7); v and byte
    need the stored template T (B, B)."""
    num = _Num(prec)
    cam8 = np.asarray(cam8, np.float64)
    half = (B - 1) // 2
    f64 = num.f64
    with mpmath.workdps(DPS), np.errstate(invalid="ignore"):
        y_, xo_, xp_ = num(y), num(xo), num(xp)
        r, ro = xp_[0:3], xo_[0:3]
        R, Ro = rotation_rrw(xp_[3:7]), rotation_rrw(xo_[3:7])
        z = R @ (y_ - r)
        zoy = Ro @ (y_ - ro)
        h, ho = project(cam8, z, num), project(cam8, zoy, num)
        a, b = np.mgrid[0:B, 0:B]
        p = np.stack([h[0] + num(b - half), h[1] + num(a - half)], -1)
        U, reach, inside = solve_ray(cam8, p, num)
        zc = [-U[..., 0] / num(cam8[2]), -U[..., 1] / num(cam8[3]), num(np.ones((B, B)))]
        Minv = _inverse3(R, num)
        dW = [Minv[i, 0] * zc[0] + Minv[i, 1] * zc[1] + Minv[i, 2] * zc[2] for i in range(3)]
        nW = ro - y_
        d = y_ - r
        numer = nW @ d
        den = nW[0] * dW[0] + nW[1] * dW[1] + nW[2] * dW[2]
        nn, nd, ndW = _norm(nW, num), _norm(d, num), _norm(dW, num)
        m_lam = numer * den / (nn * nn * nd * ndW)
        m_lam = np.where(inside, m_lam, np.nan)
        lam_ok = inside & (m_lam > 0).astype(bool)
        lam = numer / np.where(lam_ok, den, 1)
        X = np.stack([r[i] + lam * dW[i] for i in range(3)], -1)
        e = X - ro
        zo = np.einsum("ij,abj->abi", Ro, e)
        Xo = _norm([e[..., i] for i in range(3)], num)
        m_zo = np.where(lam_ok, zo[..., 2] / np.where(lam_ok, Xo, 1), np.nan)
        valid = lam_ok & (m_zo > 0).astype(bool)
        zs = np.where(valid[..., None], zo, num(np.array([0.0, 0.0, 1.0])))
        gp = project(cam8, zs, num)
        src = np.stack([gp[..., 0] - ho[0] + half, gp[..., 1] - ho[1] + half], -1)
        out = dict(
            src=np.where(valid[..., None], f64(src), np.nan), valid=valid, p=f64(p),
            X=np.where(lam_ok[..., None], f64(X), np.nan),
            m_reach=f64(reach), m_lam=f64(m_lam), m_zo=f64(m_zo),
            k_plane=np.where(lam_ok, f64(nn * ndW / np.abs(np.where(lam_ok, den, 1))), np.nan),
            k_num=float(f64(nn * nd / abs(numer))) if numer != 0 else np.inf,
            Xr=np.where(lam_ok, f64(np.abs(lam) * ndW), np.nan), Xo=np.where(lam_ok, f64(Xo), np.nan),
            zo2=np.where(lam_ok, f64(zo[..., 2]), np.nan), lam=np.where(lam_ok, f64(lam), np.nan),
            rho_p=f64(num.sqrt(U[..., 0] ** 2 + U[..., 1] ** 2)),
            rho_g=np.where(valid, f64(_undistorted(cam8, zs, num)), np.nan),
            g=np.where(valid, f64(num.sqrt(gp[..., 0] ** 2 + gp[..., 1] ** 2)), np.nan),
            h=f64(h), ho=f64(ho), rho_h=float(f64(_undistorted(cam8, z, num))),
            rho_ho=float(f64(_undistorted(cam8, zoy, num))), y_r=float(f64(nd)), z2=float(f64(z[2])),
            y_xo=float(f64(_norm(y_ - ro, num))), zo2_y=float(f64(zoy[2])))
        v = byte = tie = None
        if T is not None:
            Tn = num(np.asarray(T, np.float64))
            sx = np.minimum(np.maximum(np.where(valid, src[..., 0], 0), 0), B - 1)
            sy = np.minimum(np.maximum(np.where(valid, src[..., 1], 0), 0), B - 1)
            fl = _floor(num)
            x0 = np.minimum(f64(fl(sx)).astype(np.int64), B - 2)
            y0 = np.minimum(f64(fl(sy)).astype(np.int64), B - 2)
            fx, fy = sx - num(x0), sy - num(y0)
            vv = ((1 - fy) * ((1 - fx) * Tn[y0, x0] + fx * Tn[y0, x0 + 1])
                  + fy * ((1 - fx) * Tn[y0 + 1, x0] + fx * Tn[y0 + 1, x0 + 1]))
            # v itself and its distance to the nearest k + 1/2, both rounded to FP64 only at the end
            byte = np.where(valid, f64(fl(vv + mpmath.mpf(1) / 2 if num.prec == "mp" else vv + 0.5)), -1).astype(np.int64)
            tie = np.abs(vv - (fl(vv) + (mpmath.mpf(1) / 2 if num.prec == "mp" else 0.5)))
            v = np.where(valid, f64(vv), np.nan)
            tie = np.where(valid, f64(tie), np.nan)
        out["v"], out["byte"], out["tie_gap"] = v, byte, (tie if T is not None else None)
    return Truth(**out)
