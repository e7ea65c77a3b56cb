"""Relocalisation (include/sl2b200.h, sl2_relocalise) restated in NumPy, steps 2-6, in the order of csrc/reloc.cu
reloc_kernel: bearings, the splitmix64 hypothesis sequence, Kneip's P3P, support, winner, Gauss-Newton refinement,
recount.  The inlier tests run the camera model of camera_ref one IEEE double operation at a time in the kernel's
order; the P3P, whose cube roots and trigonometry differ between libraries in the last bits, is followed up to
rounding.  Fed the device's matches, it gives the device's decisions whenever no squared distance lies within reach of
a last-bit difference of fl(tau * tau): `margin` says how far the closest one was."""
import math

import numpy as np

from camera_ref import camera_points, reprojection_d2, rrw

HYPOTHESES = 1024
GN_ITERS = 5
MASK64 = (1 << 64) - 1


def splitmix64(x):
    z = (x + 0x9E3779B97F4A7C15) & MASK64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & MASK64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & MASK64
    return z ^ (z >> 31)


def triple(h, k):
    """The three distinct match indices of hypothesis h among k >= 3 matches."""
    i0 = splitmix64(3 * h) % k
    i1 = splitmix64(3 * h + 1) % (k - 1)
    i2 = splitmix64(3 * h + 2) % (k - 2)
    if i1 >= i0:
        i1 += 1
    if i2 >= min(i0, i1):
        i2 += 1
    if i2 >= max(i0, i1):
        i2 += 1
    return i0, i1, i2


def unproject(cam8, z):
    """Camera::Unproject (camera.cpp:133-157) of the pixels z (k, 2), divided by its norm: unit bearings (k, 3)."""
    fku, fkv, u0, v0, kd1 = (float(v) for v in cam8[2:7])
    z = np.asarray(z, np.float64)
    c0, c1 = z[:, 0] - u0, z[:, 1] - v0
    radius2 = c0 * c0 + c1 * c1
    with np.errstate(invalid="ignore"):
        factor = np.sqrt(1.0 - 2.0 * kd1 * radius2)
    b = np.stack([(c0 / factor) / (-fku), (c1 / factor) / (-fkv), np.ones_like(c0)], axis=1)
    nb = np.sqrt(b[:, 0] * b[:, 0] + b[:, 1] * b[:, 1] + b[:, 2] * b[:, 2])
    return b / nb[:, None]


def _cubic_max_root(a, b, c):
    a3 = a / 3.0
    P, Q = b - a * a3, 2.0 * a3 * a3 * a3 - a3 * b + c
    D = 0.25 * Q * Q + P * P * P / 27.0
    if D > 0.0:
        sD = math.sqrt(D)
        t = np.cbrt(-0.5 * Q + sD) + np.cbrt(-0.5 * Q - sD)
    else:
        rr = math.sqrt(max(-P / 3.0, 0.0))
        cs = min(max(-0.5 * Q / (rr * rr * rr), -1.0), 1.0) if rr > 0.0 else 0.0
        t = 2.0 * rr * math.cos(math.acos(cs) / 3.0)
    m = float(t) - a3
    for _ in range(2):
        f, fp = ((m + a) * m + b) * m + c, (3.0 * m + 2.0 * a) * m + b
        if fp != 0.0:
            m -= f / fp
    return m


def quartic_roots(a):
    """Real roots of a[0] x^4 + ... + a[4] (Ferrari), in the kernel's order, Newton-polished."""
    if not abs(a[0]) > 0.0:
        return []
    B, C, D, E = a[1] / a[0], a[2] / a[0], a[3] / a[0], a[4] / a[0]
    BB = B * B
    p, q = C - 0.375 * BB, D - 0.5 * B * C + 0.125 * BB * B
    r = E - 0.25 * B * D + 0.0625 * BB * C - 3.0 / 256.0 * BB * BB
    m = _cubic_max_root(p, 0.25 * p * p - r, -0.125 * q * q)
    y = []
    if not m > 0.0:
        disc = p * p - 4.0 * r
        if disc >= 0.0:
            sd = math.sqrt(disc)
            for t2 in (0.5 * (-p + sd), 0.5 * (-p - sd)):
                if t2 >= 0.0:
                    y += [math.sqrt(t2), -math.sqrt(t2)]
    else:
        s = math.sqrt(2.0 * m)
        qs = q / (2.0 * s)
        for bq, cq in ((-s, 0.5 * p + m + qs), (s, 0.5 * p + m - qs)):
            disc = bq * bq - 4.0 * cq
            if disc >= 0.0:
                sd = math.sqrt(disc)
                y += [0.5 * (-bq + sd), 0.5 * (-bq - sd)]
    poly = lambda x: (((a[0] * x + a[1]) * x + a[2]) * x + a[3]) * x + a[4]  # noqa: E731
    out = []
    for yi in y:
        x = yi - 0.25 * B
        f = poly(x)
        for _ in range(3):
            fp = ((4.0 * a[0] * x + 3.0 * a[1]) * x + 2.0 * a[2]) * x + a[3]
            if not fp != 0.0:
                break
            xn = x - f / fp
            fn = poly(xn)
            if not abs(fn) < abs(f):
                break
            x, f = xn, fn
        out.append(x)
    return out


def rot_to_quat(R):
    """Row-major rotation -> unit quaternion (w, x, y, z), w >= 0 (Shepperd)."""
    tr = R[0][0] + R[1][1] + R[2][2]
    if tr > 0.0:
        s = 2.0 * math.sqrt(tr + 1.0)
        w, x, y, z = 0.25 * s, (R[2][1] - R[1][2]) / s, (R[0][2] - R[2][0]) / s, (R[1][0] - R[0][1]) / s
    elif R[0][0] > R[1][1] and R[0][0] > R[2][2]:
        s = 2.0 * math.sqrt(1.0 + R[0][0] - R[1][1] - R[2][2])
        w, x, y, z = (R[2][1] - R[1][2]) / s, 0.25 * s, (R[0][1] + R[1][0]) / s, (R[0][2] + R[2][0]) / s
    elif R[1][1] > R[2][2]:
        s = 2.0 * math.sqrt(1.0 + R[1][1] - R[0][0] - R[2][2])
        w, x, y, z = (R[0][2] - R[2][0]) / s, (R[0][1] + R[1][0]) / s, 0.25 * s, (R[1][2] + R[2][1]) / s
    else:
        s = 2.0 * math.sqrt(1.0 + R[2][2] - R[0][0] - R[1][1])
        w, x, y, z = (R[1][0] - R[0][1]) / s, (R[0][2] + R[2][0]) / s, (R[1][2] + R[2][1]) / s, 0.25 * s
    n = math.sqrt(w * w + x * x + y * y + z * z)
    if w < 0.0:
        n = -n
    return [w / n, x / n, y / n, z / n]


def p3p(Pw, fb):
    """Kneip, Scaramuzza, Siegwart (CVPR 2011): the poses xp = (r, qWR) (lists of 7) under which the world points
    Pw[i] lie along the unit camera-frame bearings fb[i]; [] for a degenerate triple; every pose finite."""
    P1, P2, P3 = (np.array(p, np.float64) for p in Pw)
    f1, f2, f3 = (np.array(f, np.float64) for f in fb)
    v1, v2 = P2 - P1, P3 - P1
    with np.errstate(all="ignore"):
        if not np.linalg.norm(np.cross(v1, v2)) > 1e-10 * np.linalg.norm(v1) * np.linalg.norm(v2):
            return []
        for a, c in ((f1, f2), (f1, f3), (f2, f3)):
            if not np.linalg.norm(np.cross(a, c)) > 1e-10:
                return []

        def frame(f1, f2):
            e3 = np.cross(f1, f2)
            e3 = e3 / np.linalg.norm(e3)
            T = np.stack([f1, np.cross(e3, f1), e3])
            return T, T @ f3

        T, f3t = frame(f1, f2)
        if f3t[2] > 0.0:
            f1, f2, P1, P2 = f2, f1, P2, P1
            T, f3t = frame(f1, f2)
        d_12 = float(np.linalg.norm(P2 - P1))
        n1 = (P2 - P1) / d_12
        d31 = P3 - P1
        n3 = np.cross(n1, d31)
        n3 = n3 / np.linalg.norm(n3)
        N = np.stack([n1, np.cross(n3, n1), n3])
        p_1, p_2 = float(N[0] @ d31), float(N[1] @ d31)
        f_1, f_2 = float(f3t[0] / f3t[2]), float(f3t[1] / f3t[2])
        cos_beta = float(f1 @ f2)
        b = 1.0 / (1.0 - cos_beta * cos_beta) - 1.0
        b = -math.sqrt(b) if cos_beta < 0.0 else math.sqrt(b)
        f_1_pw2, f_2_pw2, p_1_pw2, p_2_pw2 = f_1 * f_1, f_2 * f_2, p_1 * p_1, p_2 * p_2
        p_1_pw3, p_2_pw3 = p_1_pw2 * p_1, p_2_pw2 * p_2
        p_1_pw4, p_2_pw4 = p_1_pw3 * p_1, p_2_pw3 * p_2
        d_12_pw2, b_pw2 = d_12 * d_12, b * b
        fac = [
            -f_2_pw2 * p_2_pw4 - p_2_pw4 * f_1_pw2 - p_2_pw4,
            2 * p_2_pw3 * d_12 * b + 2 * f_2_pw2 * p_2_pw3 * d_12 * b - 2 * f_2 * p_2_pw3 * f_1 * d_12,
            -f_2_pw2 * p_2_pw2 * p_1_pw2 - f_2_pw2 * p_2_pw2 * d_12_pw2 * b_pw2 - f_2_pw2 * p_2_pw2 * d_12_pw2
            + f_2_pw2 * p_2_pw4 + p_2_pw4 * f_1_pw2 + 2 * p_1 * p_2_pw2 * d_12 + 2 * f_1 * f_2 * p_1 * p_2_pw2 * d_12 * b
            - p_2_pw2 * p_1_pw2 * f_1_pw2 + 2 * p_1 * p_2_pw2 * f_2_pw2 * d_12 - p_2_pw2 * d_12_pw2 * b_pw2
            - 2 * p_1_pw2 * p_2_pw2,
            2 * p_1_pw2 * p_2 * d_12 * b + 2 * f_2 * p_2_pw3 * f_1 * d_12 - 2 * f_2_pw2 * p_2_pw3 * d_12 * b
            - 2 * p_1 * p_2 * d_12_pw2 * b,
            -2 * f_2 * p_2_pw2 * f_1 * p_1 * d_12 * b + f_2_pw2 * p_2_pw2 * d_12_pw2 + 2 * p_1_pw3 * d_12
            - p_1_pw2 * d_12_pw2 + f_2_pw2 * p_2_pw2 * p_1_pw2 - p_1_pw4 - 2 * f_2_pw2 * p_2_pw2 * p_1 * d_12
            + p_2_pw2 * f_1_pw2 * p_1_pw2 + f_2_pw2 * p_2_pw2 * d_12_pw2 * b_pw2,
        ]
        out = []
        for cos_theta in quartic_roots(fac):
            cot_alpha = (-f_1 * p_1 / f_2 - cos_theta * p_2 + d_12 * b) / (-f_1 * cos_theta * p_2 / f_2 + p_1 - d_12)
            sin_theta = math.sqrt(1.0 - cos_theta * cos_theta) if cos_theta * cos_theta <= 1.0 else math.nan
            sin_alpha = math.sqrt(1.0 / (cot_alpha * cot_alpha + 1.0))
            cos_alpha = math.sqrt(1.0 - sin_alpha * sin_alpha)
            if cot_alpha < 0.0:
                cos_alpha = -cos_alpha
            k1 = d_12 * sin_alpha * (sin_alpha * b + cos_alpha)
            Cn = np.array([d_12 * cos_alpha * (sin_alpha * b + cos_alpha), cos_theta * k1, sin_theta * k1])
            Rn = np.array([[-cos_alpha, -sin_alpha * cos_theta, -sin_alpha * sin_theta],
                           [sin_alpha, -cos_alpha * cos_theta, -cos_alpha * sin_theta],
                           [0.0, -sin_theta, cos_theta]])
            r = P1 + N.T @ Cn
            q = rot_to_quat((N.T @ Rn.T @ T).tolist())
            xp = list(r) + q
            if all(math.isfinite(v) for v in xp):
                out.append(xp)
    return out


def project(cam8, xp, y):
    """h and dh/dz (Camera::ProjectionJacobian) of the points y (k, 3) seen from xp, for the refinement."""
    fku, fkv, u0, v0, kd1 = (float(v) for v in cam8[2:7])
    zc = camera_points(xp, y)
    uc, vc = -fku * zc[:, 0] / zc[:, 2], -fkv * zc[:, 1] / zc[:, 2]
    r2 = uc * uc + vc * vc
    distor = 1.0 + 2.0 * kd1 * r2
    f = np.sqrt(distor)
    h = np.stack([uc / f + u0, vc / f + v0], axis=1)
    du = np.zeros((len(y), 2, 3))
    du[:, 0, 0] = -fku / zc[:, 2]
    du[:, 0, 2] = fku / zc[:, 2] * zc[:, 0] / zc[:, 2]
    du[:, 1, 1] = -fkv / zc[:, 2]
    du[:, 1, 2] = fkv / zc[:, 2] * zc[:, 1] / zc[:, 2]
    dh = np.einsum("ki,kj->kij", np.stack([uc, vc], 1), np.stack([uc, vc], 1)) * (-2.0 * kd1 / (f * distor))[:, None, None]
    dh += np.eye(2)[None] / f[:, None, None]
    return h, np.einsum("kij,kjl->kil", dh, du), zc


def quat_mul(a, b):
    aw, ax, ay, az = a
    bw, bx, by, bz = b
    return [aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
            aw * by + ay * bw + az * bx - ax * bz, aw * bz + az * bw + ax * by - ay * bx]


def refine(cam8, xp, y, z):
    """GN_ITERS Gauss-Newton steps over (dr, dtheta) with RWR' = RWR Exp(dtheta), on the matches y, z."""
    xp = [float(v) for v in xp]
    for _ in range(GN_ITERS):
        h, J, zc = project(cam8, xp, y)
        RRW = np.array(rrw(xp))
        Zx = np.zeros((len(y), 3, 3))
        Zx[:, 0, 1], Zx[:, 0, 2] = -zc[:, 2], zc[:, 1]
        Zx[:, 1, 0], Zx[:, 1, 2] = zc[:, 2], -zc[:, 0]
        Zx[:, 2, 0], Zx[:, 2, 1] = -zc[:, 1], zc[:, 0]
        A = np.concatenate([-J @ RRW, J @ Zx], axis=2)  # (k, 2, 6)
        e = z - h
        H = np.einsum("kri,krj->ij", A, A)
        g = np.einsum("kri,kr->i", A, e)
        try:
            L = np.linalg.cholesky(H)
        except np.linalg.LinAlgError:
            break
        d = np.linalg.solve(L.T, np.linalg.solve(L, g))
        ang = float(np.linalg.norm(d[3:]))
        sc = math.sin(0.5 * ang) / ang if ang > 0.0 else 0.5
        q = quat_mul(xp[3:7], [math.cos(0.5 * ang), sc * d[3], sc * d[4], sc * d[5]])
        n = math.sqrt(sum(v * v for v in q))
        if q[0] < 0.0:
            n = -n
        new = [xp[i] + d[i] for i in range(3)] + [v / n for v in q]
        if not all(math.isfinite(v) for v in new):
            break
        xp = new
    return xp


def relocalise(cam8, y, z, tau, min_inliers):
    """Steps 2-6 for the k matches (y (k, 3) map points, z (k, 2) match pixels, in feature-index order).  Returns a
    dict: support (per (hypothesis, pose) index), win (index or -1), win_sup, win_mask, pose (refined; NaN without a
    hypothesis), mask (inliers of the refined pose), inliers, rms, status, margin (the smallest |d2 - fl(tau tau)|
    of every inlier decision taken)."""
    y = np.asarray(y, np.float64).reshape(-1, 3)
    z = np.asarray(z, np.float64).reshape(-1, 2)
    k = len(y)
    t2 = float(tau) * float(tau)
    fb = unproject(cam8, z) if k else np.zeros((0, 3))
    margin = np.inf
    support = {}
    win, win_sup, win_pose = -1, -1, None

    def decide(xp):
        nonlocal margin
        d2 = reprojection_d2(cam8, xp, y, z)
        ok = ~np.isnan(d2)
        if ok.any():
            margin = min(margin, float(np.abs(d2[ok] - t2).min()))
        return ok & (np.nan_to_num(d2, nan=np.inf) <= t2), d2

    if k >= 3:
        for h in range(HYPOTHESES):
            t = triple(h, k)
            for s, xp in enumerate(p3p(y[list(t)], fb[list(t)])):
                m, _ = decide(xp)
                idx = 4 * h + s
                support[idx] = int(m.sum())
                if support[idx] > win_sup:
                    win, win_sup, win_pose = idx, support[idx], xp
    out = dict(support=support, win=win, win_sup=max(win_sup, 0), k=k)
    if win < 0:
        out.update(win_mask=np.zeros(k, bool), pose=np.full(7, np.nan), mask=np.zeros(k, bool), inliers=0,
                   rms=math.nan, status=0, margin=margin)
        return out
    wm, _ = decide(win_pose)
    pose = refine(cam8, win_pose, y[wm], z[wm])
    mask, d2 = decide(pose)
    n = int(mask.sum())
    out.update(win_mask=wm, win_pose=np.array(win_pose), pose=np.array(pose), mask=mask, inliers=n,
               rms=math.sqrt(float(d2[mask].sum()) / n) if n else math.nan, status=int(n >= min_inliers),
               margin=margin)
    return out
