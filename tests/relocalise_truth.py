"""Relocalisation (include/sl2b200.h, sl2_relocalise, steps 2-6) from the header's words, in extended precision
(np.longdouble; the same code in mpmath at 50 digits checks it).  None of the kernel's algorithms or operation order is
reused: the P3P is Grunert's, not Kneip's, and the model is the one of tests/rescue_truth.py.

  bearings    Camera::Unproject (camera.cpp:133-157) of the match pixel z_j, divided by its norm.
  P3P         the signed depths s_i along the three bearings with s_i^2 + s_j^2 - 2 s_i s_j cos th_ij = |P_i - P_j|^2
              (law of cosines; Grunert 1841).  s2 = u s1, s3 = v s1 turn the equations into two conics in (u, v)
              whose difference is linear in u; u put back leaves a quartic in v, formed by polynomial arithmetic and
              solved by mpmath.polyroots.  Each solution is substituted into the three equations.  The pose aligns
              the orthonormal frames of the world triangle and of the camera triangle s_i f_i.  A double root (the
              danger cylinder) is reported and has an infinite bound.  The poses with every s_i > 0 are "physical".
              The others (s and -s of each root) put one or more of the triple's own points behind the camera; the
              header's P3P (Kneip's) returns some of them, one of each pair, chosen by its geometry, so they are
              possible poses: each is scored, and one that reaches the largest support may win.
  support     match j is an inlier of a pose when the model puts y_j at depth > 0 and |z_j - h_j|^2 <= fl(tau * tau);
              every decision carries its margin |d2 - fl(tau * tau)|.
  winner      the largest support of a physical pose; among the hypotheses reaching it the lowest h (the triples of
              relocalise_ref.triple, integer arithmetic pinned by a SHA-256).  When two poses of that h reach it, the
              header's rule picks by the order of the P3P's roots: both are candidates ("order-decided"); so is every
              non-physical pose of a lower h that reaches it.  A non-physical pose above it leaves the largest support
              undecided.
  refinement  GN_ITERS Gauss-Newton steps over (dr, dtheta): r' = r + dr, q' = q Exp(dtheta) (body frame), on the
              winner's inliers, stopping when the 6 x 6 normal matrix is not positive definite.  The least-squares
              minimiser (the same steps to convergence) is given beside it.
  recount     inliers, rms and status at the refined pose.

Bounds: how far a double-precision evaluation of the same steps may lie from this truth.
  pose        of a P3P pose: P3P_C u kappa, kappa = ((1 + |J^-1| F) (1 + s_max / e_min) + |P|_max) (1 + 1 / sin_t),
              with J = dF/ds of the law-of-cosines system, F the size of its terms, s the depths, e_min the
              triangle's shortest side and sin_t the smallest sine of the angle between the triangle's plane and the
              plane through one of its edges and the camera (the angle Kneip's parametrisation solves for: its
              cos(theta) carries that angle 1 / sin(theta) times less precisely).  P3P_C is measured
              (tests/test_relocalise_truth.py asserts the worst error over the bound is at most 1).
  final       twice the winner's pose bound times how far the refinement carries it (the largest change of the refined
              pose over the change of its start, the start moved by that bound along each coordinate; 1 when the
              refinement stopped early) plus GN_C u cond(N) max(1, |r|, |y|_max), N the normal matrix at the refined
              pose.
  decision    a pose bound b pushed through the model's Jacobian A (2 x 6, over (dr, dtheta)): dh = 2 sqrt(6) |A| b
              + 64 u (|h| + |z|), and |d2 - d2~| <= 2 sqrt(d2) dh + dh^2 + 8 u max(d2, tau^2)."""
import math
import multiprocessing
import os

import mpmath
import numpy as np

from relocalise_ref import GN_ITERS, HYPOTHESES, triple
from rescue_truth import U, Ext, Mp, model

DPS = 50
P3P_C = 2.0 ** 16
GN_C = 2.0 ** 10
WORKERS = min(16, os.cpu_count() or 1)  # processes for the P3Ps of a scene's distinct triples
COLLINEAR = 1e-12  # |(P2 - P1) x (P3 - P1)| <= COLLINEAR |P2 - P1| |P3 - P1|: collinear up to the map's rounding
KERNEL_DEGENERATE = 1e-10  # the kernel's tolerance for collinear points and parallel bearings


class MpV(Mp):
    """mpmath at DPS digits, element-wise over object arrays"""

    def sqrt(self, v):
        if isinstance(v, np.ndarray):
            return np.frompyfunc(self.mp.sqrt, 1, 1)(v)
        return self.mp.sqrt(v)


def _trig(ar):
    return (np.cos, np.sin) if ar is Ext else (mpmath.cos, mpmath.sin)


def _to(ar, vals):
    """mpf or float values into the arithmetic of ar, without rounding through double"""
    vals = list(vals)
    if ar is Ext:
        return np.array([np.longdouble(mpmath.nstr(mpmath.mpf(v), 30)) for v in vals], dtype=np.longdouble)
    return np.array([mpmath.mpf(v) for v in vals], dtype=object)


@mpmath.workdps(DPS)
def bearings_mp(cam8, z):
    """Unit bearings (mpf 3-lists) of the pixels z (k, 2)."""
    fku, fkv, u0, v0, kd1 = (mpmath.mpf(float(v)) for v in cam8[2:7])
    out = []
    for zu, zv in np.asarray(z, np.float64).reshape(-1, 2):
        c0, c1 = mpmath.mpf(float(zu)) - u0, mpmath.mpf(float(zv)) - v0
        f = mpmath.sqrt(1 - 2 * kd1 * (c0 * c0 + c1 * c1))
        b = [c0 / f / (-fku), c1 / f / (-fkv), mpmath.mpf(1)]
        n = mpmath.sqrt(sum(x * x for x in b))
        out.append([x / n for x in b])
    return out


# ---- P3P from the law of cosines -------------------------------------------------------------------------------------
def _pmul(a, b):
    o = [mpmath.mpf(0)] * (len(a) + len(b) - 1)
    for i, x in enumerate(a):
        for j, y in enumerate(b):
            o[i + j] += x * y
    return o


def _padd(*ps):
    n = max(len(p) for p in ps)
    return [sum((p[i] if i < len(p) else 0) for p in ps) for i in range(n)]


def _sub(a, b):
    return [a[i] - b[i] for i in range(3)]


def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _unit(a):
    n = mpmath.sqrt(_dot(a, a))
    return [x / n for x in a]


def _frame(A, B, C):
    """columns e1 = (B - A) / |.|, e3 = e1 x (C - A) / |.|, e2 = e3 x e1"""
    e1 = _unit(_sub(B, A))
    e3 = _unit(_cross(e1, _sub(C, A)))
    e2 = _cross(e3, e1)
    return [[e1[i], e2[i], e3[i]] for i in range(3)]


def rot_to_quat_mp(R):
    """unit quaternion (w, x, y, z), w >= 0, of the rotation R (largest of the four pivots)"""
    t = [1 + R[0][0] + R[1][1] + R[2][2], 1 + R[0][0] - R[1][1] - R[2][2], 1 - R[0][0] + R[1][1] - R[2][2],
         1 - R[0][0] - R[1][1] + R[2][2]]
    i = max(range(4), key=lambda a: t[a])
    s = 2 * mpmath.sqrt(t[i])
    if i == 0:
        q = [s / 4, (R[2][1] - R[1][2]) / s, (R[0][2] - R[2][0]) / s, (R[1][0] - R[0][1]) / s]
    elif i == 1:
        q = [(R[2][1] - R[1][2]) / s, s / 4, (R[0][1] + R[1][0]) / s, (R[0][2] + R[2][0]) / s]
    elif i == 2:
        q = [(R[0][2] - R[2][0]) / s, (R[0][1] + R[1][0]) / s, s / 4, (R[1][2] + R[2][1]) / s]
    else:
        q = [(R[1][0] - R[0][1]) / s, (R[0][2] + R[2][0]) / s, (R[1][2] + R[2][1]) / s, s / 4]
    return [-v for v in q] if q[0] < 0 else q


@mpmath.workdps(DPS)
def p3p(Pw, fb):
    """The poses (r, q) under which the world points Pw (3 x 3 doubles) lie on the lines of the unit bearings fb
    (3 mpf 3-lists).  Returns (poses, double_root): poses a list of dicts pose (7 mpf), s (3 signed depths), physical
    (every s_i > 0), bound (a pose bound, inf at a double root), residual (largest |law of cosines| / its scale),
    near_degenerate (the triple lies within the kernel's degeneracy tolerances)."""
    P = [[mpmath.mpf(float(v)) for v in p] for p in Pw]
    f = fb
    a2, b2, c2 = (_dot(_sub(P[i], P[j]), _sub(P[i], P[j])) for i, j in ((1, 2), (0, 2), (0, 1)))
    ca, cb, cg = _dot(f[1], f[2]), _dot(f[0], f[2]), _dot(f[0], f[1])
    # the header's degenerate triples give no pose: coincident or collinear points (up to the rounding of the map
    # points to double) and coincident bearings
    nrm = _cross(_sub(P[1], P[0]), _sub(P[2], P[0]))
    if min(a2, b2, c2) == 0 or _dot(nrm, nrm) <= COLLINEAR ** 2 * b2 * c2:
        return [], False
    fx = min(_dot(c, c) for c in (_cross(f[0], f[1]), _cross(f[0], f[2]), _cross(f[1], f[2])))
    if fx == 0:
        return [], False
    # the header gives no tolerance; the kernel drops triples within KERNEL_DEGENERATE (relative for the points,
    # absolute for the unit bearings), so their poses are marked and counted apart
    near_degenerate = _dot(nrm, nrm) <= KERNEL_DEGENERATE ** 2 * b2 * c2 or fx <= KERNEL_DEGENERATE ** 2
    Q = [mpmath.mpf(1), -2 * cb, mpmath.mpf(1)]                  # 1 + v^2 - 2 v cos(beta)
    num = _padd([b2], [-c2 * x for x in Q], [a2 * x for x in Q], [0, 0, -b2])
    den = [-2 * b2 * cg, 2 * b2 * ca]                              # u = -num / den
    quart = _padd([b2 * x for x in _pmul(num, num)], [2 * b2 * cg * x for x in _pmul(num, den)],
                  _pmul(_padd([b2], [-c2 * x for x in Q]), _pmul(den, den)))
    scale = max(abs(x) for x in quart)
    while len(quart) > 1 and abs(quart[-1]) <= mpmath.mpf(10) ** -40 * scale:
        quart.pop()
    if len(quart) < 2:
        return [], False
    roots = mpmath.polyroots(list(reversed(quart)), maxsteps=200, extraprec=2 * DPS * 4)
    close = mpmath.mpf(10) ** (-DPS // 3)
    double_root = any(abs(roots[i] - roots[j]) <= close * max(1, abs(roots[i]))
                      for i in range(len(roots)) for j in range(i))
    out = []
    for v in roots:
        if abs(mpmath.im(v)) > close * max(1, abs(v)):
            continue
        v = mpmath.re(v)
        dv = den[0] + den[1] * v
        if dv == 0:
            continue
        u = -(num[0] + num[1] * v + num[2] * v * v) / dv
        q2 = 1 + v * v - 2 * v * cb
        if not q2 > 0:
            continue
        s1 = mpmath.sqrt(b2 / q2)
        for sg in (1, -1):
            out.append(dict(_pose(P, f, [sg * s1, sg * u * s1, sg * v * s1], (a2, b2, c2), (ca, cb, cg), double_root),
                            near_degenerate=near_degenerate))
    return out, double_root


def _pose(P, f, s, d2s, cs, double_root):
    """the pose of the signed depths s, checked against the law of cosines, and its bound"""
    a2, b2, c2 = d2s
    ca, cb, cg = cs
    # substitute into the three equations
    res, Fs = 0, 0
    for (i, j, d2, c) in ((0, 1, c2, cg), (0, 2, b2, cb), (1, 2, a2, ca)):
        res = max(res, abs(s[i] ** 2 + s[j] ** 2 - 2 * s[i] * s[j] * c - d2))
        Fs = max(Fs, s[i] ** 2 + s[j] ** 2 + 2 * s[i] * s[j] * abs(c) + d2)
    assert res <= mpmath.mpf(10) ** (-DPS // 2) * Fs, (res, Fs)
    X = [[f[i][a] * s[i] for a in range(3)] for i in range(3)]
    FP, FX = _frame(*P), _frame(*X)
    R = [[sum(FP[a][m] * FX[c][m] for m in range(3)) for c in range(3)] for a in range(3)]
    r = [P[0][a] - sum(R[a][c] * X[0][c] for c in range(3)) for a in range(3)]
    # bound from the condition of the law-of-cosines system at s
    J = mpmath.matrix([[2 * s[0] - 2 * s[1] * cg, 2 * s[1] - 2 * s[0] * cg, 0],
                       [2 * s[0] - 2 * s[2] * cb, 0, 2 * s[2] - 2 * s[0] * cb],
                       [0, 2 * s[1] - 2 * s[2] * ca, 2 * s[2] - 2 * s[1] * ca]])
    try:
        Jinv = mpmath.norm(mpmath.inverse(J), 2)
    except ZeroDivisionError:
        Jinv = mpmath.inf
    e_min = mpmath.sqrt(min(a2, b2, c2))
    Pmax = max(abs(x) for p in P for x in p)
    # the camera's elevation over the triangle's plane, seen from each edge: sin(theta) of the plane through the
    # edge and the camera against the triangle's plane (the angle Kneip's parametrisation solves for)
    sin_t = mpmath.inf
    for i, j, m in ((0, 1, 2), (0, 2, 1), (1, 2, 0)):
        n1 = _unit(_sub(P[j], P[i]))
        n3 = _unit(_cross(n1, _sub(P[m], P[i])))
        n2 = _cross(n3, n1)
        w = _sub(r, P[i])
        a, b = _dot(w, n2), _dot(w, n3)
        sin_t = min(sin_t, abs(b) / mpmath.sqrt(a * a + b * b))
    kappa = ((1 + Jinv * Fs) * (1 + max(abs(v) for v in s) / e_min) + Pmax) * (1 + 1 / sin_t)
    bound = math.inf if double_root else float(P3P_C * U * kappa)
    return dict(pose=r + rot_to_quat_mp(R), s=s, physical=min(s) > 0, bound=bound, residual=float(res / Fs))


# ---- support, refinement, recount -----------------------------------------------------------------------------------
def evaluate(ar, cam8, pose, Y, Z, t2):
    """d2 (k,), depth (k,) and A (k, 2, 6) of the matches Y (3, k), Z (2, k) (both in ar) at pose (7, in ar)."""
    h, Hxp, _, _, depth = model(ar, cam8, pose, Y)
    w, x, y, z = pose[3], pose[4], pose[5], pose[6]
    L = [[w, -x, -y, -z], [x, w, -z, y], [y, z, w, -x], [z, -y, x, w]]  # q (x) p = L(q) p
    k = Y.shape[1]
    A = np.empty((k, 2, 6), dtype=Y.dtype)
    for rr in range(2):
        for c in range(3):
            A[:, rr, c] = Hxp[rr][c]
            A[:, rr, 3 + c] = sum(Hxp[rr][3 + m] * L[m][1 + c] for m in range(4)) / 2
    e = [Z[0] - h[0], Z[1] - h[1]]
    return e[0] * e[0] + e[1] * e[1], depth, A, e, h


def _chol_solve(ar, N, g):
    """N^-1 g for the 6 x 6 N, or None when N is not positive definite"""
    n = len(g)
    L = [[0] * n for _ in range(n)]
    for j in range(n):
        s = N[j][j] - sum(L[j][m] * L[j][m] for m in range(j))
        if not s > 0:
            return None
        L[j][j] = ar.sqrt(s)
        for i in range(j + 1, n):
            L[i][j] = (N[i][j] - sum(L[i][m] * L[j][m] for m in range(j))) / L[j][j]
    y = [0] * n
    for i in range(n):
        y[i] = (g[i] - sum(L[i][m] * y[m] for m in range(i))) / L[i][i]
    d = [0] * n
    for i in reversed(range(n)):
        d[i] = (y[i] - sum(L[m][i] * d[m] for m in range(i + 1, n))) / L[i][i]
    return d


def gn_step(ar, cam8, pose, Y, Z, t2):
    """One Gauss-Newton step; (new pose, N) or (None, N) when N is not positive definite."""
    _, _, A, e, _ = evaluate(ar, cam8, pose, Y, Z, t2)
    N = [[(A[:, :, a] * A[:, :, b]).sum() for b in range(6)] for a in range(6)]
    g = [(A[:, 0, a] * e[0] + A[:, 1, a] * e[1]).sum() for a in range(6)]
    d = _chol_solve(ar, N, g)
    if d is None:
        return None, N
    cos, sin = _trig(ar)
    ang = ar.sqrt(d[3] * d[3] + d[4] * d[4] + d[5] * d[5])
    sc = sin(ang / 2) / ang if ang > 0 else ar.conv(np.array(0.5))[()]
    dq = [cos(ang / 2), sc * d[3], sc * d[4], sc * d[5]]
    w, x, y, z = pose[3:7]
    q = [w * dq[0] - x * dq[1] - y * dq[2] - z * dq[3], w * dq[1] + x * dq[0] + y * dq[3] - z * dq[2],
         w * dq[2] + y * dq[0] + z * dq[1] - x * dq[3], w * dq[3] + z * dq[0] + x * dq[2] - y * dq[1]]
    n = ar.sqrt(sum(v * v for v in q))
    if q[0] < 0:
        n = -n
    out = np.array([pose[i] + d[i] for i in range(3)] + [v / n for v in q], dtype=pose.dtype)
    return out, N


def refine(ar, cam8, pose, Y, Z, t2, iters=GN_ITERS):
    """iters Gauss-Newton steps (stopping when N is not positive definite): pose, N at the last pose, steps taken."""
    done = 0
    for _ in range(iters):
        new, _ = gn_step(ar, cam8, pose, Y, Z, t2)
        if new is None:
            break
        pose, done = new, done + 1
    _, _, A, _, _ = evaluate(ar, cam8, pose, Y, Z, t2)
    N = np.array([[float((A[:, :, a] * A[:, :, b]).sum()) for b in range(6)] for a in range(6)])
    return pose, N, done


def decisions(ar, cam8, pose, Y, Z, t2, bound):
    """inlier mask, margins |d2 - t2|, decision bounds and d2 at pose under the pose bound `bound`"""
    d2, depth, A, _, h = evaluate(ar, cam8, pose, Y, Z, t2)
    d2f = np.array([float(v) for v in d2])
    front = np.array([bool(v > 0) for v in depth], bool)
    mask = front & np.array([bool(v <= t2) for v in d2], bool)
    margin = np.where(front, np.abs(d2f - float(t2)), np.inf)
    Af = np.sqrt((np.array([[float(v) for v in a.ravel()] for a in A]).reshape(-1, 12) ** 2).sum(1))
    mag = np.array([abs(float(h[0][j])) + abs(float(h[1][j])) + abs(float(Z[0][j])) + abs(float(Z[1][j]))
                    for j in range(len(d2f))])
    dh = 2 * math.sqrt(6) * Af * bound + 64 * U * mag
    dbound = 2 * np.sqrt(d2f) * dh + dh * dh + 8 * U * np.maximum(d2f, float(t2))
    return mask, margin, dbound, d2f


def _p3p_of(args):
    y, z, fb, srt = args
    return p3p(y[list(srt)], [fb[i] for i in srt])


def truth(cam8, y, z, tau, min_inliers, ar=Ext, cache=None, hypotheses=HYPOTHESES, lsq=True):
    """Steps 2-6 for the matches y (k, 3), z (k, 2) in feature-index order.  Returns a dict:
    hyps[h] = list of P3P poses (dicts: pose (7 mpf), pose_f, bound, mask, margin, dbound, lo, hi: the support counting
    only the decisions outside their bounds, and counting them all);
    max_lo / max_hi (largest lo / hi support of a physical pose), decided (max_lo == max_hi, the winning hypothesis is
    the same under both and no non-physical pose may score more), win (lowest h at the largest support, -1 without a
    pose), win_hs (the hypotheses that may win: win and those below it whose non-physical poses reach max_lo),
    order_decided (more than one candidate);
    cands: per candidate winning pose (distinct starts), the refined pose (float and ar), its bound, mask, margin, dbound, inliers,
    rms, status, gn_steps, cond (of N), lsq (the minimiser) and gn_gap (|refined - minimiser|);
    double_roots: the hypotheses with a double root."""
    y = np.asarray(y, np.float64).reshape(-1, 3)
    z = np.asarray(z, np.float64).reshape(-1, 2)
    k = len(y)
    t2f = float(tau) * float(tau)
    cache = {} if cache is None else cache
    with mpmath.workdps(DPS):
        t2 = _to(ar, [t2f])[0]
        Y = ar.conv(y.T) if ar is Ext else _to(ar, y.T.ravel()).reshape(3, k)
        Z = ar.conv(z.T) if ar is Ext else _to(ar, z.T.ravel()).reshape(2, k)
        fb = bearings_mp(cam8, z)
        hs = list(range(hypotheses if k >= 3 else 0))
        keys = {}
        for h in hs:
            srt = sorted(triple(h, k))
            keys[h] = (np.asarray(cam8, np.float64).tobytes(), y[srt].tobytes(), z[srt].tobytes(), tuple(srt))
        todo = sorted({v for v in keys.values() if v not in cache}, key=lambda v: v[3])
        if ar is Ext and len(todo) > 64 and WORKERS > 1:  # the P3Ps of distinct triples, in worker processes
            with multiprocessing.get_context("spawn").Pool(WORKERS) as pool:  # no fork of a CUDA process
                for key, res in zip(todo, pool.map(_p3p_of, [(y, z, fb, key[3]) for key in todo], chunksize=16)):
                    cache[key] = res
        for key in todo:
            if key not in cache:
                cache[key] = _p3p_of((y, z, fb, key[3]))
        hyps, double_roots = [], []
        for h in hs:
            poses, dr = cache[keys[h]]
            if dr:
                double_roots.append(h)
            row = []
            for p in poses:
                pa = _to(ar, p["pose"])
                mask, margin, dbound, _ = decisions(ar, cam8, pa, Y, Z, t2, p["bound"])
                sure = margin > dbound
                row.append(dict(p, pose_f=np.array([float(v) for v in p["pose"]]), pose_a=pa, mask=mask,
                                margin=margin, dbound=dbound, lo=int((mask & sure).sum()), hi=int((mask | ~sure).sum())))
            hyps.append(row)
        out = dict(k=k, t2=t2f, hyps=hyps, double_roots=double_roots, cands=[], win=-1, order_decided=False)
        phys = [(h, p) for h, row in enumerate(hyps) for p in row if p["physical"]]
        if not phys:
            out.update(max_lo=0, max_hi=0, decided=True)
            return out
        max_lo, max_hi = max(p["lo"] for _, p in phys), max(p["hi"] for _, p in phys)
        win = next(h for h, p in phys if p["lo"] == max_lo)
        win_hi = next(h for h, p in phys if p["hi"] == max_hi)
        above = any(p["hi"] > max_lo for row in hyps for p in row if not p["physical"])
        out.update(max_lo=max_lo, max_hi=max_hi, win=win, decided=max_lo == max_hi and win == win_hi and not above)
        winners = [(h, s, p) for h in range(win + 1) for s, p in enumerate(hyps[h])
                   if p["lo"] == max_lo and (p["physical"] or h < win)]
        out["order_decided"] = len(winners) > 1
        out["win_hs"] = sorted({h for h, _, _ in winners})
        for h, s, p in winners:
            if any(rt_same(p["pose_f"], c["start"]) and (p["mask"] == c["win_mask"]).all() for c in out["cands"]):
                continue  # the same start: the same refinement
            m = p["mask"]
            Yi, Zi = Y[:, m], Z[:, m]
            pose, N, steps = refine(ar, cam8, p["pose_a"], Yi, Zi, t2)
            cond = float(np.linalg.cond(N)) if steps or m.sum() >= 3 else math.inf
            scale = max(1.0, float(np.abs(p["pose_f"][:3]).max()), float(np.abs(y).max()))
            # how far the refinement carries an error of the start: the start moved by its bound along each
            # coordinate, refined again (the steps contract it, quadratically when the residuals vanish)
            carry = 1.0
            if math.isfinite(p["bound"]) and steps == GN_ITERS:
                carry = 0.0
                pf = np.array([float(v) for v in pose])
                for a in range(7):
                    for sg in (1, -1):
                        st = p["pose_a"].copy()
                        st[a] = st[a] + sg * p["bound"]
                        pe = np.array([float(v) for v in refine(ar, cam8, st, Yi, Zi, t2)[0]])
                        carry = max(carry, pose_distance(pe, pf) / p["bound"])
            bound = 2 * carry * p["bound"] + GN_C * U * cond * scale
            mask, margin, dbound, d2 = decisions(ar, cam8, pose, Y, Z, t2, bound)
            n = int(mask.sum())
            c = dict(index=4 * h + s, start=p["pose_f"], pose=np.array([float(v) for v in pose]), pose_a=pose,
                     bound=bound, mask=mask, margin=margin, dbound=dbound, inliers=n, d2=d2,
                     rms=math.sqrt(float(d2[mask].sum()) / n) if n else math.nan, status=int(n >= min_inliers),
                     min_inliers=min_inliers,
                     gn_steps=steps, cond=cond, win_mask=m)
            if lsq:
                lp, _, lsteps = refine(ar, cam8, pose, Yi, Zi, t2, iters=20)
                c["lsq"] = np.array([float(v) for v in lp])
                c["gn_gap"] = pose_distance(c["pose"], c["lsq"])
            out["cands"].append(c)
        return out


def rt_same(a, b):
    return pose_distance(a, b) <= 1e-13


def pose_distance(a, b):
    """max |r - r'|, min over the sign of q of max |q -+ q'|: quaternions compared as rotations"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    dq = min(np.abs(a[3:7] - b[3:7]).max(), np.abs(a[3:7] + b[3:7]).max())
    return max(float(np.abs(a[:3] - b[:3]).max()), float(dq))
