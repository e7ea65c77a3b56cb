"""The exposure blur (include/sl2b200.h, sl2_set_stream_blur; csrc/warp.cu blur_setup, blur_job; csrc/sl2_model.cuh
quat_from_angular_velocity, patch_ray_source, patch_bilinear) restated in NumPy, one IEEE double operation at a time in
the kernel's order (NumPy's element-wise operations and Python's float operations are correctly rounded and never
fused), vectorised over the template's pixels, on top of tests/warp_ref.py and tests/normals_ref.py.

The pose at time s uses the host's sin and cos by default; the GPU tests pass `pose_fn` with the device's own poses
(the device's sin and cos need not round like the host's).  The keyword arguments `swap_order`, `centre_at_s`,
`round_samples` and `half_step` make the broken copies the tests must catch."""
import math

import numpy as np

from camera_ref import camera_points, project_point, rrw
from normals_ref import basis, normal
from warp_ref import adjugate, unproject_point

MAX_SAMPLES = 32


def _dot(a, b):
    return ((0.0 + a[0] * b[0]) + a[1] * b[1]) + a[2] * b[2]


def _mat_vec(M, v):
    return [((0.0 + M[i][0] * v[0]) + M[i][1] * v[1]) + M[i][2] * v[2] for i in range(3)]


def quat_mul(a, b):
    aw, ax, ay, az = a
    bw, bx, by, bz = b
    return (((aw * bw - ax * bx) - ay * by) - az * bz, ((aw * bx + ax * bw) + ay * bz) - az * by,
            ((aw * by + ay * bw) + az * bx) - ax * bz, ((aw * bz + az * bw) + ax * by) - ay * bx)


def quat_from_angular_velocity(av):
    """QuaternionFromAngularVelocity of the rotation vector av (the motion model's)."""
    angle = math.sqrt((av[0] * av[0] + av[1] * av[1]) + av[2] * av[2])
    if angle > 0.0:
        s = math.sin(angle / 2.0) / angle
        return (math.cos(angle / 2.0), s * av[0], s * av[1], s * av[2])
    return (1.0, 0.0, 0.0, 0.0)


def pose_at(x, s, swap_order=False):
    """The pose (7) at time s of the state x (13): x[0:7] for s = 0; r + v s and q (x) qw(omega s) otherwise."""
    x = [float(v) for v in x[:13]]
    if s == 0.0:
        return np.array(x[:7])
    r = [x[i] + x[7 + i] * s for i in range(3)]
    qw = quat_from_angular_velocity([x[10] * s, x[11] * s, x[12] * s])
    q = quat_mul(qw, x[3:7]) if swap_order else quat_mul(x[3:7], qw)
    return np.array(r + list(q))


def times(exposure, offset):
    """(s-, s_c, s+)."""
    hx = float(exposure) * 0.5
    off = float(offset)
    return off - hx, off, off + hx


class _Pose:
    """adj(RRW), r and num = nW . (y - r) of a viewing pose (PatchPose)."""

    def __init__(self, xs, y, nW):
        xs = [float(v) for v in xs]
        self.A = adjugate(rrw(xs))
        self.r = xs[:3]
        self.num = _dot(nW, [y[i] - xs[i] for i in range(3)])


def ray_source(cam8, P, Rref, rref, cref, nW, c, half):
    """patch_ray_source of the rays c (3 arrays) from the pose P into the reference camera (RRW Rref, position rref,
    centre cref): (src (..., 2), valid (...))."""
    with np.errstate(all="ignore"):
        dW = _mat_vec(P.A, c)
        t = P.num / _dot(nW, dW)
        e = [(P.r[i] + t * dW[i]) - rref[i] for i in range(3)]
        zo = np.stack(_mat_vec(Rref, e), axis=-1)
        shp = zo.shape[:-1]
        g = project_point(cam8, zo.reshape(-1, 3)).reshape(shp + (2,))
        src = np.stack([(g[..., 0] - cref[0]) + float(half), (g[..., 1] - cref[1]) + float(half)], axis=-1)
        valid = np.isfinite(t) & (t > 0.0) & (zo[..., 2] > 0.0) & np.isfinite(src).all(axis=-1)
    return src, valid


def bilinear(T, src):
    """patch_bilinear: the unrounded bilinear value of T at src (..., 2), each coordinate clamped to [0, B - 1]."""
    B = T.shape[0]
    Tf = T.astype(np.float64)
    sx = np.minimum(np.maximum(src[..., 0], 0.0), float(B - 1))
    sy = np.minimum(np.maximum(src[..., 1], 0.0), float(B - 1))
    x0 = np.minimum(np.floor(sx).astype(np.int64), B - 2)
    y0 = np.minimum(np.floor(sy).astype(np.int64), B - 2)
    fx = sx - x0.astype(np.float64)
    fy = sy - y0.astype(np.float64)
    top = (1.0 - fx) * Tf[y0, x0] + fx * Tf[y0, x0 + 1]
    bot = (1.0 - fx) * Tf[y0 + 1, x0] + fx * Tf[y0 + 1, x0 + 1]
    return (1.0 - fy) * top + fy * bot


def setup(cam8, B, y, xo, x, exposure, offset, warp, theta=(0.0, 0.0), pose_fn=None, swap_order=False,
          centre_at_s=False):
    """The per-job terms: dict(poses, ident, Rref, rref, cref, nW, h0, times, half)."""
    y = [float(v) for v in y]
    xo = [float(v) for v in xo]
    x = np.asarray(x, np.float64)
    xp = [float(v) for v in x[:7]]
    h0 = project_point(cam8, camera_points(xp, y))[0]
    nW = normal(basis(xo, y), float(theta[0]), float(theta[1])) if (theta[0] != 0.0 or theta[1] != 0.0) \
        else [xo[i] - y[i] for i in range(3)]
    if warp:
        Rref, rref = rrw(xo), xo[:3]
        cref = project_point(cam8, camera_points(xo, y))[0]
    else:
        Rref, rref, cref = rrw(xp), xp[:3], h0
    ts = times(exposure, offset)
    poses, ident, centres = [], [], []
    for s in ts:
        xs = pose_at(x, s, swap_order) if pose_fn is None or s == 0.0 else np.asarray(pose_fn(x, s), np.float64)
        poses.append(_Pose(xs, y, nW))
        ident.append((not warp) and s == 0.0)
        centres.append(project_point(cam8, camera_points([float(v) for v in xs], y))[0] if centre_at_s else h0)
    return dict(poses=poses, ident=ident, Rref=Rref, rref=rref, cref=cref, nW=nW, h0=h0, times=ts, centres=centres,
                half=(B - 1) // 2)


def sources(cam8, B, J, k, centre=None):
    """src(s_k) (B, B, 2) and validity of every output pixel, or of the centre pixel only (centre=True)."""
    half = J["half"]
    h = J["centres"][k]
    if centre:
        a = b = np.array([half])
    else:
        a, b = np.mgrid[0:B, 0:B]
    if J["ident"][k]:
        return np.stack([b.astype(np.float64), a.astype(np.float64)], -1), np.ones(b.shape, bool)
    c0, c1 = unproject_point(cam8, h[0] + (b - half).astype(np.float64), h[1] + (a - half).astype(np.float64))
    return ray_source(cam8, J["poses"][k], J["Rref"], J["rref"], J["cref"], J["nW"],
                      [c0, c1, np.ones_like(c0)], half)


def sample_count(cam8, B, J):
    """(L, K, valid) from the centre pixel's src(s+) - src(s-)."""
    sm, vm = sources(cam8, B, J, 0, centre=True)
    sp, vp = sources(cam8, B, J, 2, centre=True)
    with np.errstate(all="ignore"):
        dx = float(sp[0, 0] - sm[0, 0])
        dy = float(sp[0, 1] - sm[0, 1])
        L = math.sqrt(dx * dx + dy * dy) if math.isfinite(dx) and math.isfinite(dy) else math.nan
    ok = bool(vm[0] and vp[0]) and math.isfinite(L)
    K = int(min(float(MAX_SAMPLES), max(1.0, math.ceil(L)))) if ok else 1
    return L, K, ok


def quadratic_points(s0, s1, s2, K, half_step=False):
    """src_k (K, ..., 2) of the quadratic through src(s-), src(s_c), src(s+) at u_k = ((k + 0.5) / K) - 0.5
    (half_step, broken: k / K - 0.5)."""
    d1 = s2 - s0
    d2 = (s2 - 2.0 * s1) + s0
    out = []
    for m in range(K):
        u = (float(m) / float(K)) - 0.5 if half_step else ((float(m) + 0.5) / float(K)) - 0.5
        w2 = (2.0 * u) * u
        out.append((s1 + u * d1) + w2 * d2)
    return np.stack(out)


def blur_template(cam8, T, y, xo, x, exposure, offset, warp, theta=(0.0, 0.0), pose_fn=None, swap_order=False,
                  centre_at_s=False, round_samples=False, half_step=False):
    """-> (template (B, B) u8, valid (0 stored, 1 warped, 2 blurred), K (0 unless blurred)) of one job of a blur-on
    stream at the state x (13)."""
    T = np.asarray(T, np.uint8)
    B = T.shape[0]
    J = setup(cam8, B, y, xo, x, exposure, offset, warp, theta, pose_fn, swap_order, centre_at_s)
    L, K, ok = sample_count(cam8, B, J)
    if ok:
        s1, v1 = sources(cam8, B, J, 1)
        if K == 1:
            if v1.all():
                return (bilinear(T, s1) + 0.5).astype(np.int64).astype(np.uint8), 2, 1
        else:
            s0, v0 = sources(cam8, B, J, 0)
            s2, v2 = sources(cam8, B, J, 2)
            if (v0 & v1 & v2).all():
                pts = quadratic_points(s0, s1, s2, K, half_step)
                acc = np.zeros((B, B))
                for m in range(K):
                    w = bilinear(T, pts[m])
                    acc = acc + (np.floor(w + 0.5) if round_samples else w)
                v = acc / float(K)
                return (v + 0.5).astype(np.int64).astype(np.uint8), 2, K
    return unblurred(cam8, T, y, xo, x, warp, theta)


def unblurred(cam8, T, y, xo, x, warp, theta=(0.0, 0.0)):
    """The fallback: the warp's template when the warp is on and valid, else the stored one."""
    T = np.asarray(T, np.uint8)
    if warp:
        import normals_ref
        out, v = normals_ref.warp_template(cam8, T, y, xo, np.asarray(x, np.float64)[:7], theta)
        if v:
            return out, 1, 0
    return T.copy(), 0, 0


def blur_templates(cam8, T, y, xo, x, exposure, offset, warp, theta=None, **kw):
    """blur_template of every feature k of T (n, B, B), y (n, 3), xo (n, 7), theta (n, 2) at the one state x."""
    out = [blur_template(cam8, T[k], y[k], xo[k], x, exposure, offset, warp,
                         (0.0, 0.0) if theta is None else tuple(float(v) for v in theta[k]), **kw)
           for k in range(len(T))]
    B = np.asarray(T).shape[-1]
    return (np.stack([o[0] for o in out]) if out else np.zeros((0, B, B), np.uint8),
            np.array([o[1] for o in out], np.uint8), np.array([o[2] for o in out], np.int32))

