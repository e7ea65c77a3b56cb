"""The planar patch warp (include/sl2b200.h, sl2_set_stream_warp; csrc/sl2_model.cuh: patch_warp_setup,
patch_warp_source, patch_sample) restated in NumPy, one IEEE double operation at a time in the kernel's order (NumPy's
element-wise operations are correctly rounded and never fused), vectorised over the template's pixels.  The camera
model is tests/camera_ref.py's, with unproject_point stated here."""
import numpy as np

from camera_ref import camera_points, project_point, rrw


def unproject_point(cam8, p0, p1):
    """unproject_point (Camera::Unproject) of the pixels (p0, p1): the camera-frame direction (x, y, 1), x and y as
    arrays (NaN where 1 - 2 kd1 r^2 < 0)."""
    fku, fkv, u0, v0, kd1 = (float(v) for v in cam8[2:7])
    with np.errstate(all="ignore"):
        c0 = np.asarray(p0, np.float64) - u0
        c1 = np.asarray(p1, np.float64) - v0
        factor = np.sqrt(1.0 - (2.0 * kd1) * (c0 * c0 + c1 * c1))
        return (c0 / factor) / (-fku), (c1 / factor) / (-fkv)


def _dot(a, b):
    return ((0.0 + a[0] * b[0]) + a[1] * b[1]) + a[2] * b[2]


def warp_source(cam8, B, y, xo, xp):
    """src (B, B, 2) positions in the stored template of every output pixel (row a, column b) and their validity
    (B, B) for the feature y (3) first seen from xo (7), at the camera pose xp (7); also h, the template's centre at
    xp."""
    half = (B - 1) // 2
    y = [float(v) for v in y]
    xo = [float(v) for v in xo]
    xp = [float(v) for v in xp]
    R, Ro = rrw(xp), rrw(xo)
    h = project_point(cam8, camera_points(xp, y))[0]
    ho = project_point(cam8, camera_points(xo, y))[0]
    d = [y[i] - xp[i] for i in range(3)]
    nW = [xo[i] - y[i] for i in range(3)]
    num = _dot(nW, d)
    a, b = np.mgrid[0:B, 0:B]
    p0 = h[0] + (b - half).astype(np.float64)
    p1 = h[1] + (a - half).astype(np.float64)
    c0, c1 = unproject_point(cam8, p0, p1)
    c = [c0, c1, np.ones_like(c0)]
    with np.errstate(all="ignore"):
        dW = [((0.0 + R[0][i] * c[0]) + R[1][i] * c[1]) + R[2][i] * c[2] for i in range(3)]
        t = num / _dot(nW, dW)
        e = [(xp[i] + t * dW[i]) - xo[i] for i in range(3)]
        zo = np.stack([((0.0 + Ro[i][0] * e[0]) + Ro[i][1] * e[1]) + Ro[i][2] * e[2] for i in range(3)], axis=-1)
        g = project_point(cam8, zo.reshape(-1, 3)).reshape(B, B, 2)
        src = np.stack([(g[..., 0] - ho[0]) + float(half), (g[..., 1] - ho[1]) + float(half)], axis=-1)
        valid = np.isfinite(t) & (t > 0.0) & (zo[..., 2] > 0.0) & np.isfinite(src).all(axis=-1)
    return src, valid, h


def sample(T, src):
    """patch_sample: bilinear sample of the B x B template T at the finite positions src (..., 2) = (column, row),
    each coordinate clamped to [0, B - 1]; the bytes (int)(v + 0.5)."""
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
    v = (1.0 - fy) * top + fy * bot
    return (v + 0.5).astype(np.int64).astype(np.uint8)


def warp_template(cam8, T, y, xo, xp):
    """The warped template (B, B) u8 of the feature (y, xo, stored template T) at the pose xp and its valid flag:
    the stored template and 0 when any pixel is invalid."""
    T = np.asarray(T, np.uint8)
    src, valid, _ = warp_source(cam8, T.shape[0], y, xo, xp)
    if not valid.all():
        return T.copy(), 0
    return sample(T, src), 1


def warp_templates(cam8, T, y, xo, xp):
    """warp_template of every feature k of T (n, B, B), y (n, 3), xo (n, 7) at the one pose xp."""
    out = [warp_template(cam8, T[k], y[k], xo[k], xp) for k in range(len(T))]
    return (np.stack([o[0] for o in out]) if out else np.zeros((0,) + T.shape[1:], np.uint8),
            np.array([o[1] for o in out], np.uint8))
