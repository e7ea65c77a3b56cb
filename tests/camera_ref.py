"""The device camera model of the match consensus and the relocalisation (csrc/sl2_model.cuh: pose_RRW, zeroed_point,
project_point, reproj_inlier) restated in NumPy, one IEEE double operation at a time in the kernels' order (NumPy's
element-wise operations are correctly rounded and never fused)."""
import numpy as np


def quat_to_R(w, x, y, z):
    """Eigen's toRotationMatrix of (w, x, y, z), row-major nested lists."""
    tx, ty, tz = 2.0 * x, 2.0 * y, 2.0 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return [[1.0 - (tyy + tzz), txy - twz, txz + twy],
            [txy + twz, 1.0 - (txx + tzz), tyz - twx],
            [txz - twy, tyz + twx, 1.0 - (txx + tyy)]]


def rrw(xp):
    """pose_RRW: the rotation of qRW = qWR^-1 (conjugate / squared norm; zero for a zero quaternion)."""
    w, x, y, z = (float(v) for v in xp[3:7])
    n2 = w * w + x * x + y * y + z * z
    if n2 > 0.0:
        w, x, y, z = w / n2, (-x) / n2, (-y) / n2, (-z) / n2
    else:
        w = x = y = z = 0.0
    return quat_to_R(w, x, y, z)


def camera_points(xp, y):
    """zeroed_point of every y (k, 3) seen from xp: RRW (y - r), rows summed from 0.0 in ascending order."""
    R = rrw(xp)
    y = np.asarray(y, np.float64).reshape(-1, 3)
    d = [y[:, i] - float(xp[i]) for i in range(3)]
    return np.stack([((0.0 + R[i][0] * d[0]) + R[i][1] * d[1]) + R[i][2] * d[2] for i in range(3)], axis=1)


def project_point(cam8, zc):
    """project_point (Camera::Project) of the camera-frame points zc (k, 3): pixels (k, 2)."""
    fku, fkv, u0, v0, kd1 = (float(v) for v in cam8[2:7])
    zc = np.asarray(zc, np.float64).reshape(-1, 3)
    with np.errstate(all="ignore"):
        uc = ((-fku) * zc[:, 0]) / zc[:, 2]
        vc = ((-fkv) * zc[:, 1]) / zc[:, 2]
        factor = np.sqrt(1.0 + (2.0 * kd1) * (uc * uc + vc * vc))
        return np.stack([uc / factor + u0, vc / factor + v0], axis=1)


def reprojection_d2(cam8, xp, y, z):
    """Squared distance of project_point(zeroed_point(y)) to z (k, 2), NaN behind the camera (reproj_inlier)."""
    zc = camera_points(xp, y)
    g = project_point(cam8, zc)
    z = np.asarray(z, np.float64).reshape(-1, 2)
    with np.errstate(all="ignore"):
        du = z[:, 0] - g[:, 0]
        dv = z[:, 1] - g[:, 1]
        d2 = du * du + dv * dv
    return np.where(zc[:, 2] > 0.0, d2, np.nan)
