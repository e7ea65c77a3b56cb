"""Inputs of the closed-form model tests, shared by the CPU tests that pin the oracle to the reference's stored outputs
(test_oracle_ref.py) and the GPU tests that replay the same outputs against the device (test_gpu_models.py), plus the
many-feature viewpoint streams of test_gpu_models.py and a float64 mirror of the visibility gates (full_feature_model.cpp
via ekf.cu) that places features and xp_org on either side of each gate.

The generators draw from their seeded PCG64 streams in a fixed order: the stored reference outputs are keyed to it."""
import numpy as np

CAMS = [np.array([320, 240, 195.0, 195.0, 162.0, 125.0, 9e-6, 1.0]),
        np.array([640, 480, 390.0, 392.0, 322.0, 247.0, 2e-6, 2.0])]
BOUND = 20.0                                   # kImageSearchBoundary_, full_feature_model.cpp:51
ANGLE_MAX = np.pi * 45.0 / 180.0               # the angle gate, in the kernel's own expression


def random_xv(rng, normalise=True):
    xv = np.zeros(13)
    xv[:3] = rng.normal(0, 0.3, 3)
    q = rng.normal(0, 1, 4)
    if normalise:
        q /= np.linalg.norm(q)
    xv[3:7] = q
    xv[7:10] = rng.normal(0, 0.2, 3)
    xv[10:13] = rng.normal(0, 0.3, 3)
    return xv


def motion_cases():
    """(xv, dt, u) of the motion-model comparison: 200 random states, a third with a non-unit q (the reference never
    renormalises q, quirk Q1), every omega component non-zero except the cfg's starting omega (data/SceneLib2.cfg:81-83)
    every 10th case, dt of 1/30, 0.05 and 0.01, a control input in every 4th case."""
    rng = np.random.default_rng(31)
    for k in range(200):
        xv = random_xv(rng, normalise=(k % 3 != 0))
        if k % 10 == 0:
            xv[10:13] = [0.0, 0.0, 0.01]
        dt = [1 / 30.0, 0.05, 0.01][k % 3]
        u = rng.normal(0, 1, 3) if k % 4 == 0 else np.zeros(3)
        yield xv, dt, u


def measurement_cases():
    """(cam8, xv, y, P (16 x 16), xp_org) of the measurement-model comparison: 300 cases over the two cameras, camera
    poses with a non-unit q, every 17th feature behind the camera, a random xp_org."""
    rng = np.random.default_rng(32)
    for k in range(300):
        cam8 = CAMS[k % 2]
        xv = random_xv(rng)
        xv[:3] *= 0.2
        xv[3:7] = [1, 0, 0, 0] + rng.normal(0, 0.15 if k % 5 else 1.0, 4)
        y = np.array([rng.uniform(-0.6, 0.6), rng.uniform(-0.4, 0.4), rng.uniform(0.3, 3.0)])
        if k % 17 == 0:
            y[2] = -abs(y[2])
        A = rng.normal(0, 1, (16, 16))
        P = A @ A.T * 1e-4 + 1e-6 * np.eye(16)
        xp_org = random_xv(rng)[:7]
        xp_org[:3] *= 0.2
        xp_org[3:7] = [1, 0, 0, 0] + rng.normal(0, 0.3, 4)
        yield cam8, xv, y, P, xp_org


def particle_cases():
    """(cam8, xv, ypi, P (19 x 19), lambda (9)) of the particle-prediction comparison: 120 cases over the two cameras,
    camera poses with a non-unit q, a ray from near the camera centre, 9 sorted depths per ray."""
    rng = np.random.default_rng(57)
    for k in range(120):
        cam8 = CAMS[k % 2]
        xv = random_xv(rng)
        xv[:3] *= 0.2
        xv[3:7] = [1, 0, 0, 0] + rng.normal(0, 0.15, 4)
        hh = np.array([rng.uniform(-0.5, 0.5), rng.uniform(-0.4, 0.4), 1.0])
        ypi = np.concatenate([xv[:3] + rng.normal(0, 0.05, 3), hh / np.linalg.norm(hh)])
        A = rng.normal(0, 1, (19, 19))
        P = A @ A.T * 1e-4 + 1e-6 * np.eye(19)
        lam = np.sort(rng.uniform(0.3, 6.0, 9))
        yield cam8, xv, ypi, P, lam


# ---- float64 mirror of the geometry of predict_feature / visibility_test (ekf.cu) -----------------------------------
def quat_inverse(q):
    return np.array([q[0], -q[1], -q[2], -q[3]]) / (q @ q)


def quat_to_R(q):
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def quat_mul(a, b):
    return np.array([a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3],
                     a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
                     a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3],
                     a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1]])


def world_to_camera(xp):
    """z = M (y - r) with M = R(q^-1): the camera-frame point of zeroedyi (also for a non-unit q)."""
    return quat_to_R(quat_inverse(xp[3:7]))


def gate_map(xp):
    """The vector the viewpoint gates use for a pose xp: R(q) R(q^-1) (y - r) (the identity map for a unit q)."""
    return quat_to_R(xp[3:7]) @ world_to_camera(xp)


def gates(xp, y, xp_org):
    """(distance ratio, view angle) of the distance and angle gates, as visibility_test forms them."""
    a, b = gate_map(xp) @ (y - xp[:3]), gate_map(xp_org) @ (y - xp_org[:3])
    ma, mb = np.sqrt(a @ a), np.sqrt(b @ b)
    return ma / mb, abs(np.arccos(np.clip((a @ b) / (ma * mb), -1.0, 1.0)))


def project(cam8, z):
    fku, fkv, u0, v0, kd1 = cam8[2:7]
    uc, vc = -fku * z[0] / z[2], -fkv * z[1] / z[2]
    f = np.sqrt(1 + 2 * kd1 * (uc * uc + vc * vc))
    return np.array([uc / f + u0, vc / f + v0])


def unproject(cam8, h, depth):
    """Camera-frame point at `depth` (its z) whose projection is h (camera.cpp:132-157)."""
    fku, fkv, u0, v0, kd1 = cam8[2:7]
    cu, cv = h[0] - u0, h[1] - v0
    f = np.sqrt(1 - 2 * kd1 * (cu * cu + cv * cv))
    return np.array([cu / f / -fku * depth, cv / f / -fkv * depth, depth])


def visibility_code(cam8, xp, y, xp_org, h):
    """The failure code of visibility_test: 1 / 2 outside the search bound in u / v, 4 distance ratio, 8 view angle,
    16 behind the camera."""
    code = 0
    if h[0] < BOUND or h[0] > int(cam8[0]) - 1 - BOUND:
        code |= 1
    if h[1] < BOUND or h[1] > int(cam8[1]) - 1 - BOUND:
        code |= 2
    if (world_to_camera(xp) @ (y - xp[:3]))[2] <= 0:
        code |= 16
    ratio, angle = gates(xp, y, xp_org)
    if ratio > 2.0 or ratio < 0.5:
        code |= 4
    if angle > ANGLE_MAX:
        code |= 8
    return code


def _rotate_about(v, axis, angle):
    axis = axis / np.linalg.norm(axis)
    return v * np.cos(angle) + np.cross(axis, v) * np.sin(angle) + axis * (axis @ v) * (1 - np.cos(angle))


def place_xp_org(rng, xp, y, ratio, angle, unit_q=True):
    """An xp_org whose gates give (ratio, angle) for the feature at y seen from pose xp: b = gate vector of xp_org."""
    a = gate_map(xp) @ (y - xp[:3])
    perp = np.cross(a, rng.normal(size=3))
    b = _rotate_about(a, perp, angle) / ratio
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    if not unit_q:
        q *= rng.uniform(0.85, 1.15)
    xo = np.zeros(7)
    xo[3:7] = q
    xo[:3] = y - np.linalg.solve(gate_map(xo), b)
    return xo


# margins of the near-threshold cases: the ratio / distance / pixel gates are + - x / sqrt only and must agree with the
# oracle at any margin; the angle gate goes through acos, which may differ from glibc by an ulp or two, so its margins
# stay above 1e-12 except in the streams with `probe` set
NEAR = (1e-3, 1e-6, 1e-9, 2e-12)
PROBE = (3e-14, 1e-14, 3e-15, 1e-15, 3e-16)


def viewpoint_stream(seed, nf, cam8, unit_q=True, probe=False, ties=4):
    """One stream of `nf` features seen from a random full-orientation pose: features placed by pixel (inside the
    image, within a pixel of the 20 px search bound on each side, outside it) and depth (some behind the camera), each
    with its own xp_org on either side of the distance-ratio and angle gates, some just at their thresholds; `ties`
    features repeat an earlier feature's y, xp_org and covariance blocks (exact ties in trace S); a dense SPD P whose
    scales spread over three orders of magnitude.  Returns dict(x, P, xp_org, design) where design[i] names the
    feature's pixel / gate case."""
    rng = np.random.default_rng(seed)
    W, H = int(cam8[0]), int(cam8[1])
    xv = np.zeros(13)
    xv[:3] = rng.normal(0, 0.5, 3)
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    xv[3:7] = q if unit_q else q * rng.uniform(0.9, 1.1)
    xv[7:10] = rng.normal(0, 0.05, 3)
    xv[10:13] = rng.normal(0, 0.2, 3)
    Minv = np.linalg.inv(world_to_camera(xv))
    lo, hi = (BOUND, BOUND), (W - 1 - BOUND, H - 1 - BOUND)
    y = np.zeros((nf, 3))
    xo = np.zeros((nf, 7))
    design = []
    src = {}
    for i in range(nf):
        if i >= nf - ties and i >= 2 * ties:       # exact duplicate of an earlier feature
            j = int(rng.integers(0, i - ties))
            y[i], xo[i], src[i] = y[j], xo[j], j
            design.append(("tie", j))
            continue
        kind = rng.choice(["inside", "edge", "outside"], p=[0.6, 0.25, 0.15])
        h = np.array([rng.uniform(lo[0] + 2, hi[0] - 2), rng.uniform(lo[1] + 2, hi[1] - 2)])
        if kind == "edge":                         # within a pixel of the bound, either side, in u or v or both
            for c in ([0], [1], [0, 1])[int(rng.integers(0, 3))]:
                h[c] = (lo[c] if rng.random() < 0.5 else hi[c]) + rng.uniform(-1, 1)
        elif kind == "outside":
            c = int(rng.integers(0, 2))
            h[c] = rng.uniform(-30, lo[c] - 1) if rng.random() < 0.5 else rng.uniform(hi[c] + 1, (W, H)[c] + 30)
        depth = rng.uniform(0.5, 4.0)
        if rng.random() < 0.1:
            depth = -depth                         # behind the camera (same pixel)
            kind = "behind"
        y[i] = xv[:3] + Minv @ unproject(cam8, h, depth)
        g = rng.choice(["pass", "ratio", "angle", "near_ratio", "near_angle", "both"],
                       p=[0.45, 0.1, 0.1, 0.15, 0.15, 0.05])
        ratio, angle = rng.uniform(0.6, 1.8), rng.uniform(0, 0.7)
        if g == "ratio":
            ratio = rng.uniform(2.2, 4) if rng.random() < 0.5 else rng.uniform(0.25, 0.45)
        elif g == "angle":
            angle = rng.uniform(0.85, 2.5)
        elif g == "both":
            ratio, angle = rng.uniform(2.2, 4), rng.uniform(0.85, 2.5)
        elif g == "near_ratio":
            m = NEAR[int(rng.integers(0, len(NEAR)))] * (1 if rng.random() < 0.5 else -1)
            ratio = (2.0 if rng.random() < 0.5 else 0.5) * (1 + m)
        elif g == "near_angle":
            m = (PROBE if probe else NEAR)[int(rng.integers(0, len(PROBE if probe else NEAR)))]
            angle = ANGLE_MAX + m * (1 if rng.random() < 0.5 else -1)
        xo[i] = place_xp_org(rng, xv, y[i], ratio, angle, unit_q=rng.random() < 0.8)
        design.append((kind, g))
    # dense SPD covariance, scales over three orders of magnitude; a tie copies the rows / columns of its source
    n = 13 + 3 * nf
    d = 10.0 ** rng.uniform(-3.5, -0.5, n)
    A = rng.standard_normal((n, 12))
    for i, j in src.items():
        d[13 + 3 * i:16 + 3 * i] = d[13 + 3 * j:16 + 3 * j]
        A[13 + 3 * i:16 + 3 * i] = A[13 + 3 * j:16 + 3 * j]
    c = A @ A.T
    s = 1.0 / np.sqrt(np.diag(c))
    c = 0.6 * c * s[:, None] * s[None, :] + 0.4 * np.eye(n)
    P = d[:, None] * c * d[None, :]
    P = 0.5 * (P + P.T)
    for i, j in src.items():                       # make the copied blocks identical to the last bit
        bi, bj = slice(13 + 3 * i, 16 + 3 * i), slice(13 + 3 * j, 16 + 3 * j)
        P[:13, bi] = P[:13, bj]
        P[bi, :13] = P[bj, :13]
        P[bi, bi] = P[bj, bj]
    x = np.concatenate([xv, y.ravel()])
    return dict(x=x, P=P, xp_org=xo, design=design, cam8=cam8, probe=probe)


def viewpoint_streams(cam8=CAMS[0], count=24, cap=128):
    """`count` streams for one context of capacity `cap`: map sizes from 1 to `cap`, every 5th stream with a non-unit
    camera q, streams 7 and 19 probing the angle gate closer than 1e-12."""
    sizes = [cap, 1, 2, 3] + [int(v) for v in np.random.default_rng(77).integers(5, cap, count - 4)]
    return [viewpoint_stream(9000 + s, sizes[s], cam8, unit_q=(s % 5 != 4), probe=s in (7, 19),
                             ties=min(4, sizes[s] // 3)) for s in range(count)]
