"""A rendered jolt for the accelerometer (tests/warp_scene.py's texture and renderer): a camera about 0.5 m from the
textured plane, tilted so that gravity (along the world's -y axis) lies along none of its axes, translates and turns
slowly; then a constant world acceleration of JOLT m/s^2 acts over `span` frame intervals and its opposite over the
next `span` (a shove that starts and stops), and the slow motion resumes.  Over each frame interval the acceleration is constant,
so the true position is r + v dt + a dt^2 / 2.  A sample is the specific force over the interval seen through R_ac, the
bias and noise drawn from cov: f = R_ac R(q)^T (a - g) + b + noise, with q the orientation at the interval's middle."""
from dataclasses import dataclass

import numpy as np

from gyro_scene import qmul
from warp_scene import CAM, DT, PLANE_Z, make_texture, quat_axis, quat_R, rays, render
from scenelib2_b200 import synth

GRAVITY = np.array([0.0, -9.81, 0.0])   # m/s^2, world frame
JOLT = np.array([30.0, 18.0, 0.0])       # m/s^2, world frame: about 3.6 g, nearly along the plane
V0 = np.array([0.03, -0.02, 0.01])       # m/s: the slow drift (world)
OMEGA = np.array([0.02, -0.03, 0.015])   # rad/s: the slow turn (body; |omega| > 0)
TILT = quat_axis([1.0, 0.6, 0.2], np.radians(18.0))  # frame 0's orientation


@dataclass
class JoltScene:
    cam8: np.ndarray
    boxsize: int
    n_select: int
    poses: np.ndarray    # (T + 1, 7) true poses r, q (w, x, y, z)
    accel: np.ndarray    # (T, 3) true world acceleration over frame interval [k, k + 1]
    frames: np.ndarray   # (T + 1, H, W) u8
    xp_org: np.ndarray
    patches: np.ndarray
    x0: np.ndarray
    P0: np.ndarray
    jolt: int            # the first step (1-based: the step that consumes frame jolt) whose interval holds +JOLT
    search_override: tuple = (0.0, 0.0, 0.0)
    delta_t: float = DT


def make_jolt_scene(steps=16, jolt=6, span=2, n_features=40, n_select=12, seed=2, margin=60, sigma=4.0, depth=0.5):
    rng = np.random.default_rng(0x6E7C00 + seed)
    cam8 = CAM.copy()
    B, half = 11, 5
    tex = make_texture(rng, sigma)
    acc = np.zeros((steps, 3))
    acc[jolt - 1:jolt - 1 + span] = JOLT
    acc[jolt - 1 + span:jolt - 1 + 2 * span] = -JOLT
    poses = np.zeros((steps + 1, 7))
    poses[0, 3:] = TILT
    axis = quat_R(TILT) @ np.array([0.0, 0.0, 1.0])
    poses[0, :3] = np.array([0.0, 0.0, PLANE_Z]) - depth / axis[2] * axis  # the optical axis meets the plane at depth
    v = V0.copy()
    for k in range(steps):
        poses[k + 1, :3] = poses[k, :3] + v * DT + 0.5 * acc[k] * DT * DT
        v = v + acc[k] * DT
        poses[k + 1, 3:] = qmul(poses[k, 3:], quat_axis(OMEGA, np.linalg.norm(OMEGA) * DT))
    frames = np.stack([render(cam8, p, tex, rng) for p in poses])
    pix = synth._feature_pixels(rng, int(cam8[0]), int(cam8[1]), n_features, margin)
    d = rays(cam8, poses[0])[pix[:, 1], pix[:, 0]]
    y = poses[0, :3] + ((PLANE_Z - poses[0, 2]) / d[:, 2])[:, None] * d
    patches = np.stack([frames[0][py - half:py + half + 1, px - half:px + half + 1] for px, py in pix])
    x0 = np.concatenate([poses[0], V0, OMEGA, y.ravel()])
    n = x0.size
    sd = np.concatenate([np.full(3, 1e-3), np.full(4, 1e-3), np.full(3, 1e-2), np.full(3, 1e-2),
                         np.full(n - 13, 1e-3)])
    return JoltScene(cam8=cam8, boxsize=B, n_select=n_select, poses=poses, accel=acc, frames=frames,
                     xp_org=np.tile(poses[0], (n_features, 1)), patches=patches, x0=x0, P0=np.diag(sd * sd),
                     jolt=jolt)


def accel_samples(sc, R_ac, bias, cov, seed=0):
    """(T, 3): the sample of step t + 1 (frame interval [t, t + 1]) = R_ac R(q_mid)^T (a - g) + b + noise(cov)."""
    rng = np.random.default_rng(0x6E7D00 + seed)
    out = np.zeros((len(sc.accel), 3))
    for k in range(len(sc.accel)):
        q = qmul(sc.poses[k, 3:], quat_axis(OMEGA, np.linalg.norm(OMEGA) * DT / 2))
        out[k] = np.asarray(R_ac) @ (quat_R(q).T @ (sc.accel[k] - GRAVITY)) + np.asarray(bias)
    return out + rng.multivariate_normal(np.zeros(3), cov, size=len(out))
