"""A rendered hand-held "whip" for the gyroscope update (tests/warp_scene.py's texture and renderer): a camera at the
origin looking at the textured plane turns slowly, then its yaw rate jumps by WHIP rad/s for one frame and drops back.
The true body rates are known per frame interval, so a gyro sample is R_gc omega_true + b + noise drawn from cov."""
from dataclasses import dataclass

import numpy as np

from warp_scene import CAM, DT, PLANE_Z, make_texture, quat_axis, rays, render
from scenelib2_b200 import synth

WHIP = 2.0                               # rad/s: the yaw-rate change within one frame, and back
BASE = np.array([0.03, 0.12, -0.02])     # rad/s: the slow turn before and after (body frame; |omega| > 0)


@dataclass
class WhipScene:
    cam8: np.ndarray
    boxsize: int
    n_select: int
    poses: np.ndarray    # (T + 1, 7) true poses r, q (w, x, y, z)
    omega: np.ndarray    # (T, 3) true body rate over frame interval [k, k + 1]
    frames: np.ndarray   # (T + 1, H, W) u8
    xp_org: np.ndarray
    patches: np.ndarray
    x0: np.ndarray
    P0: np.ndarray
    whip: int            # the step (1-based: the step that consumes frame whip) whose interval holds the jump
    search_override: tuple = (0.0, 0.0, 0.0)
    delta_t: float = DT


def qmul(a, b):
    w1, x1, y1, z1 = a
    w2, x2, y2, z2 = b
    return np.array([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                     w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2])


def make_whip_scene(steps=16, whip=8, n_features=40, n_select=12, seed=0, margin=60, sigma=4.0):
    rng = np.random.default_rng(0x6E7A00 + seed)
    cam8 = CAM.copy()
    B, half = 11, 5
    tex = make_texture(rng, sigma)
    omega = np.tile(BASE, (steps, 1))
    omega[whip - 1, 1] += WHIP  # the interval [whip - 1, whip]: consumed by step `whip`
    poses = np.zeros((steps + 1, 7))
    poses[0, 3] = 1.0
    for k in range(steps):
        w = omega[k]
        poses[k + 1, 3:] = qmul(poses[k, 3:], quat_axis(w, np.linalg.norm(w) * DT))
    frames = np.stack([render(cam8, p, tex, rng) for p in poses])
    pix = synth._feature_pixels(rng, int(cam8[0]), int(cam8[1]), n_features, margin)
    d = rays(cam8, poses[0])[pix[:, 1], pix[:, 0]]
    y = ((PLANE_Z - poses[0, 2]) / d[:, 2])[:, None] * d
    patches = np.stack([frames[0][py - half:py + half + 1, px - half:px + half + 1] for px, py in pix])
    x0 = np.concatenate([poses[0], np.zeros(3), omega[0], y.ravel()])
    n = x0.size
    sd = np.concatenate([np.full(3, 1e-3), np.full(4, 1e-3), np.full(3, 1e-2), np.full(3, 1e-2),
                         np.full(n - 13, 1e-3)])
    return WhipScene(cam8=cam8, boxsize=B, n_select=n_select, poses=poses, omega=omega, frames=frames,
                     xp_org=np.tile(poses[0], (n_features, 1)), patches=patches, x0=x0, P0=np.diag(sd * sd),
                     whip=whip)


def gyro_samples(sc, R_gc, bias, cov, seed=0):
    """(T, 3): the sample of step t + 1 (frame interval [t, t + 1]) = R_gc omega_true + b + noise(cov)."""
    rng = np.random.default_rng(0x6E7B00 + seed)
    noise = rng.multivariate_normal(np.zeros(3), cov, size=len(sc.omega))
    return sc.omega @ np.asarray(R_gc).T + np.asarray(bias) + noise
