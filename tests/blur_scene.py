"""A rendered fast yaw for the exposure blur (tests/warp_scene.py's texture, rays and renderer): a camera at the origin
looking at the textured plane yaws back and forth about its y axis with a peak rate of PEAK rad/s.  Each frame is the
rounded mean of SUB noise-free renders at equally spaced times over the exposure, with the noise added once; the camera
stamps the end of its exposure, so the exposure of frame k is [t_k - EXPOSURE, t_k] and the blur's offset is
-EXPOSURE / 2.  The templates are cut from a sharp render at t_0; the initial state holds the true pose and rate, and a
gyro sample is the true mean rate over each frame interval."""
from dataclasses import dataclass

import numpy as np

from warp_scene import CAM, DT, PLANE_Z, make_texture, quat_axis, rays
from scenelib2_b200 import synth

PEAK = 3.0               # rad/s: the peak yaw rate
PERIOD = 0.4             # s: one back-and-forth
EXPOSURE = 1.0 / 60.0    # s
OFFSET = -EXPOSURE / 2   # the frame's time stamps the end of the exposure
SUB = 64                 # renders averaged per frame
T0 = 0.01                # s: the time of frame 0 (a nonzero rate there)


def yaw(t):
    """The yaw angle (rad) at time t: A (1 - cos(2 pi t / PERIOD)), whose rate peaks at PEAK."""
    return PEAK * PERIOD / (2 * np.pi) * (1 - np.cos(2 * np.pi * t / PERIOD))


def rate(t):
    return PEAK * np.sin(2 * np.pi * t / PERIOD)


def pose(t):
    return np.concatenate([np.zeros(3), quat_axis([0, 1, 0], yaw(t))])


@dataclass
class BlurScene:
    cam8: np.ndarray
    boxsize: int
    times: np.ndarray    # (T + 1,) frame times
    poses: np.ndarray    # (T + 1, 7) true poses at the frame times
    omega: np.ndarray    # (T, 3) true mean body rate over frame interval [k, k + 1]
    streak: np.ndarray   # (T + 1,) px: the true streak of the image centre in frame k
    frames: np.ndarray   # (T + 1, H, W) u8
    y: np.ndarray
    xp_org: np.ndarray
    patches: np.ndarray
    x0: np.ndarray
    P0: np.ndarray
    delta_t: float = DT


def _render_float(cam8, p, tex):
    d = rays(cam8, p)
    t = (PLANE_Z - p[2]) / d[..., 2]
    X, Y = p[0] + t * d[..., 0], p[1] + t * d[..., 1]
    n = tex.shape[0]
    from warp_scene import EXTENT, TEXEL
    gx = np.clip((X + EXTENT) / TEXEL, 0, n - 1.000001)
    gy = np.clip((Y + EXTENT) / TEXEL, 0, n - 1.000001)
    x0, y0 = np.floor(gx).astype(int), np.floor(gy).astype(int)
    fx, fy = gx - x0, gy - y0
    return ((1 - fy) * ((1 - fx) * tex[y0, x0] + fx * tex[y0, x0 + 1])
            + fy * ((1 - fx) * tex[y0 + 1, x0] + fx * tex[y0 + 1, x0 + 1]))


def blurred_frame(cam8, t, tex, rng):
    acc = 0.0
    for j in range(SUB):
        acc = acc + _render_float(cam8, pose(t - EXPOSURE + (j + 0.5) / SUB * EXPOSURE), tex)
    val = np.round(acc / SUB) + rng.integers(-2, 3, acc.shape)
    return np.clip(val, 0, 255).astype(np.uint8)


def make_blur_scene(steps=24, n_features=40, seed=0, margin=60, sigma=4.0):
    rng = np.random.default_rng(0xB1A400 + seed)
    cam8 = CAM.copy()
    B, half = 11, 5
    tex = make_texture(rng, sigma)
    times = T0 + np.arange(steps + 1) * DT
    poses = np.stack([pose(t) for t in times])
    omega = np.zeros((steps, 3))
    omega[:, 1] = (yaw(times[1:]) - yaw(times[:-1])) / DT
    streak = cam8[2] * np.abs(yaw(times) - yaw(times - EXPOSURE))
    frames = np.stack([blurred_frame(cam8, t, tex, rng) for t in times])
    sharp = np.clip(np.round(_render_float(cam8, poses[0], tex)) + rng.integers(-2, 3, frames[0].shape), 0, 255)
    sharp = sharp.astype(np.uint8)
    pix = synth._feature_pixels(rng, int(cam8[0]), int(cam8[1]), n_features, margin)
    d = rays(cam8, poses[0])[pix[:, 1], pix[:, 0]]
    y = ((PLANE_Z - poses[0, 2]) / d[:, 2])[:, None] * d
    patches = np.stack([sharp[py - half:py + half + 1, px - half:px + half + 1] for px, py in pix])
    x0 = np.concatenate([poses[0], np.zeros(3), [0.0, rate(T0), 0.0], y.ravel()])
    n = x0.size
    sd = np.concatenate([np.full(3, 1e-3), np.full(4, 1e-3), np.full(3, 1e-2), np.full(3, 1e-2),
                         np.full(n - 13, 1e-3)])
    return BlurScene(cam8=cam8, boxsize=B, times=times, poses=poses, omega=omega, streak=streak, frames=frames, y=y,
                     xp_org=np.tile(poses[0], (n_features, 1)), patches=patches, x0=x0, P0=np.diag(sd * sd))


def true_state(sc, k):
    """The true 13-number state at frame k: pose, v = 0 and the body rate at the exposure's middle."""
    return np.concatenate([sc.poses[k], np.zeros(3), [0.0, rate(sc.times[k] + OFFSET), 0.0]])
