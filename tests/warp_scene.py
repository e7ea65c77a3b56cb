"""Rendered scenes for the planar patch warp (pure NumPy, seeded): a band-limited texture on the plane z = PLANE_Z,
seen by a camera that rolls, approaches the plane or orbits the map's centre.  Every pixel of a frame is the texture
where that pixel's ray (the device camera model's unproject_point: Camera::Unproject of the reference) meets the
plane, sampled bilinearly, plus +-2 grey levels of noise.  Templates are cut from frame 0; a feature's y is the ray of
its template's centre pixel met with the plane, and its xp_org is the frame-0 pose.  The initial state holds the true
pose, v and omega, so a filter that keeps its matches follows the trajectory."""
from dataclasses import dataclass

import numpy as np

from warp_ref import unproject_point
from scenelib2_b200 import synth

PLANE_Z = 2.0       # m: the textured plane, fronto-parallel to the frame-0 camera at the origin
TEXEL = 0.004       # m per texel of the texture
EXTENT = 3.0        # m: the texture covers [-EXTENT, EXTENT]^2 of the plane (edge texels repeat beyond)
DT = 1.0 / 30.0
CAM = synth.camera_params(320, 240)  # the reference's calibration (kd1 != 0)


@dataclass
class WarpScene:
    name: str
    cam8: np.ndarray
    boxsize: int
    poses: np.ndarray    # (T, 7) true camera poses r, q (w, x, y, z)
    v: np.ndarray        # (3,) true initial velocity (world)
    omega: np.ndarray    # (3,) true angular velocity (body)
    frames: np.ndarray   # (T, H, W) u8
    y: np.ndarray        # (N, 3)
    xp_org: np.ndarray   # (N, 7)
    patches: np.ndarray  # (N, B, B) u8
    pix: np.ndarray      # (N, 2) template centres in frame 0
    x0: np.ndarray       # initial state: true pose, v, omega, y
    P0: np.ndarray


def quat_axis(axis, angle):
    a = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    return np.concatenate([[np.cos(angle / 2)], np.sin(angle / 2) * a])


def quat_R(q):
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def trajectory(kind, steps):
    """True poses (steps + 1, 7), initial v (world) and omega (body) of `kind` at DT: 'roll' (40 degrees about the
    optical axis), 'approach' (to half the distance to the plane, along the axis) or 'orbit' (35 degrees about the map's centre)."""
    T = steps * DT
    t = np.arange(steps + 1) * DT
    poses = np.zeros((steps + 1, 7))
    if kind == "roll":
        w = np.radians(40.0) / T
        for k, tk in enumerate(t):
            poses[k, 3:] = quat_axis([0, 0, 1], w * tk)
        return poses, np.zeros(3), np.array([0.0, 0.0, w])
    if kind == "approach":  # with 1 degree of roll: the motion model's Jacobian needs |omega| > 0
        vz = 0.5 * PLANE_Z / T
        w = np.radians(1.0) / T
        poses[:, 2] = vz * t
        for k, tk in enumerate(t):
            poses[k, 3:] = quat_axis([0, 0, 1], w * tk)
        return poses, np.array([0.0, 0.0, vz]), np.array([0.0, 0.0, w])
    if kind == "orbit":
        w = np.radians(35.0) / T
        c = np.array([0.0, 0.0, PLANE_Z])
        for k, tk in enumerate(t):
            phi = w * tk
            poses[k, :3] = c + PLANE_Z * np.array([-np.sin(phi), 0.0, -np.cos(phi)])
            poses[k, 3:] = quat_axis([0, 1, 0], phi)
        return poses, np.array([-PLANE_Z * w, 0.0, 0.0]), np.array([0.0, w, 0.0])
    raise ValueError(kind)


def make_texture(rng, sigma):
    n = int(round(2 * EXTENT / TEXEL)) + 1
    return synth.make_texture(rng, n, n, sigma=sigma).astype(np.float64)


def rays(cam8, pose):
    """World ray directions (H, W, 3) of every pixel of the camera at pose."""
    H, W = int(cam8[1]), int(cam8[0])
    v, u = np.mgrid[0:H, 0:W].astype(np.float64)
    c0, c1 = unproject_point(cam8, u, v)
    return np.stack([c0, c1, np.ones_like(c0)], axis=-1) @ quat_R(pose[3:]).T


def render(cam8, pose, tex, rng):
    d = rays(cam8, pose)
    r = pose[:3]
    t = (PLANE_Z - r[2]) / d[..., 2]
    X = r[0] + t * d[..., 0]
    Y = r[1] + t * d[..., 1]
    n = tex.shape[0]
    gx = np.clip((X + EXTENT) / TEXEL, 0, n - 1.000001)
    gy = np.clip((Y + EXTENT) / TEXEL, 0, n - 1.000001)
    x0, y0 = np.floor(gx).astype(int), np.floor(gy).astype(int)
    fx, fy = gx - x0, gy - y0
    val = ((1 - fy) * ((1 - fx) * tex[y0, x0] + fx * tex[y0, x0 + 1])
           + fy * ((1 - fx) * tex[y0 + 1, x0] + fx * tex[y0 + 1, x0 + 1]))
    val = np.round(val) + rng.integers(-2, 3, val.shape)
    return np.clip(val, 0, 255).astype(np.uint8)


def make_warp_scene(kind, steps=40, n_features=48, boxsize=11, seed=0, margin=70, sigma=4.0):
    rng = np.random.default_rng(0x3A9F00 + seed)
    cam8 = CAM.copy()
    B, half = boxsize, (boxsize - 1) // 2
    tex = make_texture(rng, sigma)
    poses, v, omega = trajectory(kind, steps)
    frames = np.stack([render(cam8, p, tex, rng) for p in poses])
    pix = synth._feature_pixels(rng, int(cam8[0]), int(cam8[1]), n_features, margin)
    d = rays(cam8, poses[0])[pix[:, 1], pix[:, 0]]
    y = poses[0, :3] + ((PLANE_Z - poses[0, 2]) / d[:, 2])[:, None] * d
    patches = np.stack([frames[0][py - half:py + half + 1, px - half:px + half + 1] for px, py in pix])
    x0 = np.concatenate([poses[0], v, omega, y.ravel()])
    n = x0.size
    sd = np.concatenate([np.full(3, 1e-3), np.full(4, 1e-3), np.full(3, 1e-2), np.full(3, 1e-2),
                         np.full(n - 13, 1e-3)])
    return WarpScene(name=kind, cam8=cam8, boxsize=B, poses=poses, v=v, omega=omega, frames=frames, y=y,
                     xp_org=np.tile(poses[0], (n_features, 1)), patches=patches, pix=pix, x0=x0,
                     P0=np.diag(sd * sd))


def angle_deg(q1, q2):
    """The rotation angle between the orientations q1 and q2 in degrees."""
    q1, q2 = q1 / np.linalg.norm(q1), q2 / np.linalg.norm(q2)
    return float(np.degrees(2 * np.arccos(min(1.0, abs(float(q1 @ q2))))))
