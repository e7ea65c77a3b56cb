"""A rendered slanted plane for the patch normals (pure NumPy, seeded): warp_scene's texture on a plane through (0, 0,
PLANE_Z) tilted by TILT degrees about the y axis away from the frame-0 line of sight, so a feature's fixed normal
(facing the frame-0 camera) is about TILT wrong.  The camera moves on an arc about the plane's centre from the frame-0
pose toward the head-on view.  Pixels, templates, features and the initial state are made as warp_scene makes them.
Also the true tilt theta of a feature on a plane of known normal."""
import numpy as np

import normals_ref
import warp_scene
from scenelib2_b200 import synth
from warp_scene import DT, EXTENT, PLANE_Z, TEXEL, WarpScene, quat_axis, rays

TILT = 45.0  # degrees


def plane_normal(tilt_deg):
    """The plane's unit normal, on the side of the frame-0 camera at the origin."""
    t = np.radians(tilt_deg)
    return np.array([-np.sin(t), 0.0, -np.cos(t)])


def arc(steps, end_deg):
    """Poses (steps + 1, 7), v and omega of the arc of radius PLANE_Z about (0, 0, PLANE_Z) from 0 to end_deg."""
    T = steps * DT
    w = np.radians(end_deg) / T
    c = np.array([0.0, 0.0, PLANE_Z])
    poses = np.zeros((steps + 1, 7))
    for k in range(steps + 1):
        phi = w * k * DT
        poses[k, :3] = c + PLANE_Z * np.array([-np.sin(phi), 0.0, -np.cos(phi)])
        poses[k, 3:] = quat_axis([0, 1, 0], phi)
    return poses, np.array([-PLANE_Z * w, 0.0, 0.0]), np.array([0.0, w, 0.0])


def render(cam8, pose, tex, rng, n):
    """The frame of the camera at pose: the texture of the plane through (0, 0, PLANE_Z) with unit normal n, in the
    plane's own axes (e1 in the x-z plane, e2 = y), sampled bilinearly, plus +-2 grey levels of noise."""
    d = rays(cam8, pose)
    r = pose[:3]
    P0 = np.array([0.0, 0.0, PLANE_Z])
    t = ((P0 - r) @ n) / (d @ n)
    X = r + t[..., None] * d - P0
    e2 = np.array([0.0, 1.0, 0.0])
    e1 = np.cross(e2, n)
    m = tex.shape[0]
    gx = np.clip((X @ e1 + EXTENT) / TEXEL, 0, m - 1.000001)
    gy = np.clip((X @ e2 + EXTENT) / TEXEL, 0, m - 1.000001)
    x0, y0 = np.floor(gx).astype(int), np.floor(gy).astype(int)
    fx, fy = gx - x0, gy - y0
    val = ((1 - fy) * ((1 - fx) * tex[y0, x0] + fx * tex[y0, x0 + 1])
           + fy * ((1 - fx) * tex[y0 + 1, x0] + fx * tex[y0 + 1, x0 + 1]))
    val = np.round(val) + rng.integers(-2, 3, val.shape)
    return np.clip(val, 0, 255).astype(np.uint8)


def make_slanted_scene(steps=40, end_deg=40.0, tilt_deg=TILT, n_features=32, boxsize=11, seed=0, margin=70,
                       sigma=4.0):
    rng = np.random.default_rng(0x4E0B00 + seed)
    cam8 = warp_scene.CAM.copy()
    B, half = boxsize, (boxsize - 1) // 2
    n = plane_normal(tilt_deg)
    tex = warp_scene.make_texture(rng, sigma)
    poses, v, omega = arc(steps, end_deg)
    frames = np.stack([render(cam8, p, tex, rng, n) for p in poses])
    pix = synth._feature_pixels(rng, int(cam8[0]), int(cam8[1]), n_features, margin)
    d = rays(cam8, poses[0])[pix[:, 1], pix[:, 0]]
    P0 = np.array([0.0, 0.0, PLANE_Z])
    y = poses[0, :3] + (((P0 - poses[0, :3]) @ n) / (d @ n))[:, None] * d
    patches = np.stack([frames[0][py - half:py + half + 1, px - half:px + half + 1] for px, py in pix])
    x0 = np.concatenate([poses[0], v, omega, y.ravel()])
    sd = np.concatenate([np.full(3, 1e-3), np.full(4, 1e-3), np.full(3, 1e-2), np.full(3, 1e-2),
                         np.full(x0.size - 13, 1e-3)])
    return WarpScene(name="slanted", cam8=cam8, boxsize=B, poses=poses, v=v, omega=omega, frames=frames, y=y,
                     xp_org=np.tile(poses[0], (n_features, 1)), patches=patches, pix=pix, x0=x0,
                     P0=np.diag(sd * sd))


def true_theta(y, xo, n):
    """The tilt theta whose nW(theta) is parallel to the unit normal n (the basis of normals_ref.basis)."""
    n0, E1, E2 = (np.array(v) for v in normals_ref.basis(xo, y))
    a = n @ n0
    return np.array([(n @ E1) / a, (n @ E2) / a])


def normal_angle_deg(y, xo, theta, n):
    """The angle between nW(theta) and the unit normal n, in degrees."""
    nW = np.array(normals_ref.normal(normals_ref.basis(xo, y), float(theta[0]), float(theta[1])))
    c = abs(nW @ n) / np.linalg.norm(nW)
    return float(np.degrees(np.arccos(min(1.0, c))))
