"""Deterministic synthetic inputs for the SceneLib2 hot path (BASELINE.md §3, SURVEY.md §8(d)).

Frames are band-limited noise textures (uniform noise, Gaussian blur sigma = 1.5 px, contrast
stretched so that every BxB window has sigma >= 10); templates are cut from frame 0 at the
features' projected pixel; frame t is frame 0 under a global integer shift |d| <= 3 px plus
i.i.d. +-2 grey-level noise (d_t is a random walk with steps <= 1 px), so the true match of
feature i in frame t is pix_i + d_t.
The 3-D scene is consistent with the reference's camera model (camera.cpp:90-114, inverse
:132-157) so that the EKF's predicted measurement h_i lands on pix_i at t = 0.

Seeds: 0x5CE7E1B2 ^ (config_id << 16) ^ stream_id  (numpy PCG64).
Pure numpy; no oracle, no CUDA.
"""
from dataclasses import dataclass, field

import numpy as np

SEED0 = 0x5CE7E1B2

# BASELINE.json configs (C1..C4; C5 = 8 x C3, one stream per GPU)
CONFIGS = {
    "C1": dict(config_id=1, width=320, height=240, n_features=20, boxsize=11, radius=None,
               n_select=10, margin=31),
    "C2": dict(config_id=2, width=320, height=240, n_features=50, boxsize=11, radius=20,
               n_select=50, margin=31),
    "C3": dict(config_id=3, width=640, height=480, n_features=100, boxsize=15, radius=40,
               n_select=100, margin=56),
    "C4": dict(config_id=4, width=320, height=240, n_features=100, boxsize=11, radius=20,
               n_select=100, margin=31),
}


def camera_params(width, height):
    """(width,height,fku,fkv,u0,v0,kd1,sd): data/SceneLib2.cfg:24-31 scaled with resolution."""
    s = width / 320.0
    return np.array([width, height, 195.0 * s, 195.0 * s, 162.0 * s, 125.0 * s, 9e-6 / (s * s), 1.0])


def project(cam8, yr):
    """camera.cpp:90-114 (ideal camera frame point -> distorted pixel)."""
    fku, fkv, u0, v0, kd1 = cam8[2], cam8[3], cam8[4], cam8[5], cam8[6]
    uc = -fku * yr[..., 0] / yr[..., 2]
    vc = -fkv * yr[..., 1] / yr[..., 2]
    f = np.sqrt(1 + 2 * kd1 * (uc * uc + vc * vc))
    return np.stack([uc / f + u0, vc / f + v0], axis=-1)


def unproject(cam8, h, depth):
    """camera.cpp:132-157 scaled to a given depth along the optical axis."""
    fku, fkv, u0, v0, kd1 = cam8[2], cam8[3], cam8[4], cam8[5], cam8[6]
    cu, cv = h[..., 0] - u0, h[..., 1] - v0
    f = np.sqrt(1 - 2 * kd1 * (cu * cu + cv * cv))
    return np.stack([cu / f / -fku * depth, cv / f / -fkv * depth, depth * np.ones_like(cu)], axis=-1)


def _gauss_kernel(sigma):
    r = int(np.ceil(4 * sigma))
    x = np.arange(-r, r + 1, dtype=np.float64)
    k = np.exp(-0.5 * (x / sigma) ** 2)
    return k / k.sum()


def make_texture(rng, height, width, sigma=1.5):
    """uint8 texture whose local standard deviation is comfortably above the sigma >= 10 gate."""
    k = _gauss_kernel(sigma)
    r = len(k) // 2
    a = rng.random((height + 2 * r, width + 2 * r))
    a = np.apply_along_axis(lambda m: np.convolve(m, k, mode="valid"), 1, a)
    a = np.apply_along_axis(lambda m: np.convolve(m, k, mode="valid"), 0, a)
    a = (a - a.mean()) / a.std()
    return np.clip(128.0 + 56.0 * a, 0, 255).astype(np.uint8)


def shift_image(img, dx, dy):
    """out[y, x] = img[y - dy, x - dx] with edge replication."""
    h, w = img.shape
    ys = np.clip(np.arange(h) - dy, 0, h - 1)
    xs = np.clip(np.arange(w) - dx, 0, w - 1)
    return img[np.ix_(ys, xs)]


@dataclass
class Scene:
    name: str
    cam8: np.ndarray
    delta_t: float
    boxsize: int
    n_select: int
    search_override: tuple          # (P00,P01,P11) or (0,0,0)
    x0: np.ndarray                  # (n,)   [xv(13) | y_0 | y_1 ...]
    P0: np.ndarray                  # (n,n)
    xp_org: np.ndarray              # (N,7)
    patches: np.ndarray             # (N,B,B) u8
    pix: np.ndarray                 # (N,2) int, template centre in frame 0
    frames: np.ndarray              # (T,H,W) u8
    shifts: np.ndarray              # (T,2) int
    meta: dict = field(default_factory=dict)

    @property
    def n_features(self):
        return self.patches.shape[0]

    @property
    def n(self):
        return self.x0.size

    @property
    def width(self):
        return int(self.cam8[0])

    @property
    def height(self):
        return int(self.cam8[1])


def _feature_pixels(rng, width, height, n, margin):
    """n distinct integer pixels on a jittered grid inside [margin, dim-1-margin]."""
    w, h = width - 2 * margin, height - 2 * margin
    cols = int(np.ceil(np.sqrt(n * w / h)))
    rows = int(np.ceil(n / cols))
    cw, ch = w / cols, h / rows
    cells = [(r, c) for r in range(rows) for c in range(cols)]
    idx = rng.permutation(len(cells))[:n]
    pts = []
    for i in sorted(idx):
        r, c = cells[i]
        px = margin + int(c * cw + rng.integers(0, max(1, int(cw))))
        py = margin + int(r * ch + rng.integers(0, max(1, int(ch))))
        pts.append((min(px, width - 1 - margin), min(py, height - 1 - margin)))
    return np.array(pts, dtype=np.int64)


def make_prior_covariance(rng, n, sig_r=0.010, sig_q=0.005, sig_v=0.05, sig_w=0.05, sig_y=0.020,
                          rank=16, mix=0.3):
    """Dense SPD prior: D (mix * Chat + (1-mix) I) D with a rank-`rank` correlation part.
    Scaled so that innovation sigmas are ~6-7 px at 320x240 (3 sigma ~ +-20 px)."""
    d = np.concatenate([np.full(3, sig_r), np.full(4, sig_q), np.full(3, sig_v), np.full(3, sig_w),
                        np.full(n - 13, sig_y)])
    a = rng.standard_normal((n, rank))
    c = a @ a.T
    s = 1.0 / np.sqrt(np.diag(c))
    c = c * s[:, None] * s[None, :]
    corr = mix * c + (1.0 - mix) * np.eye(n)
    p = d[:, None] * corr * d[None, :]
    return 0.5 * (p + p.T)


def make_scene(name="C2", stream_id=0, n_frames=8, known_patches=None, override=True,
               n_features=None, seed_extra=0, camera=None, delta_t=None):
    """Build the synthetic scene of one camera stream for BASELINE config `name`.  `camera` (width, height, fku, fkv,
    u0, v0, kd1, sd) renders it for that camera and image instead of the config's; `delta_t` sets its frame period
    (default 0.033333333).  With both left at None the scene is the config's own, draw for draw."""
    cfg = dict(CONFIGS[name])
    if n_features is not None:
        cfg["n_features"] = n_features
        cfg["n_select"] = min(cfg["n_select"], n_features) if name != "C1" else cfg["n_select"]
    rng = np.random.default_rng((SEED0 ^ (cfg["config_id"] << 16) ^ stream_id) + (seed_extra << 40))
    if camera is None:
        cam8 = camera_params(cfg["width"], cfg["height"])
    else:
        cam8 = np.array(camera, dtype=np.float64).reshape(8)
        cfg["width"], cfg["height"] = int(cam8[0]), int(cam8[1])
    W, H, N, B = cfg["width"], cfg["height"], cfg["n_features"], cfg["boxsize"]
    half = (B - 1) // 2

    frame0 = make_texture(rng, H, W)
    pix = _feature_pixels(rng, W, H, N, cfg["margin"])
    if camera is not None:
        # the camera model reaches only the pixels with 2 kd1 r^2 < 1 (r: distance to the principal point; the
        # undistortion of camera.cpp:132-157): with strong distortion, pull features towards the principal point
        pp = cam8[4:6]
        r2 = ((pix - pp) ** 2).sum(axis=1)
        far = 2.0 * cam8[6] * r2 > 0.8
        if far.any():
            scale = np.sqrt(0.8 / (2.0 * cam8[6] * r2[far]))
            pix[far] = np.floor(pp + (pix[far] - pp) * scale[:, None]).astype(np.int64)

    # C1: the first four features are the reference's known target corners
    # (data/SceneLib2.cfg:267-305) drawn with the shipped 11x11 templates.
    xv0 = np.array([0.0, 0.0, -0.60, 1.0, 0.0, 0.0, 0.0, 0.0, 0.0, -0.02, 0.0, 0.0, 0.01])
    if name != "C1":
        xv0[9] = -0.005
    y = np.zeros((N, 3))
    depth = rng.uniform(0.45, 1.1, size=N)
    start = 0
    if name == "C1" and known_patches is not None:
        known_y = np.array([[0.105, 0.07425, 0.0], [-0.105, 0.07425, 0.0],
                            [0.105, -0.07425, 0.0], [-0.105, -0.07425, 0.0]])
        hk = project(cam8, known_y - xv0[:3])
        for i in range(4):
            pix[i] = np.round(hk[i]).astype(np.int64)
            y[i] = known_y[i]
            px, py = pix[i]
            frame0[py - half:py + half + 1, px - half:px + half + 1] = known_patches[i]
        start = 4
    for i in range(start, N):
        yr = unproject(cam8, pix[i].astype(np.float64), depth[i])
        y[i] = xv0[:3] + yr  # q = identity: world = camera axes

    patches = np.stack([frame0[py - half:py + half + 1, px - half:px + half + 1].copy()
                        for px, py in pix])

    shifts = np.zeros((n_frames, 2), dtype=np.int64)
    frames = np.zeros((n_frames, H, W), dtype=np.uint8)
    for t in range(n_frames):
        if t > 0:  # bounded random walk: at most 1 px per frame, |d| <= 3 px
            shifts[t] = np.clip(shifts[t - 1] + rng.integers(-1, 2, size=2), -3, 3)
        noise = rng.integers(-2, 3, size=(H, W))
        f = shift_image(frame0, int(shifts[t, 0]), int(shifts[t, 1])).astype(np.int64) + noise
        frames[t] = np.clip(f, 0, 255).astype(np.uint8)

    n = 13 + 3 * N
    x0 = np.concatenate([xv0, y.reshape(-1)])
    P0 = make_prior_covariance(rng, n)
    xp_org = np.tile(xv0[:7], (N, 1))
    if cfg["radius"] is not None and override:
        r = float(cfg["radius"])
        search_override = (9.0 / (r * r), 0.0, 9.0 / (r * r))
    else:
        search_override = (0.0, 0.0, 0.0)
    return Scene(name=name, cam8=cam8, delta_t=0.033333333 if delta_t is None else float(delta_t), boxsize=B, n_select=cfg["n_select"],
                 search_override=search_override, x0=x0, P0=P0, xp_org=xp_org, patches=patches,
                 pix=pix, frames=frames, shifts=shifts,
                 meta=dict(config=cfg, stream_id=stream_id, depth=depth))


def algorithmic_search_bytes(boxsize, radius):
    """SURVEY.md §8(d): window + template + 24 B params + 16 B result, per feature."""
    w = 2 * radius + boxsize
    return w * w + boxsize * boxsize + 40


def ekf_structured_flops(n, m):
    """SURVEY.md §8(d) structured-minimum FLOPs of one EKF update (nz = 10 non-zeros per H row)."""
    nz = 10
    return (2 * m * nz * n + 2 * m * nz * m + m ** 3 / 3.0 + 2 * m * m * n + n * n * m
            + 2 * n * m + 2 * m * m)


def write_reference_case(directory, sc, Pxx):
    """A scene in the reference's own input format: `key = value;` cfg (data/SceneLib2.cfg), one PGM template per
    known feature (feature.cpp:119 reads them with cv::imread) and the frames as raw 8-bit gray.  Returns the cfg path."""
    import os
    lines = ["cam.width = %d;" % sc.width, "cam.height = %d;" % sc.height,
             "cam.fku = %d;" % sc.cam8[2], "cam.fkv = %d;" % sc.cam8[3], "cam.u0 = %d;" % sc.cam8[4],
             "cam.v0 = %d;" % sc.cam8[5], "cam.kd1 = %r;" % float(sc.cam8[6]), "cam.sd = 1;",
             "params.delta_t = %r;   # frame period" % sc.delta_t,
             "params.number_of_features_to_select = %d;" % sc.n_select,
             "params.number_of_features_to_keep_visible = 12;"]
    names = ["rw_x", "rw_y", "rw_z", "qwr_w", "qwr_x", "qwr_y", "qwr_z", "vw_x", "vw_y", "vw_z",
             "ww_x", "ww_y", "ww_z"]
    for k, nm in enumerate(names):
        lines.append("state.%s = %r;" % (nm, float(sc.x0[k])))
    for i in range(13):
        for j in range(13):
            lines.append("state.pxx%d_%d = %r;" % (i, j, float(Pxx[i, j])))
    for i in range(sc.n_features):
        p = "f%d" % (i + 1)
        y = sc.x0[13 + 3 * i:16 + 3 * i]
        lines += ["%s.yi_x = %r;" % (p, float(y[0])), "%s.yi_y = %r;" % (p, float(y[1])),
                  "%s.yi_z = %r;" % (p, float(y[2]))]
        for k in range(7):
            lines.append("%s.xp_org_%d = %r;" % (p, k, float(sc.xp_org[i, k])))
        lines.append("%s.identifier = patch%d.pgm;" % (p, i))
        with open(os.path.join(directory, "patch%d.pgm" % i), "wb") as f:
            f.write(b"P5\n%d %d\n255\n" % (sc.boxsize, sc.boxsize) + sc.patches[i].tobytes())
    lines.append("device.max_features = %d;" % max(sc.n_features, 4))
    cfg = os.path.join(directory, "case.cfg")
    open(cfg, "w").write("\n".join(lines) + "\n")
    sc.frames.tofile(os.path.join(directory, "frames.raw"))
    return cfg
