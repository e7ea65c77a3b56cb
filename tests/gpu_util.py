"""Helpers shared by the GPU parity tests (CUDA path through the C ABI vs the CPU oracle)."""
import dataclasses

import numpy as np

import scenelib2_b200 as sl2
from model_cases import quat_to_R
from scenelib2_b200 import synth

# north star: "FP state/covariance within 1e-5 relative".  The tests hold the CUDA path to a
# much tighter bound (different summation order only) so that real bugs cannot hide.
RTOL_NORTH_STAR = 1e-5
RTOL_TEST = 1e-8
# the step's measurement predictions against the oracle's: x carries its (summation-order) error into h and S.  Over
# the GPU suite on an H100 the worst were 8.5e-13 px and 5.2e-13 relative; the bounds leave a factor of ~10
H_ATOL_STEP = 1e-11         # px
S_RTOL_STEP = 1e-11
# worst (h px, S relative) deviation check_streams_against_oracle has seen in this process
WORST_PREDICTION = [0.0, 0.0]


def oracle_slam_from_scene(oracle, sc):
    cfg = oracle.make_config(width=sc.width, height=sc.height, fku=sc.cam8[2], fkv=sc.cam8[3],
                             u0=sc.cam8[4], v0=sc.cam8[5], kd1=sc.cam8[6], sd=sc.cam8[7],
                             delta_t=sc.delta_t, n_select=sc.n_select, boxsize=sc.boxsize,
                             search_override=sc.search_override)
    s = oracle.Slam(cfg)
    for i in range(sc.n_features):
        s.add_feature(sc.x0[13 + 3 * i:16 + 3 * i], sc.xp_org[i], sc.patches[i])
    s.set_state(sc.x0, sc.P0)
    return s


def ctx_from_scenes(scenes, frame_slots=1, **kw):
    cfg = sl2.config_for_scene(scenes[0], num_streams=len(scenes), frame_slots=frame_slots, **kw)
    ctx = sl2.Context(cfg)
    for s, sc in enumerate(scenes):
        sl2.load_scene(ctx, s, sc)
    return ctx


def ring_block(img, H, W, rng):
    """An H x W ring block with the stream's image in its top-left and fresh noise everywhere else."""
    out = rng.integers(0, 256, (H, W), dtype=np.uint8)
    out[:img.shape[0], :img.shape[1]] = img
    return out


def step_frames(ctx, frames, slot=0):
    """One fused step of every stream on `frames` (a frame set, e.g. num_streams x H x W) in ring slot `slot`."""
    ctx.set_frames(slot, frames)
    ctx.step(slot)
    ctx.sync()


def stream_result(ctx, s, jacobians=False, camera=False):
    """What the getters show of stream s: x, P and the feature getters; with `jacobians` also the features'
    dh_dxv, dh_dy, R and nu; with `camera` also the stream config (as float64) and the map size."""
    x, P = ctx.get_state(s)
    out = dict(x=x, P=P, **ctx.features(s))
    if jacobians:
        out.update(zip(("dh_dxv", "dh_dy", "R", "nu"), ctx.feature_jacobians(s)))
    if camera:
        sc = ctx.stream_config(s)
        out["cam"] = np.array([getattr(sc, k) for k, _ in sl2.Sl2StreamConfig._fields_], np.float64)
        out["nf"] = np.array([ctx.num_features(s)])
    return out


def assert_same_bytes(a, b, where, keys=None):
    """a[k] and b[k] have the same shape, dtype and bytes for every k in `keys`; without `keys`, a and b have the
    same key set and every key is compared."""
    if keys is None:
        assert a.keys() == b.keys(), where
        keys = a
    for k in keys:
        assert a[k].shape == b[k].shape and a[k].dtype == b[k].dtype, (where, k)
        assert a[k].tobytes() == b[k].tobytes(), (where, k)


def ctx_for_image(image, patches, radius=20, boxsize=None):
    """Context with one stream whose frame is `image` and whose templates are `patches`."""
    patches = np.ascontiguousarray(patches, np.uint8)
    n, B = patches.shape[0], patches.shape[1]
    cfg = sl2.default_config()
    cfg.width, cfg.height = image.shape[1], image.shape[0]
    cfg.boxsize = B
    cfg.max_features = max(n, 1)
    cfg.search_tile_radius = radius
    ctx = sl2.Context(cfg)
    ctx.set_features(0, np.zeros((n, 3)), np.tile([0, 0, 0, 1, 0, 0, 0.0], (n, 1)), patches)
    ctx.set_frame(0, 0, image)
    return ctx


def state_err(xg, Pg, xo, Po):
    """Largest error relative to the natural scale sqrt(P_ii P_jj) (covariance) / sigma_i (state)."""
    d = np.sqrt(np.abs(np.diag(Po))) + 1e-300
    eP = np.abs(Pg - Po) / (d[:, None] * d[None, :])
    ex = np.abs(xg - xo) / np.maximum(np.abs(xo), d)
    return float(ex.max()), float(eP.max())


def assert_state_close(xg, Pg, xo, Po, rtol=RTOL_TEST):
    ex, eP = state_err(xg, Pg, xo, Po)
    assert ex <= rtol, "state error %.3e" % ex
    assert eP <= rtol, "covariance error %.3e" % eP
    return ex, eP


def check_streams_against_oracle(ctx, oracles, picks, scenes_of, frame):
    """Step the oracle of every stream in `picks` on `frame` of its scene and compare it with the stream's state after
    the fused step: map size, selection, flags, match positions and counters exactly, the step's predictions h and S
    of every feature at H_ATOL_STEP / S_RTOL_STEP, x and P at RTOL_TEST, P exactly symmetric.  Returns the worst
    (state, covariance) errors."""
    worst = (0.0, 0.0)
    for s in picks:
        o = oracles[s]
        o.step(scenes_of(s).frames[frame])
        fg, fo = ctx.features(s), o.features()
        assert ctx.num_features(s) == o.num_features, s
        assert (fg["select_rank"] == fo["select_rank"]).all() and (fg["flags"] == fo["flags"]).all(), s
        ok = (fo["flags"] & 2) > 0
        assert (fg["z"][ok] == fo["z"][ok]).all(), s
        assert (fg["attempted"] == fo["attempted"]).all() and (fg["successful"] == fo["successful"]).all(), s
        if len(fo["h"]):
            eh = float(np.abs(fg["h"] - fo["h"]).max())
            eS = float((np.abs(fg["S"] - fo["S"]).max(axis=1) / np.abs(fo["S"]).max(axis=1)).max())
            WORST_PREDICTION[0], WORST_PREDICTION[1] = max(WORST_PREDICTION[0], eh), max(WORST_PREDICTION[1], eS)
            assert eh <= H_ATOL_STEP and eS <= S_RTOL_STEP, (s, eh, eS)
        xg, Pg = ctx.get_state(s)
        e = assert_state_close(xg, Pg, *o.get_state())
        worst = (max(worst[0], e[0]), max(worst[1], e[1]))
        assert np.abs(Pg - Pg.T).max() == 0.0, s
    return worst


def quat_left(q):
    """L(q): q (x) p = L(q) p for quaternions (w, x, y, z)."""
    w, x, y, z = q
    return np.array([[w, -x, -y, -z], [x, w, -z, y], [y, z, w, -x], [z, -y, x, w]])


def rigid_transform(n, q_w):
    """T of rigid_transform_scene for a state of size n: blockdiag(R_w, L(q_w), R_w, I3, R_w, R_w, ...)."""
    R = quat_to_R(q_w)
    T = np.eye(n)
    T[0:3, 0:3] = R
    T[3:7, 3:7] = quat_left(q_w)
    T[7:10, 7:10] = R
    for k in range(13, n, 3):
        T[k:k + 3, k:k + 3] = R
    return T


def rigid_transform_scene(sc, q_w, t_w):
    """The scene in a world moved by the rigid motion (R_w = R(q_w), t_w): r, y and the position of xp_org map to
    R_w (.) + t_w, q and the q of xp_org to q_w (x) q, v to R_w v; omega is a body-frame rate (qnew = q (x) q(omega dt))
    and stays.  P becomes T P T^T (rigid_transform), made exactly symmetric.  The camera sees the same image, so the
    transformed scene tracks the same frames."""
    q_w = np.asarray(q_w, np.float64) / np.linalg.norm(q_w)
    t_w = np.asarray(t_w, np.float64)
    R = quat_to_R(q_w)
    x = sc.x0.copy()
    x[0:3] = R @ x[0:3] + t_w
    x[3:7] = quat_left(q_w) @ x[3:7]
    x[7:10] = R @ x[7:10]
    x[13:] = (x[13:].reshape(-1, 3) @ R.T + t_w).ravel()
    T = rigid_transform(x.size, q_w)
    P = T @ sc.P0 @ T.T
    xp = sc.xp_org.copy()
    xp[:, :3] = xp[:, :3] @ R.T + t_w
    xp[:, 3:7] = xp[:, 3:7] @ quat_left(q_w).T
    return dataclasses.replace(sc, x0=x, P0=0.5 * (P + P.T), xp_org=xp, meta=dict(sc.meta, rigid=(q_w, t_w)))


def untransform_state(x, P, q_w, t_w):
    """x and P of a run of rigid_transform_scene(sc, q_w, t_w) mapped back to the frame of sc."""
    R = quat_to_R(q_w)
    T = rigid_transform(x.size, q_w)
    xb = T.T @ x
    xb[0:3] -= R.T @ t_w
    for k in range(13, x.size, 3):
        xb[k:k + 3] -= R.T @ t_w
    return xb, T.T @ P @ T


def update_variant(cap, nf, bad=0, out_of_view=False, stream_id=0, n_frames=12):
    """C4-sized scene of `nf` features for a context of capacity `cap` that selects up to `cap` features, so that
    every visible feature is selected.  The templates of `bad` features (spread over the map) are replaced by random
    bytes: they are selected but never found, so K = nf - bad measurements per step, and the default
    min_attempts = 10 culls them at step 10.  `out_of_view` moves every feature to the side of the view: nothing is
    selected (K = 0 with nf > 0)."""
    sc = synth.make_scene("C4", stream_id=stream_id, n_frames=n_frames, n_features=nf)
    sc.n_select = cap
    if bad:
        idx = np.linspace(0, nf - 1, bad).round().astype(int)
        assert len(set(idx)) == bad
        patches = sc.patches.copy()
        rng = np.random.default_rng(1000 + stream_id)
        patches[idx] = rng.integers(0, 256, patches[idx].shape, dtype=np.uint8)
        sc.patches = patches
    if out_of_view:
        sc.x0 = sc.x0.copy()
        sc.x0[13:] += np.tile([3.0, 0.0, 0.0], nf)
    sc.meta["variant"] = (nf, bad, out_of_view)
    return sc


def large_variant(nf, in_view, bad=0, stream_id=0, n_frames=12, n_select=sl2.lib.SL2_MAX_MEASURED):
    """C4-sized scene of nf features; features >= in_view moved to the side of the view, `bad` templates (spread over
    the features in view) replaced by random bytes."""
    sc = synth.make_scene("C4", stream_id=stream_id, n_frames=n_frames, n_features=nf)
    sc.n_select = n_select
    if bad:
        idx = np.linspace(0, in_view - 1, bad).round().astype(int)
        assert len(set(idx)) == bad
        patches = sc.patches.copy()
        rng = np.random.default_rng(2000 + stream_id)
        patches[idx] = rng.integers(0, 256, patches[idx].shape, dtype=np.uint8)
        sc.patches = patches
    if in_view < nf:
        sc.x0 = sc.x0.copy()
        sc.x0[13 + 3 * in_view:] += np.tile([3.0, 0.0, 0.0], nf - in_view)
    sc.meta["variant"] = (nf, in_view, bad)
    return sc


def camera(width, height, focal=1.0, shift=(0.0, 0.0), kd1=1.0, sd=1.0):
    """A calibration derived from the reference's (synth.camera_params) for a width x height image."""
    c = synth.camera_params(width, height)
    c[2:4] *= focal
    c[4] += shift[0]
    c[5] += shift[1]
    c[6] *= kd1
    c[7] = sd
    return c


# calibrations that fit a 320x240 ring (the benchmark's C4 shape)
CAMS_320 = [camera(320, 240), camera(320, 240, focal=1.3, shift=(9.0, -7.0), kd1=3.0), camera(288, 224, focal=0.9),
            camera(320, 240, sd=2.0)]


def random_measurements(rng, n, nf, K):
    """K random measured features of a map of nf (state size n): the host rows of sl2_ekf_update and the dense H and
    R of kalman.cpp."""
    feats = rng.permutation(nf)[:K].astype(np.int32)
    Hxv = np.zeros((2 * K, 13))
    Hxv[:, :7] = rng.standard_normal((2 * K, 7)) * 60
    Hy = rng.standard_normal((2 * K, 3)) * 300
    var = rng.uniform(1, 4, K)
    R = np.zeros((K, 2, 2))
    R[:, 0, 0] = R[:, 1, 1] = var
    nu = rng.standard_normal(2 * K) * 2
    H = np.zeros((2 * K, n))
    H[:, :13] = Hxv
    for k, f in enumerate(feats):
        H[2 * k:2 * k + 2, 13 + 3 * f:16 + 3 * f] = Hy[2 * k:2 * k + 2]
    return feats, Hxv, Hy, R, nu, H, np.kron(np.diag(var), np.eye(2))


def patch_snapshot_field(blob, name, index, value):
    """The blob with element `index` of per-feature section `name` replaced."""
    h = sl2.read_snapshot(blob)
    layout, _ = sl2.lib.snapshot_layout(h["nfeat"], h["boxsize"])
    off, _, dt = layout[name]
    b = bytearray(blob)
    b[off + index * np.dtype(dt).itemsize:off + (index + 1) * np.dtype(dt).itemsize] = np.array([value], dt).tobytes()
    return bytes(b)


# ---- update-shape regimes: every launch regime of one capacity against recorded oracle runs --------------------------
def record_oracle(oracle, scenes, T, states=True):
    """One oracle per variant stepped over the T frames (threads across variants); per variant and step: map size,
    features, and (states) x and P."""
    slams = [oracle_slam_from_scene(oracle, sc) for sc in scenes]
    nthreads = max(1, min(len(slams), oracle.usable_cpus()))
    traj = [[] for _ in slams]
    for t in range(T):
        oracle.run_slams(slams, [sc.frames[t][None] for sc in scenes], 1, nthreads)
        for rec, o in zip(traj, slams):
            rec.append(dict(nf=o.num_features, f=o.features(), xP=o.get_state() if states else None))
    return traj


class Replay:
    """A recorded oracle trajectory with the surface check_streams_against_oracle uses (each step() advances one
    recorded step; the frames are those the trajectory was recorded on)."""

    def __init__(self, steps):
        self.steps, self.t = steps, -1

    def step(self, frame):
        self.t += 1

    @property
    def num_features(self):
        return self.steps[self.t]["nf"]

    def features(self):
        return self.steps[self.t]["f"]

    def get_state(self):
        return self.steps[self.t]["xP"]


def run_regimes(scenes, cap, regimes, T, snap_steps, traj):
    """Every regime (name, B, step groups) of one capacity: stream s of a B-stream context of capacity `cap` runs the
    variant scenes[(5 s) % U] (neighbouring streams hold different variants; U coprime to 5) for T steps.  The first
    stream of every variant and streams 0, nsm - 1, nsm and B - 1 are checked against the variant's recorded oracle
    trajectory `traj` at every step; after the last step every stream is bit-identical to the first stream of its
    variant, and at every step of `snap_steps` every variant is bit-identical across the regimes.  Returns the
    snapshots {(regime, step): {variant: stream_result}} and the worst (state, covariance) error of each regime."""
    import torch
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    U = len(scenes)
    scene_of = lambda s: scenes[(s * 5) % U]  # noqa: E731
    snaps, worst = {}, {}
    for name, B, groups in regimes:
        first = {}
        for s in range(B):
            first.setdefault((s * 5) % U, s)
        assert len(first) == U
        picks = sorted(({0, nsm - 1, nsm, B - 1} & set(range(B))) | set(first.values()))
        ctx = ctx_from_scenes([scene_of(s) for s in range(B)], frame_slots=2, max_features=cap)
        try:
            if groups > 1:
                ctx.set_step_groups(groups)
            replays = {s: Replay(traj[(s * 5) % U]) for s in picks}
            worst[name] = (0.0, 0.0)
            for t in range(T):
                step_frames(ctx, np.stack([scene_of(s).frames[t] for s in range(B)]), t % 2)
                w = check_streams_against_oracle(ctx, replays, picks, scene_of, t)
                worst[name] = (max(worst[name][0], w[0]), max(worst[name][1], w[1]))
                if t in snap_steps:
                    snaps[name, t] = {u: stream_result(ctx, s) for u, s in first.items()}
            for s in range(B):
                u = (s * 5) % U
                if s != first[u]:
                    assert_same_bytes(stream_result(ctx, s), snaps[name, T - 1][u],
                                      (name, "stream", s, "variant", scenes[u].meta["variant"]))
        finally:
            ctx.close()
    names = [name for name, _, _ in regimes]
    for name in names[1:]:
        for t in snap_steps:
            for u in range(U):
                assert_same_bytes(snaps[name, t][u], snaps[names[0], t][u],
                                  (name, "vs", names[0], "step", t, "variant", scenes[u].meta["variant"]))
    return snaps, worst


def random_puinv(rng, n, lo, hi, iso_fraction=0.5):
    out = np.zeros((n, 3))
    for i in range(n):
        a, b = rng.uniform(lo, hi, 2)
        r = 0.0 if rng.random() < iso_fraction else rng.uniform(-0.8, 0.8)
        if rng.random() < iso_fraction:
            b = a
        Si = np.linalg.inv(np.array([[a * a / 9, r * a * b / 9], [r * a * b / 9, b * b / 9]]))
        out[i] = [Si[0, 0], Si[0, 1], Si[1, 1]]
    return out


__all__ = ["sl2", "synth", "np"]
