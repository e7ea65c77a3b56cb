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
