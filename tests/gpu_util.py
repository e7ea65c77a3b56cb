"""Helpers shared by the GPU parity tests (CUDA path through the C ABI vs the CPU oracle)."""
import numpy as np

import scenelib2_b200 as sl2
from scenelib2_b200 import synth

# north star: "FP state/covariance within 1e-5 relative".  The tests hold the CUDA path to a
# much tighter bound (different summation order only) so that real bugs cannot hide.
RTOL_NORTH_STAR = 1e-5
RTOL_TEST = 1e-8


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
    the fused step: map size, selection, flags, match positions and counters exactly, x and P at RTOL_TEST, P exactly
    symmetric.  Returns the worst (state, covariance) errors."""
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
        xg, Pg = ctx.get_state(s)
        e = assert_state_close(xg, Pg, *o.get_state())
        worst = (max(worst[0], e[0]), max(worst[1], e[1]))
        assert np.abs(Pg - Pg.T).max() == 0.0, s
    return worst


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
