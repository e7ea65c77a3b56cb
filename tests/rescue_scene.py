"""Scenes for the consensus rescue (sl2_set_stream_rescue): a settled map, some features whose position is still
uncertain (as a depth ray converted by sl2_append_feature leaves them), and distractors.

  settled map    synth scene with feature sigmas / 10 and camera sigmas x 2 (the consensus tests' converged map)
  new features   `new`: estimate = truth + e, e ~ N(0, sigma^2 I) per feature, and the covariance of y = r + e with e
                 independent of the state: P[y, :] = P[r, :], P[y, y] = P[r, r] + sigma^2 I.  That is the covariance
                 column (Pcol) a converted ray gives, cross terms to the camera included.
  distractors    `wrong`: the true location occluded by noise, the template pasted OFFSET px away (|OFFSET| = 10.8 px),
                 every frame; with `spread`, each distractor at its own direction, 11 px away, so that the distractors
                 do not agree with each other.
A match is correct iff z = pix + shift[t]."""
import numpy as np

from scenelib2_b200 import synth

OFFSET = (9, -6)


def rescue_scene(name="C2", stream_id=0, n_frames=16, n_features=None, new=(), sigma=0.05, wrong=(), seed=0,
                 camera=None, sc=None, spread=False):
    if sc is None:
        sc = synth.make_scene(name, stream_id=stream_id, n_frames=n_frames, n_features=n_features, camera=camera)
    rng = np.random.default_rng(4242 + 131 * stream_id + seed)
    d = np.concatenate([np.full(13, 2.0), np.full(sc.n - 13, 0.1)])
    P = d[:, None] * sc.P0 * d[None, :]
    x = sc.x0.copy()
    new = list(new)
    for f in new:  # rows / columns of the camera position, then the feature's own uncertainty
        p = 13 + 3 * f
        P[p:p + 3, :] = P[0:3, :]
        P[:, p:p + 3] = P[:, 0:3]
    for f in new:
        p = 13 + 3 * f
        for g in new:
            q = 13 + 3 * g
            P[p:p + 3, q:q + 3] = P[0:3, 0:3]
        P[p:p + 3, p:p + 3] += sigma * sigma * np.eye(3)
        e = rng.standard_normal(3) * sigma
        x[p:p + 3] = sc.x0[p:p + 3] + e
    sc.P0 = 0.5 * (P + P.T)
    sc.x0 = x
    B = sc.boxsize
    half = (B - 1) // 2
    frames = sc.frames.copy()
    nrng = np.random.default_rng(777 + stream_id)
    off = {}
    for f in wrong:
        a = nrng.uniform(0.0, 2.0 * np.pi)
        off[f] = np.round(11.0 * np.array([np.cos(a), np.sin(a)])).astype(np.int64) if spread else np.array(OFFSET)
    for t in range(len(frames)):
        for f in wrong:
            u, v = sc.pix[f] + sc.shifts[t]
            frames[t, v - half - 2:v + half + 3, u - half - 2:u + half + 3] = nrng.integers(0, 256, (B + 4, B + 4))
        for f in wrong:
            u, v = sc.pix[f] + sc.shifts[t] + off[f]
            frames[t, v - half:v + half + 1, u - half:u + half + 1] = sc.patches[f]
    sc.frames = frames
    sc.meta["new"] = new
    sc.meta["wrong"] = list(wrong)
    return sc


def truth(sc, t):
    return sc.pix + sc.shifts[t]
