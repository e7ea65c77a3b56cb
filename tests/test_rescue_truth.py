"""The consensus rescue's gate against its definition (tests/rescue_truth.py, np.longdouble): the extended-precision
truth is checked against the same definition at 50 digits (mpmath); the op-for-op restatement of the device's gate
(tests/rescue_ref.py), fed the state of a double-precision update 1, stays within q_band of the truth, and its
decisions equal the truth's wherever the truth's q is farther than q_band from chi2."""
import math

import mpmath
import numpy as np
import pytest

import rescue_oracle as ro
import rescue_ref
import rescue_truth as rt
from rescue_scene import rescue_scene


def case(seed, nf, n_inl, k, spread=4.0):
    """Prior x, P of a settled map with uncertain new features; the features k .. k + n_inl - 1 are inliers (z = h +
    about one sigma, rounded), the first k are rejected matches (z = h + 0.5 to `spread` innovation sigmas)."""
    rng = np.random.default_rng(seed)
    sc = rescue_scene("C2", n_frames=1, n_features=nf, new=range(0, min(k, nf)), sigma=0.03, seed=seed)
    x, P = sc.x0.copy(), sc.P0.copy()
    z = np.zeros((nf, 2))
    for i in range(nf):
        p = rescue_ref.predict(sc.cam8, x, x[13 + 3 * i:16 + 3 * i], P, 13 + 3 * i)
        a = rng.uniform(0, 2 * np.pi)
        r = rng.uniform(0.5, spread) if i < k else rng.uniform(0.0, 1.0)
        z[i] = np.round(p["h"] + np.linalg.cholesky(p["S"]) @ (r * np.array([np.cos(a), np.sin(a)])))
    rej = list(range(k))
    inl = list(range(k, k + n_inl))
    return sc.cam8, x, P, inl, z[inl], rej, z[rej]


def test_extended_truth_equals_50_digits():
    cam8, x, P, inl, zi, rej, zr = case(1, 6, 4, 2)
    q_ext, ok_ext, _ = rt.truth(cam8, x, P, inl, zi, rej, zr, 5.991)
    with mpmath.workdps(50):
        q_mp, ok_mp, _ = rt.truth(cam8, x, P, inl, zi, rej, zr, mpmath.mpf(5.991), ar=rt.Mp())
        for a, b in zip(q_ext, q_mp):
            assert abs(mpmath.mpf(float(a)) - b) <= mpmath.mpf(1e-15) * max(abs(b), 1)
    assert (ok_ext == ok_mp).all()


@pytest.mark.parametrize("seed", range(4))
def test_restatement_within_the_band_and_decisions_equal_the_truth(seed):
    cam8, x, P, inl, zi, rej, zr = case(10 + seed, 24, 16, 8)
    q_t, _, cond = rt.truth(cam8, x, P, inl, zi, rej, zr, 0.0)
    q_t = np.array([float(v) for v in q_t])
    x1, P1, _ = rt.update_1(rt.F64, cam8, x, P, inl, zi)
    n, m1 = x.size, 2 * len(inl)
    pos = (13 + 3 * np.array(rej)).astype(np.int32)
    _, q_r, _ = rescue_ref.gate(cam8, x1, P1, pos, zr, 0.0)
    band = np.array([rt.q_band(v, n, m1, cond) for v in q_t])
    assert (np.abs(q_r - q_t) <= band).all(), (np.abs(q_r - q_t) / band).max()
    held = 0
    for chi2 in sorted(q_t) + [float(np.median(q_t)), 5.991]:
        ok_r, _, _ = rescue_ref.gate(cam8, x1, P1, pos, zr, chi2)
        _, ok_t, _ = rt.truth(cam8, x, P, inl, zi, rej, zr, chi2)
        far = np.abs(q_t - chi2) > band
        assert (ok_r[far] == ok_t[far]).all(), chi2
        held += int(far.sum())
    assert held > 0


def test_a_nan_q_is_never_rescued_by_the_truth_or_the_restatement():
    cam8, x, P, inl, zi, rej, zr = case(3, 6, 0, 2)
    p = 13 + 3 * rej[0]
    P = P.copy()
    P[p:p + 3, p:p + 3] -= 10.0 * np.eye(3)  # S' of feature 0 indefinite
    pos = (13 + 3 * np.array(rej)).astype(np.int32)
    ok_r, q_r, _ = rescue_ref.gate(cam8, x, P, pos, zr, 1e300)
    assert math.isnan(q_r[0]) and not ok_r[0] and ok_r[1]
    ok_o, q_o, _, _ = ro.gate(cam8, x, P, pos, zr, 1e300)
    assert math.isnan(q_o[0]) and not ok_o[0] and ok_o[1]
    with np.errstate(invalid="ignore"):
        q_t, ok_t, _ = rt.truth(cam8, x, P, [], np.zeros((0, 2)), rej, zr, 1e300)
    assert math.isnan(float(q_t[0])) and not ok_t[0] and ok_t[1]
