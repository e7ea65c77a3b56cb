"""The consensus rescue on the CPU: the NumPy restatement of the gate (rescue_ref) against the oracle's
(rescue_oracle.gate, built on oracle/models.hpp), constructed edges (the chi2 knife edge, k = 0, 1, 2 and all rejected,
a point behind the camera), broken copies of the restatement that the tests must catch, and the whole step of the
rescue oracle: off is the consensus oracle's step, and on a settled map with uncertain new features the rescue keeps
the features the consensus alone loses."""
import math

import numpy as np
import pytest

import consensus_oracle as co
import rescue_oracle as ro
import rescue_ref
from rescue_scene import rescue_scene, truth

CHI2 = 5.991


def make_case(seed, k, nf=20):
    """A settled state with nf features and the first k as rejected matches: z = the prediction + an offset of 0.5 to
    4 innovation sigmas in a random direction, rounded to whole pixels like a match."""
    rng = np.random.default_rng(seed)
    sc = rescue_scene("C2", n_frames=1, n_features=nf, new=range(nf - 4, nf), sigma=0.03, seed=seed)
    x, P = sc.x0.copy(), sc.P0.copy()
    x[13:] += rng.standard_normal(x.size - 13) * 0.002
    pos = (13 + 3 * np.arange(k)).astype(np.int32)
    z = np.zeros((k, 2))
    for j in range(k):
        p = rescue_ref.predict(sc.cam8, x, x[pos[j]:pos[j] + 3], P, int(pos[j]))
        a = rng.uniform(0, 2 * np.pi)
        v = rng.uniform(0.5, 4.0) * np.array([np.cos(a), np.sin(a)])
        z[j] = np.round(p["h"] + np.linalg.cholesky(p["S"]) @ v)
    return sc.cam8, x, P, pos, z


def both(cam8, x, P, pos, z, chi2):
    ok_r, q_r, preds = rescue_ref.gate(cam8, x, P, pos, z, chi2)
    ok_o, q_o, h_o, S_o = ro.gate(cam8, x, P, pos, z, chi2)
    return ok_r, q_r, preds, ok_o, q_o, h_o, S_o


@pytest.mark.parametrize("seed", range(6))
def test_restatement_equals_the_oracle_bit_for_bit(seed):
    cam8, x, P, pos, z = make_case(seed, 12)
    ok_r, q_r, preds, ok_o, q_o, h_o, S_o = both(cam8, x, P, pos, z, CHI2)
    assert (ok_r == ok_o).all()
    assert q_r.tobytes() == q_o.tobytes()
    assert np.array([p["h"] for p in preds]).tobytes() == h_o.tobytes()
    assert np.array([p["S"] for p in preds]).tobytes() == S_o.tobytes()
    assert 0 < ok_r.sum() < len(ok_r)  # the cases exercise both outcomes


@pytest.mark.parametrize("k", [0, 1, 2, 20])
def test_small_and_full_k(k):
    cam8, x, P, pos, z = make_case(100 + k, k, nf=20)
    ok_r, q_r, _, ok_o, q_o, _, _ = both(cam8, x, P, pos, z, CHI2)
    assert ok_r.shape == (k,) and (ok_r == ok_o).all() and q_r.tobytes() == q_o.tobytes()


def test_chi2_knife_edge():
    cam8, x, P, pos, z = make_case(7, 8)
    _, q, _ = rescue_ref.gate(cam8, x, P, pos, z, CHI2)
    for j in range(len(pos)):
        at = q[j]
        below = np.nextafter(at, -np.inf)  # q one double above chi2
        for chi2, want in ((at, True), (below, False)):
            ok_r, _, _, ok_o, _, _, _ = both(cam8, x, P, pos[j:j + 1], z[j:j + 1], chi2)
            assert ok_r[0] == want and ok_o[0] == want, (j, chi2)


def test_point_behind_the_camera_is_never_rescued():
    cam8, x, P, pos, z = make_case(8, 3)
    # move feature 1 behind the camera (the camera looks along -z from x[0:3] with q = identity) while its match
    # stays where its mirrored point projects: q can be small, the depth is not > 0
    p = pos[1]
    x[p:p + 3] = x[0:3] - (x[p:p + 3] - x[0:3])
    h = rescue_ref.predict(cam8, x, x[p:p + 3], P, int(p))
    assert h["depth"] < 0.0
    z[1] = np.round(h["h"])
    ok_r, q_r, _, ok_o, _, _, _ = both(cam8, x, P, pos, z, 1e6)
    assert q_r[1] <= 1e6 and not ok_r[1] and not ok_o[1]
    assert ok_r[0] and ok_r[2]


def test_nan_is_never_rescued():
    S = np.array([[-1.0, 0.0], [0.0, 1.0]])
    assert math.isnan(rescue_ref.q_of([1.0, 1.0], [0.0, 0.0], S))


# ---- broken copies of the restatement --------------------------------------------------------------------------
def _mutant_prior_S(cam8, x, P, pos, z, chi2, x0, P0):
    preds = [rescue_ref.predict(cam8, x, x[p:p + 3], P, int(p)) for p in pos]
    prior = [rescue_ref.predict(cam8, x0, x0[p:p + 3], P0, int(p)) for p in pos]
    return np.array([rescue_ref.q_of(z[j], preds[j]["h"], prior[j]["S"]) <= chi2 for j in range(len(pos))])


def _mutant_prior_h(cam8, x, P, pos, z, chi2, x0, P0):
    preds = [rescue_ref.predict(cam8, x, x[p:p + 3], P, int(p)) for p in pos]
    prior = [rescue_ref.predict(cam8, x0, x0[p:p + 3], P0, int(p)) for p in pos]
    return np.array([rescue_ref.q_of(z[j], prior[j]["h"], preds[j]["S"]) <= chi2 for j in range(len(pos))])


def _mutant_strict(cam8, x, P, pos, z, chi2, x0, P0):
    _, q, _ = rescue_ref.gate(cam8, x, P, pos, z, chi2)
    return q < chi2


def test_mutations_are_caught():
    """Each broken copy disagrees with the oracle on some case: the prior S instead of S', h at the prior x instead of
    x', and < for <=."""
    caught = {m.__name__: False for m in (_mutant_prior_S, _mutant_prior_h, _mutant_strict)}
    for seed in range(4):
        cam8, x0, P0, pos, z = make_case(200 + seed, 12)
        # x', P': a Kalman update of the camera position from a direct observation (what an update 1 does to x, P)
        n = x0.size
        H = np.zeros((3, n))
        H[:, 0:3] = np.eye(3)
        S = H @ P0 @ H.T + np.eye(3) * 1e-6
        K = P0 @ H.T @ np.linalg.inv(S)
        x = x0 + K @ np.array([0.004, -0.003, 0.002])
        P = P0 - K @ S @ K.T
        P = 0.5 * (P + P.T)
        ok, q, _, _ = ro.gate(cam8, x, P, pos, z, CHI2)
        for m in (_mutant_prior_S, _mutant_prior_h):
            if (m(cam8, x, P, pos, z, CHI2, x0, P0) != ok).any():
                caught[m.__name__] = True
        j = int(np.argmin(np.abs(q - CHI2)))
        ok_e, _, _, _ = ro.gate(cam8, x, P, pos[j:j + 1], z[j:j + 1], q[j])
        if _mutant_strict(cam8, x, P, pos[j:j + 1], z[j:j + 1], q[j], x0, P0)[0] != ok_e[0]:
            caught["_mutant_strict"] = True
    assert all(caught.values()), caught


# ---- the whole step ---------------------------------------------------------------------------------------------
def test_chi2_zero_is_the_consensus_oracle_step():
    sc = rescue_scene("C2", n_frames=8, n_features=30, new=range(24, 30), sigma=0.03, wrong=[3])
    a = ro.slam_from_scene(sc, 2.5, 0.0)
    b = co.slam_from_scene(sc, 2.5)
    for t in range(8):
        a.step(sc.frames[t])
        b.step(sc.frames[t])
        fa, fb = a.features(), b.features()
        for k in fa:
            assert fa[k].tobytes() == fb[k].tobytes(), (t, k)
        xa, Pa = a.get_state()
        xb, Pb = b.get_state()
        assert xa.tobytes() == xb.tobytes() and Pa.tobytes() == Pb.tobytes(), t


def capability(name, nf, new, wrong, sigma, chi2, T=15):
    """The rescue oracle over T steps: per step (new features' matches rejected, rescued, distractors rescued), and at
    the end the new features kept and their position sigmas."""
    sc = rescue_scene(name, n_frames=T + 1, n_features=nf, new=new, sigma=sigma, wrong=wrong)
    o = ro.slam_from_scene(sc, 2.5, chi2)
    new, wrong = set(new), set(wrong)
    rows = []
    for t in range(T):
        o.step(sc.frames[t])
        f = o.features()
        lab, tr = f["label"], truth(sc, t)
        correct = [(f["z"][i] == tr[l]).all() for i, l in enumerate(lab)]
        rej = sum(1 for i, l in enumerate(lab) if l in new and f["flags"][i] & 4 and correct[i])
        res = o.rescued()
        rows.append((rej, len(res & new), len(res & wrong)))
    x, P = o.get_state()
    f = o.features()
    sig = [math.sqrt(np.trace(P[13 + 3 * i:16 + 3 * i, 13 + 3 * i:16 + 3 * i]) / 3)
           for i, l in enumerate(f["label"]) if l in new]
    return rows, sig


def test_capability_on_the_oracle():
    """C4 map, 8 new features with sigma 3 cm (cross terms to the camera), distractors on two settled features."""
    new, wrong = range(92, 100), [5, 50]
    off, sig_off = capability("C4", 100, new, wrong, 0.03, 0.0)
    on, sig_on = capability("C4", 100, new, wrong, 0.03, CHI2)
    assert off[0][0] >= 5 and on[0][0] == 0          # consensus only: most correct new matches rejected at first
    assert on[0][1] >= 6                              # the rescue takes them back on the first step
    assert len(sig_off) <= 6 and len(sig_on) == 8     # consensus only: the cull deletes some; rescue: all kept
    assert max(sig_on) < 0.02                         # and their positions settle
    assert all(r[2] == 0 for r in on)                 # a distractor is never rescued
