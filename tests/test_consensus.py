"""The match consensus of the test oracle (tests/consensus_oracle.cpp, on top of oracle/; include/sl2b200.h
sl2_set_stream_consensus) against an independent restatement in Python floats: masks, supports and winners bit for
bit over random cases and constructed ones (k = 0, 1, 2; all matches agreeing; two equal-support clusters; a point
behind the camera; tau on the knife edge of a chosen pair).  Its whole step with tau = 0 is byte-identical to the
oracle's own step."""
import math

import numpy as np
import pytest

import consensus_oracle as co
from camera_ref import project_point, quat_to_R
from consensus_ref import restated
from oracle import pyoracle as po
from scenelib2_b200 import synth

CAM8 = synth.camera_params(320, 240)


# ---- cases ---------------------------------------------------------------------------------------------------------
def _quat(rng, spread):
    q = np.array([1.0, *rng.normal(0.0, spread, 3)])
    return q / np.linalg.norm(q)


def make_case(rng, k, nf=None, outliers=(), offset=(9.0, -6.0), P=None, camera_pts=None, xv=None, cam8=CAM8):
    """k matched features of a map of nf, in a random rank order: the oracle's predictions (h, dh/dxv, dh/dy, S) of
    the predicted state for the camera cam8, z = round(h) (+-1 px) and, for the matches in `outliers`, z shifted by
    `offset`."""
    nf = nf or k + 3
    n = 13 + 3 * nf
    if xv is None:
        xv = np.concatenate([rng.normal(0.0, 0.05, 3), _quat(rng, 0.05), rng.normal(0.0, 0.02, 6)])
    if camera_pts is None:
        d = rng.uniform(0.5, 1.5, nf)
        camera_pts = np.stack([rng.uniform(-0.35, 0.35, nf) * d, rng.uniform(-0.25, 0.25, nf) * d, d], axis=1)
    R = np.array(quat_to_R(*xv[3:7]))
    x = np.concatenate([xv, (xv[:3] + camera_pts @ R.T).ravel()])
    if P is None:
        P = synth.make_prior_covariance(rng, n, sig_y=0.01)
    feats = rng.permutation(nf)[:k]
    pos = 13 + 3 * feats
    h, S, dxp, dy = np.zeros((k, 2)), np.zeros((k, 2, 2)), np.zeros((k, 2, 7)), np.zeros((k, 2, 3))
    for j, p in enumerate(pos):
        hj, dxv, dyj, _, Sj = po.predict_feature(cam8, xv, x[p:p + 3], P[:13, :13], P[:13, p:p + 3],
                                                 P[p:p + 3, p:p + 3])
        h[j], S[j], dxp[j], dy[j] = hj, Sj, dxv[:, :7], dyj
    z = np.round(h) + rng.integers(-1, 2, (k, 2))
    for j in outliers:
        z[j] += offset
    return dict(cam8=cam8, x=x, P=P, pos=pos.astype(np.int32), z=z, h=h, S=S, dh_dxp=dxp, dh_dy=dy)


def both(case, tau):
    """The oracle's and the restatement's answers, asserted identical; returns (keep, support, winner, d2)."""
    keep, sup, win = co.consensus(case["cam8"], case["x"], case["P"], case["pos"], case["z"], case["h"], case["S"],
                                  case["dh_dxp"], case["dh_dy"], tau)
    rk, rs, rw, d2 = restated(case["cam8"], case["x"], case["P"], case["pos"], case["z"], case["h"], case["S"],
                              case["dh_dxp"], case["dh_dy"], tau)
    assert (keep == rk).all() and (sup == rs).all() and win == rw, (keep, rk, sup, rs, win, rw)
    return keep, sup, win, d2


def test_random_cases_agree_bit_for_bit():
    rng = np.random.default_rng(11)
    rejected = nothing = 0
    for t in range(60):
        k = int(rng.integers(0, 25))
        out = rng.permutation(k)[:int(rng.integers(0, max(1, k // 3) + 1))]
        case = make_case(rng, k, outliers=out, offset=rng.uniform(-15, 15, 2).round())
        keep, _, win, _ = both(case, float(rng.choice([1.5, 2.0, 3.0, 5.0])))
        rejected += int((~keep).sum())
        nothing += int(win < 0)
    assert rejected > 0 and nothing > 0


def test_small_k():
    rng = np.random.default_rng(12)
    keep, sup, win, _ = both(make_case(rng, 0), 3.0)
    assert keep.size == 0 and win == -1
    keep, sup, win, _ = both(make_case(rng, 1), 3.0)
    assert keep.tolist() == [True] and win == -1 and sup[0] <= 1
    keep, sup, win, _ = both(make_case(rng, 2), 3.0)  # two agreeing matches
    assert keep.all() and win == 0 and sup.tolist() == [2, 2]
    keep, sup, win, _ = both(make_case(rng, 2, outliers=[1], offset=(14.0, 9.0)), 2.0)  # no two agree
    assert keep.all() and win == -1 and sup.max() < 2


def test_all_matches_agreeing():
    rng = np.random.default_rng(13)
    for k in (3, 8, 20):
        keep, sup, win, _ = both(make_case(rng, k), 3.0)
        assert keep.all() and win == int(np.argmax(sup)) and sup[win] == k


def _cluster_case(rng, k):
    """Features on one fronto-parallel plane, only the camera position uncertain: a match moves the camera and with it
    every prediction by about the same pixels.  Matches of even rank are shifted by +7 px, odd ranks by -7 px."""
    nf = k
    d = 1.0
    pts = np.stack([rng.uniform(-0.3, 0.3, nf) * d, rng.uniform(-0.2, 0.2, nf) * d, np.full(nf, d)], axis=1)
    xv = np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0])
    P = np.zeros((13 + 3 * nf, 13 + 3 * nf))
    P[0, 0] = P[1, 1] = 0.05 ** 2
    case = make_case(rng, k, nf=nf, P=P, camera_pts=pts, xv=xv)
    case["z"] = np.round(case["h"]) + np.where(np.arange(k) % 2 == 0, 7.0, -7.0)[:, None] * [1.0, 0.0]
    return case


def test_two_equal_clusters_lowest_rank_wins():
    rng = np.random.default_rng(14)
    for k in (4, 6, 10):
        keep, sup, win, _ = both(_cluster_case(rng, k), 2.5)
        even = np.arange(k) % 2 == 0
        assert (sup == k // 2).all(), sup   # every hypothesis explains exactly its own cluster
        assert win == 0 and (keep == even).all()


def behind_camera_case(rng, k=6):
    """Feature of rank 2 moved behind the camera (its prediction stays finite: the projection mirrors), its z set to
    exactly that mirrored projection."""
    case = make_case(rng, k, nf=k)
    p = case["pos"][2]
    xv = case["x"][:13]
    R = np.array(quat_to_R(*xv[3:7]))
    c = R.T @ (case["x"][p:p + 3] - xv[:3])
    case["x"][p:p + 3] = xv[:3] + R @ (c * [1.0, 1.0, -1.0])
    case["P"][p:p + 3, :] = 0.0
    case["P"][:, p:p + 3] = 0.0
    case["P"][p:p + 3, p:p + 3] = np.eye(3) * 1e-4
    zc = R.T @ (case["x"][p:p + 3] - xv[:3])
    case["z"][2] = np.round(project_point(CAM8, zc)[0])
    return case


def test_point_behind_the_camera_is_never_an_inlier():
    k = 6
    case = behind_camera_case(np.random.default_rng(15), k)
    keep, sup, win, d2 = both(case, 1000.0)  # a radius that takes every point in front of the camera
    assert np.isnan(d2[:, 2]).all()
    assert win >= 0 and not keep[2] and keep[np.arange(k) != 2].all()


def test_tau_on_the_knife_edge():
    rng = np.random.default_rng(16)
    case = make_case(rng, 8, outliers=[5], offset=(4.0, 3.0))
    keep, _, win, d2 = both(case, 3.0)
    assert win >= 0
    # the winner's inlier farthest from its prediction: the one decision a slightly smaller tau flips
    j = int(np.nanargmax(np.where(keep & (np.arange(8) != win), d2[win], np.nan)))
    s = math.sqrt(d2[win, j])
    taus = [s]
    for _ in range(2):
        taus = [np.nextafter(taus[0], 0.0)] + taus + [np.nextafter(taus[-1], np.inf)]
    sups = {}
    for tau in taus:  # the doubles around sqrt(d2): j leaves the inlier set of `win` where fl(tau * tau) drops below d2
        _, sup, _, _ = both(case, float(tau))
        sups[float(tau) * float(tau) >= d2[win, j]] = int(sup[win])
    assert sups.keys() == {False, True} and sups[True] == sups[False] + 1


def _oracle(sc):
    cfg = po.make_config(width=sc.width, height=sc.height, fku=sc.cam8[2], fkv=sc.cam8[3], u0=sc.cam8[4],
                         v0=sc.cam8[5], kd1=sc.cam8[6], sd=sc.cam8[7], delta_t=sc.delta_t, n_select=sc.n_select,
                         boxsize=sc.boxsize, search_override=sc.search_override)
    s = po.Slam(cfg)
    for i in range(sc.n_features):
        s.add_feature(sc.x0[13 + 3 * i:16 + 3 * i], sc.xp_org[i], sc.patches[i])
    s.set_state(sc.x0, sc.P0)
    return s


@pytest.mark.parametrize("name", ["C1", "C2"])
def test_slam_tau_zero_is_the_oracle_step(name):
    sc = synth.make_scene(name, n_frames=4, n_features=24)
    a, b = _oracle(sc), co.slam_from_scene(sc, 0.0)
    for t in range(4):
        a.step(sc.frames[t])
        b.step(sc.frames[t])
        fa, fb = a.features(), b.features()
        for key in fa:
            assert fa[key].tobytes() == fb[key].tobytes(), (t, key)
        for u, v in zip(a.get_state(), b.get_state()):
            assert u.tobytes() == v.tobytes()
