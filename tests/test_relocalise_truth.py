"""The relocalisation restatement (tests/relocalise_ref.py) against the relocalisation from its definition
(tests/relocalise_truth.py): random scenes on C1 and C3 with their kd1 and on a wide camera whose bearings reach past
90 degrees, 0-60 % outliers, and constructed ones (two clusters of equal support, rotations through each of the four
branches of a rotation-to-quaternion conversion, matches behind the camera, a triple near theta = 0 of Kneip's
parametrisation).  Broken copies of the restatement must each fail a named check."""
import math

import numpy as np
import pytest

import relocalise_cases as rc
import relocalise_ref as rr
import relocalise_truth as rt

TAU = 2.0
MIN_INLIERS = 4
CACHE = {}   # truth P3P per sorted triple
SCENES = {}  # name -> (scene, truth)


def build(name):
    rng = np.random.default_rng(sum(map(ord, name)))
    if name.startswith("random") or name.startswith("rounded"):
        kind, cam, k, out = name.split("-")
        cam8, B = {"C1": (rc.C1, 11), "C3": (rc.C3, 15), "wide": (rc.WIDE, 11)}[cam]
        return rc.make_scene(cam8, B, int(k), rng, outliers=int(out) / 100, jitter=0.5 if kind == "rounded" else 0.0,
                             ring=cam == "wide")
    if name == "wide-k3":
        return rc.make_scene(rc.WIDE, 11, 3, rng, z=rc.WIDE_TRIPLE)
    if name == "tie-across":
        return rc.tie_scene(rc.C1, 11, rng, rc.TIE_ACROSS)
    if name == "tie-within":
        return rc.tie_scene(rc.C1, 11, rng, rc.TIE_WITHIN)
    if name.startswith("shepperd"):
        axis = "xyz".index(name[-1])
        return rc.make_scene(rc.C1, 11, 8, rng, outliers=0.25, pose=rc.axis_pose(axis, 179.0, rng))
    if name == "behind":
        return rc.behind(rc.make_scene(rc.C1, 11, 10, rng, outliers=0.2), [1, 4, 7])
    if name == "theta0-k3":
        return rc.theta0_triple(rng)
    if name == "theta0-k4":
        sc = dict(SCENES_GET("theta0-k3")[0])
        z4 = rc.grid_pixels(rc.C1, 11, 20, rng)
        z4 = next(p for p in z4 if not (p == sc["z"]).all(axis=1).any())
        y4 = rc.exact_points(rc.C1, sc["r"], sc["q"], z4[None], [1.5])
        sc.update(y=np.vstack([sc["y"], y4]), z=np.vstack([sc["z"], z4]), good=np.ones(4, bool))
        return sc
    raise KeyError(name)


def SCENES_GET(name):
    if name not in SCENES:
        sc = build(name)
        SCENES[name] = (sc, rt.truth(sc["cam8"], sc["y"], sc["z"], TAU, MIN_INLIERS, cache=CACHE))
    return SCENES[name]


NAMES = ["random-C1-12-0", "random-C1-14-30", "rounded-C1-12-25", "random-C3-14-60", "random-wide-12-20", "wide-k3", "tie-across", "tie-within",
         "shepperd-x", "shepperd-y", "shepperd-z", "behind", "theta0-k3", "theta0-k4"]
STATS = {}


# ---- the truth's own arithmetic -----------------------------------------------------------------------------------------
def test_ext_agrees_with_mp():
    """The truth in np.longdouble and in mpmath at 50 digits: the same decisions, d2 and refined pose to 1e-15."""
    sc, _ = SCENES_GET("random-C1-14-30")
    n = 6
    T = {}
    for ar in (rt.Ext, rt.MpV()):
        T[ar is rt.Ext] = rt.truth(sc["cam8"], sc["y"][:n], sc["z"][:n], TAU, MIN_INLIERS, ar=ar, cache=CACHE,
                                   hypotheses=4, lsq=False)
    e, m = T[True], T[False]
    worst = 0.0
    for re_, rm in zip(e["hyps"], m["hyps"]):
        for pe, pm in zip(re_, rm):
            assert (pe["mask"] == pm["mask"]).all()
            fin = np.isfinite(pe["margin"])
            assert (fin == np.isfinite(pm["margin"])).all()
            worst = max(worst, float(np.abs(pe["margin"][fin] - pm["margin"][fin]).max(initial=0.0)))
    ce, cm = e["cands"][0], m["cands"][0]
    dp = rt.pose_distance(ce["pose"], cm["pose"])
    print("Ext against Mp: |d2| %.2e px^2, final pose %.2e" % (worst, dp))
    assert worst <= 1e-14 and dp <= 1e-15 and (ce["mask"] == cm["mask"]).all()
    assert len(e["hyps"][0]) >= 1


def test_truth_solutions_are_exact_and_the_constructions_hold():
    """Every truth P3P pose satisfies the law of cosines to 1e-25 of its scale and is physical iff its depths are
    positive; every construction's good match lies
    on the construction's pose; the wide camera has bearings more than 90 degrees apart; the tie clusters are the
    only all-cluster hypotheses, at the hypotheses they are chosen for; the theta -> 0 triple loses precision in
    Kneip's P3P."""
    for name in NAMES:
        sc, T = SCENES_GET(name)
        for row in T["hyps"]:
            for p in row:
                assert p["residual"] <= 1e-25 and p["physical"] == (min(p["s"]) > 0)
    sc, _ = SCENES_GET("random-wide-12-20")
    b = rr.unproject(sc["cam8"], sc["z"])
    assert (b @ b.T).min() < -0.3
    b = rr.unproject(rc.WIDE, rc.WIDE_TRIPLE)
    i, j, _ = rr.triple(0, 3)
    assert b[i] @ b[j] < -0.3  # the first hypothesis's f1, f2 are more than 90 degrees apart
    assert rc.hypotheses_inside(rc.TIE_K, rc.TIE_ACROSS[0]) == [7]
    assert rc.hypotheses_inside(rc.TIE_K, rc.TIE_ACROSS[1]) == [258]
    assert rc.hypotheses_inside(rc.TIE_K, rc.TIE_WITHIN[0]) == [0]
    assert rc.hypotheses_inside(rc.TIE_K, rc.TIE_WITHIN[1]) == [256]
    print("theta -> 0 triple: Kneip's error %.2e" % SCENES_GET("theta0-k3")[0]["kneip_error"])


@pytest.mark.parametrize("name", NAMES)
def test_restatement_equals_the_truth(name):
    sc, T = SCENES_GET(name)
    stats = {}
    fails = rc.check_restatement(rr, sc, T, TAU, MIN_INLIERS, stats)
    STATS[name] = stats
    print("%s: %s; pose error / bound %.2e, smallest margin / bound %.2e, beyond the bound %d, lost %d, near-degenerate "
          "%d, unexplained %d, double roots %d" % (
              name, rc.report(T), stats.get("pose", 0.0), stats.get("margin", np.inf), len(stats.get("imprecise", [])),
              stats.get("lost", 0), stats.get("near_degenerate", 0), stats.get("unexplained", 0),
              len(T["double_roots"])))
    assert not fails, fails
    assert not beyond_the_bound(name, stats), beyond_the_bound(name, stats)
    assert T["decided"]
    c = T["cands"][0]
    if name.startswith("tie"):  # cluster A's pose, support 4 for each cluster
        assert T["win"] == rc.hypotheses_inside(rc.TIE_K, sc["good"].nonzero()[0])[0] and T["max_lo"] == 4
        hB = rc.hypotheses_inside(rc.TIE_K, rc.TIE_ACROSS[1] if name == "tie-across" else rc.TIE_WITHIN[1])[0]
        assert max(p["lo"] for p in T["hyps"][hB]) == 4
    if name.startswith("theta0-k3"):
        assert T["max_lo"] == 3 and c["status"] == 0
    if "theta0" not in name and not name.startswith("tie") and not name.startswith("rounded"):
        assert (c["mask"] == sc["good"]).all()
        assert rt.pose_distance(c["pose"], np.concatenate([sc["r"], sc["q"]])) < 5e-3


def beyond_the_bound(name, stats):
    """the restatement's P3P poses farther from their truth pose than its bound"""
    return stats.get("imprecise", [])


def test_lost_poses_only_change_nothing():
    """Over every scene: every truth pose has a restatement pose within 1e-6, and within its bound except on the
    theta -> 0 triple; Kneip's poses that no truth pose explains are counted (the checks above fail if one of them
    could win)."""
    for name in NAMES:
        if name not in STATS:
            sc, T = SCENES_GET(name)
            STATS[name] = {}
            assert not rc.check_restatement(rr, sc, T, TAU, MIN_INLIERS, STATS[name])
    lost = sum(s.get("lost", 0) for s in STATS.values())
    unexplained = sum(s.get("unexplained", 0) for s in STATS.values())
    poses = sum(len(row) for name in NAMES for row in SCENES_GET(name)[1]["hyps"])
    margin = min(s.get("margin", np.inf) for s in STATS.values())
    worst = max(s.get("pose", 0.0) for s in STATS.values())
    print("truth poses %d, physical ones with no restatement pose within 1e-6 %d; Kneip poses no truth pose explains "
          "%d; worst pose error / bound %.2e; smallest margin / bound %.2e" % (poses, lost, unexplained, worst, margin))
    assert worst <= 1.0 and lost == 0


# ---- broken copies of the restatement ---------------------------------------------------------------------------------
NO_DEPTH = """from camera_ref import camera_points, project_point, rrw


def reprojection_d2(cam8, xp, y, z):
    d = np.asarray(z, np.float64).reshape(-1, 2) - project_point(cam8, camera_points(xp, y))
    return d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]
"""
MUTATIONS = {
    "ties reduced by warp": ("                if support[idx] > win_sup:",
                             "                if support[idx] > win_sup or (support[idx] == win_sup and h % 8 < "
                             "(win // 4) % 8):"),
    "the last max wins": ("if support[idx] > win_sup:", "if support[idx] >= win_sup:"),
    "no depth > 0 test": ("from camera_ref import camera_points, reprojection_d2, rrw\n", NO_DEPTH),
    "bearings without the distortion factor": ("factor = np.sqrt(1.0 - 2.0 * kd1 * radius2)",
                                               "factor = np.ones_like(radius2)"),
    "a world-frame rotation increment": ("q = quat_mul(xp[3:7], [math.cos(0.5 * ang), sc * d[3], sc * d[4], sc * d[5]])",
                                         "q = quat_mul([math.cos(0.5 * ang), sc * d[3], sc * d[4], sc * d[5]], xp[3:7])"),
    "GN over all matches": ("pose = refine(cam8, win_pose, y[wm], z[wm])", "pose = refine(cam8, win_pose, y, z)"),
    "the recount at the P3P pose": ("mask, d2 = decide(pose)", "mask, d2 = decide(win_pose)"),
    "a triple off by one in its splitmix input": ("i0 = splitmix64(3 * h) % k", "i0 = splitmix64(3 * h + 1) % k"),
    "the cos beta sign dropped": ("b = -math.sqrt(b) if cos_beta < 0.0 else math.sqrt(b)", "b = math.sqrt(b)"),
    "the f3t swap skipped": ("if f3t[2] > 0.0:", "if False:"),
}


def mutant(old, new):
    src = open(rr.__file__).read()
    assert src.count(old) == 1, old
    mod = type(rr)("relocalise_mutant")
    mod.__file__ = rr.__file__
    exec(compile(src.replace(old, new), rr.__file__, "exec"), mod.__dict__)
    return mod


def test_mutations_are_caught():
    caught = {}
    for what, (old, new) in MUTATIONS.items():
        mod = mutant(old, new)
        for name in NAMES:
            sc, T = SCENES_GET(name)
            fails = rc.check_restatement(mod, sc, T, TAU, MIN_INLIERS)
            if fails:
                caught[what] = (name, sorted({f[0] for f in fails}))
                break
        print("%-45s %s" % (what, "caught on %s by %s" % caught[what] if what in caught else "NOT CAUGHT"))
    assert sorted(caught) == sorted(MUTATIONS)
