"""Relocalisation on the device (sl2_relocalise; csrc/reloc.cu reloc_kernel) on scenes built directly, with no fused
step: the map from tests/relocalise_cases.py's exact constructions (set_features, set_state), the camera by
set_stream_config, and a flat frame (no window passes the sigma >= 10 gate) with distinct noise templates pasted a box
apart at the match pixels.  The full-image search must find exactly the pasted centres; then the result is held to the
truth of tests/relocalise_truth.py under its decision rule, and to the restatement of tests/relocalise_ref.py (equal
decisions, the pose within 1e-9).  Cases: k = 0, 1, 2, 3 and an empty map; k at the 32-match words of the inlier mask
up to 256 with unmatched features between the matches; min_inliers at the refined count and one above it; two
clusters of equal support, across warps and within one warp; collinear maps, duplicate templates, points behind the
camera; rotations through every quaternion branch, a wide camera, a theta -> 0 triple; a call listing streams 2 and 0
with their own cameras around an unlisted stream 1; probes 1e-3 .. 1e-7 px^2 either side of fl(tau^2)."""
import numpy as np
import pytest

import relocalise_cases as rc
import relocalise_ref as rr
import relocalise_truth as rt
import scenelib2_b200 as sl2
from gpu_util import CAMS_320

TAU = 2.0
MIN_INLIERS = 4
V = (0.0, 0.0, 0.0)
OMEGA = (0.0, 0.0, 1e-3)
PXX = np.diag([1e-4] * 3 + [1e-4] * 4 + [2.5e-3] * 6)
CACHE = {}


def make_ctx(cams, cap, B, slots=1):
    c0 = cams[0]
    cfg = sl2.default_config()
    cfg.num_streams, cfg.frame_slots = len(cams), slots
    cfg.width, cfg.height = int(max(c[0] for c in cams)), int(max(c[1] for c in cams))
    cfg.boxsize, cfg.max_features = B, cap
    cfg.number_of_features_to_select = min(cap, sl2.lib.SL2_MAX_MEASURED)
    cfg.search_tile_radius = 20
    cfg.fku, cfg.fkv, cfg.u0, cfg.v0, cfg.kd1, cfg.sd = [float(v) for v in c0[2:8]]
    ctx = sl2.Context(cfg)
    for s, c in enumerate(cams):
        ctx.set_stream_config(s, ctx.stream_config(s), width=int(c[0]), height=int(c[1]), fku=c[2], fkv=c[3], u0=c[4],
                              v0=c[5], kd1=c[6], sd=c[7])
    return ctx


def install(ctx, s, sc, B, rng, nfeat=None, unmatched=(), dup=None, slot=0):
    """Stream s: features = the scene's matches in order, with unmatched features (templates not pasted) inserted at
    the feature indices `unmatched`; dup = (i, j): feature j gets feature i's template.  Returns the matched features."""
    k = len(sc["z"])
    nfeat = k + len(unmatched) if nfeat is None else nfeat
    M = np.array([f for f in range(nfeat) if f not in set(unmatched)], np.int64)
    assert len(M) == k
    y = rng.uniform(-1, 1, (nfeat, 3)) + [0, 0, 2]
    y[M] = sc["y"]
    T = rng.integers(0, 256, (nfeat, B, B), dtype=np.uint8)
    if dup is not None:
        T[M[dup[1]]] = T[M[dup[0]]]
    x = np.concatenate([[0, 0, 0, 1, 0, 0, 0], V, OMEGA, y.ravel()])
    ctx.set_features(s, y, np.tile([0, 0, 0, 1, 0, 0, 0.0], (nfeat, 1)), T)
    ctx.set_state(s, x, np.eye(len(x)) * 1e-4)
    W, H = int(sc["cam8"][0]), int(sc["cam8"][1])
    frame = np.full((H, W), 128, np.uint8)
    half = (B - 1) // 2
    for j, f in enumerate(M):
        if dup is not None and j == dup[1]:
            continue
        u, v = (int(a) for a in sc["z"][j])
        frame[v - half:v + half + 1, u - half:u + half + 1] = T[f]
    ctx.set_frame(s, slot, frame)
    return M


def call(ctx, ids=(0,), slot=0, min_inliers=MIN_INLIERS):
    return ctx.relocalise(list(ids), slot, TAU, min_inliers, V, OMEGA, PXX)


def truth_of(sc, min_inliers=MIN_INLIERS):
    return rt.truth(sc["cam8"], sc["y"], sc["z"], TAU, min_inliers, cache=CACHE)


def check(ctx, s, res, zuv, fl, sc, M, T, min_inliers=MIN_INLIERS, before=None, decided=True):
    """search, truth, restatement and the state write (or, without acceptance, the unchanged snapshot `before`);
    decided: the truth must decide the winner (with probes near tau, a P3P pose's decisions may lie within their
    bounds, and then the support is compared with the restatement only)"""
    nf = ctx.num_features(s)
    fl, zuv = fl[:nf], zuv[:nf]
    assert (np.flatnonzero(fl & 1) == M).all() and res["matches"] == len(M)
    assert (zuv[M] == sc["z"]).all()  # the search finds the pasted centres
    assert not (fl & 2)[np.setdiff1d(np.arange(nf), M)].any()
    fails = rc.check_device(res, fl, M, T)
    assert not fails, fails
    assert T["decided"] or not decided, rc.report(T)
    ref = rr.relocalise(sc["cam8"], sc["y"], sc["z"], TAU, min_inliers)
    assert ref["margin"] > 1e-9, ref["margin"]
    assert res["support"] == ref["win_sup"] and res["inliers"] == ref["inliers"] and res["status"] == ref["status"]
    assert (((fl[M] & 2) > 0) == ref["mask"]).all()
    if ref["win"] < 0:
        assert np.isnan(res["pose"]).all() and np.isnan(res["rms_px"]) and res["support"] == 0 and res["inliers"] == 0
    else:
        scale = np.concatenate([np.maximum(1.0, np.abs(ref["pose"][:3])), np.ones(4)])
        assert (np.abs(res["pose"] - ref["pose"]) <= 1e-9 * scale).all(), (res["pose"], ref["pose"])
        if ref["inliers"]:
            assert abs(res["rms_px"] - ref["rms"]) <= 1e-9 * max(1.0, ref["rms"])
    if res["status"] == 1:
        x, P = ctx.get_state(s)
        assert x[:7].tobytes() == res["pose"].tobytes() and (x[7:10] == V).all() and (x[10:13] == OMEGA).all()
        assert (P[:13, :13] == PXX).all() and (P[:13, 13:] == 0).all() and (P[13:, :13] == 0).all()
    elif before is not None:
        assert ctx.save_stream(s) == before
    print(rc.report(T))


def run_one(cams, B, sc, cap, rng, min_inliers=MIN_INLIERS, **kw):
    ctx = make_ctx(cams, cap, B)
    try:
        M = install(ctx, 0, sc, B, rng, **kw)
        before = ctx.save_stream(0)
        T = truth_of(sc, min_inliers)
        res, zuv, fl = call(ctx, min_inliers=min_inliers)
        check(ctx, 0, res[0], zuv[0], fl[0], sc, M, T, min_inliers, before)
        return res[0], T
    finally:
        ctx.close()


# ---- small k -------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("k", [0, 1, 2, 3])
def test_small_k(k):
    rng = np.random.default_rng(100 + k)
    sc = rc.make_scene(rc.C1, 11, k, rng)
    res, T = run_one([rc.C1], 11, sc, 8, rng, unmatched=[0, k + 1] if k else [0, 1, 2])
    if k < 3:
        assert res["support"] == 0 and res["inliers"] == 0 and res["status"] == 0
        assert np.isnan(res["pose"]).all() and np.isnan(res["rms_px"])
    else:  # every hypothesis is the one triple: a refined truth P3P pose with support 3
        assert res["support"] == 3 and res["status"] == 0 and T["cands"]


@pytest.mark.gpu
def test_empty_map():
    rng = np.random.default_rng(7)
    ctx = make_ctx([rc.C1], 8, 11)
    try:
        ctx.set_features(0, np.zeros((0, 3)), np.zeros((0, 7)), np.zeros((0, 11, 11), np.uint8))
        ctx.set_state(0, np.concatenate([[0, 0, 0, 1, 0, 0, 0], V, OMEGA]), np.eye(13) * 1e-4)
        ctx.set_frame(0, 0, rng.integers(0, 256, (240, 320), dtype=np.uint8))
        before = ctx.save_stream(0)
        res, zuv, fl = call(ctx)
        r = res[0]
        assert r["matches"] == 0 and r["support"] == 0 and r["inliers"] == 0 and r["status"] == 0
        assert np.isnan(r["pose"]).all() and np.isnan(r["rms_px"])
        assert (zuv[0] == -1).all() and (fl[0] == 0).all() and ctx.save_stream(0) == before
    finally:
        ctx.close()


# ---- k at the inlier mask's 32-match words ---------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("k", [4, 31, 32, 33, 64, 65, 255, 256])
def test_mask_word_boundaries(k):
    rng = np.random.default_rng(200 + k)
    sc = rc.make_scene(rc.C3, 15, k, rng)
    bad = [j for j in (31, 32, 63, 255) if j < k]
    out = rc.make_scene(rc.C3, 15, k, rng, outliers=1.0, z=sc["z"])
    sc["y"][bad] = out["y"][bad]
    sc["good"][bad] = False
    extra = min(3, 256 - k)  # unmatched features between the matches, as many as fit
    unmatched = sorted(rng.choice(k + extra, extra, replace=False).tolist())
    res, T = run_one([rc.C3], 15, sc, 256, rng, unmatched=unmatched)
    assert res["status"] == 1 and res["inliers"] == k - len(bad) == T["max_lo"]


# ---- min_inliers at the refined count -----------------------------------------------------------------------------------
@pytest.mark.gpu
def test_min_inliers_at_the_refined_count():
    rng = np.random.default_rng(300)
    sc = rc.make_scene(rc.C1, 11, 20, rng, outliers=0.25)
    n = int(sc["good"].sum())
    ctx = make_ctx([rc.C1], 32, 11)
    try:
        M = install(ctx, 0, sc, 11, rng, unmatched=[3])
        before = ctx.save_stream(0)
        x0, P0 = ctx.get_state(0)
        T = truth_of(sc, n + 1)
        assert T["cands"][0]["inliers"] == n
        res, zuv, fl = call(ctx, min_inliers=n + 1)
        assert res[0]["status"] == 0 and res[0]["inliers"] == n
        check(ctx, 0, res[0], zuv[0], fl[0], sc, M, T, n + 1, before)
        T = truth_of(sc, n)
        res, zuv, fl = call(ctx, min_inliers=n)
        assert res[0]["status"] == 1
        check(ctx, 0, res[0], zuv[0], fl[0], sc, M, T, n)
        x, P = ctx.get_state(0)
        assert (x[13:] == x0[13:]).all() and P[13:, 13:].tobytes() == P0[13:, 13:].tobytes()
    finally:
        ctx.close()


# ---- ties ----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("which", ["across", "within"])
def test_two_cluster_tie_goes_to_the_lowest_hypothesis(which):
    """Clusters A and B of support 4: A's only hypothesis comes first (h = 7 in warp 7 against B's h = 258 in warp 2;
    h = 0 against h = 256, both in warp 0), so the pose is A's."""
    clusters = rc.TIE_ACROSS if which == "across" else rc.TIE_WITHIN
    rng = np.random.default_rng(400 + len(which))
    sc = rc.tie_scene(rc.C1, 11, rng, clusters)
    res, T = run_one([rc.C1], 11, sc, 64, rng)
    assert res["support"] == 4 and T["win"] == rc.hypotheses_inside(rc.TIE_K, clusters[0])[0]
    (ra, qa), (rb, qb) = sc["poses"]
    assert rt.pose_distance(res["pose"], np.concatenate([ra, qa])) < 1e-6
    assert rt.pose_distance(res["pose"], np.concatenate([rb, qb])) > 1e-2


# ---- degenerate maps and matches --------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_collinear_map_gives_no_pose():
    rng = np.random.default_rng(500)
    sc = rc.make_scene(rc.C1, 11, 8, rng)
    t = np.linspace(-1, 1, 8)
    sc["y"] = np.stack([0.3 * t, 0.1 + 0.2 * t, 2.0 + 0.5 * t], axis=1)
    res, T = run_one([rc.C1], 11, sc, 8, rng)
    assert T["win"] == -1 and res["support"] == 0 and np.isnan(res["pose"]).all()


@pytest.mark.gpu
def test_duplicate_templates_and_points_behind_the_camera():
    rng = np.random.default_rng(501)
    sc = rc.make_scene(rc.C1, 11, 12, rng, outliers=1 / 6)
    j0, j1 = np.flatnonzero(sc["good"])[:2]
    sc["z"][j1] = sc["z"][j0]  # one paste, two features: the same match pixel, parallel bearings
    sc["good"][j1] = False
    rc.behind(sc, [int(j) for j in np.flatnonzero(sc["good"])[2:4]])
    res, T = run_one([rc.C1], 11, sc, 16, rng, dup=(j0, j1))
    assert res["status"] == 1 and res["inliers"] == sc["good"].sum()


# ---- geometry branches -------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", ["shepperd-w", "shepperd-x", "shepperd-y", "shepperd-z", "wide", "wide-k3", "theta0-k3",
                                  "theta0-k4"])
def test_geometry_branches(case):
    rng = np.random.default_rng(sum(map(ord, case)))
    cam8 = rc.WIDE if case.startswith("wide") else rc.C1
    if case.startswith("shepperd"):
        pose = rc.axis_pose("xyz".index(case[-1]), 179.0, rng) if case[-1] != "w" else rc.axis_pose(0, 20.0, rng)
        sc = rc.make_scene(cam8, 11, 10, rng, outliers=0.2, pose=pose)
    elif case == "wide-k3":  # the first hypothesis's cos(beta) < 0
        sc = rc.make_scene(cam8, 11, 3, rng, z=rc.WIDE_TRIPLE)
    elif case == "wide":
        sc = rc.make_scene(cam8, 11, 12, rng, outliers=0.2, ring=True)
        b = rr.unproject(cam8, sc["z"])
        assert (b @ b.T).min() < -0.3  # bearings more than 90 degrees apart
    else:
        sc = rc.theta0_triple(rng)
        if case == "theta0-k4":
            z4 = next(p for p in rc.grid_pixels(rc.C1, 11, 20, rng) if not (p == sc["z"]).all(axis=1).any())
            sc.update(y=np.vstack([sc["y"], rc.exact_points(rc.C1, sc["r"], sc["q"], z4[None], [1.5])]),
                      z=np.vstack([sc["z"], z4]), good=np.ones(4, bool))
    res, T = run_one([cam8], 11, sc, 16, rng)
    if case in ("theta0-k3", "wide-k3"):
        assert res["support"] == 3 and res["status"] == 0
    else:
        assert res["status"] == 1 and res["inliers"] == sc["good"].sum()
        assert rt.pose_distance(res["pose"], np.concatenate([sc["r"], sc["q"]])) < 1e-6


# ---- one call, several streams -----------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_streams_listed_out_of_order_with_their_own_cameras():
    cams = [CAMS_320[0], CAMS_320[2], CAMS_320[1]]
    rng = np.random.default_rng(600)
    ctx = make_ctx(cams, 32, 11)
    try:
        scs = [rc.make_scene(c, 11, 14 + 2 * s, rng, outliers=0.2) for s, c in enumerate(cams)]
        Ms = [install(ctx, s, scs[s], 11, rng, unmatched=[2 * s + 1]) for s in range(3)]
        before = [ctx.save_stream(s) for s in range(3)]
        res, zuv, fl = call(ctx, ids=(2, 0))
        for i, s in enumerate((2, 0)):
            check(ctx, s, res[i], zuv[i], fl[i], scs[s], Ms[s], truth_of(scs[s]))
            assert res[i]["status"] == 1
        assert ctx.save_stream(1) == before[1]
        # each stream's result is the one it gets alone
        ctx.load_streams(before)
        for i, s in enumerate((2, 0)):
            alone, za, fa = call(ctx, ids=(s,))
            assert alone[0].tobytes() == res[i].tobytes() and (za[0] == zuv[i]).all() and (fa[0] == fl[i]).all()
    finally:
        ctx.close()


# ---- probes near tau ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_probes_near_tau():
    """Probe matches whose truth d2 at the refined pose lies 1e-3, 1e-5 and 1e-7 px^2 either side of fl(tau^2): the
    device's decisions equal the restatement's, and the truth's wherever the margin exceeds its bound; the rest are
    reported."""
    rng = np.random.default_rng(900)
    sc, T = rc.probe_scene(rc.C1, 11, rng, TAU, cache=CACHE)
    c, P = T["cands"][0], sc["probes"]
    ctx = make_ctx([rc.C1], 96, 11)
    try:
        M = install(ctx, 0, sc, 11, rng, unmatched=[5])
        res, zuv, fl = call(ctx)
        check(ctx, 0, res[0], zuv[0], fl[0], sc, M, T, decided=False)
        inl = (fl[0][M] & 2) > 0
        sure = c["margin"][P] > c["dbound"][P]
        for j, off, s, d in zip(P, rc.PROBE_OFFSETS, sure, inl[P]):
            print("probe %+.0e px^2: truth d2 - tau^2 %+.3e, bound %.1e, device inlier %d%s" % (
                off, c["d2"][j] - TAU * TAU, c["dbound"][j], d, "" if s else " (within the bound: reported)"))
        assert (np.abs(c["d2"][P] - TAU * TAU - np.array(rc.PROBE_OFFSETS)) <= 1e-3 * np.abs(rc.PROBE_OFFSETS)).all()
        assert sure[:2].all() and (inl[P][sure] == (np.array(rc.PROBE_OFFSETS) < 0)[sure]).all()
    finally:
        ctx.close()
