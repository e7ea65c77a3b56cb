"""Relocalisation scenes built from their definition, and the checks that hold a relocalisation (the restatement of
tests/relocalise_ref.py, or the device) to the truth of tests/relocalise_truth.py.

A scene is k matches (y_j, z_j) in feature-index order.  z_j are integer pixels on a grid a box apart (so the patch
search can find pasted templates there).  A match consistent with a pose has y_j = r + R(q) X_j, X_j = d (x_u, y_u, 1)
with (x_u, y_u) Camera::Unproject's undistorted point of z_j (the exact inverse of Camera::Project), formed in mpmath
and rounded once; it reprojects to z_j up to that rounding.  An outlier's y is built the same way for another pixel
at least 20 px from z_j."""
import math

import mpmath
import numpy as np

import relocalise_ref as rr
import relocalise_truth as rt
from model_cases import quat_to_R
from scenelib2_b200 import synth

# two clusters of 4 matches among k = 40 whose only all-cluster hypotheses are:
TIE_K = 40
TIE_ACROSS = ((0, 23, 29, 36), (1, 5, 8, 38))  # h = 7 (round 0, warp 7) and h = 258 (round 1, warp 2)
TIE_WITHIN = ((0, 2, 15, 33), (1, 5, 23, 25))  # h = 0 (round 0, warp 0) and h = 256 (round 1, warp 0)
# a 320 x 240 camera wide enough for bearings more than 90 degrees apart (the distortion doubles the corner radius)
WIDE = np.array([320.0, 240.0, 80.0, 80.0, 162.0, 125.0, 9e-6, 1.0])
# three pixels of it whose first hypothesis (matches 1, 2, 0) has its first two bearings more than 90 degrees apart
WIDE_TRIPLE = np.array([[300.0, 12.0], [8.0, 125.0], [300.0, 232.0]])
C1 = synth.camera_params(320, 240)
C3 = synth.camera_params(640, 480)


def hypotheses_inside(k, S):
    S = set(S)
    return [h for h in range(rr.HYPOTHESES) if set(rr.triple(h, k)) <= S]


def in_model(cam8, p):
    """the pixels p (n, 2) inside Camera::Unproject's domain (1 - 2 kd1 r^2 > 0), with a margin"""
    r2 = (p[:, 0] - cam8[4]) ** 2 + (p[:, 1] - cam8[5]) ** 2
    return 2 * cam8[6] * r2 < 0.9


def grid_pixels(cam8, B, n, rng, ring=False):
    """n distinct integer pixels a box apart, a box's half from the image edges, in random order (ring: the
    quarter of them farthest from the principal point)"""
    half = (B - 1) // 2
    us = np.arange(half, int(cam8[0]) - half, B)
    vs = np.arange(half, int(cam8[1]) - half, B)
    cells = np.stack(np.meshgrid(us, vs, indexing="ij"), -1).reshape(-1, 2).astype(np.float64)
    cells = cells[in_model(cam8, cells)]
    if ring:
        r2 = (cells[:, 0] - cam8[4]) ** 2 + (cells[:, 1] - cam8[5]) ** 2
        cells = cells[np.argsort(-r2)[:len(cells) // 4]]
    return cells[rng.permutation(len(cells))[:n]]


@mpmath.workdps(rt.DPS)
def exact_points(cam8, r, q, z, depth):
    """y (n, 3): the points at camera depths `depth` that project to the pixels z (n, 2) from the pose (r, q)."""
    fku, fkv, u0, v0, kd1 = (mpmath.mpf(float(v)) for v in cam8[2:7])
    w, x, yq, zq = (mpmath.mpf(float(v)) for v in q)
    n = mpmath.sqrt(w * w + x * x + yq * yq + zq * zq)
    w, x, yq, zq = w / n, x / n, yq / n, zq / n
    R = [[1 - 2 * (yq * yq + zq * zq), 2 * (x * yq - w * zq), 2 * (x * zq + w * yq)],
         [2 * (x * yq + w * zq), 1 - 2 * (x * x + zq * zq), 2 * (yq * zq - w * x)],
         [2 * (x * zq - w * yq), 2 * (yq * zq + w * x), 1 - 2 * (x * x + yq * yq)]]
    out = np.zeros((len(z), 3))
    for j, ((zu, zv), d) in enumerate(zip(np.asarray(z, np.float64), depth)):
        c0, c1 = mpmath.mpf(float(zu)) - u0, mpmath.mpf(float(zv)) - v0
        f = mpmath.sqrt(1 - 2 * kd1 * (c0 * c0 + c1 * c1))
        d = mpmath.mpf(float(d))
        X = [d * c0 / f / (-fku), d * c1 / f / (-fkv), d]
        for a in range(3):
            out[j, a] = float(mpmath.mpf(float(r[a])) + sum(R[a][c] * X[c] for c in range(3)))
    return out


def random_pose(rng):
    q = rng.standard_normal(4)
    q /= np.linalg.norm(q)
    return rng.uniform(-1.0, 1.0, 3), q if q[0] >= 0 else -q


def axis_pose(axis, deg, rng):
    """a rotation of deg degrees about the axis (0, 1, 2), tilted by a little under a degree"""
    a = np.zeros(3)
    a[axis] = 1.0
    a += rng.uniform(-0.01, 0.01, 3)
    a /= np.linalg.norm(a)
    h = math.radians(deg) / 2
    q = np.concatenate([[math.cos(h)], math.sin(h) * a])
    return rng.uniform(-1.0, 1.0, 3), q


def make_scene(cam8, B, k, rng, outliers=0.0, pose=None, depth=(0.5, 3.0), z=None, jitter=0.0, ring=False):
    """k matches seen from pose (default random), a fraction `outliers` of them outliers; good marks the others.
    jitter > 0: a good match's point projects up to jitter px from z in each coordinate (z is its rounding for 0.5)."""
    r, q = random_pose(rng) if pose is None else pose
    z = grid_pixels(cam8, B, k, rng, ring) if z is None else np.asarray(z, np.float64)
    good = np.ones(k, bool)
    good[rng.permutation(k)[:int(round(outliers * k))]] = False
    seen = z + rng.uniform(-jitter, jitter, z.shape)
    for j in np.flatnonzero(~good):
        while True:
            p = np.array([rng.uniform(10, cam8[0] - 10), rng.uniform(10, cam8[1] - 10)])
            if np.hypot(*(p - z[j])) >= 20.0 and in_model(cam8, p[None])[0]:
                break
        seen[j] = p
    y = exact_points(cam8, r, q, seen, rng.uniform(depth[0], depth[1], k))
    return dict(cam8=np.asarray(cam8, np.float64), y=y, z=z, r=r, q=q, good=good)


def tie_scene(cam8, B, rng, clusters):
    """TIE_K matches: cluster A consistent with one pose, cluster B with another, the rest outliers of both"""
    sc = make_scene(cam8, B, TIE_K, rng, outliers=1.0)
    for C in clusters:
        r, q = random_pose(rng)
        idx = list(C)
        sc["y"][idx] = exact_points(cam8, r, q, sc["z"][idx], rng.uniform(0.5, 3.0, len(idx)))
        sc.setdefault("poses", []).append((r, q))
    sc["good"][:] = False
    sc["good"][list(clusters[0])] = True
    return sc


def behind(sc, idx):
    """matches idx moved behind the camera of the scene's pose, to the mirror point: the same pixel, depth < 0"""
    R = quat_to_R(sc["q"])
    for j in idx:
        sc["y"][j] = sc["r"] - (sc["y"][j] - sc["r"])
        assert ((sc["y"][j] - sc["r"]) @ R)[2] < 0
    sc["good"][list(idx)] = False
    return sc


PROBE_OFFSETS = (1e-3, -1e-3, 1e-5, -1e-5, 1e-7, -1e-7)  # px^2 from fl(tau^2), at the truth's final pose


def probe_scene(cam8, B, rng, tau, k_good=60, cache=None):
    """k_good exact matches of one pose, then one probe match per PROBE_OFFSETS: an integer pixel whose map point the
    truth's refined pose projects sqrt(fl(tau^2) + offset) px away.  The probes move the refined pose (those inside
    tau join the refinement, and the winning hypothesis may hold one), so they are placed by fixed-point iteration:
    the truth names the winning hypothesis; then, for that triple, its P3P pose at the largest support, the matches
    inside tau there, the refinement on them, and the probes' map points put on the rays of their targets under the
    refined pose, until the pose stops moving; the truth is asked again until it names the same winner.  Returns the
    scene and its truth."""
    n = k_good + len(PROBE_OFFSETS)
    sc = make_scene(cam8, B, n, rng)
    t2 = float(tau) * float(tau)
    P = np.arange(k_good, n)
    ang = rng.uniform(0, 2 * np.pi, len(P))
    rho = np.sqrt(t2 + np.array(PROBE_OFFSETS))
    depth = rng.uniform(0.8, 2.5, len(P))
    Z = rt.Ext.conv(sc["z"].T)
    T = rt.truth(cam8, sc["y"], sc["z"], tau, 4, cache=cache, lsq=False)
    for _ in range(4):
        win = T["win"]
        pose = T["cands"][0]["pose"]
        for _ in range(60):
            target = sc["z"][P] + rho[:, None] * np.stack([np.cos(ang), np.sin(ang)], 1)
            sc["y"][P] = exact_points(cam8, pose[:3], pose[3:], target, depth)
            Y = rt.Ext.conv(sc["y"].T)
            t = sorted(rr.triple(win, n))
            poses, _ = rt.p3p(sc["y"][t], rt.bearings_mp(cam8, sc["z"][t]))
            best = None
            for p in poses:
                pa = rt._to(rt.Ext, p["pose"])
                inside = rt.decisions(rt.Ext, cam8, pa, Y, Z, t2, 0.0)[0]
                if p["physical"] and (best is None or inside.sum() > best[1].sum()):
                    best = (pa, inside)
            new = rt.refine(rt.Ext, cam8, best[0], Y[:, best[1]], Z[:, best[1]], t2)[0]
            new = np.array([float(v) for v in new])
            moved = rt.pose_distance(new, pose)
            pose = new
            if moved == 0.0:
                break
        T = rt.truth(cam8, sc["y"], sc["z"], tau, 4, cache=cache)
        if T["win"] == win:
            break
    sc["good"][P] = np.array(PROBE_OFFSETS) < 0
    sc["probes"] = P
    return sc, T


def theta0_triple(rng):
    """three exact matches on C1 at integer pixels whose best restatement pose is more than 1e-9 from the pose they
    were built from (Kneip's theta -> 0)"""
    for _ in range(100000):
        r, q = random_pose(rng)
        sc = make_scene(C1, 11, 3, rng, pose=(r, q), depth=(0.3, 3.0))
        sols = rr.p3p(sc["y"], rr.unproject(C1, sc["z"]))
        err = min([rt.pose_distance(s, np.concatenate([r, q])) for s in sols] + [np.inf])
        if 1e-9 < err < 1e-3:
            sc["kneip_error"] = err
            return sc
    raise AssertionError("no theta -> 0 triple")



# ---- checks -----------------------------------------------------------------------------------------------------------
NEAR = 1e-6  # a restatement pose this close to a truth pose is that pose, however imprecisely computed


def _within(margin, dbound):
    return margin <= dbound


def _recount_failures(T, pose, mask, inliers, rms, status, fails, who):
    """the refined pose, its inliers, rms and status against the truth's candidates (any of them when order-decided)"""
    if not T["cands"]:
        if not (np.isnan(pose).all() and inliers == 0 and math.isnan(rms) and status == 0):
            fails.append(("no pose", "%s: %s %d %s %d" % (who, pose, inliers, rms, status)))
        return None
    dist = [rt.pose_distance(pose, c["pose"]) for c in T["cands"]]
    c = T["cands"][int(np.argmin(dist))]
    if not min(dist) <= c["bound"]:
        fails.append(("final pose", "%s: %.3g > bound %.3g" % (who, min(dist), c["bound"])))
        return c
    sure = ~_within(c["margin"], c["dbound"])
    if (mask[sure] != c["mask"][sure]).any():
        fails.append(("recount", "%s: inlier mask differs at %s" % (who, np.flatnonzero(sure & (mask != c["mask"])))))
    lo, hi = int((c["mask"] & sure).sum()), int((c["mask"] | ~sure).sum())
    if not (lo <= inliers <= hi and status == int(inliers >= c["min_inliers"])):
        fails.append(("recount", "%s: inliers %d status %d, truth %d..%d, min_inliers %d" % (
            who, inliers, status, lo, hi, c["min_inliers"])))
    if sure.all():
        if inliers != c["inliers"] or status != c["status"]:
            fails.append(("recount", "%s: inliers %d status %d, truth %d %d" % (who, inliers, status, c["inliers"],
                                                                               c["status"])))
        elif inliers:
            band = float(c["dbound"][c["mask"]].sum()) / inliers
            tol = band / (2 * c["rms"]) if c["rms"] > 0 else math.sqrt(band)
            if not abs(rms - c["rms"]) <= tol + 1e-12 * c["rms"]:
                fails.append(("rms", "%s: %.17g truth %.17g (bound %.3g)" % (who, rms, c["rms"], tol)))
    return c


def check_restatement(mod, sc, T, tau, min_inliers, stats=None):
    """The restatement `mod` (relocalise_ref or a broken copy of it) on scene sc against its truth T.  Returns the
    failed checks as (name, detail).  A truth pose with a restatement pose within NEAR is found; its error over its
    bound goes into stats["pose"] (the worst), and a ratio above 1 into stats["imprecise"] as (h, sorted triple,
    ratio), with the decisions then compared outside the bounds scaled by that ratio.  stats also collects the smallest
    decision margin over its bound, the physical truth poses no restatement pose is near ("lost"; those of a triple
    the kernel's degeneracy tolerances drop are counted apart, "near_degenerate") and the restatement poses near no
    truth pose ("unexplained")."""
    stats = {} if stats is None else stats
    cam8, y, z = sc["cam8"], sc["y"], sc["z"]
    k = len(y)
    fails = []
    out = mod.relocalise(cam8, y, z, tau, min_inliers)
    t2 = float(tau) * float(tau)
    fb = mod.unproject(cam8, z) if k else np.zeros((0, 3))
    for h, row in enumerate(T["hyps"]):
        t = list(mod.triple(h, k))
        K = mod.p3p(y[t], fb[t])
        for p in row:
            d = [rt.pose_distance(kp, p["pose_f"]) for kp in K]
            if not d or min(d) > NEAR:
                if p["physical"]:
                    key = "near_degenerate" if p["near_degenerate"] else "lost"
                    stats[key] = stats.get(key, 0) + 1
                continue
            ratio = min(d) / p["bound"]
            stats["pose"] = max(stats.get("pose", 0.0), ratio)
            stats.setdefault("ratios", []).append((tuple(sorted(t)), ratio))
            if ratio > 1:
                stats.setdefault("imprecise", []).append((h, tuple(sorted(t)), ratio))
            dbound = p["dbound"] * max(1.0, ratio)
            d2 = mod.reprojection_d2(cam8, K[int(np.argmin(d))], y, z)
            mask = ~np.isnan(d2) & (np.nan_to_num(d2, nan=np.inf) <= t2)
            sure = ~_within(p["margin"], dbound)
            stats["margin"] = min(stats.get("margin", np.inf), float((p["margin"] / dbound).min()))
            if (mask[sure] != p["mask"][sure]).any():
                fails.append(("decisions", "h %d: %s" % (h, np.flatnonzero(sure & (mask != p["mask"])))))
        for s, kp in enumerate(K):
            if not any(rt.pose_distance(kp, p["pose_f"]) <= NEAR for p in row):
                # a pose no truth pose explains (Kneip's precision loss) may not take the win
                sup = out["support"].get(4 * h + s, 0)
                stats["unexplained"] = stats.get("unexplained", 0) + 1
                if T["decided"] and (sup > T["max_lo"] or (sup == T["max_lo"] and h < T["win"])):
                    fails.append(("extra poses", "h %d pose %d: support %d, the winner's %d at h %d" % (
                        h, s, sup, T["max_lo"], T["win"])))
    if T["decided"]:
        if out["win_sup"] != T["max_lo"] or (T["win"] >= 0) != (out["win"] >= 0) or \
                (T["win"] >= 0 and out["win"] // 4 not in T["win_hs"]):
            fails.append(("winner", "h %d support %d, truth h %d support %d" % (out["win"] // 4, out["win_sup"],
                                                                              T["win"], T["max_lo"])))
    _recount_failures(T, out["pose"], out["mask"], out["inliers"], out["rms"], out["status"], fails, "restatement")
    return fails


def check_device(res, flags, M, T):
    """sl2_relocalise's result res, flags (per feature) and matched features M against the truth T of its matches."""
    fails = []
    if T["decided"] and res["support"] != T["max_lo"]:
        fails.append(("winner", "support %d, truth %d" % (res["support"], T["max_lo"])))
    mask = (flags[M] & 2) > 0
    _recount_failures(T, res["pose"], mask, int(res["inliers"]), float(res["rms_px"]), int(res["status"]), fails,
                      "device")
    return fails


def report(T):
    """the truth's undecided decisions (within their bounds), as one line"""
    c = T["cands"][0] if T["cands"] else None
    near = [] if c is None else np.flatnonzero(_within(c["margin"], c["dbound"])).tolist()
    return "k %d: support %d..%d at h %d%s, %d undecided final decisions %s%s" % (
        T["k"], T["max_lo"], T["max_hi"], T["win"], " (order-decided)" if T["order_decided"] else "", len(near),
        near, "" if c is None else ", final bound %.2e, GN gap to the minimiser %.2e" % (c["bound"],
                                                                                       c.get("gn_gap", math.nan)))
