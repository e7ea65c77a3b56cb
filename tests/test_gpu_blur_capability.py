"""What the exposure blur buys on a rendered fast yaw (tests/blur_scene.py): first on the CPU, the oracle's search on
the blurred frames with the warped stored templates against blur_ref's templates at the true state; then on the device,
one context whose streams track the same frames with the gyro on and the blur off, on, and mis-set (half and twice the
exposure, the offset's sign flipped).  The thresholds come from a measured device run (DESIGN.md, the blur's row)."""
import numpy as np
import pytest

import blur_ref
import blur_scene as bs
import warp_ref
from camera_ref import camera_points, project_point
from warp_scene import angle_deg

SIGMA = 3.0  # px: the search ellipse of the rehearsal, puinv = I / SIGMA^2
SCENE = {}


def scene():
    if "s" not in SCENE:
        SCENE["s"] = bs.make_blur_scene()
    return SCENE["s"]


def rehearse(sc):
    """Per frame with a true streak >= 3 px: the fractions of the visible features the oracle's search matches within
    2 px of their true position, with the warped stored templates and with blur_ref's templates."""
    from oracle import pyoracle as po
    out = []
    B, half = sc.boxsize, (sc.boxsize - 1) // 2
    for k in range(1, len(sc.frames)):
        if sc.streak[k] < 3.0:
            continue
        x = bs.true_state(sc, k)
        h = np.stack([project_point(sc.cam8, camera_points(x[:7], y))[0] for y in sc.y])
        vis = (h[:, 0] > 20) & (h[:, 0] < sc.cam8[0] - 21) & (h[:, 1] > 20) & (h[:, 1] < sc.cam8[1] - 21)
        idx = np.flatnonzero(vis)
        stored, _ = warp_ref.warp_templates(sc.cam8, sc.patches[idx], sc.y[idx], sc.xp_org[idx], x[:7])
        blurred, valid, _ = blur_ref.blur_templates(sc.cam8, sc.patches[idx], sc.y[idx], sc.xp_org[idx], x,
                                                    bs.EXPOSURE, bs.OFFSET, True)
        puinv = np.tile([1 / SIGMA ** 2, 0.0, 1 / SIGMA ** 2], (len(idx), 1))
        row = [k, float(sc.streak[k])]
        for T in (stored, blurred):
            u, v, found, _ = po.elliptical_search(sc.frames[k], T, h[idx], puinv)
            err = np.hypot(u - h[idx, 0], v - h[idx, 1])
            row.append(float((found.astype(bool) & (err <= 2.0)).mean()))
        out.append(row)
    return np.array(out)


def test_cpu_rehearsal_blurred_templates_match_where_stored_ones_fail():
    r = rehearse(scene())
    print("rehearsal [frame, streak px, stored, blurred]:\n", np.round(r, 3))
    # measured: stored 0.08 and blurred 0.71 of the visible features on average, blurred at least 0.325 on a frame
    assert len(r) >= 10
    assert r[:, 3].mean() >= r[:, 2].mean() + 0.5, r[:, 2:].mean(0)
    assert r[:, 3].min() >= 0.3 and (r[:, 3] >= r[:, 2]).all(), r[:, 2:]


# ---- on the device -------------------------------------------------------------------------------------------------
RUNS = {"off": None, "on": (bs.EXPOSURE, bs.OFFSET), "half": (bs.EXPOSURE / 2, bs.OFFSET / 2),
        "double": (2 * bs.EXPOSURE, 2 * bs.OFFSET), "sign": (bs.EXPOSURE, -bs.OFFSET)}


def track(sc):
    """Every run of RUNS as one stream of one context (warp and gyro on in all): per run, the matched fraction of
    the selected features on every step, and the final state."""
    import scenelib2_b200 as sl2
    names = list(RUNS)
    S = len(names)
    cfg = sl2.default_config()
    cfg.num_streams = S
    cfg.width, cfg.height = int(sc.cam8[0]), int(sc.cam8[1])
    cfg.boxsize = sc.boxsize
    cfg.max_features = len(sc.y)
    cfg.number_of_features_to_select = 16
    cfg.fku, cfg.fkv, cfg.u0, cfg.v0, cfg.kd1, cfg.sd = [float(v) for v in sc.cam8[2:8]]
    cfg.delta_t = sc.delta_t
    ctx = sl2.Context(cfg)
    try:
        for s, name in enumerate(names):
            ctx.set_features(s, sc.y, sc.xp_org, sc.patches)
            ctx.set_state(s, sc.x0, sc.P0)
            ctx.set_stream_warp(s, 1)
            ctx.set_stream_gyro(s, 1, cov=np.eye(3) * 1e-4)
            if RUNS[name] is not None:
                ctx.set_stream_blur(s, 1, *RUNS[name])
        frac = np.zeros((len(sc.frames) - 1, S))
        for t in range(1, len(sc.frames)):
            ctx.set_gyro_samples(0, np.tile(sc.omega[t - 1], (S, 1)))
            ctx.set_frames(0, np.stack([sc.frames[t]] * S))
            ctx.step(0)
            ctx.sync()
            for s in range(S):
                f = ctx.features(s)
                sel = f["select_rank"] >= 0
                frac[t - 1, s] = ((f["flags"] & 2) > 0)[sel].sum() / max(1, sel.sum())
        return {n: (frac[:, s], ctx.get_state(s)[0]) for s, n in enumerate(names)}
    finally:
        ctx.close()


@pytest.mark.gpu
def test_blur_keeps_the_matches_of_a_fast_yaw():
    sc = scene()
    res = track(sc)
    fast = sc.streak[1:] >= 3.0
    report = {}
    for name, (frac, x) in res.items():
        report[name] = dict(matched_fast=round(float(frac[fast].mean()), 3), min_fast=round(float(frac[fast].min()), 3),
                            end_deg=round(angle_deg(x[3:7], sc.poses[-1][3:]), 3))
    print("capability", report)
    # measured on an H100 (DESIGN.md): matched on fast steps off 0.724, on 0.842, half 0.825, double 0.622, sign
    # 0.769; end orientation error off 0.303, on 0.172 degrees
    on, off = report["on"], report["off"]
    assert on["matched_fast"] >= off["matched_fast"] + 0.1, report
    assert on["matched_fast"] >= 0.8 and on["min_fast"] >= off["min_fast"] and on["end_deg"] <= 0.3, report
    for name in ("double", "sign"):  # an exposure set too long or on the wrong side of the stamp helps less
        assert report[name]["matched_fast"] < on["matched_fast"], report
    assert report["half"]["matched_fast"] <= on["matched_fast"] + 0.02, report
