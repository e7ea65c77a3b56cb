"""The planar patch warp on the device (sl2_warp_templates; csrc/warp.cu warp_kernel) against the restatement
(tests/warp_ref.py) bit for bit and against the warp from its definition (tests/warp_truth.py) under the decision rule
of tests/warp_cases.py: at |q| != 1, on the exact constructions (.5 ties, the template's edges, the reach, zo[2] <= 0,
a ray parallel to the plane), at 15 x 15 on C3, on a stream with its own wide camera, at the kernel's shape edges, and
at the pose a run of fused steps with the warp on leaves."""
import numpy as np
import pytest

import scenelib2_b200 as sl2
import warp_cases as wc
import warp_ref
from test_gpu_warp import cam8_of, ctx_for, scene, scene_ctx

N = 256


def features(cam8, B, xp, n, rng, reach=0.9):
    """n features of the visibility envelope seen from the unit-q pose xp: y (n, 3), xo (n, 7), T (n, B, B)."""
    y = np.stack([wc.seen_point(cam8, xp, rng, reach=reach) for _ in range(n)])
    xo = np.stack([wc.first_view(y[k], xp, rng, rng.uniform(0.55, 1.8), rng.uniform(0, 40)) for k in range(n)])
    return y, xo, rng.integers(0, 256, (n, B, B), dtype=np.uint8)


def check(ctx, s, cam8, y, xo, T, xp, idx=None, truth_every=1):
    """The device's templates of features idx at xp: equal to the restatement byte for byte (and in valid), and to
    the truth under the rule for every truth_every-th job.  Returns the device's valid flags."""
    idx = np.arange(len(y)) if idx is None else np.asarray(idx)
    out, valid = ctx.warp_templates(s, idx, xp)
    want, wvalid = warp_ref.warp_templates(cam8, T[idx], y[idx], xo[idx], xp)
    assert (valid == wvalid).all() and out.tobytes() == want.tobytes()
    B = T.shape[1]
    for j in range(0, len(idx), truth_every):
        k = idx[j]
        D = wc.Decided(cam8, B, y[k], xo[k], xp, T[k])
        fail = D.check_template(out[j], valid[j])
        assert not fail, (j, k, fail)
    return valid


# ---- 1. non-unit q, C1 at 11 x 11 and C3 at 15 x 15 -------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["C1", "C3"])
def test_non_unit_q_equals_the_truth(name):
    n = 48
    ctx, cam8 = ctx_for(name, n)
    B = ctx.cfg.boxsize
    rng = np.random.default_rng(90 + B)
    try:
        warped = 0
        for s in wc.Q_NORMS:
            xp = wc.look_at(rng.uniform(-1, 1, 3), rng.uniform(-1, 1, 3) + [0, 0, 3.0], rng.uniform(-np.pi, np.pi))
            y, xo, T = features(cam8, B, xp, n, rng)
            xo = np.stack([wc.with_norm(x, s) for x in xo])
            ctx.set_features(0, y, xo, T)
            warped += int(check(ctx, 0, cam8, y, xo, T, wc.with_norm(xp, s)).sum())
        assert warped >= 0.9 * n * len(wc.Q_NORMS), warped
    finally:
        ctx.close()


# ---- 2. the exact constructions: the device equals the truth exactly ---------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["C1", "C3"])
def test_constructions_equal_the_truth_exactly(name):
    ctx, _ = ctx_for(name, 4)
    B = ctx.cfg.boxsize
    try:
        for cname, cam8, cB, y, xo, xp, T in wc.constructions():
            if cB != B:
                continue
            ctx.set_stream_config(0, ctx.stream_config(0), fku=cam8[2], fkv=cam8[3], u0=cam8[4], v0=cam8[5],
                                  kd1=cam8[6])
            cam = cam8_of(ctx, 0)
            assert (cam[2:7] == cam8[2:7]).all()
            T3 = np.asarray(T, np.uint8)[None]
            ctx.set_features(0, np.asarray(y)[None], np.asarray(xo)[None], T3)
            out, valid = ctx.warp_templates(0, [0], xp)
            want, wvalid = warp_ref.warp_templates(cam, T3, np.asarray(y)[None], np.asarray(xo)[None], xp)
            assert (valid == wvalid).all() and out.tobytes() == want.tobytes(), cname
            D = wc.Decided(cam, B, y, xo, xp, T)
            tr = D.tr
            if tr.valid.all():  # every byte, ties included: the chain is exact
                assert valid[0] == 1 and (out[0] == tr.byte).all(), cname
                if cname.startswith("half-shift"):
                    assert (tr.tie_gap == 0).sum() >= B
            else:               # the rows and the reach: some pixel is invalid, exactly
                assert valid[0] == 0 and (out[0] == T).all(), cname
            assert not D.check_template(out[0], valid[0]), cname
    finally:
        ctx.close()


# ---- 3. a stream other than 0 with its own wide camera --------------------------------------------------------------------
@pytest.mark.gpu
def test_stream_2_with_a_wide_camera():
    n = 96
    ctx, _ = ctx_for("C1", n, num_streams=3)
    rng = np.random.default_rng(2)
    try:
        _, wide, _ = next(c for c in wc.cameras() if c[0] == "reach")
        ctx.set_stream_config(2, ctx.stream_config(2), fku=wide[2], fkv=wide[3], kd1=wide[6])
        cam = cam8_of(ctx, 2)
        assert (cam[2:7] == wide[2:7]).all()
        for s in (1.0, 1 + 1e-3):
            xp = wc.look_at(np.zeros(3), np.array([0.1, -0.1, 2.0]), 0.4)
            y, xo, T = features(cam, 11, xp, n, rng, reach=0.999)
            xo = np.stack([wc.with_norm(x, s) for x in xo])
            ctx.set_features(2, y, xo, T)
            ctx.set_features(0, y[::-1], xo[::-1], T[::-1])
            v = check(ctx, 2, cam, y, xo, T, wc.with_norm(xp, s))
            assert 0 < v.sum() < n  # templates that straddle the reach are invalid
    finally:
        ctx.close()


# ---- 4. the kernel's shape edges: 4 warps per CTA, one job per warp -------------------------------------------------------
@pytest.mark.gpu
def test_shape_edges():
    ctx, cam8 = ctx_for("C1", N)
    rng = np.random.default_rng(4)
    try:
        xu = wc.look_at(np.zeros(3), np.array([0.1, -0.1, 2.0]), 0.2)
        xp = wc.with_norm(xu, 1 - 3.5e-5)
        y, xo, T = features(cam8, 11, xu, N, rng)
        for k in range(N):
            if k % 2:  # the first camera faces away from the feature: every plane point lies behind it (zo[2] < 0)
                xo[k] = wc.look_at(xo[k][:3], 2 * xo[k][:3] - y[k], 0.3)
            else:      # a feature whose every pixel is valid
                while not warp_ref.warp_template(cam8, T[k], y[k], xo[k], xp)[1]:
                    y1, xo1, _ = features(cam8, 11, xu, 1, rng)
                    y[k], xo[k] = y1[0], xo1[0]
        ctx.set_features(0, y, xo, T)
        for n in (1, 3, 4, 5, 8, 9, 255, 256):
            v = check(ctx, 0, cam8, y, xo, T, xp, idx=np.arange(n), truth_every=1 if n < 255 else 17)
            assert (v == (np.arange(n) % 2 == 0)).all(), n  # valid and invalid alternate within each CTA
        rep = np.array([3, 3, 7, 3, 0, 7, 255, 255, 0, 3, 128])
        check(ctx, 0, cam8, y, xo, T, xp, idx=rep)
        check(ctx, 0, cam8, y, xo, T, xp, idx=np.full(9, 6))
    finally:
        ctx.close()


# ---- 5. the fused step's pose ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_templates_at_the_fused_steps_pose_equal_the_truth():
    """After fused steps with the warp on, |q| of the stream's x has drifted from 1; the templates its search used
    (sl2_warp_templates at that x[0:7], the link that
    test_measure_stage_equals_the_oracle_search_of_templates_warped_at_non_unit_q pins)
    equal the truth under the rule."""
    sc = scene("roll")
    ctx = scene_ctx([sc])
    try:
        ctx.set_stream_warp(0, 1)
        for t in range(1, 21):
            ctx.set_frames(0, sc.frames[t][None])
            ctx.step(0)
            ctx.sync()
        x, _ = ctx.get_state(0)
        qn = float(np.linalg.norm(x[3:7]))
        snap = sl2.read_snapshot(ctx.save_stream(0))
        nf = ctx.num_features(0)
        assert nf == len(sc.y)  # no feature culled: the stored templates are the scene's
        y, xo = x[13:13 + 3 * nf].reshape(-1, 3), snap["xp_org"][:nf]
        T = np.asarray(sc.patches[:nf], np.uint8)
        print("|q| - 1 after 20 fused steps: %.3g" % (qn - 1))
        assert qn != 1.0
        valid = check(ctx, 0, sc.cam8, y, xo, T, x[:7])
        assert valid.sum() >= 0.9 * nf
    finally:
        ctx.close()
