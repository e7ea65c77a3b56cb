"""GPU: the depth-particle re-weighting (particle_kernel, particles.cu) behind sl2_measure_particles[_patch] and
sl2_measure_partial_features, at its knife edges and batch shapes.

The matches are placed exactly: a noise template is pasted at known integer positions of a texture, and every
particle's ellipse holds exactly one paste (or lies on a flat band, where the match fails), so the search returns
z = that position.  The device search is first held to oracle.smoe_search.  Then:
  - where every found particle has nu = 0 (e^-0 = 1 on both sides) the device equals oracle.particle_update bit for
    bit in prob, cumulative, keep, left and (mean, variance);
  - with general nu it equals the restatement (particle_ref) run with the device's own exp bit for bit, the oracle
    (glibc's exp) to a few ulps, and the extended-precision truth (particle_truth) within the bounds of
    particle_cases.  The device's exp is measured on the same arguments and its differences from glibc's are
    reported.
The search bounds q = nu^T S^-1 nu (its ellipse is q < 9 around the integer centre), so on the device the likelihood
cannot underflow through e^(-q/2): the subnormal and vanishing cases get there through the prior and det S.
Last, every per-particle output slot k >= K[f] of sl2_measure_partial_features keeps what the caller put there."""
import math

import numpy as np
import pytest

import particle_ref
from gpu_util import ctx_for_image, sl2, synth
from particle_truth import particle_truth
from particle_cases import bounds, compare, dyadic_probabilities, exact_case, sinv_random, threshold_cases

pytestmark = pytest.mark.gpu
W, H, B = 320, 240, 11
PASTES = [(x, y) for y in range(20, 161, 20) for x in range(20, 301, 20)]     # 15 x 8, 20 px apart
FLAT = [(x, y) for y in (200, 212, 224) for x in range(24, 297, 8)]            # centres on the flat band
EXP_STATS = {"n": 0, "differ": 0, "max_ulps": 0}
ORC = ("h", "Sinv3", "detS", "lam", "z", "found", "threshold", "prior")    # oracle.particle_update's, particle_ref's


def _impl_args(case):
    return [case[k] for k in ORC]


def scene(seed):
    """A texture with the noise template pasted (centred) at PASTES and a flat band in rows 185..239."""
    rng = np.random.default_rng(seed)
    img = synth.make_texture(rng, H, W)
    tpl = rng.integers(0, 256, (B, B), dtype=np.uint8)
    for x, y in PASTES:
        img[y - 5:y + 6, x - 5:x + 6] = tpl
    img[185:, :] = 127
    return img, tpl


def _inside(P, h, s):
    """The search's ellipse test of integer location P around the integer centre of h (sl2_score.cuh)."""
    du, dv = P[0] - math.trunc(h[0]), P[1] - math.trunc(h[1])
    return s[0] * du * du + 2 * s[1] * du * dv + s[2] * dv * dv < 9.0


def placed(rng, K, found, general=False, Sinv3=None):
    """h (K, 2), Sinv3 (K, 3) and the intended z: found particles on PASTES (cycled), others on FLAT.  general: h off
    its paste by a random nu that keeps the paste inside the ellipse; else h = z exactly (nu = 0)."""
    Sinv3 = sinv_random(rng, K, 0.7, 2.0) if Sinv3 is None else Sinv3
    z = np.zeros((K, 2), np.int32)
    h = np.zeros((K, 2))
    off = rng.integers(0, len(PASTES))
    for k in range(K):
        P = PASTES[(off + k) % len(PASTES)] if found[k] else FLAT[(off + k) % len(FLAT)]
        z[k] = P
        h[k] = P
        while general and found[k]:
            cand = np.array(P, float) + rng.normal(0, 0.8, 2)
            if _inside(P, cand, Sinv3[k]):
                h[k] = cand
                break
    return h, Sinv3, z


def device_exp(args):
    """The device's exp (the CUDA math library's, which particle_kernel calls) on FP64 arguments, via torch."""
    import torch
    t = torch.tensor(np.asarray(args, np.float64), dtype=torch.float64, device="cuda")
    return torch.exp(t).cpu().numpy()


def _ulps(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    ia, ib = a.view(np.int64), b.view(np.int64)
    return np.where(a == b, 0, np.abs(ia - ib))


def run_case(oracle, ctx, img, tpl, case, patch=False, exact=None, label=""):
    """One feature through sl2_measure_particles[_patch]: the search against the oracle and the construction, then the
    re-weighting against the oracle (bits when exact, else a few ulps), the restatement with the device's exp (bits)
    and the truth (bounds).  Returns the device's result."""
    h, Sinv3, z = case["h"], case["Sinv3"], case["z"]
    got = ctx.measure_particles(0, 0, 0, h, Sinv3, case["detS"], case["lam"], case["threshold"], case["prior"],
                                patch=tpl if patch else None)
    left, prob, gz, found, keep, cum, mv = got
    ou, ov, of, _ = oracle.smoe_search(img, tpl, Sinv3, h)
    assert (found == of).all(), label
    assert (gz[of > 0, 0] == ou[of > 0]).all() and (gz[of > 0, 1] == ov[of > 0]).all(), label
    assert (found == case["found"]).all() and (gz[found > 0] == z[found > 0]).all(), label   # the construction
    o = oracle.particle_update(*_impl_args(case))
    res = (left, prob, keep, cum, mv)
    exact = case.get("nu0", False) if exact is None else exact
    if exact:
        assert left == o[0], label
        for a, b, what in zip(res[1:], o[1:], ("prob", "keep", "cumulative", "mean_var")):
            assert np.asarray(a).tobytes() == np.asarray(b).tobytes(), (label, what)
    else:
        args = [particle_ref.exp_argument(z[k], h[k], Sinv3[k]) for k in range(len(h)) if found[k]]
        dev = device_exp(args)
        host = np.array([math.exp(a) for a in args])
        d = _ulps(dev, host)
        EXP_STATS["n"] += len(args)
        EXP_STATS["differ"] += int((d > 0).sum())
        EXP_STATS["max_ulps"] = max(EXP_STATS["max_ulps"], int(d.max()) if d.size else 0)
        table = dict(zip(args, dev))
        r = particle_ref.update(*_impl_args(case), exp=lambda a: float(table[a]))
        assert left == r[0], label
        for a, b, what in zip(res[1:], r[1:], ("prob", "keep", "cumulative", "mean_var")):
            assert np.asarray(a).tobytes() == np.asarray(b).tobytes(), (label, what, "device exp restated")
        if (keep == o[2]).all():
            assert _ulps(prob, o[1]).max() <= 64 and _ulps(cum, o[3]).max() <= 64, label
    c2 = dict(case, exact=bool(case.get("exact", False) and exact))
    prec = "mp" if c2["exact"] else "ld"       # longdouble does not hold the exact cases' probabilities exactly
    tr = particle_truth(*[case[k] for k in ("h", "Sinv3", "detS", "lam", "prior", "z", "found", "threshold")],
                        prec=prec)
    fail, _ = compare(c2, tr, bounds(c2, tr, prec), res, prec)
    assert not fail, (label, fail)
    return got


def exact_device_case(rng, p, found, lam, threshold, t=None, scale=1.0, exact=True):
    """exact_case on pasted positions (nu = 0)."""
    K = len(p)
    h, Sinv3, z = placed(rng, K, found)
    c = exact_case(p, z, found, lam, threshold, t=t, scale=scale, Sinv3=Sinv3, exact=exact)
    c["nu0"] = True
    return c


@pytest.fixture(scope="module")
def bench():
    img, tpl = scene(7)
    ctx = ctx_for_image(img, tpl[None], radius=20)
    yield img, tpl, ctx
    ctx.close()


def test_threshold_edges_are_bit_exact(oracle, bench):
    """fl(threshold / K) exactly on one particle's probability: kept; the next double above the threshold: pruned
    (K = 4, 128, 256)."""
    img, tpl, ctx = bench
    rng = np.random.default_rng(11)
    for K in (4, 128, 256):
        for name, c, j, kept in threshold_cases(rng, K):
            case = exact_device_case(rng, c["prior"], np.ones(K), c["lam"], c["threshold"])
            left, prob, _, _, keep, _, _ = run_case(oracle, ctx, img, tpl, case, label=name)
            assert bool(keep[j]) == kept and prob[j] != 0, name


def test_exact_edges_are_bit_exact(oracle, bench):
    """threshold 0, every particle pruned (the reference keeps the feature with no particles: left = 0, prob stays
    normalised, no deletion), lambda clustered to 1e-7 and all equal (the variance cancels, negative included),
    unnormalised priors, zero priors, det S over seven decades, failed matches."""
    img, tpl, ctx = bench
    rng = np.random.default_rng(12)
    K = 64
    f = np.ones(K)
    f[rng.permutation(K)[:7]] = 0
    p = np.zeros(K)
    p[f > 0] = dyadic_probabilities(rng, int(f.sum()), zeros=9)
    left, prob, _, _, keep, _, _ = run_case(oracle, ctx, img, tpl, exact_device_case(rng, p, f, np.linspace(1, 3, K),
                                                                                    0.0), label="threshold-0")
    assert left == K and keep.all()
    case = exact_device_case(rng, np.full(128, 2.0 ** -7), np.ones(128), np.linspace(1, 3, 128), 2.0)
    left, prob, _, _, keep, cum, mv = run_case(oracle, ctx, img, tpl, case, label="all-pruned")
    assert left == 0 and not keep.any() and (cum == 0).all() and (mv == 0).all() and prob.sum() == 1.0
    case = exact_device_case(rng, dyadic_probabilities(rng, 100), np.ones(100),
                             1.7 * (1 + 1e-7 * rng.uniform(-1, 1, 100)), 0.05)
    run_case(oracle, ctx, img, tpl, case, label="lambda-clustered")
    negative = 0
    for i in range(40):
        p = dyadic_probabilities(rng, 33)
        case = exact_device_case(rng, p, np.ones(33), np.full(33, 2.3 + 0.01 * i), 0.05)
        negative += run_case(oracle, ctx, img, tpl, case, label="lambda-equal")[6][1] < 0
    assert negative > 0
    run_case(oracle, ctx, img, tpl, exact_device_case(rng, dyadic_probabilities(rng, 50, zeros=6), np.ones(50),
                                                      np.linspace(0.3, 7, 50), 0.3, scale=96.0), label="unnormalised")
    t = rng.integers(-3, 9, 64)
    case = exact_device_case(rng, dyadic_probabilities(rng, 64), np.ones(64), np.linspace(0.4, 6, 64), 0.8, t=t,
                             exact=False)
    run_case(oracle, ctx, img, tpl, case, label="detS-decades")


def test_general_nu_against_truth_and_device_exp(oracle, bench):
    """nu off the paste, correlated S^-1, det S = 1 / det S^-1 over two decades, several thresholds."""
    img, tpl, ctx = bench
    rng = np.random.default_rng(13)
    differ = 0
    for i in range(12):
        K = int(rng.choice([7, 40, 100, 200, 256]))
        found = (rng.random(K) < rng.choice([1.0, 0.7])).astype(np.uint8)
        h, Sinv3, z = placed(rng, K, found, general=True)
        prior = rng.uniform(0, 1, K)
        prior[rng.random(K) < 0.1] = 0
        case = dict(h=h, Sinv3=Sinv3, detS=1.0 / (Sinv3[:, 0] * Sinv3[:, 2] - Sinv3[:, 1] ** 2),
                    lam=rng.uniform(0.3, 8, K), prior=prior, z=z, found=found,
                    threshold=float(rng.choice([0.05, 0.5, 1.0])), exact=False)
        left, prob, _, _, keep, cum, mv = run_case(oracle, ctx, img, tpl, case, label="general-%d" % i)
        o = oracle.particle_update(*_impl_args(case))
        tr = particle_truth(*[case[k] for k in ("h", "Sinv3", "detS", "lam", "prior", "z", "found", "threshold")],
                            prec="ld")
        b = bounds(case, tr, "ld")
        # a prune decision the device and the oracle take differently must be one the truth cannot fix
        assert not ((keep != o[2]) & b["decided"]).any(), i
        differ += int((keep != o[2]).sum())
    print("device exp vs glibc exp on %d likelihood arguments: %d differ, by at most %d ulp; prune decisions that "
          "differ from the oracle's: %d" % (EXP_STATS["n"], EXP_STATS["differ"], EXP_STATS["max_ulps"], differ))


def test_underflow(oracle, bench):
    """Subnormal w (prior 1e-310 on some particles), every found w subnormal (the total is subnormal and positive: the
    feature survives, as in the reference), every w exactly 0 (prior 1e-200 and det S 1e250: deletion, prob
    un-normalised, i.e. 0), failed matches mixed with found ones, all matches failed."""
    img, tpl, ctx = bench
    rng = np.random.default_rng(14)
    for nu0 in (True, False):
        K = 48
        found = np.ones(K, np.uint8)
        h, Sinv3, z = placed(rng, K, found, general=not nu0)
        base = dict(h=h, Sinv3=Sinv3, detS=1.0 / (Sinv3[:, 0] * Sinv3[:, 2] - Sinv3[:, 1] ** 2),
                    lam=np.linspace(0.5, 5, K), z=z, found=found, exact=False, nu0=nu0)
        prior = rng.uniform(0.1, 1, K)
        prior[::4] = rng.uniform(1e-312, 1e-309, len(prior[::4]))
        left, prob, *_ = run_case(oracle, ctx, img, tpl, dict(base, prior=prior, threshold=0.0), label="some-sub")
        assert left == K
        left, prob, _, _, keep, _, _ = run_case(oracle, ctx, img, tpl,
                                                dict(base, prior=rng.uniform(1e-316, 1e-312, K), threshold=0.05),
                                                label="all-sub")
        assert left > 0 and abs(prob[keep > 0].sum() - 1) < 1e-12
        vanish = dict(base, prior=np.full(K, 1e-200), detS=np.full(K, 1e250), threshold=0.05)
        left, prob, _, _, keep, cum, mv = run_case(oracle, ctx, img, tpl, vanish, label="vanish")
        assert left == 0 and (prob == 0).all() and not keep.any()
        mixed = rng.random(K) < 0.5
        h2, S2, z2 = placed(rng, K, mixed.astype(np.uint8), general=not nu0)
        run_case(oracle, ctx, img, tpl, dict(base, h=h2, Sinv3=S2, z=z2, found=mixed.astype(np.uint8),
                                             detS=1.0 / (S2[:, 0] * S2[:, 2] - S2[:, 1] ** 2),
                                             prior=rng.uniform(0, 1, K), threshold=0.9), label="mixed")
    h, Sinv3, z = placed(rng, 12, np.zeros(12))
    left, prob, *_ = run_case(oracle, ctx, img, tpl, dict(h=h, Sinv3=Sinv3, detS=np.ones(12), lam=np.ones(12),
                                                          prior=np.full(12, 1 / 12), z=z, found=np.zeros(12, np.uint8),
                                                          threshold=0.05, exact=False, nu0=True), label="all-failed")
    assert left == 0 and (prob == 0).all()


@pytest.mark.parametrize("patch", [False, True])
def test_particle_counts_across_the_block(oracle, bench, patch):
    """K through one, and either side of the warp and of particle_kernel's 128-thread stride, by feature index and
    by raw template."""
    img, tpl, ctx = bench
    rng = np.random.default_rng(15 + patch)
    for K in (1, 2, 31, 32, 33, 127, 128, 129, 255, 256):
        found = (rng.random(K) < 0.85).astype(np.uint8)
        found[0] = 1
        h, Sinv3, z = placed(rng, K, found, general=True)
        case = dict(h=h, Sinv3=Sinv3, detS=1.0 / (Sinv3[:, 0] * Sinv3[:, 2] - Sinv3[:, 1] ** 2),
                    lam=rng.uniform(0.3, 8, K), prior=rng.uniform(0.1, 1, K), z=z, found=found, threshold=0.5,
                    exact=False)
        run_case(oracle, ctx, img, tpl, case, patch=patch, label="K%d" % K)
        c0 = exact_device_case(rng, dyadic_probabilities(rng, K, lo=0.05), np.ones(K), rng.uniform(0.3, 8, K), 0.5)
        run_case(oracle, ctx, img, tpl, c0, patch=patch, label="K%d-exact" % K)


def test_other_stream_and_slot(oracle):
    """Stream 2, ring slot 1 of a three-stream, two-slot context whose other streams and slots hold different frames
    and templates."""
    img, tpl = scene(21)
    cfg = sl2.default_config()
    cfg.width, cfg.height, cfg.boxsize = W, H, B
    cfg.max_features, cfg.num_streams, cfg.frame_slots = 1, 3, 2
    cfg.search_tile_radius = 20
    ctx = sl2.Context(cfg)
    try:
        rng = np.random.default_rng(22)
        for s in range(3):
            other, otpl = scene(30 + s)
            ctx.set_features(s, np.zeros((1, 3)), np.array([[0, 0, 0, 1, 0, 0, 0.0]]), (tpl if s == 2 else otpl)[None])
            for slot in range(2):
                ctx.set_frame(s, slot, img if (s, slot) == (2, 1) else synth.make_texture(rng, H, W))
        K = 100
        found = (rng.random(K) < 0.8).astype(np.uint8)
        h, Sinv3, z = placed(rng, K, found, general=True)
        case = dict(h=h, Sinv3=Sinv3, detS=1.0 / (Sinv3[:, 0] * Sinv3[:, 2] - Sinv3[:, 1] ** 2),
                    lam=rng.uniform(0.3, 8, K), prior=rng.uniform(0.1, 1, K), z=z, found=found, threshold=0.5,
                    exact=False)
        got = ctx.measure_particles(2, 1, 0, h, Sinv3, case["detS"], case["lam"], 0.5, case["prior"])
        assert (got[3] == found).all() and (got[2][found > 0] == z[found > 0]).all()
        o = oracle.particle_update(*_impl_args(case))
        assert got[0] == o[0] and (got[4] == o[2]).all()
        c0 = exact_device_case(rng, dyadic_probabilities(rng, K), found, rng.uniform(0.3, 8, K), 0.5)
        c0["prior"][found == 0] = 0.25
        got = ctx.measure_particles(2, 1, -1, c0["h"], c0["Sinv3"], c0["detS"], c0["lam"], 0.5, c0["prior"],
                                    patch=tpl)
        o = oracle.particle_update(*_impl_args(c0))
        assert got[0] == o[0]
        for a, b in zip((got[1], got[4], got[5], got[6]), o[1:]):
            assert np.asarray(a).tobytes() == np.asarray(b).tobytes()
    finally:
        ctx.close()


# ---- sl2_measure_partial_features: shapes and the slots past K[f] ----------------------------------------------------
def partial_inputs(ctx, img, rng, F, Kmax):
    """F rays of the stream's camera (some toward pasted templates), their 13 x 6 / 6 x 6 covariance blocks,
    lambda and priors."""
    cfg = ctx.cfg
    xv = np.zeros(13)
    xv[3] = 1.0
    A = rng.normal(0, 1, (16, 16))
    P = A @ A.T * 2e-6 + 1e-8 * np.eye(16)
    ctx.set_state(0, np.concatenate([xv, [0.1, 0.1, 2.0]]), P)
    ypi = np.zeros((F, 6))
    Pxy = np.zeros((F, 13, 6))
    Pyy = np.zeros((F, 6, 6))
    for f in range(F):
        u, v = PASTES[(7 * f) % len(PASTES)]
        hh = np.array([-(u - cfg.u0) / cfg.fku, -(v - cfg.v0) / cfg.fkv, 1.0])
        ypi[f, 3:] = hh / np.linalg.norm(hh)
        Af = rng.normal(0, 1, (19, 19))
        Pf = Af @ Af.T * 2e-6 + 1e-8 * np.eye(19)
        Pxy[f], Pyy[f] = Pf[:13, 13:], Pf[13:, 13:]
    lam = np.tile(np.linspace(0.3, 8.0, Kmax), (F, 1))
    prob = rng.uniform(0.2, 1.0, (F, Kmax))
    cam8 = np.array([cfg.width, cfg.height, cfg.fku, cfg.fkv, cfg.u0, cfg.v0, cfg.kd1, cfg.sd], float)
    return cam8, xv, P, ypi, Pxy, Pyy, lam, prob


def check_partial(oracle, img, patches, cam8, xv, P, inp, K, out, prob_in, thr):
    ypi, Pxy, Pyy, lam = inp
    any_found = False
    for f in range(len(K)):
        k = int(K[f])
        if k == 0:
            assert out["left"][f] == 0 and (out["mean_var"][f] == 0).all()
            continue
        oh, oS, osi, odet = oracle.predict_particles(cam8, xv, ypi[f], lam[f, :k], P[:13, :13], Pxy[f], Pyy[f])
        assert out["h"][f, :k].tobytes() == oh.tobytes() and out["Sinv3"][f, :k].tobytes() == osi.tobytes(), f
        assert out["detS"][f, :k].tobytes() == odet.tobytes(), f
        ou, ov, of, _ = oracle.smoe_search(img, patches[f], osi, oh)
        assert (out["found"][f, :k] == of).all(), f
        z = np.column_stack([ou, ov]).astype(np.int32)
        assert (out["z"][f, :k][of > 0] == z[of > 0]).all(), f
        any_found |= bool(of.any())
        case = dict(h=oh, Sinv3=osi, detS=odet, lam=lam[f, :k], z=z, found=of, threshold=thr, prior=prob_in[f, :k],
                    exact=False)
        args = [particle_ref.exp_argument(z[j], oh[j], osi[j]) for j in range(k) if of[j]]
        table = dict(zip(args, device_exp(args))) if args else {}
        r = particle_ref.update(*_impl_args(case), exp=lambda a: float(table[a]))
        res = (out["left"][f], out["prob"][f, :k], out["keep"][f, :k], out["cumulative"][f, :k], out["mean_var"][f])
        assert res[0] == r[0], f
        for a, b in zip(res[1:], r[1:]):
            assert np.asarray(a).tobytes() == np.asarray(b).tobytes(), f
        tr = particle_truth(*[case[x] for x in ("h", "Sinv3", "detS", "lam", "prior", "z", "found", "threshold")],
                            prec="ld")
        fail, _ = compare(case, tr, bounds(case, tr, "ld"), res, "ld")
        assert not fail, (f, fail)
    assert any_found


@pytest.mark.parametrize("Ks", ["edges", "below-Kmax"])
def test_partial_features_batch_shapes(oracle, bench, Ks):
    """F = 16, Kmax = 256 in one call: K through 1, 2, 31..33, 127..129, 255, 256 with K = 0 features between them;
    and the same with Kmax above every K."""
    img, tpl, ctx = bench
    rng = np.random.default_rng(40)
    F, Kmax = 16, 256
    K = np.array([256, 0, 1, 2, 31, 0, 32, 33, 127, 128, 0, 129, 255, 64, 3, 200], np.int32)
    if Ks == "below-Kmax":
        K = np.minimum(K, 250 - np.arange(F)).astype(np.int32)
    cam8, xv, P, ypi, Pxy, Pyy, lam, prob = partial_inputs(ctx, img, rng, F, Kmax)
    patches = np.stack([tpl if f % 3 else synth.make_texture(rng, B, B) for f in range(F)])
    out = ctx.measure_partial_features(0, 0, patches, ypi, Pxy, Pyy, lam, 0.3, prob, K=K)
    check_partial(oracle, img, patches, cam8, xv, P, (ypi, Pxy, Pyy, lam), K, out, prob, 0.3)


def test_partial_features_leave_slots_past_k_alone(oracle, bench):
    """A call with every K = Kmax leaves the staging buffer full of results; a second call with smaller K, every output
    pre-filled with a sentinel, must leave slots k >= K[f] of every per-particle output (prediction: h, Sinv3, detS;
    search: z, found; re-weighting: keep, cumulative; and prob, which is in/out) exactly as they were."""
    img, tpl, ctx = bench
    rng = np.random.default_rng(41)
    F, Kmax = 12, 200
    cam8, xv, P, ypi, Pxy, Pyy, lam, prob = partial_inputs(ctx, img, rng, F, Kmax)
    patches = np.stack([tpl] * F)
    ctx.measure_partial_features(0, 0, patches, ypi, Pxy, Pyy, lam, 0.3, prob, K=np.full(F, Kmax, np.int32))
    K = np.array([0, 1, 31, 200, 57, 128, 129, 0, 3, 199, 100, 64], np.int32)
    out = {"h": np.full((F, Kmax, 2), -7.25), "Sinv3": np.full((F, Kmax, 3), -7.25), "detS": np.full((F, Kmax), -7.25),
           "z": np.full((F, Kmax, 2), -77, np.int32), "found": np.full((F, Kmax), 0xA5, np.uint8),
           "keep": np.full((F, Kmax), 0xA5, np.uint8), "cumulative": np.full((F, Kmax), -7.25)}
    prob2 = prob.copy()
    for f in range(F):
        prob2[f, K[f]:] = -3.5
    res = ctx.measure_partial_features(0, 0, patches, ypi, Pxy, Pyy, lam, 0.3, prob2, K=K, out=out)
    for f in range(F):
        k = K[f]
        for name, a in out.items():
            assert res[name] is a
            tail = a[f, k:]
            assert (tail == (-77 if name == "z" else 0xA5 if a.dtype == np.uint8 else -7.25)).all(), (name, f, k)
        assert (res["prob"][f, k:] == -3.5).all(), f
    check_partial(oracle, img, patches, cam8, xv, P, (ypi, Pxy, Pyy, lam), K, res, prob2, 0.3)
