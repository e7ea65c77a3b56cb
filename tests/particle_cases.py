"""Cases and checks shared by tests/test_particle_truth.py (CPU) and tests/test_gpu_particles.py (GPU): constructors
of particle sets whose arithmetic is exact up to the prune, and the bounds an FP64 implementation of the re-weighting
must meet against particle_truth, with the comparison that applies them."""
import math

import numpy as np

import particle_ref
from particle_truth import truth_ld

U = 2.0 ** -53            # unit roundoff of FP64
TINY = 2.0 ** -1074       # subnormal spacing
LD = np.longdouble
HALF = LD(2) ** -1075     # not a double: RN rounds at or below it to 0


# ---- case constructors -----------------------------------------------------------------------------------------------
def det_for_c(t):
    """A det S for which the kernel's 1 / sqrt(fl(2 pi) det S) is exactly 2^-t: fl(fl(2 pi) det S) = 4^t."""
    d = 4.0 ** t / particle_ref.TWO_PI
    for step in range(-4, 5):
        x = d
        for _ in range(abs(step)):
            x = math.nextafter(x, math.inf if step > 0 else -math.inf)
        if particle_ref.TWO_PI * x == 4.0 ** t and 1.0 / math.sqrt(particle_ref.TWO_PI * x) == 2.0 ** -t:
            return x
    raise AssertionError("no det S with c = 2^-%d" % t)


def dyadic_probabilities(rng, K, m=20, zeros=0, pinned=None, lo=0.2):
    """K probabilities n_k 2^-m summing to exactly 1 (integers n_k >= 0, drawn in proportion to U(lo, 1)); `zeros` of
    them 0; pinned = (j, n_j) fixes one.  Every partial sum is exact in FP64."""
    n = rng.uniform(lo, 1.0, K)
    n[rng.permutation(K)[:zeros]] = 0.0
    total = 2 ** m
    fixed = 0
    if pinned is not None:
        n[pinned[0]] = 0.0
        fixed = pinned[1]
    n = np.floor(n / n.sum() * (total - fixed)).astype(np.int64)
    if pinned is not None:
        n[pinned[0]] = fixed
    free = [k for k in range(K) if n[k] > 0 and (pinned is None or k != pinned[0])]
    n[free[0]] += total - n.sum()
    assert n.sum() == total and (n >= 0).all()
    return n.astype(np.float64) * 2.0 ** -m


def sinv_random(rng, K, lo=0.7, hi=3.0):
    """K symmetric positive definite S^-1 = (S00, S01, S11) of standard deviations lo..hi px, |rho| up to 0.8."""
    a, b = rng.uniform(lo, hi, K), rng.uniform(lo, hi, K)
    r = rng.uniform(-0.8, 0.8, K)
    det = (a * b) ** 2 * (1 - r * r)
    return np.column_stack([b * b / det, -r * a * b / det, a * a / det])


def exact_case(p, z, found, lam, threshold, t=None, scale=1.0, Sinv3=None, exact=True):
    """nu = 0 for every particle (h = z), det S_k with c_k = 2^-t_k exactly, prior_k = p_k 2^t_k scale: every
    operation before the prune has an exact FP64 result (q = 0, e^-0 = 1, w_k = p_k scale, dyadic sums), so the
    normalised probabilities are p (renormalised over the found particles) on the device, on the CPU and, when every
    found particle has the same t, in the truth.  `exact` states that last condition."""
    K = len(p)
    t = np.zeros(K, int) if t is None else np.asarray(t)
    z = np.asarray(z, np.int32).reshape(K, 2)
    return dict(h=z.astype(np.float64), Sinv3=np.tile([1.0, 0.0, 1.0], (K, 1)) if Sinv3 is None else Sinv3,
                detS=np.array([det_for_c(int(v)) for v in t]), lam=np.asarray(lam, np.float64),
                prior=np.asarray(p) * 2.0 ** t * scale, z=z, found=np.asarray(found, np.uint8),
                threshold=float(threshold), exact=exact)


def threshold_cases(rng, K):
    """fl(threshold / K) equal to one particle's normalised probability p_j = 2^-a (kept), and the next double above
    the threshold (pruned); the other particles straddle p_j."""
    a = int(np.log2(K)) + 2
    j = K // 3
    p = dyadic_probabilities(rng, K, pinned=(j, 2 ** (20 - a)), lo=0.05)
    thr = p[j] * K
    assert thr / K == p[j]
    lam = np.linspace(0.5, 4.5, K)
    z = rng.integers(20, 300, (K, 2)).astype(np.int32)
    up = math.nextafter(thr, math.inf)
    assert up / K > p[j]
    return [("at-threshold-K%d" % K, exact_case(p, z, np.ones(K), lam, thr), j, True),
            ("above-threshold-K%d" % K, exact_case(p, z, np.ones(K), lam, up), j, False)]


# ---- bounds ----------------------------------------------------------------------------------------------------------
def _rn_hi(x):
    """An upper bound on RN(x), x >= 0: |RN(x) - x| <= u x + 2^-1075, and RN(x) = 0 for x <= 2^-1075 (ties to even)."""
    return np.where(x <= HALF, LD(0), x * (1 + LD(U)) + LD(HALF))


def _rn_lo(x):
    """A lower bound on RN(x), x >= 0: RN(x) >= TINY for x > 2^-1075."""
    return np.where(x <= HALF, LD(0), np.maximum(x * (1 - LD(U)) - LD(HALF), LD(TINY)))


def bounds(case, tr, prec="mp"):
    """Bounds on what an implementation that rounds every operation to nearest (exp within 1 ulp of the correctly
    rounded value) computes, from the truth's exact values:
      w_lo, w_hi : the interval of the computed w_k = fl(prior fl(c fl(exp(-fl(q) / 2)))).  q: nu rounds once,
                   the quadratic form rounds four times along every term, so |q_hat - q| <= gamma_6 qa
                   (qa = |nu|^T |S^-1| |nu|) and exp's argument is off by <= 3.01 u qa; exp adds one ulp
                   (<= 2u y + 2^-1074) to its rounded value; c = 1 / sqrt(fl(2 pi) det S) is off by <= 3.01 u
                   (fl(2 pi), the product, the sqrt, the division); each product rounds once, to 0 at or below
                   2^-1075 (the subnormal spacing is where the absolute terms come from);
      p1         : |p1_hat - p1| after the first normalisation: the total of K terms, serial, (K - 1) u;
      decided    : per particle, whether the prune decision is fixed (|p1 - thr| > the p1 bound; exact cases: always);
      prob, cum  : after the second normalisation over the kept set (K' terms), or p1 for pruned particles, or w;
      mean, var  : each product rounds once (lambda^2 once more), serial sums of K' terms; the variance
                   E[lambda^2] - mean^2 inherits both, so its bound is a multiple of E[lambda^2], not of the variance.
    Returns a dict; 'delete' is True / False where the deletion decision is fixed, None where it is not."""
    t = truth_ld(tr, prec)
    K = len(case["prior"])
    found = np.asarray(case["found"]).astype(bool)
    prior = np.asarray(case["prior"], np.float64).astype(LD)
    e = t.e
    de = LD(3.01 * U) * t.qa
    y_hi, y_lo = _rn_hi(e * (1 + de)), _rn_lo(e * np.maximum(1 - de, 0))
    e_hi, e_lo = y_hi + 2 * LD(U) * y_hi + LD(TINY), np.maximum(y_lo - 2 * LD(U) * y_lo - LD(TINY), 0)
    c_hi, c_lo = t.c * (1 + LD(3.01 * U)), t.c * (1 - LD(3.01 * U))
    w_hi = np.where(found, _rn_hi(prior * _rn_hi(c_hi * e_hi)), LD(0))
    w_lo = np.where(found, _rn_lo(prior * _rn_lo(c_lo * e_lo)), LD(0))
    dw = np.maximum(w_hi - t.w, t.w - w_lo)
    b = dict(w_lo=w_lo, w_hi=w_hi, dw=dw)
    b["delete"] = True if (w_hi == 0).all() else (False if (w_lo > 0).any() else None)
    b["decided"] = np.ones(K, bool)
    b["prob"], b["cum"] = dw.copy(), np.zeros(K, LD)
    b["mean"] = b["var"] = LD(0)
    if tr.deleted:
        return b
    T = t.w.sum()
    dT = dw.sum() + (K - 1) * LD(U) * w_hi.sum()
    D = (dw + t.p1 * dT) / (T - dT) if T > dT else np.full(K, LD(np.inf))
    dp1 = D + LD(U) * (t.p1 + D) + LD(HALF)
    if case["exact"]:
        dp1 = np.zeros(K, LD)
    b["p1"] = dp1
    b["decided"] = np.abs(t.margin) > dp1 if not case["exact"] else np.ones(K, bool)
    kept = tr.keep
    b["prob"] = dp1.copy()
    if not kept.any():
        return b
    Kk = int(kept.sum())
    p2 = np.where(kept, t.p1 / t.p1[kept].sum(), LD(0))
    T2 = t.p1[kept].sum()
    dT2 = dp1[kept].sum() + (Kk - 1) * LD(U) * (t.p1[kept] + dp1[kept]).sum()
    D2 = (dp1 + p2 * dT2) / (T2 - dT2) if T2 > dT2 else np.full(K, LD(np.inf))
    dp2 = np.where(kept, D2 + LD(U) * (p2 + D2) + LD(HALF), LD(0))
    b["prob"] = np.where(kept, dp2, dp1)
    hi = np.where(kept, p2 + dp2, LD(0))
    n = np.cumsum(kept)
    b["cum"] = np.where(kept, np.cumsum(dp2) + np.maximum(n - 1, 0) * LD(U) * np.cumsum(hi), LD(0))
    lam = np.abs(np.asarray(case["lam"], np.float64).astype(LD))
    dmu = (dp2 * lam).sum() + (Kk + 1) * LD(U) * (hi * lam).sum() + Kk * LD(HALF)
    de2 = (dp2 * lam * lam).sum() + (Kk + 2) * LD(U) * (hi * lam * lam).sum() + Kk * LD(HALF)
    mu, e2 = abs(t.mean), t.e2
    b["mean"] = dmu
    b["var"] = de2 + 2 * mu * dmu + dmu * dmu + LD(U) * (mu + dmu) ** 2 + LD(U) * (e2 + de2 + (mu + dmu) ** 2)
    return b


# ---- the checks ------------------------------------------------------------------------------------------------------
def compare(case, tr, b, got, prec="mp"):
    """got = (left, prob, keep, cumulative, (mean, var)) of an implementation -> (failures, worst errors).  failures
    holds ("decision", ...) and ("value", ...) entries.  Values are compared where the implementation's decisions
    equal the truth's (a decision inside its bound may go either way, and then the values differ by design)."""
    left, prob, keep, cum, mv = got
    t = truth_ld(tr, prec)
    keep = np.asarray(keep).astype(bool)
    prob = np.asarray(prob, np.float64)
    fail = []
    # deleted: nothing kept and prob left un-normalised (every particle pruned also leaves nothing kept, but normalised)
    deleted = left == 0 and not keep.any() and abs(float(prob.sum()) - 1.0) > 1e-6
    if b["delete"] is not None and deleted != b["delete"]:
        fail.append(("decision", "deletion %s, truth %s" % (deleted, tr.deleted)))
    if not tr.deleted and not deleted:
        bad = (keep != tr.keep) & b["decided"]
        if bad.any():
            k = int(np.flatnonzero(bad)[0])
            fail.append(("decision", "particle %d kept %s, truth %s (margin %.3e, bound %.3e)"
                         % (k, keep[k], tr.keep[k], float(t.margin[k]), float(b["p1"][k]))))
        elif left != int(keep.sum()):
            fail.append(("decision", "left %d, %d kept" % (left, int(keep.sum()))))
    worst = {}
    if fail or deleted != tr.deleted or (keep != tr.keep).any():
        return fail, worst
    if tr.deleted:
        want_prob = t.w
    elif tr.keep.any():
        want_prob = np.where(tr.keep, t.w / t.w[tr.keep].sum(), t.p1)
    else:
        want_prob = t.p1
    want_cum = np.where(tr.keep, np.cumsum(np.where(tr.keep, want_prob, LD(0))), LD(0))
    checks = [("prob", prob.astype(LD), want_prob, b["prob"]),
              ("cumulative", np.asarray(cum, np.float64).astype(LD), want_cum, b["cum"]),
              ("mean", LD(mv[0]), t.mean, b["mean"]), ("variance", LD(mv[1]), t.var, b["var"])]
    for name, g, want, bound in checks:
        err = np.abs(g - want)
        over = err > bound
        if np.any(over):
            i = int(np.flatnonzero(np.atleast_1d(over))[0])
            fail.append(("value", "%s[%d] off by %.3e, bound %.3e" % (name, i, float(np.atleast_1d(err)[i]),
                                                                      float(np.atleast_1d(bound)[i]))))
        with np.errstate(divide="ignore", invalid="ignore"):
            rel = np.where(bound > 0, err / bound, np.where(err > 0, np.inf, 0))
        worst[name] = max(float(np.max(rel)), 0.0)
    return fail, worst
