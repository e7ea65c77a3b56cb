"""The two restatements of the depth-particle re-weighting (particle_ref.update in Python floats,
oracle.particle_update in C++) against the re-weighting from its definition in extended precision (particle_truth):
every value within a bound derived from the operation count, and the decisions (deletion, the kept set) equal the
truth's wherever the truth's margin lies outside that bound.  The cases are constructed knife edges (a probability
exactly at fl(threshold / K), all particles pruned, threshold 0, clustered lambda, subnormal and vanishing
likelihoods, failed matches) and random ones.  Deliberately broken copies of the restatement must fail the checks."""
import functools
import math

import numpy as np
import pytest

import particle_ref
from oracle import pyoracle as po
from particle_cases import (LD, bounds, compare, dyadic_probabilities, exact_case, sinv_random, threshold_cases)
from particle_truth import particle_truth, truth_ld

_MEAN_VAR = particle_ref.mean_var
KEYS = ("h", "Sinv3", "detS", "lam", "prior", "z", "found", "threshold")   # particle_truth's arguments
ORC = ("h", "Sinv3", "detS", "lam", "z", "found", "threshold", "prior")    # oracle.particle_update's, particle_ref's


def _ints(rng, K):
    return rng.integers(20, 300, (K, 2)).astype(np.int32)


def q_case(rng, K, qs, found=None, prior=None, threshold=0.05, lam=None, Sinv3=None):
    """Particles at chosen Mahalanobis distances q_k = nu^T S^-1 nu (nu along a random direction; h = z - nu rounds,
    so q is close to, not exactly, the target); det S = 1 / det S^-1."""
    z = _ints(rng, K)
    Sinv3 = sinv_random(rng, K) if Sinv3 is None else Sinv3
    ang = rng.uniform(0, 2 * np.pi, K)
    d = np.column_stack([np.cos(ang), np.sin(ang)])
    dSd = Sinv3[:, 0] * d[:, 0] ** 2 + 2 * Sinv3[:, 1] * d[:, 0] * d[:, 1] + Sinv3[:, 2] * d[:, 1] ** 2
    nu = d * np.sqrt(np.asarray(qs, np.float64) / dSd)[:, None]
    if prior is None:
        prior = rng.uniform(0.2, 1.0, K)
        prior /= prior.sum()
    return dict(h=z - nu, Sinv3=Sinv3, detS=1.0 / (Sinv3[:, 0] * Sinv3[:, 2] - Sinv3[:, 1] ** 2),
                lam=np.linspace(0.5, 5.0, K) if lam is None else np.asarray(lam, np.float64),
                prior=np.asarray(prior, np.float64), z=z,
                found=np.ones(K, np.uint8) if found is None else np.asarray(found, np.uint8),
                threshold=float(threshold), exact=False)


def _negative_variance(p):
    """An equal lambda for all the particles of probabilities p whose one-pass variance E[lambda^2] - mean^2 comes out
    below 0 in FP64 (the exact variance is 0)."""
    for i in range(1000):
        lam = 2.3 + 0.01 * i
        if particle_ref.mean_var(list(p), [1] * len(p), [lam] * len(p))[1] < 0:
            return lam
    raise AssertionError("no lambda with a negative one-pass variance")


@functools.lru_cache(maxsize=None)
def cases():
    """[(name, case)]"""
    rng = np.random.default_rng(2024)
    out = []
    for K in (4, 128, 256):
        out += [(name, c) for name, c, _, _ in threshold_cases(rng, K)]
    K = 64
    f = np.ones(K)
    f[rng.permutation(K)[:7]] = 0
    p = np.zeros(K)
    p[f > 0] = dyadic_probabilities(rng, int(f.sum()), zeros=9)   # zero priors, and failed matches
    out.append(("threshold-0", exact_case(p, _ints(rng, K), f, np.linspace(1, 3, K), 0.0)))
    out.append(("all-pruned", exact_case(np.full(128, 2.0 ** -7), _ints(rng, 128), np.ones(128),
                                         np.linspace(1, 3, 128), 2.0)))
    out.append(("unnormalised-prior", exact_case(dyadic_probabilities(rng, 50, zeros=6), _ints(rng, 50), np.ones(50),
                                                 np.linspace(0.3, 7, 50), 0.3, scale=96.0)))
    out.append(("tiny-prior-scale", exact_case(dyadic_probabilities(rng, 40), _ints(rng, 40), np.ones(40),
                                               np.linspace(0.3, 7, 40), 0.5, scale=2.0 ** -900)))
    t = rng.integers(-3, 9, 64)    # det S over 4^12 ~ 7 decades; exact on FP64, not in the truth (c_k differ by ~u)
    out.append(("detS-decades", exact_case(dyadic_probabilities(rng, 64), _ints(rng, 64), np.ones(64),
                                           np.linspace(0.4, 6, 64), 0.8, t=t, exact=False)))
    out.append(("lambda-clustered", exact_case(dyadic_probabilities(rng, 100), _ints(rng, 100), np.ones(100),
                                               1.7 * (1 + 1e-7 * rng.uniform(-1, 1, 100)), 0.05)))
    p = dyadic_probabilities(rng, 33)
    out.append(("lambda-equal", exact_case(p, _ints(rng, 33), np.ones(33), np.full(33, _negative_variance(p)), 0.05)))
    # general nu
    out.append(("q-general-detS-decades", q_case(rng, 60, rng.uniform(0, 12, 60), threshold=0.8,
                                                 Sinv3=sinv_random(rng, 60, 0.05, 40.0))))
    out.append(("lambda-clustered-general", q_case(rng, 90, rng.uniform(0, 9, 90),
                                                   lam=3.1 * (1 + 1e-7 * rng.uniform(-1, 1, 90)))))
    qs = rng.uniform(0, 9, 40)
    qs[::3] = rng.uniform(1425, 1470, len(qs[::3]))
    out.append(("some-subnormal", q_case(rng, 40, qs, threshold=1e-30)))
    out.append(("all-subnormal", q_case(rng, 24, rng.uniform(1415, 1460, 24))))
    out.append(("all-vanish", q_case(rng, 16, rng.uniform(1500, 1600, 16))))
    found = (rng.random(48) < 0.5).astype(np.uint8)
    out.append(("failed-and-found", q_case(rng, 48, rng.uniform(0, 9, 48), found=found, threshold=0.9)))
    out.append(("all-failed", q_case(rng, 12, rng.uniform(0, 9, 12), found=np.zeros(12))))
    out.append(("far-normal", q_case(rng, 30, rng.uniform(300, 1300, 30), threshold=0.3)))
    for i in range(18):       # random
        K = int(rng.choice([1, 2, 3, 7, 16, 31, 33, 64, 100, 127, 129, 256]))
        qs = rng.exponential(2.0, K) * rng.choice([1.0, 5.0])
        found = (rng.random(K) < rng.choice([1.0, 0.8, 0.5])).astype(np.uint8)
        prior = rng.uniform(0.0, 1.0, K) * rng.choice([1.0, 1e-3, 40.0])
        prior[rng.random(K) < 0.1] = 0.0
        out.append(("random-%d-K%d" % (i, K),
                    q_case(rng, K, qs, found=found, prior=prior,
                           threshold=float(rng.choice([0.05, 0.3, 0.8, 1.0, 1.5])),
                           lam=rng.uniform(0.3, 8.0, K), Sinv3=sinv_random(rng, K, 0.3, 20.0))))
    return out


def _args(case):
    return [case[k] for k in KEYS]


def _impl_args(case):
    return [case[k] for k in ORC]


@functools.lru_cache(maxsize=None)
def truths(prec="mp"):
    return [particle_truth(*_args(c), prec=prec) for _, c in cases()]


def test_truth_precisions_agree():
    """The mpmath truth (50 digits) is the definition; the longdouble one, which the GPU tests use, must give the same
    decisions, and values within what longdouble's 64-bit significand allows: the exponent -q/2 carries a relative
    error of a few 2^-64 into e^(-q/2), so per case |ld - mp| <= 2^-64 (16 + 4 max qa) relative (the variance relative
    to E[lambda^2]).  That is at least 2^11 times tighter than the FP64 bounds the truth is used with."""
    worst = {}
    for (name, c), tm in zip(cases(), truths("mp")):
        tl = particle_truth(*_args(c), prec="ld")
        assert tl.deleted == tm.deleted and (tl.keep == tm.keep).all(), name
        m = truth_ld(tm, "mp")
        allowed = LD(2.0 ** -64) * (16 + 4 * (m.qa.max() if len(m.qa) else 0))
        for key, scale in (("w", m.w), ("p1", m.p1), ("mean", m.mean), ("var", m.e2)):
            a, r = np.asarray(getattr(m, key), LD), np.asarray(getattr(tl, key), LD)
            s = np.abs(np.asarray(scale, LD))
            with np.errstate(divide="ignore", invalid="ignore"):
                rel = np.where(s != 0, np.abs(a - r) / s, np.where(a == r, LD(0), LD(np.inf)))
            assert (rel <= allowed).all(), (name, key, float(rel.max()), float(allowed))
            worst[key] = max(worst.get(key, 0.0), float(np.max(rel)) if rel.size else 0.0)
    print("longdouble vs mpmath truth over %d cases, worst relative difference: %s (variance relative to E[lambda^2])"
          % (len(cases()), {k: "%.2e" % v for k, v in worst.items()}))


def test_constructions_hold():
    """The exact cases are what they claim: the truth's normalised probabilities are FP64 numbers, and the threshold
    cases put fl(threshold / K) exactly on p_j (kept) or one double above the threshold (pruned)."""
    rng = np.random.default_rng(2024)
    for K in (4, 128, 256):
        for name, c, j, kept in threshold_cases(rng, K):
            tr = particle_truth(*_args(c), prec="mp")
            m = truth_ld(tr, "mp")
            assert (m.p1 == np.asarray(m.p1, np.float64).astype(LD)).all(), name
            assert bool(tr.keep[j]) == kept, name
            assert (tr.thr == float(m.p1[j])) == kept, name
    for (name, c), tr in zip(cases(), truths()):
        if c["exact"] and not tr.deleted:
            m = truth_ld(tr, "mp")
            assert (m.p1 == np.asarray(m.p1, np.float64).astype(LD)).all(), name
    names = {n: tr for (n, _), tr in zip(cases(), truths())}
    assert names["all-pruned"].left == 0 and not names["all-pruned"].deleted
    eq = dict(cases())["lambda-equal"]
    assert po.particle_update(*_impl_args(eq))[4][1] < 0.0      # the oracle's variance too
    assert names["all-vanish"].deleted and names["all-failed"].deleted
    sub = names["all-subnormal"]
    assert not sub.deleted and (np.asarray(truth_ld(sub, "mp").w, LD) < LD(2.0 ** -1022)).all()


def test_restatement_equals_oracle_bit_for_bit():
    for name, c in cases():
        a, o = particle_ref.update(*_impl_args(c)), po.particle_update(*_impl_args(c))
        assert a[0] == o[0], name
        for x, y, what in zip(a[1:], o[1:], ("prob", "keep", "cumulative", "mean_var")):
            assert np.asarray(x).tobytes() == np.asarray(y).tobytes(), (name, what)


@pytest.mark.parametrize("which", ["restated", "oracle"])
def test_values_and_decisions_equal_the_truth(which):
    impl = particle_ref.update if which == "restated" else po.particle_update
    worst, undecided, pruned, deleted = {}, [], 0, 0
    for (name, c), tr in zip(cases(), truths()):
        b = bounds(c, tr)
        fail, w = compare(c, tr, b, impl(*_impl_args(c)))
        assert not fail, (name, fail)
        for k, v in w.items():
            worst[k] = max(worst.get(k, 0.0), v)
        if not tr.deleted and not b["decided"].all():
            undecided.append(name)
        pruned += int((~tr.keep).sum()) if not tr.deleted else 0
        deleted += tr.deleted
    print("%s: worst error / bound over %d cases: %s; cases with a prune decision inside its bound: %s"
          % (which, len(cases()), {k: "%.2e" % v for k, v in worst.items()}, undecided))
    assert pruned > 0 and deleted >= 2 and len(undecided) <= 3, undecided


# ---- the checks can see ----------------------------------------------------------------------------------------------
def _likelihood_no_coefficient(z, h, s, det, exp=math.exp):
    nu0, nu1 = float(z[0]) - h[0], float(z[1]) - h[1]
    q = nu0 * (s[0] * nu0 + s[1] * nu1) + nu1 * (s[1] * nu0 + s[2] * nu1)
    return exp(-0.5 * q)


def _likelihood_off_diagonal(sign, one_row):
    def f(z, h, s, det, exp=math.exp):
        nu0, nu1 = float(z[0]) - h[0], float(z[1]) - h[1]
        r0 = s[0] * nu0 + sign * s[1] * nu1
        r1 = (0.0 if one_row else sign * s[1] * nu0) + s[2] * nu1
        q = nu0 * r0 + nu1 * r1
        return (1.0 / math.sqrt(particle_ref.TWO_PI * det)) * exp(-0.5 * q)
    return f


def _renormalise_over_all(prob, keep, cumulative):
    total = 0.0
    for p in prob:
        total = total + p
    cum = 0.0
    for k in range(len(prob)):
        if keep[k]:
            prob[k] = prob[k] / total
            cumulative[k] = cum + prob[k]
            cum = cum + prob[k]
    return True


def _prune_keeping_cumulative(prob, keep, cumulative, thr):
    left = 0
    for k in range(len(prob)):
        if particle_ref.pruned(prob[k], thr):
            keep[k] = 0
        else:
            left += 1
    return left


def _mean_var_two_pass(prob, keep, lam):
    mean = 0.0
    for k in range(len(prob)):
        if keep[k]:
            mean = mean + prob[k] * lam[k]
    var = 0.0
    for k in range(len(prob)):
        if keep[k]:
            var = var + prob[k] * ((lam[k] - mean) * (lam[k] - mean))
    return mean, var


def _mean_var_clamped(prob, keep, lam):
    mean, var = _MEAN_VAR(prob, keep, lam)
    return mean, max(var, 0.0)


def _normalise_dbl_min(prob, keep, cumulative):
    total = 0.0
    for k in range(len(prob)):
        if keep[k]:
            total = total + prob[k]
    if total < 2.2250738585072014e-308:
        return False
    cum = 0.0
    for k in range(len(prob)):
        if keep[k]:
            prob[k] = prob[k] / total
            cumulative[k] = cum + prob[k]
            cum = cum + prob[k]
    return True


MUTATIONS = {
    "prune-at-equality": ("pruned", lambda p, thr: p <= thr),
    "threshold-over-found": ("threshold", lambda prune, prob, found: prune / float(int(np.sum(found)) or 1)),
    "threshold-over-nonzero": ("threshold", lambda prune, prob, found: prune / float(sum(p > 0 for p in prob) or 1)),
    "renormalise-over-all": ("renormalise", _renormalise_over_all),
    "pruned-keep-cumulative": ("prune", _prune_keeping_cumulative),
    "variance-two-pass": ("mean_var", _mean_var_two_pass),
    "variance-clamped": ("mean_var", _mean_var_clamped),
    "no-gaussian-coefficient": ("likelihood", _likelihood_no_coefficient),
    "off-diagonal-sign": ("likelihood", _likelihood_off_diagonal(-1.0, False)),
    "off-diagonal-one-row": ("likelihood", _likelihood_off_diagonal(1.0, True)),
    "total-below-dbl-min": ("normalise", _normalise_dbl_min),
}


@pytest.mark.parametrize("mutation", sorted(MUTATIONS))
def test_mutations_are_caught(mutation, monkeypatch):
    """Each broken copy of the restatement fails at least one check: a decision or a value against the truth, or the
    bit-for-bit comparison with the oracle."""
    attr, fn = MUTATIONS[mutation]
    if attr == "normalise":   # both normalisations, like the one function the kernel calls twice
        monkeypatch.setattr(particle_ref, "renormalise", fn)
    monkeypatch.setattr(particle_ref, attr, fn)
    caught = {}
    for (name, c), tr in zip(cases(), truths()):
        got = particle_ref.update(*_impl_args(c))
        kinds = {f[0] for f in compare(c, tr, bounds(c, tr), got)[0]}
        o = po.particle_update(*_impl_args(c))
        if got[0] != o[0] or any(np.asarray(x).tobytes() != np.asarray(y).tobytes() for x, y in zip(got[1:], o[1:])):
            kinds.add("oracle-bits")
        for k in sorted(kinds):
            caught.setdefault(k, []).append(name)
    print("%s: %s" % (mutation, {k: "%d cases, first %s" % (len(v), v[0]) for k, v in sorted(caught.items())}))
    assert caught
    if mutation not in ("variance-two-pass", "variance-clamped"):
        assert set(caught) - {"oracle-bits"}, "only the oracle comparison sees %s" % mutation
