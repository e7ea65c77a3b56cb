"""The depth-particle re-weighting (include/sl2b200.h, sl2_measure_particles / sl2_measure_partial_features) from its
definition, in extended precision: the truth that tests/test_particle_truth.py holds the restatements to and
tests/test_gpu_particles.py holds the device to.

It reads exactly the FP64 inputs particle_kernel reads (h, Sinv3 = (S00, S01, S11) of the symmetric S^-1, det S,
lambda, the prior, the integer match z and the found flag of the search, the prune threshold) and follows
monoslam.cpp:1447-1493 and feature_init_info.cpp:95-172 in this order, with exact 2 pi and exact arithmetic:
  likelihood:  nu = z - h, q = nu^T S^-1 nu, (2 pi det S)^-1/2 e^(-q/2), 0 where the match failed; w = prior * it;
  delete:      the reference deletes the feature when the FP64 total is 0.  Exactly, the total of the found particles
               is positive, so the truth's decision is the one FP64 can make: every w rounds to 0 (w <= 2^-1075);
  normalise:   p = w / sum w, cumulative sums in particle order;
  prune:       keep iff p >= fl(threshold / K) (the reference prunes p < thr, strictly; K counts every particle);
  renormalise: over the kept particles (p' = w / sum_kept w), cumulative again, pruned ones 0; nothing when none is
               kept (the reference then keeps the feature with no particles);
  moments:     mean = sum p' lambda, E[lambda^2] = sum p' lambda^2, variance E[lambda^2] - mean^2.
The returned prob follows the device's layout: p' for kept particles, the first normalisation's p for pruned ones,
w itself (un-normalised) when the feature is deleted.

Two precisions run the same code: mpmath at 50 digits (object arrays of mpf) and np.longdouble.  The first is the
definition; the second is fast enough for the GPU shapes and tests/test_particle_truth.py shows the two agree."""
import collections

import mpmath
import numpy as np

DPS = 50

Truth = collections.namedtuple(
    "Truth", "nu q qa e c w deleted thr p1 keep margin prob cumulative mean e2 var left")


class _Num:
    """Conversions and elementary functions of one precision; FP64 inputs convert exactly in both."""

    def __init__(self, prec):
        self.prec = prec
        if prec == "mp":
            self.dtype = object
            self._mpf = np.vectorize(mpmath.mpf, otypes=[object])
            self._sqrt = np.vectorize(mpmath.sqrt, otypes=[object])
            self._exp = np.vectorize(mpmath.exp, otypes=[object])
            self.pi = mpmath.pi
            self.half_tiny = mpmath.mpf(2) ** -1075   # half the subnormal spacing: a w at or below it rounds to 0
        elif prec == "ld":
            self.dtype = np.longdouble
            self.pi = np.longdouble("3.14159265358979323846264338327950288")
            self.half_tiny = np.longdouble(2) ** -1075
        else:
            raise ValueError(prec)

    def __call__(self, a):
        a = np.asarray(a, np.float64)
        return self._mpf(a) if self.prec == "mp" else a.astype(np.longdouble)

    def sqrt(self, a):
        return self._sqrt(a) if self.prec == "mp" else np.sqrt(a)

    def exp(self, a):
        return self._exp(a) if self.prec == "mp" else np.exp(a)

    def f64(self, a):
        """The FP64 rounding of a (mpf -> float is round to nearest)."""
        a = np.asarray(a, dtype=self.dtype)
        if self.prec == "mp":
            return np.array([float(v) for v in a.ravel()], np.float64).reshape(a.shape)
        return a.astype(np.float64)

    def ld(self, a):
        """a in longdouble (what the bounds are computed in)."""
        a = np.asarray(a, dtype=self.dtype)
        if self.prec == "mp":
            return np.array([np.longdouble(mpmath.nstr(v, 25)) for v in a.ravel()], np.longdouble).reshape(a.shape)
        return a


def particle_truth(h, Sinv3, detS, lam, prior, z, found, threshold, prec="mp"):
    """One feature's K particles -> Truth.  Every field is in the precision `prec` (object arrays of mpf or
    longdouble) except: deleted, keep (bool), thr (the FP64 threshold), prob and cumulative (their FP64 roundings),
    left (int).  margin[k] = p1[k] - thr, the distance of the prune decision from its edge."""
    num = _Num(prec)
    h = np.asarray(h, np.float64).reshape(-1, 2)
    Sinv3 = np.asarray(Sinv3, np.float64).reshape(-1, 3)
    K = h.shape[0]
    found = np.asarray(found).astype(bool).reshape(K)
    thr = float(threshold) / float(K) if K else 0.0
    with mpmath.workdps(DPS):
        nu = num(np.asarray(z, np.float64).reshape(K, 2)) - num(h)
        s00, s01, s11 = num(Sinv3[:, 0]), num(Sinv3[:, 1]), num(Sinv3[:, 2])
        n0, n1 = nu[:, 0], nu[:, 1]
        q = s00 * n0 * n0 + 2 * s01 * n0 * n1 + s11 * n1 * n1
        qa = abs(s00) * n0 * n0 + 2 * abs(s01) * abs(n0 * n1) + abs(s11) * n1 * n1
        e = num.exp(-q / 2)
        c = 1 / num.sqrt(2 * num.pi * num(detS))
        w = np.where(found, num(prior) * c * e, num(np.zeros(K)))
        lamx = num(lam)
        deleted = bool((w <= num.half_tiny).all())
        keep = np.zeros(K, bool)
        cum = num(np.zeros(K))
        mean = e2 = var = num(0.0)
        if deleted:
            p1 = num(np.zeros(K))
            margin = num(np.zeros(K))
            prob = w
        else:
            p1 = w / w.sum()
            margin = p1 - num(thr)
            keep = (p1 >= num(thr)).astype(bool)
            prob = p1.copy()
            if keep.any():
                prob[keep] = w[keep] / w[keep].sum()
                cum[keep] = np.cumsum(prob[keep])
                mean = (prob[keep] * lamx[keep]).sum()
                e2 = (prob[keep] * lamx[keep] * lamx[keep]).sum()
                var = e2 - mean * mean
        return Truth(nu, q, qa, e, c, w, deleted, thr, p1, keep, margin, num.f64(prob), num.f64(cum), mean, e2, var,
                     int(keep.sum()))


def truth_ld(truth, prec):
    """The truth's high-precision fields as longdouble (the bounds are computed in longdouble)."""
    num = _Num(prec)
    return truth._replace(**{k: num.ld(getattr(truth, k)) for k in
                             ("nu", "q", "qa", "e", "c", "w", "p1", "margin", "mean", "e2", "var")})
