"""The depth-particle re-weighting restated in particle_kernel's operation order (particles.cu), in Python floats:
every operation rounded on its own (never fused), every sum serial in particle order, glibc's exp unless another is
passed in.  On the CPU it equals oracle.particle_update bit for bit (tests/test_particle_truth.py).  The steps are
separate functions so that the mutation checks can replace one at a time."""
import math

import numpy as np

TWO_PI = 6.283185307179586476925286766559   # fl(2 pi), the constant particle_kernel and the reference multiply by


def likelihood(z, h, s, det, exp=math.exp):
    """monoslam.cpp:1456-1478 for one found particle: z (2 ints), h (2), s = (S00, S01, S11) of S^-1, det S."""
    nu0, nu1 = float(z[0]) - h[0], float(z[1]) - h[1]
    r0 = s[0] * nu0 + s[1] * nu1
    r1 = s[1] * nu0 + s[2] * nu1
    q = nu0 * r0 + nu1 * r1
    return (1.0 / math.sqrt(TWO_PI * det)) * exp(-0.5 * q)


def normalise(prob, keep, cumulative):
    """feature_init_info.cpp:95-119 over the kept particles; False when their total is 0."""
    total = 0.0
    for k in range(len(prob)):
        if keep[k]:
            total = total + prob[k]
    if total == 0.0:
        return False
    cum = 0.0
    for k in range(len(prob)):
        if keep[k]:
            prob[k] = prob[k] / total
            cumulative[k] = cum + prob[k]
            cum = cum + prob[k]
    return True


def renormalise(prob, keep, cumulative):
    """prune_particle_vector's closing normalisation (feature_init_info.cpp:140)."""
    return normalise(prob, keep, cumulative)


def threshold(prune, prob, found):
    """feature_init_info.cpp:128: the threshold over the particle count before pruning."""
    return prune / float(len(prob))


def pruned(p, thr):
    return p < thr


def prune(prob, keep, cumulative, thr):
    """feature_init_info.cpp:126-139 -> the number kept."""
    left = 0
    for k in range(len(prob)):
        if pruned(prob[k], thr):
            keep[k] = 0
            cumulative[k] = 0.0
        else:
            left += 1
    return left


def mean_var(prob, keep, lam):
    """feature_init_info.cpp:152-172, scalar lambda."""
    mean = e2 = 0.0
    for k in range(len(prob)):
        if keep[k]:
            mean = mean + prob[k] * lam[k]
            e2 = e2 + prob[k] * (lam[k] * lam[k])
    return mean, e2 - mean * mean


def exp_argument(z, h, s):
    """-0.5 q of likelihood(), the argument its exp is evaluated at."""
    nu0, nu1 = float(z[0]) - h[0], float(z[1]) - h[1]
    return -0.5 * (nu0 * (s[0] * nu0 + s[1] * nu1) + nu1 * (s[1] * nu0 + s[2] * nu1))


def update(h, Sinv3, detS, lam, z, found, prune_threshold, prior, exp=math.exp):
    """One feature -> left, prob, keep, cumulative, (mean, variance): oracle.particle_update's outputs.  `exp` is
    glibc's by default; the GPU tests pass the device's, measured on the same arguments."""
    h = np.asarray(h, np.float64).reshape(-1, 2)
    Sinv3 = np.asarray(Sinv3, np.float64).reshape(-1, 3)
    z = np.asarray(z).reshape(-1, 2)
    K = h.shape[0]
    prob = [float(p) for p in prior]
    keep = [1] * K
    cumulative = [0.0] * K
    for k in range(K):
        lk = likelihood(z[k], (float(h[k, 0]), float(h[k, 1])), [float(v) for v in Sinv3[k]],
                        float(detS[k]), exp) if found[k] else 0.0
        prob[k] = prob[k] * lk
    mv = (0.0, 0.0)
    if not normalise(prob, keep, cumulative):
        left, keep = 0, [0] * K
    else:
        left = prune(prob, keep, cumulative, threshold(float(prune_threshold), prob, found))
        renormalise(prob, keep, cumulative)
        mv = mean_var(prob, keep, [float(v) for v in lam])
    return (left, np.array(prob), np.array(keep, np.uint8), np.array(cumulative), np.array(mv))
