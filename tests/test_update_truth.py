"""The extended-precision truth of the EKF update (update_truth.py) and the conditioning sweep built on it, on the CPU:
the longdouble update against mpmath at 50 digits, every mechanism at its designed cond(S), and the FP64 Cholesky
yardstick growing like cond(S) eps.  The oracle's explicit-inverse error is printed beside it, not asserted: past
cond(S) ~ 1e5 it exceeds 1e-5 and stops being a reference (DESIGN.md §4)."""
import math
import os

import numpy as np
import pytest

import update_truth as ut

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# FP64 Cholesky yardstick: err <= C64 max(cond(S), 10) eps over the sweep.  Worst measured on the sweep: 905
# (mechanism A at cond 1e4, m = 126: the cancellation P - Y^T Y of the inflated camera block); a factor of ~3.3 left.
C64 = 3000.0
WORST64 = [0.0]


def test_longdouble_has_a_64_bit_mantissa():
    nmant = np.finfo(np.longdouble).nmant
    assert nmant >= 63, ("np.longdouble has a %d-bit mantissa on this platform; the update's truth needs x87 extended "
                         "precision (63 bits) or more" % nmant)


@pytest.mark.parametrize("nf,K", [(5, 3), (16, 8)])
def test_truth_matches_mpmath(oracle, nf, K):
    """The longdouble update against the same sequence at 50 digits, before and after upd_finish's normalisation and
    symmetrisation: within 1e3 eps_ld cond(S)."""
    for mech in ut.MECHANISMS:
        for c in (1e2, 1e6, 1e10):
            case = ut.conditioned_case(np.random.default_rng([nf, K, 7]), nf, K, mech, c)
            args = (case.x, case.P) + ut.rows_of(case)
            k = ut.kalman_ld(*args)
            ex, eP = ut.mp_err(k, *ut.kalman_mp(*args))
            print("\n%s cond %8.2e: longdouble vs 50 digits  x %.2e  P %.2e" % (mech, k.cond, ex, eP), end="")
            assert max(ex, eP) <= 1e3 * ut.EPS_LD * k.cond, (mech, c, ex, eP)
            # and with upd_finish's J P J^T and symmetrisation, on the same J (of x rounded to FP64)
            xo, Po = ut.kalman_mp(*args)
            xf = np.asarray(k.x, np.float64)
            ex, eP = ut.mp_err(k._replace(P=ut.finish(xf, k.P)), xo, ut.finish_mp(xf, Po))
            assert max(ex, eP) <= 1e3 * ut.EPS_LD * k.cond, ("finish", mech, c, ex, eP)


@pytest.mark.parametrize("shape", ut.SWEEP_SHAPES, ids=lambda s: "cap%d_nf%d_K%d" % s)
def test_sweep_reaches_its_conditioning_and_the_yardstick_grows_like_cond(oracle, shape):
    """Every mechanism reaches its designed cond(S) within 10x (measured on the extended-precision S), its posterior
    is a covariance, and the FP64 Cholesky update stays within C64 cond(S) eps of the truth."""
    _, nf, K = shape
    print("\nnf %d K %d (n = %d, m = %d)\nmech  target   cond(S)   FP64 chol  /cond eps   oracle" % (
        nf, K, 13 + 3 * nf, 2 * K), end="")
    for mech in ut.MECHANISMS:
        for c in ut.SWEEP_CONDS:
            case = ut.sweep_case(nf, K, mech, c)
            assert case.P.shape == (13 + 3 * nf,) * 2 and (case.P == case.P.T).all()
            assert len(set(case.feats.tolist())) == K and (np.sort(case.feats) != case.feats).any() or K == 1
            args = (case.x, case.P) + ut.rows_of(case)
            t = ut.truth_update(*args)
            ch = ut.chol64_update(*args)
            e64 = max(ut.update_err(ch.x, ch.P, t.x, t.P))
            eo = max(ut.update_err(*ut.oracle_update(*args), t.x, t.P))
            r = e64 / (max(t.cond, 10.0) * ut.EPS)
            WORST64[0] = max(WORST64[0], r)
            print("\n  %s  %6.0e  %8.2e  %9.2e  %9.2f  %9.2e" % (mech, c, t.cond, e64, r, eo), end="")
            assert c / 10 <= t.cond <= c * 10, (mech, c, t.cond)
            assert (np.diag(t.P) >= 0).all(), (mech, c)
            assert r <= C64, (mech, c, e64, t.cond)
            if mech == "A" and c == ut.A_ZERO_PYY_COND:   # known features: their blocks stay exactly 0
                assert (case.P[13:, :] == 0).all() and (t.P[13:, :] == 0).all()
    print("\nworst FP64 Cholesky error / (cond eps) so far: %.2f" % WORST64[0])


def test_scene_conditioning(oracle):
    """cond(S) of the first update of the default C1, C2 and C4 scenes, where the oracle-parity tests sit on the
    sweep (printed); each is well inside the range where the oracle's explicit inverse is accurate."""
    from gpu_util import oracle_slam_from_scene, synth
    kp = np.load(os.path.join(G, "known_patches.npy"))
    for name, kw in (("C1", dict(known_patches=kp)), ("C2", dict()), ("C4", dict())):
        sc = synth.make_scene(name, n_frames=1, **kw)
        o = oracle_slam_from_scene(oracle, sc)
        o.predict()
        o.select()
        o.measure(sc.frames[0])
        rows = ut.slam_rows(o, sc.cam8)
        assert len(rows[2]) > 0, name
        t = ut.truth_update(*rows)
        print("\n%s: m = %3d  cond(S) = %.2e  NIS = %.2f" % (name, 2 * len(rows[2]), t.cond, t.nis), end="")
        assert t.cond < 1e5, name
        assert math.isfinite(t.logdet)
