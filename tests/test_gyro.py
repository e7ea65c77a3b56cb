"""The gyroscope update on the CPU: the op-for-op restatement (tests/gyro_ref.py) against the extended-precision truth
(tests/gyro_truth.py), constructed cases, broken copies the comparison must catch, and the sl2_stream_gyro layout."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import gyro_ref as gr
import gyro_truth as gt
import scenelib2_b200.lib as mirror

from gyro_truth import bound

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def make_case(rng, n, pww, aniso, cov_scale, resid, R=None, cov_corr=True):
    """A positive definite P of size n whose omega block has eigenvalues pww * (1, sqrt(aniso), aniso), consistent
    cross terms, R_gc (random unless given), a correlated (or diagonal) anisotropic cov and a sample whose residual
    from R_gc omega + b has scale resid."""
    A = rng.standard_normal((n, n)) * 0.1
    Q = Rotation.random(random_state=int(rng.integers(1 << 30))).as_matrix()
    ev = pww * np.array([1.0, aniso ** 0.5, aniso])
    Bn = A[10:13] / np.linalg.norm(A[10:13], axis=1, keepdims=True)
    A[10:13] = Q @ np.diag(np.sqrt(ev)) @ Bn
    P = A @ A.T + np.diag(np.r_[np.full(10, 1e-4), np.zeros(3), np.full(n - 13, 1e-4)])
    P = 0.5 * (P + P.T)
    if R is None:
        R = Rotation.random(random_state=int(rng.integers(1 << 30))).as_matrix()
    Cq = Rotation.random(random_state=int(rng.integers(1 << 30))).as_matrix() if cov_corr else np.eye(3)
    cov = Cq @ np.diag(cov_scale * np.array([1.0, 0.3, 0.05])) @ Cq.T
    cov = 0.5 * (cov + cov.T)
    x = rng.standard_normal(n)
    b = rng.standard_normal(3) * 0.01
    z = R @ x[10:13] + b + rng.standard_normal(3) * resid
    return x, P, R, b, cov, z


CASES = [(n, pww, aniso, ident)
         for n in (13, 16, 313, 781) for pww, aniso in ((1e-12, 1.0), (1e-4, 0.1), (1.0, 1e-4), (1e4, 1e-12))
         for ident in (True, False)]


@pytest.mark.parametrize("n,pww,aniso,ident", CASES)
def test_restatement_within_the_bound_of_the_truth(n, pww, aniso, ident):
    rng = np.random.default_rng(int(n * 7 + np.log10(pww) * 3 + ident + 100))
    worst_cond = 0.0
    for rep in range(2 if n > 300 else 4):
        cov_scale = 1e-12 if pww == 1e4 else 10.0 ** rng.uniform(-12, -3)
        x, P, R, b, cov, z = make_case(rng, n, pww, aniso, cov_scale, 10.0 ** rng.uniform(-4, 0),
                                       R=np.eye(3) if ident else None, cov_corr=rep % 2 == 0)
        xr, Pr, q, st = gr.update(x, P, R, b, cov, z)
        assert st == 1
        tr = gt.update(x, P, R, b, cov, z)
        lim = bound(tr, x, R, b, z)
        e = gt.errors(xr, Pr, q, tr)
        assert max(e) <= lim, (rep, e, lim)
        assert (Pr == Pr.T).all()  # bit-symmetric from a symmetric P
        worst_cond = max(worst_cond, gt.cond(tr[3]))
    if pww == 1e4:
        assert worst_cond > 1e11  # the ill-conditioned end is reached


def test_truth_agrees_with_50_digits():
    """The extended-precision truth is within a hundredth of the restatement's bound of the 50-digit update: a
    yardstick that is far finer than what it measures."""
    rng = np.random.default_rng(50)
    for pww, aniso in ((1.0, 0.1), (1e4, 1e-8)):
        x, P, R, b, cov, z = make_case(rng, 16, pww, aniso, 1e-6, 0.1)
        tr = gt.update(x, P, R, b, cov, z)
        xm, Pm, qm = gt.mp_update(x, P, R, b, cov, z)
        ld = lambda v: np.longdouble(str(v))  # noqa: E731
        e = gt.errors(np.array([ld(xm[i]) for i in range(16)]),
                      np.array([[ld(Pm[i, j]) for j in range(16)] for i in range(16)]), ld(qm), tr)
        assert max(e) <= bound(tr, x, R, b, z) / 100, e


# ---- constructions ---------------------------------------------------------------------------------------------------
def test_zero_q_omega_cross_terms_leave_the_pose_bit_unchanged():
    rng = np.random.default_rng(7)
    x, P, R, b, cov, z = make_case(rng, 40, 1.0, 0.1, 1e-4, 0.5)
    P[0:7, 10:13] = 0.0
    P[10:13, 0:7] = 0.0
    xr, Pr, q, st = gr.update(x, P, R, b, cov, z)
    assert st == 1 and q > 0
    assert xr[0:7].tobytes() == x[0:7].tobytes()
    assert Pr[0:7, 0:7].tobytes() == np.ascontiguousarray(P[0:7, 0:7]).tobytes()
    assert not np.array_equal(xr[10:13], x[10:13])


def test_a_huge_covariance_changes_almost_nothing():
    rng = np.random.default_rng(8)
    x, P, R, b, cov, z = make_case(rng, 40, 1.0, 0.1, 1e-4, 0.5)
    xr, Pr, q, st = gr.update(x, P, R, b, cov * 1e24, z)
    assert st == 1
    assert np.abs(xr - x).max() <= 1e-14 * np.abs(x).max()
    assert np.abs(Pr - P).max() <= 1e-14 * np.abs(P).max()


@pytest.mark.parametrize("how", ["negative", "nan", "inf_rate"])
def test_a_non_positive_definite_s_is_skipped(how):
    rng = np.random.default_rng(9)
    x, P, R, b, cov, z = make_case(rng, 20, 1.0, 0.1, 1e-4, 0.5)
    if how == "negative":
        P[11, 11] = -1.0
    elif how == "nan":
        P[12, 10] = P[10, 12] = np.nan
    else:
        z = np.array([np.inf, 0.0, 0.0])
    xr, Pr, q, st = gr.update(x, P, R, b, cov, z)
    assert st == 2 and q == 0.0
    assert xr.tobytes() == x.tobytes() and Pr.tobytes() == P.tobytes()


# ---- broken copies the truth comparison catches --------------------------------------------------------------------
@pytest.mark.parametrize("broken", [dict(transpose_R=True), dict(flip_bias=True), dict(bad_W=True),
                                    dict(nis_terms=2)], ids=["R_transposed", "bias_flipped", "W_from_updated_P",
                                                             "missing_nis_term"])
def test_broken_copies_are_caught(broken):
    rng = np.random.default_rng(11)
    x, P, R, b, cov, z = make_case(rng, 40, 1.0, 0.1, 1e-4, 0.5)
    b = b + 0.05
    tr = gt.update(x, P, R, b, cov, z)
    assert max(gt.errors(*gr.update(x, P, R, b, cov, z)[:3], tr)) <= bound(tr, x, R, b, z)
    assert max(gt.errors(*gr.update(x, P, R, b, cov, z, **broken)[:3], tr)) > 1e6 * bound(tr, x, R, b, z)


# ---- ABI -------------------------------------------------------------------------------------------------------------
def test_gyro_struct_matches_header(tmp_path):
    """sizeof and every field's offset and size of sl2_stream_gyro, as the host C compiler lays it out from the
    header, equal the ctypes mirror's."""
    M = mirror.Sl2StreamGyro
    fields = [f for f, _ in M._fields_]
    assert fields == ["on", "reserved", "R_gc", "bias", "cov"]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "sl2b200.h"', "int main(void) {",
             '  printf("sizeof %zu\\n", sizeof(sl2_stream_gyro));']
    lines += ['  printf("%s %%zu %%zu\\n", offsetof(sl2_stream_gyro, %s), sizeof(((sl2_stream_gyro *)0)->%s));'
              % (f, f, f) for f in fields]
    src, exe = tmp_path / "gyro_layout.c", tmp_path / "gyro_layout"
    src.write_text("\n".join(lines + ["  return 0;", "}"]) + "\n")
    subprocess.check_call([os.environ.get("CC", "cc"), "-std=c99", "-I", os.path.join(ROOT, "include"), "-o", str(exe),
                           str(src)])
    out = {ln.split()[0]: tuple(int(v) for v in ln.split()[1:])
           for ln in subprocess.check_output([str(exe)], text=True).splitlines()}
    assert out["sizeof"] == (C.sizeof(M),) == (176,)
    for f, t in M._fields_:
        assert out[f] == (getattr(M, f).offset, C.sizeof(t)), f
    for name in ("sl2_set_stream_gyro", "sl2_get_stream_gyro", "sl2_set_gyro_samples", "sl2_gyro_update",
                 "sl2_get_gyro_results"):
        assert name in mirror.EXPORTS
