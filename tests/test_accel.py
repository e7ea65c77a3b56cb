"""The accelerometer's motion prediction on the CPU: the op-for-op restatement (tests/accel_ref.py) against the
extended-precision truth (tests/accel_truth.py), D against central differences, the reference's control form, skipped
samples, broken copies the comparison must catch, and the sl2_stream_accel layout."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import accel_ref as ar
import accel_truth as at
import scenelib2_b200.lib as mirror

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPS = at.OPS


def make_case(rng, n, cond, unit_q=True):
    """A state of size n with a rotated q (unit or not), a P whose eigenvalues spread over `cond`, a setting with its
    own R_ac, bias, correlated cov, gravity along a world axis and sd_a, and a sample of a few g."""
    x = np.zeros(n)
    x[:3] = rng.normal(0, 0.5, 3)
    q = Rotation.random(random_state=int(rng.integers(1 << 30))).as_quat()[[3, 0, 1, 2]]
    x[3:7] = q if unit_q else q * rng.uniform(0.9, 1.1)
    x[7:10] = rng.normal(0, 0.3, 3)
    x[10:13] = rng.normal(0, 0.5, 3)
    x[13:] = rng.normal(0, 1.0, n - 13)
    Qr = np.linalg.qr(rng.standard_normal((n, n)))[0]
    P = (Qr * np.logspace(0, -np.log10(cond), n)) @ Qr.T * 1e-2
    P = 0.5 * (P + P.T)
    R = Rotation.random(random_state=int(rng.integers(1 << 30))).as_matrix()
    Cq = Rotation.random(random_state=int(rng.integers(1 << 30))).as_matrix()
    cov = Cq @ np.diag(10.0 ** rng.uniform(-4, 0) * np.array([1.0, 0.4, 0.1])) @ Cq.T
    cov = 0.5 * (cov + cov.T)
    setting = dict(R_ac=R, bias=rng.normal(0, 0.05, 3), cov=cov, gravity=np.array([0.0, 0.0, -9.81]),
                   sd_a=float(rng.uniform(0.0, 2.0)))
    f = rng.normal(0, 15.0, 3)
    return x, P, setting, f


def compare(x, P, dt, setting, f, **broken):
    sk = ar.reference_skeleton(x[:13], dt)
    xr, Pr, a, st = ar.predict(x, P, dt, setting, f, sk, **broken)
    tr = at.predict(x, P, dt, setting, f, sk)
    return st, at.errors(xr, Pr, x, P, dt, setting, f, tr)


CASES = [(n, cond, unit) for n in (13, 16, 313, 781) for cond in (1.0, 1e8, 1e14) for unit in (True, False)]


@pytest.mark.parametrize("n,cond,unit", CASES)
def test_restatement_within_the_bound_of_the_truth(n, cond, unit):
    rng = np.random.default_rng(int(n * 3 + np.log10(cond) + unit))
    for rep in range(1 if n > 300 else 3):
        x, P, setting, f = make_case(rng, n, cond, unit)
        dt = [1 / 30.0, 0.05, 0.01][rep % 3]
        st, (ex, eP) = compare(x, P, dt, setting, f)
        assert st == 1
        assert ex <= OPS and eP <= OPS, (rep, ex, eP)


def test_truth_agrees_with_50_digits():
    """The extended-precision truth is within a hundredth of the restatement's bound of the 50-digit prediction."""
    rng = np.random.default_rng(50)
    for cond, unit in ((1.0, True), (1e10, False)):
        x, P, setting, f = make_case(rng, 16, cond, unit)
        sk = ar.reference_skeleton(x[:13], 1 / 30.0)
        tr = at.predict(x, P, 1 / 30.0, setting, f, sk)
        xm, Pm = at.mp_predict(x, P, 1 / 30.0, setting, f, sk)
        ld = lambda v: np.longdouble(str(v))  # noqa: E731
        xs = np.array([ld(xm[i]) for i in range(16)])
        Ps = np.array([[ld(Pm[i, j]) for j in range(16)] for i in range(16)])
        sx, SP = at.scales(x, P, 1 / 30.0, setting, f, tr)
        u = float(np.finfo(np.float64).eps)
        assert (np.abs((xs - tr[0]).astype(np.float64)) / (sx + 1e-300)).max() <= OPS * u / 100
        assert (np.abs((Ps - tr[1]).astype(np.float64)) / (SP + 1e-300)).max() <= OPS * u / 100


def test_D_against_central_differences():
    """D is the reference's dRq_times_a_by_dq: the derivative of the homogeneous form Rh(q) f_c = R(q) f_c +
    (|q|^2 - 1) f_c, so it equals central differences of Rh(q) f_c in every coordinate, and of R(q) f_c itself along
    every direction tangent to |q| = 1 (where the update's normalisation keeps q)."""
    rng = np.random.default_rng(3)
    for unit in (True, False):
        x, P, setting, f = make_case(rng, 13, 1.0, unit)
        q = x[3:7]
        fc = np.asarray(setting["R_ac"]).T @ (f - setting["bias"])
        D = np.array(ar.dRq_times_a_by_dq(q, list(fc)))
        Rv = lambda p: np.array(ar.quat_to_R(*p)) @ fc  # noqa: E731
        h, tol = 1e-6, 1e-7 * max(1.0, np.abs(fc).max())
        for k in range(4):
            e = np.eye(4)[k] * h
            fd = (Rv(q + e) + ((q + e) @ (q + e) - 1) * fc - Rv(q - e) - ((q - e) @ (q - e) - 1) * fc) / (2 * h)
            assert np.abs(fd - D[:, k]).max() <= tol, k
        if unit:
            for _ in range(4):
                t = rng.standard_normal(4)
                t -= (t @ q) * q
                t *= h / np.linalg.norm(t)
                assert np.abs((Rv(q + t) - Rv(q - t)) / (2 * h) - D @ t / h).max() <= tol


def test_a_sample_at_the_bias_is_the_reference_control_form_with_gravity():
    """f = b, cov -> 0 and sd_a = 4: f_c = 0 exactly, so D = 0 and a = g; the prediction is the reference's with u = g
    plus the 1/2 g dt^2 term in r, and its Q the reference's within rounding."""
    rng = np.random.default_rng(4)
    x, P, setting, _ = make_case(rng, 40, 1e4)
    setting.update(cov=np.eye(3) * 1e-40, sd_a=4.0, gravity=np.array([0.3, -9.7, 1.2]))
    dt = 1 / 30.0
    xr, Pr, a, st = ar.predict(x, P, dt, setting, setting["bias"])
    assert st == 1 and a == list(setting["gravity"])
    fv, F, Gn = ar.reference_skeleton(x[:13], dt, u=setting["gravity"])
    want_x = x.copy()
    want_x[:13] = fv
    want_x[:3] = fv[:3] + setting["gravity"] * ((0.5 * dt) * dt)
    assert xr.tobytes() == want_x.tobytes()
    want_P, _ = ar.covariance_passes(P, F, Gn, dt)
    u = float(np.finfo(np.float64).eps)
    scale = np.abs(F) @ np.abs(P[:13, :13]) @ np.abs(F).T
    assert (np.abs(Pr[:13, :13] - want_P[:13, :13]) <= 4 * u * scale).all()
    assert Pr[:13, 13:].tobytes() == want_P[:13, 13:].tobytes()


@pytest.mark.parametrize("how", ["huge_force", "nan_q"])
def test_a_non_finite_prediction_is_skipped_as_the_reference(how):
    rng = np.random.default_rng(5)
    x, P, setting, f = make_case(rng, 25, 1e2)
    if how == "huge_force":
        f = np.array([1.7e308, 1.7e308, -1.7e308])
        setting["bias"] = -f * 0.5  # f - b overflows
    else:
        x[5] = np.nan
    xr, Pr, a, st = ar.predict(x, P, 1 / 30.0, setting, f)
    assert st == 2 and a == [0.0] * 3
    xo, Po, _, so = ar.predict(x, P, 1 / 30.0, setting, None)
    assert so == 0
    assert xr.tobytes() == xo.tobytes() and Pr.tobytes() == Po.tobytes()


@pytest.mark.parametrize("broken", [dict(transpose_R=True), dict(flip_gravity=True), dict(drop_half=True),
                                    dict(dqbar=True)],
                         ids=["R_ac_transposed", "gravity_flipped", "half_term_dropped", "D_with_dqbar"])
def test_broken_copies_are_caught(broken):
    rng = np.random.default_rng(11)
    x, P, setting, f = make_case(rng, 40, 1e4)
    st, e = compare(x, P, 1 / 30.0, setting, f)
    assert max(e) <= OPS
    st, e = compare(x, P, 1 / 30.0, setting, f, **broken)
    assert max(e) > 1e6 * OPS, e


def test_accel_struct_matches_header(tmp_path):
    """sizeof and every field's offset and size of sl2_stream_accel, as the host C compiler lays it out from the
    header, equal the ctypes mirror's."""
    M = mirror.Sl2StreamAccel
    fields = [f for f, _ in M._fields_]
    assert fields == ["on", "reserved", "R_ac", "bias", "cov", "gravity", "sd_a"]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "sl2b200.h"', "int main(void) {",
             '  printf("sizeof %zu\\n", sizeof(sl2_stream_accel));']
    lines += ['  printf("%s %%zu %%zu\\n", offsetof(sl2_stream_accel, %s), sizeof(((sl2_stream_accel *)0)->%s));'
              % (f, f, f) for f in fields]
    src, exe = tmp_path / "accel_layout.c", tmp_path / "accel_layout"
    src.write_text("\n".join(lines + ["  return 0;", "}"]) + "\n")
    subprocess.check_call([os.environ.get("CC", "cc"), "-std=c99", "-I", os.path.join(ROOT, "include"), "-o", str(exe),
                           str(src)])
    out = {ln.split()[0]: tuple(int(v) for v in ln.split()[1:])
           for ln in subprocess.check_output([str(exe)], text=True).splitlines()}
    assert out["sizeof"] == (C.sizeof(M),) == (208,)
    for f, t in M._fields_:
        assert out[f] == (getattr(M, f).offset, C.sizeof(t)), f
    for name in ("sl2_set_stream_accel", "sl2_get_stream_accel", "sl2_set_accel_samples", "sl2_accel_predict",
                 "sl2_get_accel_results"):
        assert name in mirror.EXPORTS
