"""CPU checks of the stream recovery (include/sl2b200.h, sl2_set_stream_recovery): the decision rule's restatement
(tests/recovery_ref.py) at its edges, broken copies of it each caught by a named check, the layout of the new structs
against the header, and the argument check that sl2_relocalise and sl2_set_stream_recovery share."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import recovery_ref as rv
import scenelib2_b200.lib as mirror

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def tries(out):
    return [t for t, (_, tried, _) in enumerate(out) if tried]


# ---- named checks: each holds the restatement (or a broken copy of it) to one edge of the rule -----------------------
def check_lost_after_one(broken=()):
    """lost_after = 1: the first failed step declares the stream lost and tries on that same step."""
    cfg = dict(lost_after=1, min_matches=5, retry_period=1)
    out = rv.run(cfg, [9, 9, 4, 9, 9], broken=broken)
    assert [s["lost"] for s, _, _ in out] == [0, 0, 1, 1, 1]
    assert tries(out) == [2, 3, 4]  # retry_period = 1: every lost step tries
    assert [sel for _, _, sel in out] == [True, True, True, False, False]
    assert out[2][0]["failed_steps"] == 1 and out[2][0]["lost_steps"] == 0
    assert [s["lost_steps"] for s, _, _ in out[2:]] == [0, 1, 2]


def check_knife_edge(broken=()):
    """n = min_matches - 1 fails, n = min_matches does not; a success clears the count."""
    cfg = dict(lost_after=2, min_matches=6, retry_period=1)
    out = rv.run(cfg, [5, 6, 5, 6, 5, 5], broken=broken)
    assert [s["failed_steps"] for s, _, _ in out] == [1, 0, 1, 0, 1, 2]
    assert tries(out) == [5] and out[5][0]["lost"] == 1


def check_retry_period(broken=()):
    """A lost stream tries on the declaring step, then on every retry_period-th step after it."""
    cfg = dict(lost_after=3, min_matches=4, retry_period=4)
    out = rv.run(cfg, [0] * 14, broken=broken)
    assert tries(out) == [2, 6, 10]
    assert [s["attempted"] for s, _, _ in out] == [int(t in (2, 6, 10)) for t in range(14)]
    assert [sel for _, _, sel in out] == [True] * 3 + [False] * 11


def check_accepted_on_declaring_step(broken=()):
    """A try accepted on the step that declares the loss: tracking again at once, counts zero, selection resumes."""
    cfg = dict(lost_after=2, min_matches=3, retry_period=5)
    out = rv.run(cfg, [0, 0, 9, 0], accepted=lambda t: t == 1, broken=broken)
    s1 = out[1][0]
    assert out[1][1] and s1 == dict(lost=0, failed_steps=0, lost_steps=0, attempted=1, recoveries=1)
    assert out[2][2] and out[2][0]["attempted"] == 0 and out[3][0]["failed_steps"] == 1


def check_accepted_after_retries(broken=()):
    """A rejected try keeps the stream lost; the next due try is accepted."""
    cfg = dict(lost_after=1, min_matches=1, retry_period=2)
    out = rv.run(cfg, [0, 0, 0, 7, 7, 7], accepted=lambda t: t == 2, broken=broken)
    assert tries(out) == [0, 2]
    assert [s["lost"] for s, _, _ in out] == [1, 1, 0, 0, 0, 0]
    assert out[0][0]["recoveries"] == 0 and out[2][0]["recoveries"] == 1 and out[3][0]["failed_steps"] == 0


def check_off_while_lost(broken=()):
    """Turning the feature off while lost resumes selection at once and clears the state."""
    cfg = dict(lost_after=1, min_matches=2, retry_period=9)
    out = rv.run(cfg, [0, 0, 0, 5], off_at=2, broken=broken)
    assert [sel for _, _, sel in out] == [True, False, True, True]
    assert out[2][0] == rv.fresh() and not out[2][1] and not out[3][1]


CHECKS = {f.__name__: f for f in (check_lost_after_one, check_knife_edge, check_retry_period,
                                  check_accepted_on_declaring_step, check_accepted_after_retries,
                                  check_off_while_lost)}
# the check that catches each broken copy
CAUGHT_BY = {
    "select_while_lost": "check_retry_period",
    "off_keeps_lost": "check_off_while_lost",
    "retry_before_count": "check_retry_period",
    "fail_at_min": "check_knife_edge",
    "failures_accumulate": "check_knife_edge",
    "late_declaration": "check_lost_after_one",
    "no_try_on_declaration": "check_accepted_on_declaring_step",
    "keep_failed_on_accept": "check_accepted_on_declaring_step",
}


@pytest.mark.parametrize("name", sorted(CHECKS))
def test_restatement_passes(name):
    CHECKS[name]()


@pytest.mark.parametrize("broken", rv.BROKEN)
def test_broken_copies_are_caught(broken):
    assert set(CAUGHT_BY) == set(rv.BROKEN)
    with pytest.raises(AssertionError):
        CHECKS[CAUGHT_BY[broken]](broken=(broken,))


def test_off_never_moves():
    cfg = dict(lost_after=0, min_matches=0, retry_period=0)
    out = rv.run(cfg, [0] * 6)
    assert all(s == rv.fresh() and not tried and sel for s, tried, sel in out)


def test_reset_keeps_the_past():
    st = dict(lost=1, failed_steps=3, lost_steps=7, attempted=1, recoveries=2)
    assert rv.reset(st) == dict(lost=0, failed_steps=0, lost_steps=0, attempted=1, recoveries=2)


# ---- ABI -------------------------------------------------------------------------------------------------------------
def _c_layout(tmp_path, struct, fields):
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "sl2b200.h"', "int main(void) {",
             '  printf("sizeof %%zu\\n", sizeof(%s));' % struct]
    lines += ['  printf("%s %%zu %%zu\\n", offsetof(%s, %s), sizeof(((%s *)0)->%s));' % (f, struct, f, struct, f)
              for f in fields]
    src, exe = tmp_path / (struct + ".c"), tmp_path / struct
    src.write_text("\n".join(lines + ["  return 0;", "}"]) + "\n")
    subprocess.check_call([os.environ.get("CC", "cc"), "-std=c99", "-I", os.path.join(ROOT, "include"), "-o", str(exe),
                           str(src)])
    return {ln.split()[0]: tuple(int(v) for v in ln.split()[1:])
            for ln in subprocess.check_output([str(exe)], text=True).splitlines()}


@pytest.mark.parametrize("struct, M, names, size", [
    ("sl2_stream_recovery", mirror.Sl2StreamRecovery,
     ["lost_after", "min_matches", "retry_period", "reserved", "reloc", "Pxx"], 16 + 64 + 8 * 169),
    ("sl2_recovery_result", mirror.Sl2RecoveryResult,
     ["lost", "failed_steps", "lost_steps", "attempted", "recoveries", "last"], 24 + 80),
])
def test_structs_match_header(tmp_path, struct, M, names, size):
    assert [f for f, _ in M._fields_] == names
    out = _c_layout(tmp_path, struct, names)
    assert out["sizeof"] == (C.sizeof(M),) == (size,)
    for f, t in M._fields_:
        assert out[f] == (getattr(M, f).offset, C.sizeof(t)), f
    if M is mirror.Sl2RecoveryResult:
        dt = mirror.RECOVERY_RESULT_DTYPE
        assert dt.itemsize == size and [dt.fields[f][1] for f in names] == [getattr(M, f).offset for f in names]
    for name in ("sl2_set_stream_recovery", "sl2_get_stream_recovery", "sl2_get_recovery_results"):
        assert name in mirror.EXPORTS


# ---- the shared argument check ------------------------------------------------------------------------------------------
HARNESS = r"""
#include <stdio.h>
#include <string.h>
#include <string>
#include "sl2b200.h"
namespace sl2 { std::string reloc_params_error(const sl2_reloc_params *p, const double *Pxx); }
int main() {
  /* one case per line on stdin: inlier_px min_inliers reserved v0 v1 v2 w0 w1 w2, then the 169 entries of Pxx */
  sl2_reloc_params p;
  double P[169];
  while (scanf("%lf %d %d %lf %lf %lf %lf %lf %lf", &p.inlier_px, &p.min_inliers, &p.reserved, &p.v[0], &p.v[1],
               &p.v[2], &p.omega[0], &p.omega[1], &p.omega[2]) == 9) {
    for (int i = 0; i < 169; ++i) scanf("%lf", &P[i]);
    printf("[%s]\n", sl2::reloc_params_error(&p, P).c_str());
  }
  return 0;
}
"""


@pytest.fixture(scope="module")
def checker(tmp_path_factory):
    import __graft_entry__ as g
    g.build()
    d = tmp_path_factory.mktemp("reloc_check")
    src, exe = d / "check.cpp", d / "check"
    src.write_text(HARNESS)
    libdir = os.path.dirname(mirror.LIB_PATH)
    subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++17", "-I", os.path.join(ROOT, "include"), "-o",
                           str(exe), str(src), "-L" + libdir, "-lsl2b200", "-Wl,-rpath," + libdir])

    def run(cases):
        txt = "\n".join(" ".join(repr(float(v)) if isinstance(v, float) else str(v) for v in c) for c in cases)
        out = subprocess.check_output([str(exe)], input=txt + "\n", text=True).splitlines()
        return [ln[1:-1] for ln in out]
    return run


def _case(tau=2.0, min_inliers=6, reserved=0, v=(0.0, 0.0, 0.0), omega=(0.0, 0.0, 1e-3), Pxx=None):
    P = np.diag([1e-4] * 7 + [2.5e-3] * 6) if Pxx is None else Pxx
    return [tau, min_inliers, reserved, *v, *omega, *np.asarray(P, np.float64).flatten(order="F")]


def test_shared_check_rejects_each_bad_field(checker):
    asym = np.diag([1e-4] * 13)
    asym[0, 1] = 1e-9
    neg = np.diag([1e-4] * 13)
    neg[0, 0] = -1e-3
    nan = np.diag([1e-4] * 13)
    nan[2, 2] = np.nan
    inf = np.diag([1e-4] * 13)
    inf[12, 12] = np.inf
    bad = {"tau=0": _case(tau=0.0), "tau<0": _case(tau=-1.0), "tau=nan": _case(tau=float("nan")),
           "tau=inf": _case(tau=float("inf")), "min_inliers=3": _case(min_inliers=3), "reserved": _case(reserved=1),
           "v nan": _case(v=(0.0, float("nan"), 0.0)), "omega inf": _case(omega=(0.0, 0.0, float("inf"))),
           "omega=0": _case(omega=(0.0, 0.0, 0.0)), "asymmetric": _case(Pxx=asym), "not psd": _case(Pxx=neg),
           "nan Pxx": _case(Pxx=nan), "inf Pxx": _case(Pxx=inf)}
    good = {"default": _case(), "min_inliers=4": _case(min_inliers=4), "psd, singular": _case(Pxx=np.zeros((13, 13))),
            "tiny omega": _case(omega=(1e-150, 0.0, 0.0))}
    msgs = checker(list(bad.values()) + list(good.values()))
    assert len(msgs) == len(bad) + len(good)
    for name, m in zip(list(bad) + list(good), msgs):
        assert (m != "") == (name in bad), (name, m)
