"""The planar patch warp's restatement (tests/warp_ref.py) against the warp from its definition in extended precision
(tests/warp_truth.py) under the bounds and decision rule of tests/warp_cases.py: src within its bound, and the
validity flags and bytes the rule decides equal to the truth's.  The cases: the C1 / C2 / C4 camera at 11 x 11 and
15 x 15, C3's at 15 x 15 and a camera whose reach cuts into its image; features of the visibility envelope at |q| of
xp and xo = 1, 1 +- 3.5e-5, 1 +- 1e-3, 0.97, 1.03 and 1.2; planes seen nearly edge-on; distance ratios of 0.5 and 2;
and constructions whose FP64 chain is exact (ties, the template's edges, a ray parallel to the plane, zo[2] <= 0, the
model's reach).  Deliberately broken copies of the restatement must fail a check."""
import functools
import os
import types

import numpy as np
import pytest

import warp_cases as wc
import warp_ref
from warp_truth import warp_truth

HERE = os.path.dirname(os.path.abspath(__file__))


@functools.lru_cache(maxsize=None)
def decided():
    return [(c, wc.Decided(*c[1:])) for c in wc.random_cases()]


@functools.lru_cache(maxsize=None)
def decided_constructions():
    return [(c, wc.Decided(*c[1:])) for c in wc.constructions()]


def failures(ref, case, D):
    """The checks a restatement module fails on one case ("index": it read outside the template)."""
    _, cam8, B, y, xo, xp, T = case
    try:
        src, valid, _, X = ref.warp_points(cam8, B, y, xo, xp)
        out, ov = ref.warp_template(cam8, T, y, xo, xp)
    except IndexError as e:
        return [("index", str(e))]
    return D.check(src, valid, X, out, ov)


def exact_failures(ref, case, D):
    """A construction whose chain is exact: every pixel's flag, src and byte (.5 ties included) equal the truth's."""
    _, cam8, B, y, xo, xp, T = case
    try:
        src, valid, _, _ = ref.warp_points(cam8, B, y, xo, xp)
        out, ov = ref.warp_template(cam8, T, y, xo, xp)
        tr = D.tr
        fail = []
        if not (valid == tr.valid).all():
            fail.append(("exact", "flags differ"))
        elif not (src[valid] == tr.src[valid]).all():
            fail.append(("exact", "src differs"))
        elif not (ref.sample(np.asarray(T, np.uint8), np.where(valid[..., None], src, 0.0))[valid]
                  == tr.byte[valid]).all():
            fail.append(("exact", "bytes differ"))
        elif (ov, out.tobytes()) != (D.template()[1], D.template()[0].tobytes()):
            fail.append(("exact", "template differs"))
    except IndexError as e:
        return [("index", str(e))]
    return fail


EXACT = ("half-shift-11", "half-shift-15", "edges-11", "edges-15", "beyond-11", "beyond-15")


# ---- the truth --------------------------------------------------------------------------------------------------------
def test_longdouble_truth_agrees_with_mpmath():
    """The mpmath truth (50 digits) is the definition; the longdouble one the other checks use gives the same flags
    and bytes, and src, v and the margins to within a few FP64 ulps of the values."""
    worst_src, worst_v, n = 0.0, 0.0, 0
    picks = decided()[::7] + decided_constructions()
    for case, D in picks:
        tm = warp_truth(*case[1:], prec="mp")
        tl = D.tr
        assert (tm.valid == tl.valid).all() and (tm.byte == tl.byte).all(), case[0]
        v = tm.valid
        worst_src = max(worst_src, float((np.abs(tm.src - tl.src)[v] / (1 + np.abs(tm.src[v]))).max(initial=0)))
        worst_v = max(worst_v, float((np.abs(tm.v - tl.v)[v] / 256).max(initial=0)))
        for m in ("m_reach", "m_lam", "m_zo"):
            a, b = getattr(tm, m), getattr(tl, m)
            assert ((np.isnan(a) == np.isnan(b)) & (np.sign(np.nan_to_num(a)) == np.sign(np.nan_to_num(b)))).all()
        n += 1
    print("longdouble vs mpmath over %d cases: src %.3g, v %.3g (relative to 1 + |src| and 256)"
          % (n, worst_src, worst_v))
    assert n >= 25 and worst_src <= 4 * wc.U and worst_v <= 4 * wc.U


def test_newton_ray_round_trips():
    """The truth's ray is a solution: Project of X (the plane point it meets) from xp is p, and X lies on the plane
    (mpmath, on every construction and a sample of the random cases)."""
    from consensus_truth import _Num, project, rotation_rrw
    num = _Num("ld")
    for case, D in decided()[::11] + decided_constructions():
        _, cam8, B, y, xo, xp, T = case
        tr = D.tr
        ok = ~np.isnan(tr.X).any(-1) & (tr.lam > 0)
        xpn = num(xp)
        zc = np.einsum("ij,kj->ki", rotation_rrw(xpn[3:7]), num(tr.X[ok]) - xpn[0:3])
        back = num.f64(project(cam8, zc, num))
        assert np.abs(back - tr.p[ok]).max(initial=0) <= 1e-9, case[0]
        nW = np.asarray(xo[:3]) - np.asarray(y)
        assert np.abs((tr.X[ok] - y) @ nW).max(initial=0) <= 1e-12 * (1 + np.abs(tr.X[ok]).max(initial=0)), case[0]


# ---- the restatement against it ---------------------------------------------------------------------------------------
def test_restatement_within_the_bound():
    """src within the bound, decided flags and bytes equal, the centre pixel at (HALF, HALF) and the round trip
    (the restatement's plane point seen from xp lands on its pixel), on every random case.  Reports the worst
    error / bound ratio and the decided fractions."""
    worst, fracs, valid_px = 0.0, [], 0
    for case, D in decided():
        assert not failures(warp_ref, case, D), (case[0], failures(warp_ref, case, D))
        src, valid, _, _ = warp_ref.warp_points(*case[1:6])
        both = valid & D.tr.valid
        if both.any():
            worst = max(worst, float((np.abs(src - D.tr.src).max(-1) / D.b["src"])[both].max()))
        fracs.append(float((D.byte_decided | (D.flag_decided & ~D.tr.valid)).mean()))
        valid_px += int(D.tr.valid.sum())
    fracs = np.array(fracs)
    print("%d cases: worst |src - src_truth| / bound %.3g; decided pixels min %.4f mean %.5f; %d valid pixels"
          % (len(fracs), worst, fracs.min(), fracs.mean(), valid_px))
    assert worst <= 1.0 and fracs.min() >= 0.98 and valid_px >= 0.9 * sum(c[2] ** 2 for c, _ in decided())


def test_the_reach_cuts_into_the_wide_camera():
    """The wide camera's features reach up to the model's reach: some of their templates have pixels beyond it (which
    test_restatement_within_the_bound holds to be invalid in both) and valid pixels close to it."""
    out = [D for c, D in decided() if c[0].startswith("reach-")]
    beyond = sum(int((D.tr.m_reach <= 0).sum()) for D in out)
    near = min(float(D.tr.m_reach[D.tr.m_reach > 0].min()) for D in out)
    print("wide camera: %d pixels beyond the reach, smallest margin inside %.3g" % (beyond, near))
    assert beyond > 0 and near < 0.05


@pytest.mark.parametrize("name", EXACT)
def test_exact_constructions(name):
    """kd1 = 0, fku = fkv = 256, an integer principal point, q = (1, 0, 0, 0), a fronto-parallel plane and dyadic
    translations: the FP64 chain is exact, and every flag, src and byte equals the truth's, .5 ties (which round up)
    included."""
    case, D = next(x for x in decided_constructions() if x[0][0] == name)
    assert not exact_failures(warp_ref, case, D)
    B = case[2]
    half = (B - 1) // 2
    src = D.tr.src
    a, b = np.mgrid[0:B, 0:B]
    if name.startswith("half-shift"):
        assert (src[..., 0] == half + (b - half) / 2).all() and (src[..., 1] == half + (a - half) / 2).all()
        ties = D.tr.tie_gap == 0
        assert ties.sum() >= B and (D.tr.byte[ties] == np.floor(D.tr.v[ties]) + 1).all()
    elif name.startswith("edges"):
        assert (src[..., 0] == b).all() and (src[..., 1] == a).all()
        assert (D.tr.byte == case[6]).all()
    else:
        assert (src[..., 0] == half + 2 * (b - half)).all() and (src[..., 0] < 0).any() and (src[..., 0] > B - 1).any()
        T = np.asarray(case[6])
        clip = np.clip(half + 2 * (np.arange(B) - half), 0, B - 1)
        assert (D.tr.byte == T[np.ix_(clip, clip)]).all()


def test_rows_parallel_ray_and_zo_behind():
    """Row 0 has zo[2] < 0, row 1 zo[2] = 0 exactly, rows 2-8 are valid, row 9's rays are exactly parallel to the plane
    and row 10's meet it behind the camera: the restatement's flags equal the truth's on every pixel, the exact
    zeros included."""
    case, D = next(x for x in decided_constructions() if x[0][0] == "rows")
    tr = D.tr
    assert (tr.m_zo[0] < 0).all() and (tr.m_zo[1] == 0).all() and tr.valid[2:9].all()
    assert (tr.m_lam[9] == 0).all() and (tr.m_lam[10] < 0).all() and not tr.valid[[0, 1, 9, 10]].any()
    src, valid, _ = warp_ref.warp_source(*case[1:6])
    assert (valid == tr.valid).all()
    assert not failures(warp_ref, case, D)
    out, ov = warp_ref.warp_template(case[1], case[6], *case[3:6])
    assert ov == 0 and (out == case[6]).all()


def test_reach_edge():
    """kd1 = 1/64 on the axis: the pixels at offsets (+-4, +-4) lie exactly at the reach (margin 0 in the truth, and
    1 - 2 kd1 r^2 = 0 exactly in FP64), those beyond it and they are invalid in both, the rest valid in both and
    within the bound."""
    case, D = next(x for x in decided_constructions() if x[0][0] == "reach")
    tr = D.tr
    a, b = np.mgrid[0:11, 0:11] - 5
    r2 = a * a + b * b
    assert (tr.m_reach[r2 == 32] == 0).all() and (r2 == 32).sum() == 4
    assert (1.0 - (2.0 * case[1][6]) * 32.0) == 0.0
    assert (tr.valid == (r2 < 32)).all() and (tr.m_reach[r2 < 32] >= 3 / 32).all()
    src, valid, _ = warp_ref.warp_source(*case[1:6])
    assert (valid == tr.valid).all()
    assert not failures(warp_ref, case, D)


def test_centre_pixel_at_every_norm():
    """The centre pixel samples (HALF, HALF) within its bound at every |q| (with the earlier RRW^T ray it is off by
    about 0.01 px at |q| - 1 = 3.5e-5)."""
    seen = set()
    for case, D in decided():
        src, valid, _ = warp_ref.warp_source(*case[1:6])
        c = (case[2] - 1) // 2
        if D.tr.valid[c, c]:
            assert valid[c, c] and (np.abs(src[c, c] - c) <= D.b["src"][c, c]).all(), case[0]
            seen.add(round(float(np.linalg.norm(case[5][3:7])), 6))
    assert len(seen) == len(wc.Q_NORMS)


# ---- the checks can see -----------------------------------------------------------------------------------------------
MUTATIONS = {
    "RRW^T ray": [("A = adjugate(R)", "A = [[R[k][i] for k in range(3)] for i in range(3)]")],
    "nW from xp": [("nW = [xo[i] - y[i] for i in range(3)]", "nW = [xp[i] - y[i] for i in range(3)]")],
    "h for ho": [("(g[..., 0] - ho[0])", "(g[..., 0] - h[0])"), ("(g[..., 1] - ho[1])", "(g[..., 1] - h[1])")],
    "rows and columns swapped": [("p0 = h[0] + (b - half)", "p0 = h[0] + (a - half)"),
                                 ("p1 = h[1] + (a - half)", "p1 = h[1] + (b - half)")],
    "kd1 sign in unproject_point": [("np.sqrt(1.0 - (2.0 * kd1)", "np.sqrt(1.0 + (2.0 * kd1)")],
    "round half to even": [("return (v + 0.5).astype(np.int64)", "return np.rint(v).astype(np.int64)")],
    "clamp to B": [("np.maximum(src[..., 0], 0.0), float(B - 1))", "np.maximum(src[..., 0], 0.0), float(B))"),
                   ("np.maximum(src[..., 1], 0.0), float(B - 1))", "np.maximum(src[..., 1], 0.0), float(B))")],
    "x0 without min": [("x0 = np.minimum(np.floor(sx).astype(np.int64), B - 2)", "x0 = np.floor(sx).astype(np.int64)"),
                       ("y0 = np.minimum(np.floor(sy).astype(np.int64), B - 2)", "y0 = np.floor(sy).astype(np.int64)")],
    "no zo[2] > 0 test": [(" & (zo[..., 2] > 0.0)", "")],
}


def mutant(edits):
    """A copy of tests/warp_ref.py with the edits applied (each must match exactly once)."""
    src = open(os.path.join(HERE, "warp_ref.py")).read()
    for old, new in edits:
        assert src.count(old) == 1, old
        src = src.replace(old, new)
    mod = types.ModuleType("warp_ref_mutant")
    mod.__file__ = os.path.join(HERE, "warp_ref.py")
    exec(compile(src, mod.__file__, "exec"), mod.__dict__)
    return mod


@pytest.mark.parametrize("mutation", list(MUTATIONS))
def test_mutations_are_caught(mutation):
    """Each broken copy of the restatement fails a check on at least one case: src, valid, byte, centre or round-trip
    (random cases and constructions, under the rule), exact (the exact constructions), or index (a read outside the
    template)."""
    ref = mutant(MUTATIONS[mutation])
    caught = {}
    for case, D in decided() + decided_constructions():
        kinds = {f[0] for f in failures(ref, case, D)}
        if case[0] in EXACT:
            kinds |= {f[0] for f in exact_failures(ref, case, D)}
        for k in kinds:
            caught.setdefault(k, []).append(case[0])
    print("%s: %s" % (mutation, {k: "%d cases, first %s" % (len(v), v[0]) for k, v in sorted(caught.items())}))
    assert caught
