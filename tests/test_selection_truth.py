"""The NumPy restatement of the mutual-information selection (tests/selection_ref.py) against the greedy selection from
its definition (tests/selection_truth.py) under the derived bound (tests/selection_cases.py), on the CPU: the truth's
two precisions against each other, the restatement within the bound at every q and equal to the truth at every decided
pick and stop over the constructed problems, exactly on the exact ones, and broken copies of the restatement each
caught by a named check."""
import mpmath
import numpy as np
import pytest

import selection_cases as sc
import selection_ref as sr
import selection_truth as st

# longdouble against 50-digit mpmath: both start from the same doubles, and the longdouble evaluation is an
# evaluation of the same formula with unit roundoff 2^-64 instead of 2^-53, so its error is within the double bound
# scaled by 2^-11
LD_SCALE = 2.0 ** -11
WORST = {}


def small_cases():
    return [sc.dense(1, 12, 8), sc.dense(2, 16, 16, 0.5), sc.dense(3, 10, 10, 0.0, sig=0.3),
            sc.near_duplicates(1e-6, 1.0, 0.5, V=12, n_select=8), sc.near_duplicates(1e-9, 1e-2, 0.0, V=10, n_select=10),
            sc.stretched(1e8, V=12, n_select=6), sc.decades(V=14, n_select=10)]


@pytest.mark.parametrize("k", range(7))
def test_longdouble_agrees_with_mpmath(k):
    pb = small_cases()[k]
    P, S, A, B, R, feats, rho = sc.cpu_inputs(pb)
    ld = st.Truth(P, A, B, R, feats, rho).run(pb.n_select, pb.t, bound=sc.q_bound)
    with mpmath.workdps(50):
        mp = st.Truth(P, A, B, R, feats, rho, num=object).run(pb.n_select, pb.t)
        assert [d["pick"] for d in ld] == [d["pick"] for d in mp]
        worst, ratio = 0.0, 0.0
        for a, b in zip(ld, mp):
            for j in np.flatnonzero(a["live"]):
                hi = float(a["qx"][j])
                e = abs(mpmath.mpf(hi) + mpmath.mpf(float(a["qx"][j] - np.longdouble(hi))) - b["qx"][j])
                worst = max(worst, float(e / abs(b["qx"][j])))
                ratio = max(ratio, float(e) / (LD_SCALE * a["beta"][j, 0]))
    print(pb.name, "decisions", len(ld), "worst |q_ld - q_mp| / q_mp %.3g, / (2^-11 bound) %.3g" % (worst, ratio))
    assert ratio <= 1.0


# ---- the restatement against the truth -----------------------------------------------------------------------------
def compare(pb, select=sr.information_select, P_read=None):
    """Run `select` (the restatement, or a broken copy) on pb's arrays (P_read in place of P if given) and hold it to
    the truth followed along its picks.  Returns {check name: first failure or None} and the statistics."""
    P, S, A, B, R, feats, rho = sc.cpu_inputs(pb)
    picks, info = select(P if P_read is None else P_read, feats, rho, S, A, B, R, pb.n_select, pb.t)
    index = {int(f): k for k, f in enumerate(feats)}
    follow = [index[f] for f in picks]
    tr = st.Truth(P, A, B, R, feats, rho)
    ds = tr.run(pb.n_select, pb.t, follow=follow, bound=sc.q_bound)
    fail = {"q within bound": None, "decided picks": None, "exact picks": None}
    worst, undecided = 0.0, 0
    for r, d in enumerate(ds):
        mine = follow[r] if r < len(follow) else -1
        live = d["live"] & np.isfinite(d["q"])
        if r < len(info):
            qr = info[r]["qall"]
            with np.errstate(invalid="ignore"):
                ratio = np.abs(qr[live] - d["q"][live]) / d["beta"][live, 0]
            bad = ~(ratio <= 1.0)
            if bad.any() and fail["q within bound"] is None:
                fail["q within bound"] = (r, float(np.nanmax(np.where(np.isnan(ratio), np.inf, ratio))))
            worst = max(worst, float(np.nanmax(ratio)) if ratio.size else 0.0)
        if not sc.decided(d, pb.t):
            undecided += 1
        elif mine != d["pick"] and fail["decided picks"] is None:
            fail["decided picks"] = (r, mine, d["pick"])
    if pb.exact:  # ties decide by rank, q = t by the strict >: the truth's own picks and stop, exactly
        want = [d["pick"] for d in tr.run(pb.n_select, pb.t)]
        got = follow + ([-1] if len(follow) < min(pb.n_select, len(feats)) else [])
        if want != got:
            fail["exact picks"] = (want, got)
    return fail, dict(worst=worst, undecided=undecided, decisions=len(ds), margins=st.margins(ds, pb.t))


PROBLEMS = {pb.name: pb for pb in sc.constructions()}


@pytest.mark.parametrize("name", list(PROBLEMS) + ["dense V=64", "dense V=129"])
def test_restatement_against_the_truth(name):
    pb = PROBLEMS.get(name) or sc.dense(4, int(name.split("=")[1]), 40)
    fail, stats = compare(pb)
    WORST[name] = stats
    print(name, "decisions", stats["decisions"], "worst error/bound %.3g" % stats["worst"], "inside the bound",
          stats["undecided"], "margins (winner, threshold)", stats["margins"])
    assert fail == {"q within bound": None, "decided picks": None, "exact picks": None}, fail


def test_the_tie_constructions_pick_the_lower_rank():
    pb = sc.ties()
    P, S, A, B, R, feats, rho = sc.cpu_inputs(pb)
    picks, _ = sr.information_select(P, feats, rho, S, A, B, R, pb.n_select, pb.t)
    for a, b in sc.TIE_PAIRS:
        qa = (S[a, 0] * S[a, 3] - S[a, 1] * S[a, 1]) / (R[a] * R[a])
        qb = (S[b, 0] * S[b, 3] - S[b, 1] * S[b, 1]) / (R[b] * R[b])
        assert qa == qb and abs(S[a, 1]) == abs(S[b, 1]) and rho[a] < rho[b]
        assert picks.index(a) + 1 == picks.index(b)
    lo, hi = sc.RHO_PAIR
    assert rho[hi] < rho[lo] and picks.index(hi) + 1 == picks.index(lo)


# ---- broken copies -------------------------------------------------------------------------------------------------
def broken_select(bug):
    """selection_ref.information_select with one deliberate slip."""
    def select(P, feats, rho, S, A, B, R, n_select, t):
        feats = np.asarray(feats, np.int64)
        rho = np.asarray(rho, np.int64)
        V = len(feats)
        Aj, Bj = A[feats].astype(np.float64), B[feats].astype(np.float64)
        C00, C10, C11 = S[feats, 0].copy(), S[feats, 1].copy(), S[feats, 3].copy()
        Rj = R[feats].astype(np.float64)
        yrow = sc.NXV + 3 * feats
        nmax = min(int(n_select), V)
        g = np.zeros((V, max(nmax, 1), 2, 2))
        picked = np.zeros(V, bool)
        idx = np.arange(V)
        picks, info = [], []
        Pu = P.T if bug == "u from P transposed" else P
        for r in range(nmax):
            with np.errstate(all="ignore"):
                q = (C00 * C11 - C10 * C10) / (Rj * Rj)
                above = q >= t if bug == ">= against t" else q > t
                ok = ~picked & above & (True if bug == "C00 > 0 not tested" else C00 > 0.0)
            if not ok.any():
                info.append(dict(stop=True, q=np.nan, second=-np.inf, qall=np.where(picked, np.nan, q)))
                break
            cand = idx[ok]
            keys = (rho[cand], cand, -q[cand]) if bug == "index before rank" else (cand, rho[cand], -q[cand])
            i = int(cand[np.lexsort(keys)[0]])
            info.append(dict(stop=False, q=float(q[i]), second=-np.inf, qall=np.where(picked, np.nan, q)))
            picks.append(int(feats[i]))
            picked[i] = True
            with np.errstate(all="ignore"):
                l00 = np.sqrt(C00[i])
                l10 = C10[i] / l00
                l11 = np.sqrt(C11[i] - l10 * l10)
            yi = int(yrow[i])
            u7, uy = np.zeros((7, 2)), np.zeros((V, 3, 2))
            for c in range(2):
                acc = np.zeros(7)
                for k in range(7):
                    acc = acc + Pu[0:7, k] * Aj[i, c, k]
                for k in range(3):
                    acc = acc + Pu[0:7, yi + k] * Bj[i, c, k]
                u7[:, c] = acc
                for kk in range(3):
                    rows = yrow + kk
                    acc = np.zeros(V)
                    for k in range(7):
                        acc = acc + Pu[rows, k] * Aj[i, c, k]
                    for k in range(3):
                        acc = acc + Pu[rows, yi + k] * Bj[i, c, k]
                    uy[:, kk, c] = acc
            m = ~picked
            cj = np.zeros((V, 2, 2))
            for a in range(2):
                for b in range(2):
                    acc = np.zeros(V)
                    for k in range(7):
                        acc = acc + Aj[:, a, k] * u7[k, b]
                    for k in range(3):
                        acc = acc + Bj[:, a, k] * uy[:, k, b]
                    for p in range(r):
                        pp = max(p - 1, 0) if bug == "factors of pick r - 1" else p
                        for e in range(2):
                            acc = acc - g[:, pp, a, e] * g[i, pp, b, e]
                    cj[:, a, b] = acc
            with np.errstate(all="ignore"):
                gn = np.zeros((V, 2, 2))
                if bug == "L^-1 for L^-T":
                    for b in range(2):
                        gn[:, 0, b] = cj[:, 0, b] / l00
                        gn[:, 1, b] = (cj[:, 1, b] - gn[:, 0, b] * l10) / l11
                else:
                    for a in range(2):
                        gn[:, a, 0] = cj[:, a, 0] / l00
                        gn[:, a, 1] = (cj[:, a, 1] - gn[:, a, 0] * l10) / l11
                k11 = 0.0 if bug == "g[a][1] g[b][1] dropped" else 1.0
                n00 = C00 - gn[:, 0, 0] * gn[:, 0, 0] - k11 * gn[:, 0, 1] * gn[:, 0, 1]
                n10 = C10 - gn[:, 1, 0] * gn[:, 0, 0] - k11 * gn[:, 1, 1] * gn[:, 0, 1]
                n11 = C11 - gn[:, 1, 0] * gn[:, 1, 0] - k11 * gn[:, 1, 1] * gn[:, 1, 1]
            g[m, r] = gn[m]
            C00, C10, C11 = np.where(m, n00, C00), np.where(m, n10, C10), np.where(m, n11, C11)
        return picks, info
    return select


def poisoned(pb):
    """pb's P with the triangle the kernel never reads replaced by garbage: P[y_a, y_b] for a picked before b (a
    never-picked feature counting as last).  The kernel reads P[row, col] with the row a candidate's (or the camera's)
    and the column the pick's, so the blocks of pairs are read with the later pick as the row."""
    P, S, A, B, R, feats, rho = sc.cpu_inputs(pb)
    picks, _ = sr.information_select(P, feats, rho, S, A, B, R, pb.n_select, pb.t)
    order = {f: k for k, f in enumerate(picks)}
    Pb = P.copy()
    rng = np.random.default_rng(5)
    for a in picks:
        for b in range(len(pb.y)):
            if b != a and order.get(b, 1 << 30) > order[a]:
                ya, yb = slice(13 + 3 * a, 16 + 3 * a), slice(13 + 3 * b, 16 + 3 * b)
                Pb[ya, yb] = rng.uniform(-1.0, 1.0, (3, 3)) * 1e-2
    return Pb


MUTATIONS = [("L^-1 for L^-T", "dense", "q within bound"), ("g[a][1] g[b][1] dropped", "dense", "q within bound"),
             ("factors of pick r - 1", "dense", "q within bound"), ("index before rank", "ties", "exact picks"),
             (">= against t", "degenerate", "exact picks"), ("u from P transposed", "asymmetric", "q within bound"),
             ("C00 > 0 not tested", "degenerate", "exact picks")]


@pytest.mark.parametrize("bug,problem,check", MUTATIONS)
def test_mutations_are_caught(bug, problem, check):
    pb = {"dense": lambda: sc.dense(5, 24, 12), "asymmetric": lambda: sc.dense(5, 24, 12), "ties": sc.ties,
          "degenerate": sc.degenerate}[problem]()
    P_read = poisoned(pb) if problem == "asymmetric" else None
    good, _ = compare(pb, P_read=P_read)
    assert not any(good.values()), good  # the restatement itself passes on the same problem and P
    bad, _ = compare(pb, broken_select(bug), P_read=P_read)
    print(bug, "->", check, bad[check])
    assert bad[check] is not None, bad
