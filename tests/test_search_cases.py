"""The adversarial patch-search cases of search_cases.py (no GPU): each family is what it claims to be, the premise of the
filtered kernel holds on every candidate of them, and the oracle agrees with the reference's own code on them
(replayed from tests/golden, see tests/ref_golden.py)."""
import numpy as np
import pytest

import search_cases as sc

# |exact score - (2 - 2 rho)| over every candidate with both sigmas >= 10: the kernel's filter assumes <= 1e-9
PREMISE_BOUND = 1e-9


def _accepted(c, j, corr, sd, inside):
    """Candidates the search may accept: inside the ellipse, window sigma >= 10, template sigma >= 10, <= corrmax."""
    t = c.patches[c.feat[j]].astype(np.int64)
    ok0 = not (sc.sigma_fp64(int(t.sum()), int((t * t).sum()), c.B * c.B) < 10.0)
    return (inside > 0) & ~(sd < 10.0) & (corr <= 1e6) & ok0


@pytest.mark.parametrize("B", sc.BOXES)
def test_copies_ties_and_their_winner(oracle, B):
    c = sc.cases(B)
    assert len(c.copies) >= 5 * len(sc.SWEEP)
    for f, uv in c.copies.items():
        for u, v in uv:
            assert sc.window(c, u, v).tobytes() == c.patches[f].tobytes()
    js = sorted(c.winner)
    u, v, found, best = oracle.elliptical_search(c.image, c.patches[c.feat[js]], c.centres[js], c.pu[js])
    for k, j in enumerate(js):
        assert (u[k], v[k]) == c.winner[j] and found[k] == 1, c.labels[j]
    # the copies of a template tie exactly: every one of them scores the winner's bits
    for j in js[:12]:
        box, corr, sd, inside = oracle.score_map(c.image, c.patches[c.feat[j]], c.centres[j], c.pu[j])
        us, vs, uc, vc = box[0], box[2], box[4], box[5]
        scores = {corr[u - uc - us, v - vc - vs] for u, v in c.copies[c.feat[j]]
                  if 0 <= u - uc - us < corr.shape[0] and 0 <= v - vc - vs < corr.shape[1]}
        assert len(scores) == 1, c.labels[j]


@pytest.mark.parametrize("B", sc.BOXES)
def test_knife_edge_sums_are_exact(oracle, B):
    c = sc.cases(B)
    n = B * B
    lo, hi = sc.knife_steps(B)
    assert lo < 0 < hi and lo % 2 == 0 and hi % 2 == 0
    seen = set()
    for u, v, d, s, f in c.knife:
        g = sc.window(c, u, v).astype(np.int64)
        assert sc.window_var(g) == 100 * n * n + d
        assert s == sc.sigma_fp64(int(g.sum()), int((g * g).sum()), n)
        assert (s >= 10.0) == (d > 0 or (d == 0 and s >= 10.0))
        seen.add((d, s >= 10.0))
    assert {(lo, False), (0, False), (0, True), (hi, True)} <= seen
    # the window is the best match of its template wherever the FP64 chain accepts it, and gated otherwise
    for j in c.knife_jobs:
        u, v, d, s, f = next(k for k in c.knife if k[4] == c.feat[j])
        ou, ov, of, obest = oracle.elliptical_search(c.image, c.patches[[f]], c.centres[[j]], c.pu[[j]])
        box, corr, sd, inside = oracle.score_map(c.image, c.patches[f], c.centres[j], c.pu[j])
        k = (u - box[4] - box[0], v - box[5] - box[2])
        assert inside[k] == 1 and sd[k] == s, c.labels[j]
        if s >= 10.0 and "template" not in c.labels[j]:
            assert (ou[0], ov[0], of[0]) == (u, v, 1), c.labels[j]
        elif s < 10.0:
            assert (ou[0], ov[0]) != (u, v), c.labels[j]
    # both outcomes of the template gate
    gate = {c.labels[j] for j in c.knife_jobs if "template" in c.labels[j]}
    assert len(gate) == 2


@pytest.mark.parametrize("B", sc.BOXES)
def test_straddle_gaps_cross_the_filter_window(oracle, B):
    c = sc.cases(B)
    gaps = []
    for j in c.straddle_jobs:
        box, corr, sd, inside = oracle.score_map(c.image, c.patches[c.feat[j]], c.centres[j], c.pu[j])
        s = np.sort(corr[_accepted(c, j, corr, sd, inside)])
        assert s.size >= 2 and s[0] < 0.01, c.labels[j]
        gaps.append(s[1] - s[0])
    gaps = np.array(gaps)
    near = (gaps >= 0.5e-5) & (gaps <= 2e-5)
    assert near.sum() >= 3, np.sort(gaps)
    assert (gaps < 1e-6).sum() >= 3 and (gaps > 1e-4).sum() >= 2, np.sort(gaps)
    assert (gaps < 1e-14).any()                   # the affine copies: a tie decided by FP64 rounding


@pytest.mark.parametrize("B", sc.BOXES)
def test_filter_premise_on_every_candidate(oracle, B):
    """The approximate score 2 - 2 rho, rho from the exact integer sums, is within PREMISE_BOUND of the exact FP64
    score on every candidate of every family whose template and window sigmas are >= 10."""
    c = sc.cases(B)
    n = B * B
    worst, count = 0.0, 0
    for j in c.sample(per_family=6) + c.straddle_jobs:
        t = c.patches[c.feat[j]].astype(np.int64)
        S0, S00 = int(t.sum()), int((t * t).sum())
        if sc.sigma_fp64(S0, S00, n) < 10.0:
            continue
        box, corr, sd, inside = oracle.score_map(c.image, c.patches[c.feat[j]], c.centres[j], c.pu[j])
        if corr.size == 0:
            continue
        S1, S2, Sxy = sc.box_sums(c.image, c.patches[c.feat[j]], box)
        V0 = n * S00 - S0 * S0
        V1 = n * S2 - S1 * S1
        ok = ~(sd < 10.0)
        with np.errstate(invalid="ignore", divide="ignore"):    # flat windows (V1 = 0) are gated
            rho = (n * Sxy - S0 * S1) / np.sqrt(float(V0) * V1.astype(np.float64))
        err = np.abs(corr - (2.0 - 2.0 * rho))[ok]
        count += int(ok.sum())
        worst = max(worst, float(err.max(initial=0.0)))
    assert count > 100000
    assert worst <= PREMISE_BOUND, worst


def test_search_cases_match_reference_source(oracle, reference):
    """The oracle's elliptical search on a sample of every family (every knife job among them) and its SMOE search on
    the SMOE sets, against the reference's own MonoSLAM::elliptical_search and SearchMultipleOverlappingEllipses."""
    for B in sc.BOXES:
        c = sc.cases(B)
        for j in c.sample(per_family=5):
            f = c.feat[j]
            ok, ru, rv = reference.call("elliptical_search_ref", c.image, c.patches[f], c.centres[j], c.pu[j],
                                        live=oracle.elliptical_search_ref)
            ou, ov, of, obest = oracle.elliptical_search(c.image, c.patches[[f]], c.centres[[j]], c.pu[[j]])
            assert bool(of[0]) == bool(ok), c.labels[j]
            if obest[0] < 1e6:
                assert (ou[0], ov[0]) == (ru, rv), c.labels[j]
            else:
                assert (ru, rv) == (-7, -9), c.labels[j]      # never written without an accepted candidate
        for label, patch, pu, centres in sc.smoe_cases(B):
            a = oracle.smoe_search(c.image, patch, pu, centres)
            b = reference.call("smoe_search", c.image, patch, pu, centres)
            for x, y in zip(a[:3], b[:3]):
                assert (x == y).all(), label
