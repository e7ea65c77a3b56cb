"""NumPy restatement of the mutual-information selection (include/sl2b200.h, sl2_set_stream_selection;
csrc/select.cu, select_kernel), op for op: every product, sum and quotient is one correctly rounded float64 operation
in the kernel's order, vectorised only across candidates (independent lanes), never through np.dot.

Also the trace rule's candidate ranking (ekf.cu, predict_kernel) from the device's S and visibility."""
import numpy as np

NXV = 13


def trace_candidates(S, visible):
    """The trace rule's ranking of the visible features, cut at the first zero trace: (features ascending, their
    ranks).  S (nf, 4) column-major as stored; visible (nf,) bool."""
    score = S[:, 0] + S[:, 3]
    nf = len(score)
    rank = np.full(nf, -1, np.int64)
    r0 = 1 << 30
    nvis = int(np.count_nonzero(visible))
    for i in range(nf):
        if not visible[i]:
            continue
        si = score[i]
        rk = 0
        for j in range(nf):
            if visible[j] and (score[j] > si or (j < i and not (si > score[j]))):
                rk += 1
        rank[i] = rk
        if si == 0.0:
            r0 = min(r0, rk)
    cut = min(r0, nvis)
    feats = np.array([i for i in range(nf) if 0 <= rank[i] < cut], np.int64)
    return feats, rank[feats] if len(feats) else np.zeros(0, np.int64)


def information_select(P, feats, rho, S, A, B, R, n_select, t):
    """The picks of select_kernel.  P (n, n) the predicted covariance (both triangles equal); feats (V,) the candidates'
    feature indices, rho (V,) their trace ranks; S (nf, 4) column-major; A (nf, 2, 7) dh_dxp; B (nf, 2, 3) dh_dy;
    R (nf,) Rvar; t = exp2(2 min_bits).
    Returns (picks: feature indices in pick order, info: one dict per decision with the winning q, the runner-up q
    (-inf if none) and the stop reason; the last decision is the stop when fewer than min(n_select, V) were picked)."""
    feats = np.asarray(feats, np.int64)
    rho = np.asarray(rho, np.int64)
    V = len(feats)
    Aj, Bj = A[feats].astype(np.float64), B[feats].astype(np.float64)
    C00, C10, C11 = S[feats, 0].copy(), S[feats, 1].copy(), S[feats, 3].copy()
    Rj = R[feats].astype(np.float64)
    yrow = NXV + 3 * feats
    nmax = min(int(n_select), V)
    g = np.zeros((V, max(nmax, 1), 2, 2))
    picked = np.zeros(V, bool)
    idx = np.arange(V)
    picks, info = [], []
    for r in range(nmax):
        with np.errstate(all="ignore"):
            q = (C00 * C11 - C10 * C10) / (Rj * Rj)
            ok = ~picked & (C00 > 0.0) & (q > t)
        if not ok.any():
            with np.errstate(all="ignore"):
                best = np.max(np.where(~picked & ~np.isnan(q), q, -np.inf)) if (~picked).any() else -np.inf
            info.append(dict(stop=True, q=best, second=-np.inf, qall=np.where(picked, np.nan, q)))
            break
        cand = idx[ok]
        order = np.lexsort((cand, rho[cand], -q[cand]))
        i = int(cand[order[0]])
        second = float(q[cand[order[1]]]) if len(cand) > 1 else -np.inf
        info.append(dict(stop=False, q=float(q[i]), second=second, qall=np.where(picked, np.nan, q)))
        picks.append(int(feats[i]))
        picked[i] = True
        # L_i = chol(C_i)
        l00 = np.sqrt(C00[i])
        l10 = C10[i] / l00
        l11 = np.sqrt(C11[i] - l10 * l10)
        yi = int(yrow[i])
        # u = P H_i^T on rows 0..6 and on the three y rows of every candidate
        u7 = np.zeros((7, 2))
        uy = np.zeros((V, 3, 2))
        for c in range(2):
            acc = np.zeros(7)
            for k in range(7):
                acc = acc + P[0:7, k] * Aj[i, c, k]
            for k in range(3):
                acc = acc + P[0:7, yi + k] * Bj[i, c, k]
            u7[:, c] = acc
            for kk in range(3):
                rows = yrow + kk
                acc = np.zeros(V)
                for k in range(7):
                    acc = acc + P[rows, k] * Aj[i, c, k]
                for k in range(3):
                    acc = acc + P[rows, yi + k] * Bj[i, c, k]
                uy[:, kk, c] = acc
        # condition the unpicked candidates on the pick
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
                    for e in range(2):
                        acc = acc - g[:, p, a, e] * g[i, p, b, e]
                cj[:, a, b] = acc
        with np.errstate(all="ignore"):
            gn = np.zeros((V, 2, 2))
            for a in range(2):
                gn[:, a, 0] = cj[:, a, 0] / l00
                gn[:, a, 1] = (cj[:, a, 1] - gn[:, a, 0] * l10) / l11
            n00 = C00 - gn[:, 0, 0] * gn[:, 0, 0] - gn[:, 0, 1] * gn[:, 0, 1]
            n10 = C10 - gn[:, 1, 0] * gn[:, 0, 0] - gn[:, 1, 1] * gn[:, 0, 1]
            n11 = C11 - gn[:, 1, 0] * gn[:, 1, 0] - gn[:, 1, 1] * gn[:, 1, 1]
        g[m, r] = gn[m]
        C00 = np.where(m, n00, C00)
        C10 = np.where(m, n10, C10)
        C11 = np.where(m, n11, C11)
    return picks, info


def sinv_from_S(s00, s10, s11):
    """sl2_model.cuh sinv_from_S: the search ellipse (S^-1 00, 01, 11) of a prior S."""
    l00 = np.sqrt(s00)
    l10 = s10 / l00
    l11 = np.sqrt(s11 - l10 * l10)
    x00 = 1.0 / l00
    x10 = (0.0 - l10 * x00) / l11
    x11 = 1.0 / l11
    return x00 * x00 + x10 * x10, x10 * x11, x11 * x11


def margins(info, t):
    """The smallest relative margin between a winning q and its runner-up, and between any decisive q and t."""
    win, thr = np.inf, np.inf
    for d in info:
        q = d["q"]
        if not np.isfinite(q):
            continue
        if not d["stop"] and np.isfinite(d["second"]):
            win = min(win, (q - d["second"]) / q)
        thr = min(thr, abs(q - t) / max(abs(q), t))
    return win, thr
