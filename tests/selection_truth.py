"""The greedy mutual-information selection (include/sl2b200.h, sl2_set_stream_selection) from its definition, in
extended precision, sharing nothing with select_kernel's algebra but the candidate list.

The definition: the candidates' joint innovation covariance is 𝒮 = H P Hᵀ + R, H the dense 2V x n stack of their
measurement Jacobians (dh_dxp on the camera pose, dh_dy on the feature) and R = diag(Rvar_j I2).  After the picks
p_1 .. p_r, candidate j's conditional innovation covariance is the Schur complement of the picked block,
C_j = 𝒮_jj - 𝒮_jP 𝒮_PP⁻¹ 𝒮_Pj, and q_j = det C_j / Rvar_j².  The next pick is the unpicked j of largest q with
C_j[0, 0] > 0 and q_j > t (t = exp2(2 min_bits)), ties to the smaller trace rank rho, then the smaller candidate index;
none qualifying, or min(n_select, V) picked, ends the selection.

P is read as the kernel reads it.  The filter's P is bit-symmetric except its camera block P_xx after a motion step,
whose triangles may differ by the step's rounding until the update symmetrises them (update.cu, upd_finish).  The
kernel reads the block of 𝒮 between a candidate and an earlier pick as H_cand P H_pickᵀ (the candidate's rows of P)
and the lower entry of every 2 x 2 block (C10 = S(1, 0)); the truth reads the same blocks, so it states the same
operation on any P and equals the textbook definition on a symmetric one.

Every pick recomputes 𝒮_PP's Cholesky factor and the solve against 𝒮_P,U from scratch.  𝒮's blocks are formed from
each candidate's ten nonzero Jacobian columns, so that a NaN in one feature's P block stays in that feature's own
diagonal block, as it does in the kernel.  The same code runs in np.longdouble (x86: 64-bit significand) and on
mpmath numbers (object arrays); the caller picks the number type.  The bound on a double evaluation
(tests/selection_cases.py) is evaluated from the factors each pick leaves."""
import mpmath
import numpy as np

NXV = 13


def columns(feats):
    """The ten state columns of each candidate's measurement: (V, 10)."""
    feats = np.asarray(feats, np.int64)
    cols = np.empty((len(feats), 10), np.int64)
    cols[:, :7] = np.arange(7)
    cols[:, 7:] = NXV + 3 * feats[:, None] + np.arange(3)
    return cols


def joint_covariance(P, A, B, R, feats, num):
    """𝒮 = H P Hᵀ + R of the candidates as (V, 2, V, 2) in the number type `num` (np.longdouble or object for
    mpmath).  Only the entries of P in the candidates' columns are read."""
    cols = columns(feats)
    V = len(cols)
    cv = _conv(num)
    Hc = cv(np.concatenate([A[feats], B[feats]], axis=2))  # (V, 2, 10)
    Pr = cv(P[cols[:, :, None], cols.reshape(-1)[None, None, :]])  # (V, 10, 10 V): P[cols_a, cols_b]
    HP = np.matmul(Hc, Pr).reshape(V, 2, V, 10)  # H_a P[cols_a, cols_b]
    S = np.matmul(HP.transpose(0, 2, 1, 3), Hc.transpose(0, 2, 1)[None]).transpose(0, 2, 1, 3)  # (V, 2, V, 2)
    Rv = cv(R[feats])
    for j in range(V):
        for a in range(2):
            S[j, a, j, a] = S[j, a, j, a] + Rv[j]
    return S


def _conv(num):
    if num is object:
        return lambda a: np.vectorize(lambda v: mpmath.mpf(float(v)), otypes=[object])(np.asarray(a, np.float64))
    return lambda a: np.asarray(a, np.float64).astype(num)


def _sqrt(num):
    return np.vectorize(mpmath.sqrt, otypes=[object]) if num is object else np.sqrt


def cholesky(M, num):
    """Lower L with L Lᵀ = M (M symmetric positive definite), column by column."""
    k = M.shape[0]
    sqrt = _sqrt(num)
    L = np.zeros_like(M)
    for c in range(k):
        d = M[c, c] - np.dot(L[c, :c], L[c, :c]) if c else M[c, c]
        L[c, c] = sqrt(np.array([d], dtype=M.dtype))[0]
        if c + 1 < k:
            off = M[c + 1:, c] - (L[c + 1:, :c] @ L[c, :c] if c else 0)
            L[c + 1:, c] = off / L[c, c]
    return L


def forward(L, Bm):
    """L⁻¹ Bm by forward substitution, row by row."""
    Y = np.zeros_like(Bm)
    for k in range(L.shape[0]):
        acc = Bm[k] - (L[k, :k] @ Y[:k] if k else 0)
        Y[k] = acc / L[k, k]
    return Y


class Truth:
    """The greedy selection of one candidate list from its definition.  P (n, n) symmetric, A (nf, 2, 7), B (nf, 2, 3),
    R (nf,), feats (V,) the candidates' features ascending, rho (V,) their trace ranks.  num: np.longdouble or object
    (mpmath at the current mpmath.mp.dps)."""

    def __init__(self, P, A, B, R, feats, rho, num=np.longdouble):
        self.P, self.A, self.B, self.R = P, A, B, R
        self.feats = np.asarray(feats, np.int64)
        self.rho = np.asarray(rho, np.int64)
        self.num = num
        self.S = joint_covariance(P, A, B, R, self.feats, num)
        self.V = len(self.feats)

    def conditioned(self, picked):
        """C_j (V, 2, 2) of every candidate given the picked candidate indices (pick order), with the factors the
        bound needs: L = chol(𝒮_PP) and Y = L⁻¹ 𝒮_P,all.  Picked candidates' rows are those of the
        identity-conditioned formula too and are ignored by the caller."""
        V, S = self.V, self.S
        Sjj = np.stack([S[j, :, j, :] for j in range(V)])
        if not picked:
            return Sjj, None, None
        p = np.asarray(picked)
        Spp = S[p][:, :, p, :].reshape(2 * len(p), 2 * len(p))
        Spa = S[:, :, p, :].transpose(2, 3, 0, 1).reshape(2 * len(p), 2 * V)  # (𝒮_all,P)ᵀ: candidates as rows
        L = cholesky(Spp, self.num)
        Y = forward(L, Spa)
        Yj = Y.reshape(2 * len(p), V, 2).transpose(1, 0, 2)  # (V, 2r, 2)
        C = Sjj - np.matmul(Yj.transpose(0, 2, 1), Yj)
        return C, L, Y

    def q_of(self, C):
        Rv = _conv(self.num)(self.R[self.feats])
        return (C[:, 0, 0] * C[:, 1, 1] - C[:, 1, 0] * C[:, 1, 0]) / (Rv * Rv)

    def run(self, n_select, t, follow=None, bound=None):
        """The selection: one dict per decision with the truth's own choice `pick` (candidate index, -1 to stop),
        `q` (V,) float64 of the unpicked (NaN for picked), `C` (V, 3) float64 (C00, C10, C11), and, with `bound`
        (a function of this truth, the picks and the factors; tests/selection_cases.py), `beta` (V,) the bound on
        |q_double - q|.  With `follow` (candidate indices) the picks are conditioned on those, in that order, instead
        of the truth's own; its length, the stop included, sets the number of decisions."""
        nmax = min(int(n_select), self.V)
        picked, out = [], []
        tt = _conv(self.num)(np.array([t]))[0]
        for r in range(nmax + 1):
            C, L, Y = self.conditioned(picked)
            q = self.q_of(C)
            live = np.ones(self.V, bool)
            live[picked] = False
            pick = -1
            if r < nmax:
                best = None
                for j in np.flatnonzero(live):
                    c00, qj = C[j, 0, 0], q[j]
                    if not (c00 > 0 and qj > tt):
                        continue
                    key = (qj, -self.rho[j], -j)
                    if best is None or key > best[0]:
                        best = (key, j)
                pick = -1 if best is None else int(best[1])
            d = dict(pick=pick, picked=list(picked), live=live,
                     q=np.where(live, np.array(q, np.float64), np.nan),
                     C=np.stack([np.array(C[:, 0, 0], np.float64), np.array(C[:, 1, 0], np.float64),
                                 np.array(C[:, 1, 1], np.float64)], axis=1),
                     qx=q, Cx=C)
            if bound is not None:
                d["beta"] = bound(self, picked, C, L, Y)
            out.append(d)
            if r == nmax:
                out.pop()  # min(n_select, V) picked: no decision left
                break
            nxt = pick if follow is None else (follow[r] if r < len(follow) else -1)
            if nxt < 0:
                break
            picked.append(int(nxt))
        return out


def margins(decisions, t):
    """(winner vs runner-up, decisive q vs t) relative margins of the truth's decisions: the smallest of each."""
    win, thr = np.inf, np.inf
    for d in decisions:
        q = d["q"]
        ok = d["live"] & (d["C"][:, 0] > 0) & (q > t)
        if d["pick"] >= 0:
            qw = q[d["pick"]]
            others = np.delete(q, d["pick"])[np.delete(ok, d["pick"])]
            if len(others):
                win = min(win, (qw - others.max()) / qw)
            thr = min(thr, (qw - t) / max(qw, t))
        else:
            cand = q[d["live"] & (d["C"][:, 0] > 0) & ~np.isnan(q)]
            if len(cand):
                thr = min(thr, abs(cand.max() - t) / max(abs(cand.max()), t))
    return win, thr

