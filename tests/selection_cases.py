"""The bound on a double evaluation of the selection's q, the rule that decides where it is outside that bound, and the
constructed problems of the truth tests (tests/test_selection_truth.py on the CPU, tests/test_gpu_selection_truth.py on
the device).

The bound.  u = 2⁻⁵³, γ_k = k u / (1 - k u).  select_kernel (and tests/selection_ref.py) builds, for pick r, the
entries of a block Cholesky factorisation of 𝒮 = H P Hᵀ + R whose inputs are themselves rounded sums: the predicted
S_j (predict_kernel's func_Si: two levels of ten products), u = P H_iᵀ (ten products) and c_j = H_j u (ten more), so
every entry of 𝒮 the kernel meets is 𝒮 + E with |E| <= γ_20 (|H| |P| |H|ᵀ + R).  Each c_j then takes 2 r rank-one
downdates and C_j another 2 r; the factor's own quotients and square roots add at most four roundings.  With
K = 2 r + 24 the backward error of block Cholesky, |ΔS| <= γ_K |Ĝ| |Ĝ|ᵀ (Higham, Accuracy and Stability of Numerical
Algorithms, Thm. 10.3, applied per 2 x 2 block), and E together are
    |ΔS| <= γ_K (|H| |P| |H|ᵀ + R + |Ĝ| |Ĝ|ᵀ).
The conditioned C_j the kernel holds after r picks is the Schur complement of the picked block in 𝒮 + ΔS, so to first
order its error is W ΔS Wᵀ with W = [-Xᵀ, I], X = 𝒮_PP⁻¹ 𝒮_Pj, and
    |ΔC_j| <= γ_K ((|W| |H|) |P| (|W| |H|)ᵀ + |W| R |W|ᵀ + a aᵀ + |C_j|),   a = |X|ᵀ |L_P| + |𝒮_jP L_P⁻ᵀ|,
where L_P is the picked block's Cholesky factor and |C_j| the elementwise magnitude of the trailing block (its own
factor's |L_C| |L_C|ᵀ).  The 2 x 2 determinant then cancels: with δ the three entries of that bound,
    |Δq_j| <= (|c00| δ11 + |c11| δ00 + 2 |c10| δ10 + δ00 δ11 + δ10² + γ_3 (|c00 c11| + c10²)) / R_j² + γ_3 |q_j|,
the last two terms the determinant's and the quotient's own roundings.  The truth's factors stand in for the computed
ones (first order); every term is evaluated in float64 from the truth's longdouble factors.  Terms of order u² are
dropped: they stay below u γ_K cond(𝒮_PP) of the bound, < 1e-9 of it for every problem here.

The rule.  A decision is outside the bound when the truth's winner w has q_w - β_w > t and C00 - δ00 > 0, and every
other unpicked candidate that could qualify has q + β < q_w - β_w; a stop is outside the bound when every unpicked
candidate surely fails (C00 + δ00 <= 0, q + β <= t, or NaN).  Elsewhere a double evaluation may decide either way.

The problems.  One pinhole camera (CAM8: 320 x 240, fku = fkv = 256, principal point (160, 120) at the image centre,
kd1 = 0, sd = 1) at the identity pose at the origin: a feature at (x, y, z) with integer pixel (160 - 128 x, 120 - 128
y) at z = 2 has exact Jacobians, so mirror images of a feature give bit-equal q with C10 sign-flipped.  Every problem
is a map y and a covariance P, set directly on the device with no motion step."""
from dataclasses import dataclass

import numpy as np
from scipy.linalg import solve_triangular

from scenelib2_b200 import synth

NXV = 13
U = 2.0 ** -53
CAM8 = np.array([320.0, 240.0, 256.0, 256.0, 160.0, 120.0, 0.0, 1.0])
# the camera at the origin, q = 1, at rest but for a small angular rate: the motion model's dq/dω divides by |ω|
X_POSE = np.array([0.0, 0.0, 0.0, 1.0, 0, 0, 0, 0, 0, 0, 0, 0, 0.01])


def gamma(k):
    return k * U / (1.0 - k * U)


# ---- the bound -----------------------------------------------------------------------------------------------------
def q_bound(tr, picked, C, L, Y):
    """(V, 2): the bound β on |q_double - q| and δ00 on |C00_double - C00| of every candidate after `picked`."""
    V, r = tr.V, len(picked)
    f = tr.feats
    A, B, R = np.abs(tr.A[f]), np.abs(tr.B[f]), tr.R[f]
    aP = np.abs(tr.P)
    C64 = np.array(C, np.float64)
    c00, c10, c11 = C64[:, 0, 0], C64[:, 1, 0], C64[:, 1, 1]
    absC = np.abs(C64)
    yc = NXV + 3 * f[:, None] + np.arange(3)  # (V, 3)
    Pjj = aP[yc[:, :, None], yc[:, None, :]]  # (V, 3, 3)
    eye = np.eye(2)[None]
    if r == 0:
        h0, cols0 = A, np.arange(7)
        Rt = R[:, None, None] * eye
        chol = absC
    else:
        p = np.asarray(picked)
        L64, Y64 = np.array(L, np.float64), np.array(Y, np.float64)
        X = solve_triangular(L64, Y64, trans="T", lower=True, check_finite=False)  # 𝒮_PP⁻¹ 𝒮_P,all = L⁻ᵀ Y
        Xj = np.abs(X).reshape(2 * r, V, 2).transpose(1, 2, 0)  # (V, 2, 2r) = |X_j|ᵀ
        hx = Xj @ A[p].reshape(2 * r, 7) + A
        hp = np.einsum("vakc,kcm->vakm", Xj.reshape(V, 2, r, 2), B[p]).reshape(V, 2, 3 * r)
        h0 = np.concatenate([hx, hp], axis=2)
        cols0 = np.concatenate([np.arange(7), (NXV + 3 * f[p][:, None] + np.arange(3)).reshape(-1)])
        X4 = Xj.reshape(V, 2, r, 2)
        Rt = (X4 * R[p][None, None, :, None]).reshape(V, 2, 2 * r) @ Xj.transpose(0, 2, 1) + R[:, None, None] * eye
        a = Xj @ np.abs(L64) + np.abs(Y64).reshape(2 * r, V, 2).transpose(1, 2, 0)
        chol = a @ a.transpose(0, 2, 1) + absC
    P00 = aP[np.ix_(cols0, cols0)]
    Bt = B.transpose(0, 2, 1)
    quad = (h0 @ P00) @ h0.transpose(0, 2, 1)
    cross = (h0 @ aP[cols0][:, yc].transpose(1, 0, 2)) @ Bt
    quad += cross + cross.transpose(0, 2, 1) + (B @ Pjj) @ Bt
    M = gamma(2 * r + 24) * (quad + Rt + chol)
    d00, d10, d11 = M[:, 0, 0], M[:, 1, 0], M[:, 1, 1]
    with np.errstate(invalid="ignore"):
        q = (c00 * c11 - c10 * c10) / (R * R)
        beta = ((np.abs(c00) * d11 + np.abs(c11) * d00 + 2 * np.abs(c10) * d10 + d00 * d11 + d10 * d10
                 + gamma(3) * (np.abs(c00 * c11) + c10 * c10)) / (R * R) + gamma(3) * np.abs(q))
    return np.stack([beta, d00], axis=1)


def decided(d, t):
    """Whether the truth's decision d (selection_truth.Truth.run with the bound) lies outside the bound: any double
    evaluation within the bound decides as the truth does."""
    q, c00, live = d["q"], d["C"][:, 0], d["live"]
    beta, d00 = d["beta"][:, 0], d["beta"][:, 1]
    with np.errstate(invalid="ignore"):
        bad = np.isnan(q) | np.isnan(c00) | np.isnan(beta)
        sure_out = ~live | bad | (c00 + d00 <= 0) | (q + beta <= t)
        sure_in = live & ~bad & (c00 - d00 > 0) & (q - beta > t)
    maybe = live & ~sure_out & ~sure_in
    w = d["pick"]
    if w < 0:
        return not maybe.any()
    if not sure_in[w]:
        return False
    rivals = (sure_in | maybe)
    rivals[w] = False
    return not (q[rivals] + beta[rivals] >= q[w] - beta[w]).any()


# ---- the camera model of the problems (CPU side) -------------------------------------------------------------------
def measure(y):
    """h (nf, 2), dh_dxp (nf, 2, 7), dh_dy (nf, 2, 3), Rvar (nf,) of map points y seen by CAM8 from X_POSE: the
    camera model of sl2_model.cuh at kd1 = 0 (the quaternion columns are the derivative of the camera-frame point
    under a small rotation; with P_xx = 0 they multiply zeros)."""
    y = np.asarray(y, np.float64)
    f, u0, v0, sd = CAM8[2], CAM8[4], CAM8[5], CAM8[7]
    x_, y_, z_ = y[:, 0], y[:, 1], y[:, 2]
    h = np.stack([u0 - f * x_ / z_, v0 - f * y_ / z_], axis=1)
    J = np.zeros((len(y), 2, 3))
    J[:, 0, 0] = -f / z_
    J[:, 0, 2] = f * x_ / z_ / z_
    J[:, 1, 1] = -f / z_
    J[:, 1, 2] = f * y_ / z_ / z_
    dq = np.zeros((len(y), 3, 4))
    dq[:, :, 0] = 2 * y
    for k in range(3):
        e = np.zeros(3)
        e[k] = 1.0
        dq[:, :, k + 1] = -2 * np.cross(e, y)
    A = np.concatenate([-J, J @ dq], axis=2)
    dist = np.sqrt(((h - [u0, v0]) ** 2).sum(axis=1))
    R = (sd * (1.0 + dist / np.sqrt(u0 * u0 + v0 * v0))) ** 2
    return h, A, J, R


def cpu_inputs(pb):
    """The arrays select_kernel reads for problem pb, from the CPU model: P, S (nf, 4) column-major, A, B, R, and the
    trace rule's candidates (features ascending) with their ranks."""
    import selection_ref as sr
    _, A, B, R = measure(pb.y)
    nf = len(pb.y)
    S = np.zeros((nf, 4))
    for j in range(nf):
        cols = np.concatenate([np.arange(7), NXV + 3 * j + np.arange(3)])
        H = np.concatenate([A[j], B[j]], axis=1)
        with np.errstate(invalid="ignore"):
            Sj = H @ pb.P[np.ix_(cols, cols)] @ H.T + R[j] * np.eye(2)
        S[j] = [Sj[0, 0], Sj[1, 0], Sj[0, 1], Sj[1, 1]]
    feats, rho = sr.trace_candidates(S, np.ones(nf, bool))
    return pb.P, S, A, B, R, feats, rho


# ---- the problems ----------------------------------------------------------------------------------------------------
@dataclass
class Problem:
    name: str
    y: np.ndarray         # (nf, 3): camera frame = world (X_POSE)
    P: np.ndarray         # (n, n)
    n_select: int
    min_bits: float = 0.0
    exact: bool = False   # no correlation and exact arithmetic: every double evaluation decides like the truth

    @property
    def t(self):
        return 2.0 ** (2 * self.min_bits)

    @property
    def x(self):
        return np.concatenate([X_POSE, self.y.reshape(-1)])


def at_pixel(u, v, z=2.0):
    """The point at depth z seen at pixel (u, v)."""
    return np.array([(CAM8[4] - u) * z / CAM8[2], (CAM8[5] - v) * z / CAM8[3], z])


def grid_pixels(n, rng):
    """n distinct even pixels of the visible area (20 px from every edge), shuffled."""
    us, vs = np.arange(22, 298, 2), np.arange(22, 218, 2)
    allp = np.stack(np.meshgrid(us, vs), axis=-1).reshape(-1, 2)
    return allp[rng.permutation(len(allp))[:n]]


def yblock(P, j, v):
    P[NXV + 3 * j:NXV + 3 * j + 3, NXV + 3 * j:NXV + 3 * j + 3] = v


def zero_cov(nf):
    return np.zeros((NXV + 3 * nf, NXV + 3 * nf))


# the twins of the tie construction (lower index first, in order of decreasing q): across warps, a thread's first and
# second candidates, the warp edges and the 128-candidate stride
TIE_PAIRS = [(100, 130), (5, 133), (31, 32), (63, 64), (127, 128), (129, 250), (33, 97)]
RHO_PAIR = (10, 200)  # equal q, feature 200 the larger trace: the smaller rank wins over the smaller index


def ties(V=256, n_select=128):
    """Exact ties.  P_xx = 0, P_xy = 0, P_yy = c_j I: no pick changes another candidate's C.  Each TIE_PAIRS twin is the
    mirror image of its partner (x, y, or both negated about the principal point): bit-equal S up to the sign of C10,
    equal trace, so the lower index (its smaller rank) wins.  RHO_PAIR sits on the optical axis with S = diag(4, 4) and
    diag(2, 8) (q = 16 both, traces 8 and 10): the higher index has the smaller rank and wins.  Fillers have q below
    16; every eighth candidate has P_yy = 0 (q = 1 = t at min_bits 0: never picked)."""
    rng = np.random.default_rng(11)
    pix = grid_pixels(V, rng)
    y = np.stack([at_pixel(u, v) for u, v in pix])
    P = zero_cov(V)
    special = {j for pr in TIE_PAIRS for j in pr} | set(RHO_PAIR)
    for j in range(V):
        if j in special:
            continue
        yblock(P, j, 0.0 if j % 8 == 7 else np.eye(3) * rng.uniform(0.05, 2.0) / 16384.0)
    for k, (a, b) in enumerate(TIE_PAIRS):
        u, v = pix[a]
        mu, mv = (2 * 160 - u, v) if k % 3 == 0 else (u, 2 * 120 - v) if k % 3 == 1 else (2 * 160 - u, 2 * 120 - v)
        y[b] = at_pixel(mu, mv)
        c = 2.0 ** (12 - k) / 16384.0
        yblock(P, a, np.eye(3) * c)
        yblock(P, b, np.eye(3) * c)
    lo, hi = RHO_PAIR
    y[lo] = y[hi] = at_pixel(160, 120)
    yblock(P, lo, np.diag([3.0, 3.0, 1.0 * 16384]) / 16384.0)
    yblock(P, hi, np.diag([1.0, 7.0, 1.0 * 16384]) / 16384.0)
    return Problem("ties", y, P, n_select, 0.0, exact=True)


def degenerate(V=120, n_select=120):
    """Zero (P_yy = 0: C = R I, q = 1 = t), negative (C00 < 0 with a large q) and NaN C among valid candidates, at
    every warp position; no correlation."""
    rng = np.random.default_rng(12)
    y = np.stack([at_pixel(u, v) for u, v in grid_pixels(V, rng)])
    P = zero_cov(V)
    for j in range(V):
        k = (j + j // 32) % 4
        yblock(P, j, [0.0, -1e-2 * np.eye(3), np.nan * np.eye(3), rng.uniform(0.05, 8.0) / 16384 * np.eye(3)][k])
    return Problem("degenerate", y, P, n_select, 0.0, exact=True)


def random_map(rng, V, z=(1.5, 3.0)):
    pix = grid_pixels(V, rng).astype(np.float64) + rng.uniform(-0.9, 0.9, (V, 2))
    return np.stack([at_pixel(u, v, rng.uniform(*z)) for u, v in pix])


def dense(seed, V, n_select, min_bits=0.0, sig=1.0):
    """A dense SPD prior (synth.make_prior_covariance) over a random map, its standard deviations times sig."""
    rng = np.random.default_rng(1000 + seed)
    y = random_map(rng, V)
    P = synth.make_prior_covariance(rng, NXV + 3 * V) * sig * sig
    return Problem("dense%d_V%d" % (seed, V), y, P, n_select, min_bits)


def near_duplicates(delta, scale, min_bits, V=24, n_select=12):
    """Feature 1 is feature 0 moved by delta m, with P rows and columns equal to feature 0's, and both the map's largest
    variance; the rest of the map dense, its deviations times `scale`.  After one twin is picked the other's
    conditioned C is its own R plus R (M + R)⁻¹ M (M its share of H P Hᵀ): q in [1, 4), near 1 where M << R."""
    rng = np.random.default_rng(int(1e4 * min_bits) + int(-np.log10(delta)) * 7 + int(-np.log10(scale)))
    y = random_map(rng, V)
    y[1] = y[0] + [delta, 0.5 * delta, 0.0]
    P = synth.make_prior_covariance(rng, NXV + 3 * V) * scale * scale
    y0, y1 = slice(NXV, NXV + 3), slice(NXV + 3, NXV + 6)
    P[y0, :] *= 3.0
    P[:, y0] *= 3.0
    P[y1, :] = P[y0, :]
    P[:, y1] = P[:, y0]
    return Problem("near-dup d=%g s=%g b=%g" % (delta, scale, min_bits), y, P, n_select, min_bits)


def used_up(min_bits, V=256, n_select=128):
    """A map whose information runs out within the picks.  At min_bits 0 a settled map: camera and feature deviations
    1e-4 (m, and unit quaternion), so H P Hᵀ ~ 1e-3 px² against R >= 1 px² and every q starts near 1 = t.  At min_bits
    0.5 deviations 8e-3: the first picks have q of 300 and more, the shared camera term is used up pick by pick, and
    the last of about a hundred picks has q within 3e-3 of t = 2 before the selection stops just below it."""
    rng = np.random.default_rng(13)
    y = random_map(rng, V)
    sig = 1e-4 if min_bits == 0.0 else 8e-3
    P = synth.make_prior_covariance(rng, NXV + 3 * V, sig_r=sig, sig_q=sig, sig_v=sig, sig_w=sig, sig_y=sig)
    return Problem("used-up b=%g" % min_bits, y, P, n_select, min_bits)


def stretched(cond, V=48, n_select=16):
    """The camera's uncertainty stretched along one direction of (r, q): P_xx = 1e-8 I + lam v vᵀ with lam set so
    that cond(𝒮) is about `cond`; the map's own variance 1e-6 m², uncorrelated.  The first pick collapses every other
    candidate along v."""
    rng = np.random.default_rng(int(np.log10(cond)))
    y = random_map(rng, V)
    P = zero_cov(V)
    v = rng.standard_normal(7)
    v /= np.linalg.norm(v)
    P[:7, :7] = 1e-8 * np.eye(7) + cond / 16384.0 * np.outer(v, v)
    for j in range(V):
        yblock(P, j, 1e-6 * np.eye(3))
    return Problem("stretched cond=%g" % cond, y, P, n_select)


def decades(V=96, n_select=40):
    """P_yy over 12 decades in one map (1e-14 .. 1e-2 m²), a small dense camera block (1e-6) and correlation between
    neighbouring features."""
    rng = np.random.default_rng(14)
    y = random_map(rng, V)
    n = NXV + 3 * V
    P = zero_cov(V)
    P[:7, :7] = 1e-6 * (np.eye(7) + 0.3 * np.ones((7, 7)))
    sd = np.sqrt(10.0 ** (-14 + 12 * rng.permutation(V) / (V - 1)))
    for j in range(V):
        yblock(P, j, sd[j] ** 2 * np.eye(3))
        if j:
            c = 0.4 * sd[j] * sd[j - 1] * np.eye(3)
            P[NXV + 3 * j:NXV + 3 * j + 3, NXV + 3 * j - 3:NXV + 3 * j] = c
            P[NXV + 3 * j - 3:NXV + 3 * j, NXV + 3 * j:NXV + 3 * j + 3] = c
    assert P.shape == (n, n)
    return Problem("decades", y, P, n_select)


def constructions():
    """Every constructed problem (the CPU runs each; the device runs each as well)."""
    out = [ties(), degenerate()]
    for delta in (1e-3, 1e-6, 1e-9):
        for scale, bits in ((1e-2, 0.0), (1e-4, 0.0), (1.0, 0.5), (1.0, 1.0), (0.3, 0.5)):
            out.append(near_duplicates(delta, scale, bits))
    out += [used_up(0.0), used_up(0.5)]
    out += [stretched(c) for c in (1e4, 1e6, 1e8, 1e10)]
    out.append(decades())
    return out
