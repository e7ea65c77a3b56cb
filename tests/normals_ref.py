"""The patch normal alignment (include/sl2b200.h, sl2_set_stream_normals; csrc/normals.cu normals_kernel and
csrc/sl2_model.cuh patch_basis, patch_normal, patch_warp_forward) restated in NumPy, one IEEE double operation at a time
in the kernel's order (NumPy's element-wise operations and Python's float operations are correctly rounded and never
fused), vectorised over the template's pixels, with the warp's lane partial sums and xor-shuffle tree.  Also the warp
of a feature through its estimated normal (warp_kernel with normals on)."""
import math

import numpy as np

from camera_ref import camera_points, project_point, rrw
from warp_ref import adjugate, sample, unproject_point

LANES = 32


def _dot(a, b):
    return ((0.0 + a[0] * b[0]) + a[1] * b[1]) + a[2] * b[2]


def _mat_vec(M, v):
    return [((0.0 + M[i][0] * v[0]) + M[i][1] * v[1]) + M[i][2] * v[2] for i in range(3)]


def basis(xo, y):
    """patch_basis: nW0 = xo[0:3] - y, E1 = camera o's x axis made orthogonal to nW0 and scaled to |nW0|, E2 =
    nW0 x E1 / |nW0| (lists of floats)."""
    Ro = rrw(xo)
    n0 = [float(xo[i]) - float(y[i]) for i in range(3)]
    nn = _dot(n0, n0)
    pr = _dot(Ro[0], n0) / nn
    q = [Ro[0][i] - pr * n0[i] for i in range(3)]
    ln = math.sqrt(nn)
    sc = ln / math.sqrt(_dot(q, q))
    E1 = [q[i] * sc for i in range(3)]
    E2 = [(n0[1] * E1[2] - n0[2] * E1[1]) / ln, (n0[2] * E1[0] - n0[0] * E1[2]) / ln,
          (n0[0] * E1[1] - n0[1] * E1[0]) / ln]
    return n0, E1, E2


def normal(b, ta, tb):
    """patch_normal: nW(theta) = (nW0 + a E1) + b E2, nW0 itself at theta = (0, 0)."""
    n0, E1, E2 = b
    if ta == 0.0 and tb == 0.0:
        return list(n0)
    return [(n0[i] + ta * E1[i]) + tb * E2[i] for i in range(3)]


def project_jac(cam8, zc):
    """project: the pixels g and J = dh/dz of the camera-frame points zc (3 arrays), as sl2_model.cuh forms them."""
    fku, fkv, u0, v0, kd1 = (float(v) for v in cam8[2:7])
    z0, z1, z2 = zc
    uc = ((-fku) * z0) / z2
    vc = ((-fkv) * z1) / z2
    factor = np.sqrt(1.0 + (2.0 * kd1) * (uc * uc + vc * vc))
    g = [uc / factor + u0, vc / factor + v0]
    fku_yz, fkv_yz = fku / z2, fkv / z2
    zero = np.zeros_like(z2)
    du = [[-fku_yz, zero, (fku_yz * z0) / z2], [zero, -fkv_yz, (fkv_yz * z1) / z2]]
    dh = [[uc * uc, uc * vc], [vc * uc, vc * vc]]
    r2 = dh[0][0] + dh[1][1]
    distor = 1.0 + (2.0 * kd1) * r2
    d12 = np.sqrt(distor)
    d32 = d12 * distor
    scale = (-2.0 * kd1) / d32
    dh = [[dh[i][j] * scale for j in range(2)] for i in range(2)]
    dh[0][0] = dh[0][0] + 1.0 / d12
    dh[1][1] = dh[1][1] + 1.0 / d12
    J = [[(0.0 + dh[i][0] * du[0][j]) + dh[i][1] * du[1][j] for j in range(3)] for i in range(2)]
    return g, J


def forward(cam8, B, y, xo, x, theta):
    """patch_warp_forward of every template pixel (row r, column c; arrays of B * B in k = r B + c order): g (2),
    Jw (2), t_a, t_b and the validity (t finite and > 0, zc[2] > 0), for the feature y (3) first seen from xo (7), its
    tilt theta, into the camera at x (7)."""
    half = (B - 1) // 2
    y = [float(v) for v in y]
    xo = [float(v) for v in xo]
    x = [float(v) for v in x]
    Ro, R = rrw(xo), rrw(x)
    A = adjugate(Ro)
    ho = project_point(cam8, camera_points(xo, y))[0]
    b = basis(xo, y)
    nW = normal(b, float(theta[0]), float(theta[1]))
    yx = [y[i] - xo[i] for i in range(3)]
    nd, nE1, nE2 = _dot(nW, yx), _dot(b[1], yx), _dot(b[2], yx)
    r, c = np.divmod(np.arange(B * B), B)
    with np.errstate(all="ignore"):
        c0, c1 = unproject_point(cam8, ho[0] + (c - half).astype(np.float64), ho[1] + (r - half).astype(np.float64))
        cv = [c0, c1, np.ones_like(c0)]
        dO = _mat_vec(A, cv)
        den = _dot(nW, dO)
        t = nd / den
        e = [(xo[i] + t * dO[i]) - x[i] for i in range(3)]
        zc = _mat_vec(R, e)
        g, J = project_jac(cam8, zc)
        w = _mat_vec(R, dO)
        Jw = [(J[i][0] * w[0] + J[i][1] * w[1]) + J[i][2] * w[2] for i in range(2)]
        ta = (nE1 - t * _dot(b[1], dO)) / den
        tb = (nE2 - t * _dot(b[2], dO)) / den
        valid = np.isfinite(t) & (t > 0.0) & (zc[2] > 0.0)
    return dict(g=g, Jw=Jw, ta=ta, tb=tb, valid=valid, nW=nW, b=b)


def warp_sum(v):
    """The kernel's reduction of the per-pixel values v (k order): lane l sums k = l + 32 j in ascending j from 0.0,
    then the xor-shuffle tree over offsets 16, 8, 4, 2, 1."""
    n = v.size
    pad = np.zeros(-(-n // LANES) * LANES)
    pad[:n] = v
    P = np.zeros(LANES)
    for j in range(pad.size // LANES):
        P = P + pad[j * LANES:(j + 1) * LANES]
    lanes = np.arange(LANES)
    for off in (16, 8, 4, 2, 1):
        P = P + P[lanes ^ off]
    return float(P[0])


def frame_sample(img, u, v):
    """Bilinear sample (not rounded) of the image img (H x W u8 or wider rows) at (u, v) arrays inside it."""
    x0 = np.floor(u).astype(np.int64)
    y0 = np.floor(v).astype(np.int64)
    fx = u - x0.astype(np.float64)
    fy = v - y0.astype(np.float64)
    I = img.astype(np.float64)
    top = (1.0 - fx) * I[y0, x0] + fx * I[y0, x0 + 1]
    bot = (1.0 - fx) * I[y0 + 1, x0] + fx * I[y0 + 1, x0 + 1]
    return (1.0 - fy) * top + fy * bot


def evaluate(cam8, W, H, img, T, y, xo, x, phi, variant=None):
    """align_eval at phi: (valid, sums) with sums the 21 of J^T J (upper triangle row by row), the 6 of J^T e and e^2.
    `variant` names a deliberately broken copy (the checks of tests/test_normals.py must catch each)."""
    B = T.shape[0]
    fw = forward(cam8, B, y, xo, x, phi[:2])
    nW, b = fw["nW"], fw["b"]
    ry = [float(x[i]) - float(y[i]) for i in range(3)]
    if not (_dot(nW, b[0]) > 0.0 and _dot(nW, ry) > 0.0):
        return False, None
    with np.errstate(all="ignore"):
        tu = -phi[2] if variant == "tau_sign" else phi[2]
        tv = -phi[3] if variant == "tau_sign" else phi[3]
        gu, gv = fw["g"][0] + tu, fw["g"][1] + tv
        ok = fw["valid"] & (gu >= 1.0) & (gu < float(W - 2)) & (gv >= 1.0) & (gv < float(H - 2))
    if not ok.all():
        return False, None
    Tk = np.asarray(T, np.float64).reshape(-1)
    I = frame_sample(img, gu, gv)
    if variant == "template_gradient":  # the gradient of the template, not of the frame
        Tg = np.pad(np.asarray(T, np.float64), 1, mode="edge")
        r, c = np.divmod(np.arange(B * B), B)
        Iu = (Tg[r + 1, c + 2] - Tg[r + 1, c]) * 0.5
        Iv = (Tg[r + 2, c + 1] - Tg[r, c + 1]) * 0.5
    else:
        Iu = (frame_sample(img, gu + 1.0, gv) - frame_sample(img, gu - 1.0, gv)) * 0.5
        Iv = (frame_sample(img, gu, gv + 1.0) - frame_sample(img, gu, gv - 1.0)) * 0.5
    e = (phi[4] * I + phi[5]) - Tk
    ag = phi[4] * (Iu * fw["Jw"][0] + Iv * fw["Jw"][1])
    if variant == "tau_sign":
        Jr = [ag * fw["ta"], ag * fw["tb"], -(phi[4] * Iu), -(phi[4] * Iv), I, np.ones_like(I)]
    else:
        Jr = [ag * fw["ta"], ag * fw["tb"], phi[4] * Iu, phi[4] * Iv, I, np.ones_like(I)]
    sums = [warp_sum(Jr[p] * Jr[q]) for p in range(6) for q in range(p, 6)]
    sums += [warp_sum(Jr[p] * e) for p in range(6)]
    sums.append(warp_sum(e * e))
    return True, sums


def tri(p, q):
    return p * 6 - p * (p - 1) // 2 + (q - p)


def system(sums, phi, th0, Li, w2, variant=None):
    """align_system: H (21, upper triangle), G (6) and the cost at phi."""
    H = [s * w2 for s in sums[:21]]
    G = [s * w2 for s in sums[21:27]]
    da, db = phi[0] - th0[0], phi[1] - th0[1]
    pa, pb = Li[0] * da + Li[1] * db, Li[1] * da + Li[2] * db
    if variant == "no_prior":
        return H, G, sums[27] * w2
    H[0] = H[0] + Li[0]
    H[1] = H[1] + Li[1]
    H[6] = H[6] + Li[2]
    G[0] = G[0] + pa
    G[1] = G[1] + pb
    return H, G, sums[27] * w2 + (da * pa + db * pb)


def chol6(H):
    """chol6: the lower factor (6 x 6 nested lists) or None at a pivot that is not > 0."""
    L = [[0.0] * 6 for _ in range(6)]
    for j in range(6):
        s = H[tri(j, j)]
        for k in range(j):
            s = s - L[j][k] * L[j][k]
        if not s > 0.0:
            return None
        L[j][j] = math.sqrt(s)
        for i in range(j + 1, 6):
            t = H[tri(j, i)]
            for k in range(j):
                t = t - L[i][k] * L[j][k]
            L[i][j] = t / L[j][j]
    return L


def solve(L, G):
    u = [0.0] * 6
    for p in range(6):
        t = G[p]
        for k in range(p):
            t = t - L[p][k] * u[k]
        u[p] = t / L[p][p]
    v = [0.0] * 6
    for p in range(5, -1, -1):
        t = u[p]
        for k in range(p + 1, 6):
            t = t - L[k][p] * v[k]
        v[p] = t / L[p][p]
    return v


def marginal(L, H=None, variant=None):
    """The theta block of H^-1 from L^-1's first two columns: (S_aa, S_ab, S_bb)."""
    if variant == "theta_block":  # (H_thth)^-1: the conditional, not the marginal
        a, b, d = H[0], H[1], H[6]
        det = a * d - b * b
        return d / det, (-b) / det, a / det
    cs = []
    for m in range(2):
        c = [0.0] * 6
        for p in range(6):
            t = 1.0 if p == m else 0.0
            for k in range(p):
                t = t - L[p][k] * c[k]
            c[p] = t / L[p][p]
        cs.append(c)
    saa = sab = sbb = 0.0
    for k in range(6):
        saa = saa + cs[0][k] * cs[0][k]
        sab = sab + cs[0][k] * cs[1][k]
        sbb = sbb + cs[1][k] * cs[1][k]
    return saa, sab, sbb


def align(cam8, img, T, y, xo, x, z, theta, cov, prm, variant=None):
    """One feature's alignment (normals_kernel for a matched feature).  cam8: the stream's camera (its width x height
    bound the samples); img: the step's frame (rows of at least the stream's width); T: the stored B x B template;
    y (3), xo (7), x (7: the updated pose r+, q+), z (2) the match the update used; theta (2), cov (3) the estimate;
    prm = (max_iterations, sigma0, sigma_i, sigma_step).  Returns (theta, cov, accepted (0/1 added to count), status)
    and dict(phi, H (21), Li, w2) at the accepted phi (None when nothing was accepted)."""
    W, H = int(cam8[0]), int(cam8[1])
    max_it, _, sigma_i, sigma_step = prm
    hp = project_point(cam8, camera_points(x, y))[0]
    th0 = [float(theta[0]), float(theta[1])]
    ss = sigma_step * sigma_step
    Saa, Sab, Sbb = float(cov[0]) + ss, float(cov[1]), float(cov[2]) + ss
    det = Saa * Sbb - Sab * Sab
    Li = [Sbb / det, (-Sab) / det, Saa / det]
    w2 = 1.0 / (sigma_i * sigma_i)
    phi = [th0[0], th0[1], float(z[0]) - float(hp[0]), float(z[1]) - float(hp[1]), 1.0, 0.0]
    ok, sums = evaluate(cam8, W, H, img, T, y, xo, x, phi, variant)
    if not ok:
        return (th0, [float(v) for v in cov], 0, 3), None
    Hm, G, cost = system(sums, phi, th0, Li, w2, variant)
    accepted = 0
    for _ in range(int(max_it)):
        L = chol6(Hm)
        if L is None:
            break
        v = solve(L, G)
        nphi = [phi[p] - v[p] for p in range(6)]
        ok, sums = evaluate(cam8, W, H, img, T, y, xo, x, nphi, variant)
        if not ok:
            break
        nH, nG, ncost = system(sums, nphi, th0, Li, w2, variant)
        if not ncost < cost:
            break
        phi, Hm, G, cost = nphi, nH, nG, ncost
        accepted += 1
    L = chol6(Hm) if accepted else None
    if L is None:
        return (th0, [float(v) for v in cov], 0, 2), None
    return ([phi[0], phi[1]], list(marginal(L, Hm, variant)), 1, 1), dict(phi=phi, H=Hm, Li=Li, w2=w2, th0=th0)


def warp_source(cam8, B, y, xo, xp, theta):
    """src (B, B, 2) positions in the stored template of every output pixel (row a, column b) of a feature warped
    through nW(theta) at the pose xp, and their validity (B, B) (patch_warp_setup with theta, patch_warp_source)."""
    half = (B - 1) // 2
    y = [float(v) for v in y]
    xo = [float(v) for v in xo]
    xp = [float(v) for v in xp]
    R, Ro = rrw(xp), rrw(xo)
    A = adjugate(R)
    h = project_point(cam8, camera_points(xp, y))[0]
    ho = project_point(cam8, camera_points(xo, y))[0]
    d = [y[i] - xp[i] for i in range(3)]
    nW = normal(basis(xo, y), float(theta[0]), float(theta[1]))
    num = _dot(nW, d)
    a, b = np.mgrid[0:B, 0:B]
    with np.errstate(all="ignore"):
        c0, c1 = unproject_point(cam8, h[0] + (b - half).astype(np.float64), h[1] + (a - half).astype(np.float64))
        dW = _mat_vec(A, [c0, c1, np.ones_like(c0)])
        t = num / _dot(nW, dW)
        e = [(xp[i] + t * dW[i]) - xo[i] for i in range(3)]
        zo = np.stack(_mat_vec(Ro, e), axis=-1)
        g = project_point(cam8, zo.reshape(-1, 3)).reshape(B, B, 2)
        src = np.stack([(g[..., 0] - ho[0]) + float(half), (g[..., 1] - ho[1]) + float(half)], axis=-1)
        valid = np.isfinite(t) & (t > 0.0) & (zo[..., 2] > 0.0) & np.isfinite(src).all(axis=-1)
    return src, valid


def warp_template(cam8, T, y, xo, xp, theta):
    """The warped template (B, B) u8 and its valid flag of a feature warped through nW(theta) (warp_kernel of a stream
    with normals on; theta = 0 is warp_ref.warp_template)."""
    T = np.asarray(T, np.uint8)
    src, valid = warp_source(cam8, T.shape[0], y, xo, xp, theta)
    if not valid.all():
        return T.copy(), 0
    return sample(T, src), 1
