"""The patch normal model stated from its definition in extended precision (mpmath, 50 digits): where a template
pixel of the camera at xo lands in the camera at x through the plane of normal nW(theta) through y, as the
plane-induced homography K (R + t n^T / d) K^-1 for cameras without distortion (kd1 = 0) and by casting the pixel's
ray onto the plane for distorted ones; its derivative in theta by mpmath's differentiation; the posterior covariance
as the theta block of the inverted Hessian; and the alignment's cost, whose gradient vanishes at an accepted
iterate."""
import mpmath as mp
import numpy as np

import normals_ref

mp.mp.dps = 50


def _R(q):
    """The rotation world -> camera of the pose quaternion q (w, x, y, z) = qWR, at any norm (pose_RRW)."""
    w, x, y, z = (mp.mpf(float(v)) for v in q)
    n2 = w * w + x * x + y * y + z * z
    w, x, y, z = w / n2, -x / n2, -y / n2, -z / n2
    return mp.matrix([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                      [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                      [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def _vec(v):
    return mp.matrix([mp.mpf(float(t)) for t in v])


def _project(cam8, zc):
    fku, fkv, u0, v0, kd1 = (mp.mpf(float(v)) for v in cam8[2:7])
    uc, vc = -fku * zc[0] / zc[2], -fkv * zc[1] / zc[2]
    f = mp.sqrt(1 + 2 * kd1 * (uc * uc + vc * vc))
    return uc / f + u0, vc / f + v0


def _unproject(cam8, u, v):
    fku, fkv, u0, v0, kd1 = (mp.mpf(float(t)) for t in cam8[2:7])
    c0, c1 = u - u0, v - v0
    f = mp.sqrt(1 - 2 * kd1 * (c0 * c0 + c1 * c1))
    return mp.matrix([(c0 / f) / -fku, (c1 / f) / -fkv, 1])


def normal(y, xo, theta):
    """nW(theta) from the basis' definition: E1 = camera o's x axis orthogonal to nW0 with |E1| = |nW0|,
    E2 = nW0 x E1 / |nW0|."""
    n0 = _vec(xo[:3]) - _vec(y)
    Ro = _R(xo[3:7])
    r0 = mp.matrix([Ro[0, 0], Ro[0, 1], Ro[0, 2]])
    q = r0 - (mp.fdot(r0, n0) / mp.fdot(n0, n0)) * n0
    L = mp.sqrt(mp.fdot(n0, n0))
    E1 = q * (L / mp.sqrt(mp.fdot(q, q)))
    E2 = mp.matrix([n0[1] * E1[2] - n0[2] * E1[1], n0[2] * E1[0] - n0[0] * E1[2], n0[0] * E1[1] - n0[1] * E1[0]]) / L
    return n0 + theta[0] * E1 + theta[1] * E2


def pixel_points(cam8, B, y, xo):
    """The template's pixels p_o = ho + (c - HALF, r - HALF), k = r B + c."""
    half = (B - 1) // 2
    zo = _R(xo[3:7]) * (_vec(y) - _vec(xo[:3]))
    ho = _project(cam8, zo)
    return [(ho[0] + (k % B - half), ho[1] + (k // B - half)) for k in range(B * B)]


def forward_homography(cam8, B, y, xo, x, theta):
    """g (B * B, 2) through H = K (R_co + t_co n_o^T / d) K^-1, K of a camera without distortion."""
    assert float(cam8[6]) == 0.0
    fku, fkv, u0, v0 = (mp.mpf(float(v)) for v in cam8[2:6])
    K = mp.matrix([[-fku, 0, u0], [0, -fkv, v0], [0, 0, 1]])
    Ro, Rc = _R(xo[3:7]), _R(x[3:7])
    R_co = Rc * Ro ** -1
    t_co = Rc * (_vec(xo[:3]) - _vec(x[:3]))
    nW = normal(y, xo, [mp.mpf(float(t)) for t in theta])
    n_o = (Ro ** -1).T * nW  # the plane's normal in camera-o coordinates: n^T X = n_o^T X_o with X_o = Ro (X - xo)
    d = mp.fdot(n_o, Ro * (_vec(y) - _vec(xo[:3])))
    H = K * (R_co + t_co * n_o.T / d) * K ** -1
    out = []
    for p in pixel_points(cam8, B, y, xo):
        h = H * mp.matrix([p[0], p[1], 1])
        out.append((h[0] / h[2], h[1] / h[2]))
    return out


def forward_rays(cam8, B, y, xo, x, theta, pixels=None):
    """g (B * B, 2) by casting each pixel's ray of camera o onto the plane and projecting into camera x."""
    theta = [t if isinstance(t, mp.mpf) else mp.mpf(float(t)) for t in theta]
    nW = normal(y, xo, theta)
    Ro, Rc = _R(xo[3:7]), _R(x[3:7])
    yv, o, r = _vec(y), _vec(xo[:3]), _vec(x[:3])
    out = []
    for p in (pixel_points(cam8, B, y, xo) if pixels is None else pixels):
        dW = Ro ** -1 * _unproject(cam8, p[0], p[1])
        t = mp.fdot(nW, yv - o) / mp.fdot(nW, dW)
        out.append(_project(cam8, Rc * (o + t * dW - r)))
    return out


def warp_source(cam8, B, y, xo, xp, theta):
    """The warp's direction, frame -> template: src (B * B, 2) in the stored template of output pixel (row a, column
    b), k = a B + b, of the camera at xp: the pixel h + (b - HALF, a - HALF) cast onto the plane of normal nW(theta)
    through y and projected into camera o, minus ho, plus (HALF, HALF)."""
    half = (B - 1) // 2
    th = [mp.mpf(float(t)) for t in theta]
    nW = normal(y, xo, th)
    Rp, Ro = _R(xp[3:7]), _R(xo[3:7])
    yv, o, r = _vec(y), _vec(xo[:3]), _vec(xp[:3])
    h = _project(cam8, Rp * (yv - r))
    ho = _project(cam8, Ro * (yv - o))
    out = []
    for k in range(B * B):
        dW = Rp ** -1 * _unproject(cam8, h[0] + (k % B - half), h[1] + (k // B - half))
        t = mp.fdot(nW, yv - r) / mp.fdot(nW, dW)
        g = _project(cam8, Ro * (r + t * dW - o))
        out.append((g[0] - ho[0] + half, g[1] - ho[1] + half))
    return out


def dg_dtheta(cam8, B, y, xo, x, theta, k):
    """d g_k / d(a, b) by mpmath's differentiation of the ray-cast map: ((dgu/da, dgv/da), (dgu/db, dgv/db))."""
    p = pixel_points(cam8, B, y, xo)[k]
    a0, b0 = mp.mpf(float(theta[0])), mp.mpf(float(theta[1]))
    out = []
    for which in range(2):
        def g(t, j):
            th = [t, b0] if which == 0 else [a0, t]
            return forward_rays(cam8, B, y, xo, x, th, [p])[0][j]
        t0 = a0 if which == 0 else b0
        out.append((mp.diff(lambda t: g(t, 0), t0), mp.diff(lambda t: g(t, 1), t0)))
    return out


def marginal(H21):
    """The theta block (S_aa, S_ab, S_bb) of the inverse of the symmetric 6 x 6 H (upper triangle row by row)."""
    M = mp.matrix(6, 6)
    for p in range(6):
        for q in range(p, 6):
            M[p, q] = M[q, p] = mp.mpf(float(H21[normals_ref.tri(p, q)]))
    Mi = M ** -1
    return Mi[0, 0], Mi[0, 1], Mi[1, 1]


def gauss_newton_step(cam8, img, T, y, xo, x, phi, th0, Li, w2):
    """The Gauss-Newton step H^-1 G at phi from the definition (the image gradient as the central difference of
    bilinear samples at +-1 px), in units of each unknown's posterior sigma, with numpy's sums and solve."""
    B = T.shape[0]
    fw = normals_ref.forward(cam8, B, y, xo, x, phi[:2])
    gu, gv = fw["g"][0] + phi[2], fw["g"][1] + phi[3]
    s = lambda u, v: normals_ref.frame_sample(img, u, v)  # noqa: E731
    I = s(gu, gv)
    Iu, Iv = (s(gu + 1, gv) - s(gu - 1, gv)) / 2, (s(gu, gv + 1) - s(gu, gv - 1)) / 2
    e = phi[4] * I + phi[5] - np.asarray(T, np.float64).reshape(-1)
    dg = phi[4] * (Iu * fw["Jw"][0] + Iv * fw["Jw"][1])
    J = np.stack([dg * fw["ta"], dg * fw["tb"], phi[4] * Iu, phi[4] * Iv, I, np.ones_like(I)], axis=1)
    L = np.array([[Li[0], Li[1]], [Li[1], Li[2]]])
    H = J.T @ J * w2
    H[:2, :2] += L
    G = J.T @ e * w2
    G[:2] += L @ (np.array(phi[:2]) - np.array(th0))
    return np.linalg.solve(H, G) / np.sqrt(np.diag(np.linalg.inv(H)))


def cost(cam8, img, T, y, xo, x, phi, th0, Li, w2):
    """The alignment's cost at phi from its definition, with the forward map that forward_rays checks: sum e^2 w2 +
    dt^T L dt (float64)."""
    B = T.shape[0]
    fw = normals_ref.forward(cam8, B, y, xo, x, phi[:2])
    gu, gv = fw["g"][0] + phi[2], fw["g"][1] + phi[3]
    I = normals_ref.frame_sample(img, gu, gv)
    e = (phi[4] * I + phi[5]) - np.asarray(T, np.float64).reshape(-1)
    da, db = phi[0] - th0[0], phi[1] - th0[1]
    return float((e * e).sum() * w2 + (Li[0] * da * da + 2 * Li[1] * da * db + Li[2] * db * db))


def gradient(cam8, img, T, y, xo, x, phi, th0, Li, w2, h=1e-6):
    """The cost's gradient at phi by central differences."""
    g = np.zeros(6)
    for i in range(6):
        up, dn = list(phi), list(phi)
        up[i] += h
        dn[i] -= h
        g[i] = (cost(cam8, img, T, y, xo, x, up, th0, Li, w2) - cost(cam8, img, T, y, xo, x, dn, th0, Li, w2)) / (2 * h)
    return g
