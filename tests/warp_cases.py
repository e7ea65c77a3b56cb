"""Error bounds, the decision rule and the cases for holding the planar patch warp (the restatement tests/warp_ref.py,
and through it the device) to its definition (tests/warp_truth.py).

The bound on |src - src_truth| follows the header's FP64 chain operation by operation (u = 2^-53, first order, then
doubled for the second-order terms).  Its conditioning terms:
  e_R   the entry error of RRW: quat_inverse (|q|^2: 7 ops, one division) and quat_to_R (a product and two sums per
        entry of magnitude 2 |q^-1|^2): 30 u max(1, |q|^-2); Rn = |1 - m^2| + m^2 (m = 1 / |q|) bounds |RRW|;
  h     z = RRW (y - r) (one subtraction, a 3-term row): |dz| <= (4 u + 3 e_R) Rn |y - r|; Project (two products and a
        division per coordinate, the radius, a square root, a division and a sum): |dh| <= f (4 u + 3 e_R) Rn
        (|y - r| / z[2]) (1 + rho / f) + 8 u rho + 2 u |h|, rho the undistorted radius, f = max(fku, fkv);
  p     p = h + offset: |dp| <= |dh| + u |p|;
  ray   unproject_point: the reach term 1 / (1 - 2 kd1 r^2) =: k_reach (the square root's argument), and the radial
        derivative of the inverse distortion, k_reach^(3/2) / f_min per pixel of |dp|; its own rounding
        k_reach (10 u kd1 r^2 + u) + 5 u; adj(RRW) (2 e_R + 3 u per entry, relative to its smallest singular value:
        times cond(RRW)) and its product (3 u);
  plane X = r + t dW: a ray turned by e moves X by |X - r| e (1 + k_plane), k_plane = |nW| |dW| / |nW . dW| (the
        ray-plane angle); t's numerator (5 u |nW| |y - r|, over |num|: k_num) and denominator (4 u k_plane); the sums
        3 u (|r| + |xo| + |X - r|);
  src   zo = RRW(xo) (X - xo): |dzo| <= Rn_o |dX| + (4 u + 3 e_Ro) Rn_o |X - xo|; Project as for h with the depth term
        |X - xo| / zo[2]; ho as h (depth term |y - xo| / zo[2] of y); src = (g - ho) + HALF: 2 u (|g| + |ho| + HALF).
The bound on v carries |d src| through the largest neighbour difference of the cells src can lie in (the bilinear
interpolant is Lipschitz with that constant in each coordinate) and adds the bilinear's own rounding (12 u 256).  A byte
is compared only where v lies further than that bound from every k + 1/2; a validity flag only where the margin of
each of its decisions (the reach, lam > 0, zo[2] > 0) exceeds that margin's bound."""
import numpy as np
from scipy.spatial.transform import Rotation

from camera_ref import rrw
from consensus_truth import _Num, project, rotation_rrw
from warp_truth import warp_truth

U = 2.0 ** -53


def _rrw_terms(q):
    m2 = 1.0 / float(np.dot(q, q))
    return 30 * U * max(1.0, m2), abs(1.0 - m2) + m2


def _cond_rrw(q):
    s = np.linalg.svd(np.array(rrw(np.concatenate([np.zeros(3), q]))), compute_uv=False)
    return float(s[0] / s[-1])


def bounds(cam8, B, y, xo, xp, tr):
    """-> dict of per-pixel bounds (B, B): src (on |src - src_truth|, each coordinate), reach, lam, zo (on the margins
    m_reach, m_lam, m_zo) and X (on |X - X_truth|, for the round trip)."""
    cam8, y, xo, xp = (np.asarray(a, np.float64) for a in (cam8, y, xo, xp))
    half = (B - 1) // 2
    f, fmin, kd1 = max(cam8[2], cam8[3]), min(cam8[2], cam8[3]), cam8[6]
    e_R, Rn = _rrw_terms(xp[3:7])
    e_Ro, Rn_o = _rrw_terms(xo[3:7])
    E_h = (f * (4 * U + 3 * e_R) * Rn * (tr.y_r / tr.z2) * (1 + tr.rho_h / f) + 8 * U * tr.rho_h
           + 2 * U * np.linalg.norm(tr.h))
    E_ho = (f * (4 * U + 3 * e_Ro) * Rn_o * (tr.y_xo / tr.zo2_y) * (1 + tr.rho_ho / f) + 8 * U * tr.rho_ho
            + 2 * U * np.linalg.norm(tr.ho))
    E_p = E_h + U * np.linalg.norm(tr.p, axis=-1)
    r2 = ((tr.p - cam8[4:6]) ** 2).sum(-1)
    with np.errstate(all="ignore"):
        k_reach = np.where(tr.m_reach > 0, 1.0 / tr.m_reach, np.inf)
        e_ray = (k_reach ** 1.5 * E_p / fmin + k_reach * (10 * U * kd1 * r2 + U) + 5 * U
                 + _cond_rrw(xp[3:7]) * (2 * e_R + 3 * U) + 3 * U)
        E_X = (tr.Xr * (e_ray * (1 + tr.k_plane) + 5 * U * tr.k_num + 4 * U * tr.k_plane + 2 * U)
               + 3 * U * (np.linalg.norm(xp[:3]) + np.linalg.norm(xo[:3]) + tr.Xr))
        E_zo = Rn_o * E_X + (4 * U + 3 * e_Ro) * Rn_o * tr.Xo
        E_g = f * E_zo / tr.zo2 * (1 + tr.rho_g / f) + 8 * U * tr.rho_g + U * tr.g
        src = 2 * (E_g + E_ho + 2 * U * (tr.g + np.linalg.norm(tr.ho) + half))
        reach = 2 * (2 * kd1 * (5 * U * r2 + 2 * np.sqrt(r2) * E_p + E_p ** 2) + U)
        lam = 2 * (2 * e_ray + 12 * U)
        zo = 2 * (E_zo / tr.Xo + U)
    return dict(src=src, reach=reach, lam=lam, zo=zo, X=2 * E_X)


def cell_lipschitz(T, src, b):
    """The largest neighbour difference over the cells (x0 = min(floor(s), B - 2)) that the clamped positions within
    b of src can lie in."""
    T = np.asarray(T, np.float64)
    B = T.shape[0]
    D = np.maximum.reduce([np.abs(T[:-1, 1:] - T[:-1, :-1]), np.abs(T[1:, 1:] - T[1:, :-1]),
                           np.abs(T[1:, :-1] - T[:-1, :-1]), np.abs(T[1:, 1:] - T[:-1, 1:])])

    def cell(s):
        return np.minimum(np.floor(np.clip(s, 0.0, B - 1.0)), B - 2).astype(np.int64)
    out = np.zeros(src.shape[:-1])
    for dx in (-b, b):
        for dy in (-b, b):
            out = np.maximum(out, D[cell(src[..., 1] + dy), cell(src[..., 0] + dx)])
    return out


class Decided:
    """The truth of one feature's warp, its bounds and the decision rule: which flags and bytes may be compared."""

    def __init__(self, cam8, B, y, xo, xp, T, prec="ld"):
        self.tr = tr = warp_truth(cam8, B, y, xo, xp, T, prec)
        self.b = b = bounds(cam8, B, y, xo, xp, tr)
        self.T = np.asarray(T, np.uint8)
        self.cam8, self.xp = np.asarray(cam8, np.float64), np.asarray(xp, np.float64)
        f = max(cam8[2], cam8[3])
        _, Rn = _rrw_terms(self.xp[3:7])
        with np.errstate(all="ignore"):  # X off by |dX| moves its projection by f Rn |dX| / depth (1 + rho / f)
            self.b_rt = 2 * f * Rn * b["X"] / tr.lam * (1 + tr.rho_p / f) + 4 * U * np.linalg.norm(tr.p, axis=-1)
        reach_d = np.abs(tr.m_reach) > b["reach"]
        lam_d = np.abs(tr.m_lam) > b["lam"]
        zo_d = np.abs(tr.m_zo) > b["zo"]
        # decided valid: every decision decided and true; decided invalid: one decided and false
        self.flag_decided = ((reach_d & lam_d & zo_d & tr.valid)
                             | (reach_d & (tr.m_reach <= 0))
                             | (reach_d & (tr.m_reach > 0) & lam_d & (tr.m_lam <= 0))
                             | (reach_d & lam_d & (tr.m_lam > 0) & zo_d & (tr.m_zo <= 0)))
        bs = np.where(tr.valid, b["src"], np.inf)
        srcz = np.where(tr.valid[..., None], tr.src, 0.0)
        bsz = np.where(tr.valid, bs, 0.0)
        self.b_v = 2 * cell_lipschitz(self.T, srcz, np.nan_to_num(bsz, posinf=1e300)) * bs + 12 * U * 256
        self.byte_decided = tr.valid & self.flag_decided & (tr.tie_gap > self.b_v)
        self.template_decided = bool(self.flag_decided.all())

    def template(self):
        """The warped template and valid flag the truth decides on (only meaningful where template_decided)."""
        if self.tr.valid.all():
            return self.tr.byte.astype(np.uint8), 1
        return self.T.copy(), 0

    def check(self, src, valid, X=None, out=None, out_valid=None):
        """-> failures [(check, text)] of a chain's per-pixel src (B, B, 2) and validity (B, B) (and its plane points X
        for the round trip, and its warped template and flag) against the truth under the rule."""
        tr, b, fail = self.tr, self.b, []
        if ((valid != tr.valid) & self.flag_decided).any():
            fail.append(("valid", "%d decided flags differ" % int(((valid != tr.valid) & self.flag_decided).sum())))
        both = valid & tr.valid & self.flag_decided
        err = np.abs(src - tr.src).max(axis=-1)
        if (err[both] > b["src"][both]).any() or np.isnan(err[both]).any():
            worst = np.nanmax(err[both] / b["src"][both])
            fail.append(("src", "src off by %.3g of the bound" % worst))
        B = tr.valid.shape[0]
        c = (B - 1) // 2
        if tr.valid[c, c] and valid[c, c] and not (np.abs(src[c, c] - c) <= b["src"][c, c]).all():
            fail.append(("centre", "the centre pixel samples %s" % src[c, c]))
        if X is not None:
            # the chain's plane point seen from xp lands on its pixel (Project in extended precision)
            ok = both & np.isfinite(X).all(-1)
            num = _Num("ld")
            xp = num(self.xp)
            zc = np.einsum("ij,kj->ki", rotation_rrw(xp[3:7]), num(X[ok]) - xp[0:3])
            d = np.abs(num.f64(project(self.cam8, zc, num)) - tr.p[ok]).max(axis=-1)
            lim = self.b_rt[ok]
            if (d > lim).any():
                fail.append(("round-trip", "plane point off its pixel by %.3g px (%.3g of the bound)"
                             % (d.max(), (d / lim).max())))
        if out is not None:
            fail += self.check_template(out, out_valid)
        return fail

    def check_template(self, out, out_valid):
        """-> failures of a warped template (B, B) and its valid flag: the flag where every pixel's flag is decided,
        the decided bytes of a valid one, the stored bytes of an invalid one."""
        if not self.template_decided:
            return []
        want, wv = self.template()
        if int(out_valid) != wv:
            return [("valid", "template flag %d, truth %d" % (out_valid, wv))]
        if wv:
            bad = (out != want) & self.byte_decided
            return [("byte", "%d decided bytes differ" % int(bad.sum()))] if bad.any() else []
        return [] if (out == self.T).all() else [("byte", "an invalid feature's bytes are not its stored template")]


# ---- cases -----------------------------------------------------------------------------------------------------------
C1 = (320, 240, 11)
C3 = (640, 480, 15)
Q_NORMS = (1.0, 1 + 3.5e-5, 1 - 3.5e-5, 1 + 1e-3, 1 - 1e-3, 0.97, 1.03, 1.2)


def cameras():
    """(name, cam8, B): the C1 / C2 / C4 camera (320 x 240, kd1 = 9e-6) at 11 x 11 and 15 x 15, C3's (640 x 480) at
    15 x 15, and a per-stream camera whose reach (2 kd1 r^2 < 1: r < 129 px) cuts into its 320 x 240 image."""
    from scenelib2_b200 import synth
    c1, c3 = synth.camera_params(320, 240), synth.camera_params(640, 480)
    wide = c1.copy()
    wide[2], wide[3], wide[6] = 240.0, 240.0, 3e-5
    return [("C1", c1, 11), ("C1-15", c1, 15), ("C3", c3, 15), ("reach", wide, 11)]


def look_at(pos, target, roll):
    """The unit-quaternion pose at pos whose optical axis points at target, rolled by `roll` about it."""
    z = (target - pos) / np.linalg.norm(target - pos)
    a = np.array([1.0, 0.0, 0.0]) if abs(z[0]) < 0.9 else np.array([0.0, 1.0, 0.0])
    x = np.cross(a, z)
    x /= np.linalg.norm(x)
    R = np.stack([x, np.cross(z, x), z], axis=1) @ Rotation.from_rotvec([0, 0, roll]).as_matrix()
    qx, qy, qz, qw = Rotation.from_matrix(R).as_quat()
    return np.concatenate([pos, [qw, qx, qy, qz]])


def seen_point(cam8, xp, rng, margin=30, reach=0.9):
    """A world point that the camera at xp (unit q) sees at a random pixel `margin` inside its image and inside
    `reach` of the model's reach (in radius), 0.5-3 m away."""
    c = np.asarray(cam8[4:6])
    while True:
        px = np.array([rng.uniform(margin, cam8[0] - 1 - margin), rng.uniform(margin, cam8[1] - 1 - margin)])
        if 2 * cam8[6] * ((px - c) ** 2).sum() < reach ** 2:
            break
    f = np.sqrt(1 - 2 * cam8[6] * ((px - c) ** 2).sum())
    zc = np.array([(px[0] - c[0]) / f / -cam8[2], (px[1] - c[1]) / f / -cam8[3], 1.0]) * rng.uniform(0.5, 3.0)
    return xp[:3] + np.array(rrw(xp)).T @ zc


def first_view(y, xp, rng, ratio, angle_deg):
    """xo: a unit-q pose looking at y (up to 4 degrees off its axis, any roll) from `ratio` times xp's distance, its
    direction turned from xp's by angle_deg."""
    view = xp[:3] - y
    axis = np.cross(view, rng.standard_normal(3))
    dirn = Rotation.from_rotvec(axis / np.linalg.norm(axis) * np.radians(angle_deg)).as_matrix() @ view
    pos = y + dirn * ratio
    off = Rotation.from_rotvec(rng.standard_normal(3) * np.radians(4) / np.sqrt(3)).as_matrix() @ (y - pos)
    return look_at(pos, pos + off, rng.uniform(-np.pi, np.pi))


def with_norm(x, s):
    x = np.array(x, np.float64)
    x[3:7] *= s
    return x


def random_cases(per=4, seed=5):
    """[(name, cam8, B, y, xo, xp, T)]: on every camera and at every |q| (of xp and xo both), `per` features of the
    visibility envelope (distance ratio 0.55-1.8, up to 40 degrees, any roll; on the wide camera up to the model's
    reach); then planes viewed nearly edge-on (80,
    86 and 89 degrees) and distance ratios of exactly 0.5 and 2."""
    rng = np.random.default_rng(seed)
    out = []
    for cname, cam8, B in cameras():
        for s in Q_NORMS:
            xp = look_at(rng.uniform(-1, 1, 3), rng.uniform(-1, 1, 3) + [0, 0, 3.0], rng.uniform(-np.pi, np.pi))
            for k in range(per):  # the wide camera's features up to its reach, so that templates straddle it
                y = seen_point(cam8, xp, rng, reach=0.999 if cname == "reach" else 0.9)
                xo = first_view(y, xp, rng, rng.uniform(0.55, 1.8), rng.uniform(0, 40))
                T = rng.integers(0, 256, (B, B))
                out.append(("%s-q%.6g-%d" % (cname, s, k), cam8, B, y, with_norm(xo, s), with_norm(xp, s), T))
        xp = look_at(rng.uniform(-1, 1, 3), rng.uniform(-1, 1, 3) + [0, 0, 3.0], rng.uniform(-np.pi, np.pi))
        for ang in (80.0, 86.0, 89.0):
            y = seen_point(cam8, xp, rng)
            out.append(("%s-edge-on-%g" % (cname, ang), cam8, B, y, first_view(y, xp, rng, 1.0, ang), xp,
                        rng.integers(0, 256, (B, B))))
        for ratio in (0.5, 2.0):
            for s in (1.0, 1.03):
                y = seen_point(cam8, xp, rng)
                out.append(("%s-ratio-%g-q%g" % (cname, ratio, s), cam8, B, y,
                            with_norm(first_view(y, xp, rng, ratio, 20.0), s), with_norm(xp, s),
                            rng.integers(0, 256, (B, B))))
    return out


# ---- exact constructions: kd1 = 0 (but for the reach), fku = fkv = 256, principal point (160, 120) ----------------------
CAM_EXACT = np.array([320.0, 240.0, 256.0, 256.0, 160.0, 120.0, 0.0, 1.0])
Y_AXIS, XO_AXIS = np.array([0.0, 0.0, 2.0]), np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0])


def constructions(rng=None):
    """[(name, cam8, B, y, xo, xp, T)] whose FP64 chain is exact except where stated:
      half-shift-B   the camera at half the distance, moved by a dyadic step parallel to the fronto-parallel plane
                     z = 2: output offset d samples d / 2, every odd pair sum an exact .5 tie;
      edges-B        the camera moved by a dyadic step parallel to the plane: src = (b, a), the edge columns exactly at
                     0 and B - 1 (x0 = B - 2, fx = 1);
      beyond-B       the camera at twice the distance: src = HALF + 2 (b - HALF, a - HALF), clamped beyond the edges;
      rows           the plane y = 0 seen from (0, -1/32, 0), first seen from (0, -1, 2) with q = (1, -1, 0, 0)
                     (|q|^2 = 2, RRW = (I + R(90 deg)) / 2): row 0 has zo[2] < 0, row 1 zo[2] = 0 exactly, rows 2-8
                     are valid, row 9's rays are exactly parallel to the plane and row 10's meet it behind the camera;
      reach          kd1 = 1/64 on the axis: the pixels at offsets (+-4, +-4) lie exactly at the model's reach
                     (2 kd1 r^2 = 1), those further out beyond it, the rest inside with a margin of at least 3/32 (the
                     chain is exact up to the reach decisions only)."""
    rng = np.random.default_rng(17) if rng is None else rng
    out = []
    for B in (11, 15):
        T = rng.integers(0, 256, (B, B))
        out.append(("half-shift-%d" % B, CAM_EXACT, B, Y_AXIS, XO_AXIS, np.array([0.25, -0.5, 1.0, 1, 0, 0, 0]), T))
        out.append(("edges-%d" % B, CAM_EXACT, B, Y_AXIS, XO_AXIS, np.array([0.25, -0.5, 0.0, 1, 0, 0, 0]), T))
        out.append(("beyond-%d" % B, CAM_EXACT, B, Y_AXIS, XO_AXIS, np.array([0.25, -0.5, -2.0, 1, 0, 0, 0]), T))
    out.append(("rows", CAM_EXACT, 11, np.zeros(3) + [0, 0, 2.0], np.array([0, -1.0, 2.0, 1, -1, 0, 0]),
                np.array([0, -1 / 32, 0, 1, 0, 0, 0]), rng.integers(0, 256, (11, 11))))
    cam_r = CAM_EXACT.copy()
    cam_r[6] = 1 / 64
    out.append(("reach", cam_r, 11, Y_AXIS, XO_AXIS, np.array([0.0, 0.0, 0.5, 1, 0, 0, 0]),
                rng.integers(0, 256, (11, 11))))
    return out
