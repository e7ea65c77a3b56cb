"""Adversarial cases for the patch search (csrc/search.cu, csrc/smoe.cu): deterministic images, templates and jobs
aimed at the places where its filter, its tiling and its tie-break can go wrong.  No GPU and no test module needed.

cases(B) returns, for B = 11 or 15, one 320 x 240 image, the templates and a job list (feature index, centre, PuInv),
each job labelled with the edge it aims at.  The families:

- copy:     byte-identical copies of a template inside one ellipse, placed from the kernel's geometry (the tile
            sizes of every radius of SWEEP, strip slots 0 and V - 1, strips cut short by the tile, both sides of a
            tile boundary in u and in v).  The expected winner, the copy with the largest u-major scan index inside
            the ellipse, is computed here from the rules alone (copy_winner).
- straddle: near-copies (one to a dozen pixels moved by +-1) of templates whose sigma runs from 10 to ~120, so that
            the exact scores of the best and the runner-up differ by ~1e-7 .. 1e-3, across the filter's 1e-5 window;
            and affine copies a g + b, which tie with the template in FP64 to ~1e-16.
- knife:    windows whose integer variance n S2 - S1^2 is exactly 100 n^2 (sigma = 10, where the kernel's FP32 filter
            hands the decision to the FP64 chain), with both FP64 outcomes (sigma rounds below 10 or not), and the
            nearest values on either side, placed where they are the best match; templates built the same way, for
            the template gate.  n S2 - S1^2 is even and congruent to -S1^2 modulo n, so 100 n^2 +- 1 never occurs:
            the neighbours are the nearest values that can (KNIFE_STEPS).
- geometry: PuInv(1,1) on both sides of the 1e-7 and 1e7 guards of the column-interval shortcut, rotated ellipses
            up to |rho| = 0.999, ellipses whose column minimum is 9 up to rounding, ellipses with half-extents up to
            1e6 px (box clamped on all four sides, the whole image searched), centres outside the image, negative
            and on .5.
- gated:    a template with sigma < 10, and an ellipse whose windows all have sigma < 10.

smoe_cases(B) gives the SMOE search sets (K <= 256 ellipses per call) on the same image.

Every PuInv is positive definite and every half-extent below 2^31: a NaN or overflowing half-extent is undefined
behaviour in the reference's (int) cast, so such ellipses are not part of these cases.
"""
import functools
import math
from dataclasses import dataclass, field

import numpy as np

W, H = 320, 240
BOXES = (11, 15)
SWEEP = (1, 2, 3, 5, 8, 13, 20, 33, 57, 87)   # search_tile_radius values the suite runs
SMEM_OPTIN = 227 * 1024                         # dynamic shared memory a CTA may opt in to on an H100
SEARCH_WARPS, STRIP = 4, 8                      # SL2_SEARCH_WARPS, SL2_STRIP
FLAT = (slice(150, 212), slice(236, 304))       # rows / columns of the low-contrast corner (gated windows)
WHOLE = 1.0e6                                   # half-extent (px) of the ellipses that cover the whole image


# ---- the kernel's geometry, restated -------------------------------------------------------------------------------
def filter_strip(B):
    """Candidates per strip of the filtered search (filter_strip in search.cu)."""
    return 8 if B <= 11 else 16


def tile_size(B, radius):
    """TMA tile (bytes, rows) of a context with search_tile_radius = radius (sl2_create)."""
    return min((2 * radius + B + 30) & ~15, 256), min(2 * radius + B, 255)


def search_layout(B, radius):
    """(TCW, TCH, dynamic shared memory of a search CTA) as search_layout / search_smem_bytes compute them."""
    tw, th = tile_size(B, radius)
    tcw, tch = tw - 15 - B + 1, th - B + 1
    tile_bytes = (tw * th + 16 + 127) // 128 * 128
    list_bytes = (tcw * ((tch + STRIP - 1) // STRIP) * 4 + 15) // 16 * 16
    vtab = max(tch * 16, (tcw * 4 + 15) // 16 * 16)
    per_warp = (tile_bytes + list_bytes + 16 + vtab + 127) // 128 * 128
    return tcw, tch, SEARCH_WARPS * per_warp


def largest_radius(B, optin=SMEM_OPTIN):
    r = 1
    while search_layout(B, r + 1)[2] <= optin:
        r += 1
    return r


def search_box(B, centre, pu, truncate=False):
    """(us, uf, vs, vf, uc, vc) of monoslam.cpp:416-439 (rounded centre) / smoe.cpp:118-147 (truncated centre)."""
    P00, P01, P11 = (float(x) for x in pu)
    hw = int(3.0 / math.sqrt(P00 - P01 * P01 / P11))
    hh = int(3.0 / math.sqrt(P11 - P01 * P01 / P00))
    uc = int(float(centre[0])) if truncate else int(float(centre[0]) + 0.5)
    vc = int(float(centre[1])) if truncate else int(float(centre[1]) + 0.5)
    half = (B - 1) // 2
    us, uf, vs, vf = -hw, hw, -hh, hh
    if uc + us - half < 0:
        us = half - uc
    if uc + uf - half > W - B:
        uf = W - B - uc + half
    if vc + vs - half < 0:
        vs = half - vc
    if vc + vf - half > H - B:
        vf = H - B - vc + half
    return us, uf, vs, vf, uc, vc


def inside(pu, urel, vrel):
    """The 3-sigma test of monoslam.cpp:453-454 with the reference's operation order."""
    P00, P01, P11 = (float(x) for x in pu)
    u, v = float(urel), float(vrel)
    return P00 * u * u + 2 * P01 * u * v + P11 * v * v < 9.0


def sigma_fp64(S1, S2, n):
    """sigma of improc.cpp:99-110 from the integer sums (Python floats are IEEE doubles: same bits as the kernel)."""
    m = S1 / n
    return math.sqrt(S2 / n - m * m)


def window_var(win):
    """n S2 - S1^2 of a window, exact."""
    g = np.asarray(win, np.int64).ravel()
    return int(g.size * (g * g).sum() - g.sum() ** 2)


def knife_steps(B):
    """The values of n S2 - S1^2 - 100 n^2 nearest to 0 from below and from above that a B x B window can have."""
    n = B * B
    qr = {(s * s) % n for s in range(n)}
    ok = [d for d in range(-200, 201) if d % 2 == 0 and (-d) % n in qr]
    return max(d for d in ok if d < 0), min(d for d in ok if d > 0)


def pu_from(sx, sy, rho):
    """PuInv of the covariance with standard deviations sx, sy (px) and correlation rho (3 sigma: half-extent 3 sx)."""
    sx, sy, rho = float(sx), float(sy), float(rho)
    det = sx * sx * sy * sy * (1.0 - rho * rho)     # closed form: the same bits on every machine
    return np.array([sy * sy / det, -rho * sx * sy / det, sx * sx / det])


def circle(half_extent):
    p = 9.0 / (half_extent * half_extent)
    return np.array([p, 0.0, p])


def copy_winner(B, centre, pu, copies):
    """The copy with the largest scan index inside the box and the ellipse: the reference's `corr <= corrmax` keeps
    the last of equal scores.  None when no copy is inside."""
    us, uf, vs, vf, uc, vc = search_box(B, centre, pu)
    rows = vf - vs + 1
    best = None
    for (u, v) in copies:
        ur, vr = u - uc, v - vc
        if us <= ur <= uf and vs <= vr <= vf and inside(pu, ur, vr):
            idx = (ur - us) * rows + (vr - vs)
            if best is None or idx > best[0]:
                best = (idx, u, v)
    return None if best is None else (best[1], best[2])


def box_sums(image, patch, box):
    """Exact integer S1, S2 and Sxy of every candidate of `box` (us, uf, vs, vf, uc, vc), u-major like score_map."""
    us, uf, vs, vf, uc, vc = box
    B = patch.shape[0]
    half = (B - 1) // 2
    nu, nv = uf - us + 1, vf - vs + 1
    x0, y0 = uc + us - half, vc + vs - half
    reg = image[y0:y0 + nv + B - 1, x0:x0 + nu + B - 1].astype(np.int64)
    S1 = np.zeros((nv, nu), np.int64)
    S2 = np.zeros((nv, nu), np.int64)
    Sxy = np.zeros((nv, nu), np.int64)
    p = patch.astype(np.int64)
    for dy in range(B):
        for dx in range(B):
            r = reg[dy:dy + nv, dx:dx + nu]
            S1 += r
            S2 += r * r
            Sxy += p[dy, dx] * r
    return S1.T, S2.T, Sxy.T


# ---- construction ----------------------------------------------------------------------------------------------------
@dataclass
class Cases:
    B: int
    image: np.ndarray
    patches: np.ndarray
    feat: np.ndarray
    centres: np.ndarray
    pu: np.ndarray
    labels: list
    copies: dict = field(default_factory=dict)     # template -> [(u, v)] of its byte-identical copies
    winner: dict = field(default_factory=dict)     # copy job -> (u, v) expected
    knife: list = field(default_factory=list)      # (u, v, d, sigma, template) of every knife window
    knife_jobs: list = field(default_factory=list)
    straddle_jobs: list = field(default_factory=list)

    def family(self, j):
        return self.labels[j].split("/")[0]

    def jobs(self, fam=None):
        return [j for j in range(len(self.labels)) if fam is None or self.family(j) == fam]

    def sample(self, per_family=4):
        """A few jobs of every family, every knife job among them."""
        out = []
        for fam in ("copy", "straddle", "knife", "geometry", "gated"):
            js = self.jobs(fam)
            out += js if fam == "knife" else js[::max(1, len(js) // per_family)][:per_family]
        return out


class _Builder:
    def __init__(self, B, seed):
        self.B, self.half = B, (B - 1) // 2
        self.rng = np.random.default_rng(seed)
        self.img = self.rng.integers(0, 256, (H, W), dtype=np.uint8)
        flat = self.img[FLAT]
        flat[:] = 100
        flat[:, flat.shape[1] // 2:] += self.rng.integers(0, 8, (flat.shape[0], flat.shape[1] - flat.shape[1] // 2),
                                                          dtype=np.uint8)
        self.occ = np.zeros((H, W), bool)
        self.occ[FLAT] = True
        self.patches, self.feat, self.centres, self.pu, self.labels = [], [], [], [], []
        self.copies, self.winner = {}, {}
        self.knife, self.knife_jobs, self.straddle_jobs = [], [], []

    def free(self, u, v):
        h = self.half
        return h <= u < W - h and h <= v < H - h and not self.occ[v - h:v + h + 1, u - h:u + h + 1].any()

    def paste(self, win, u, v):
        h = self.half
        assert self.free(u, v), (u, v)
        self.img[v - h:v + h + 1, u - h:u + h + 1] = win
        self.occ[v - h:v + h + 1, u - h:u + h + 1] = True

    def template(self, t):
        self.patches.append(np.asarray(t, np.uint8))
        return len(self.patches) - 1

    def job(self, f, centre, pu, label):
        self.feat.append(f)
        self.centres.append(np.asarray(centre, np.float64))
        self.pu.append(np.asarray(pu, np.float64))
        self.labels.append(label)
        return len(self.labels) - 1

    def random_template(self, sigma=None, lo=0, hi=255):
        if sigma is None:
            return self.rng.integers(lo, hi + 1, (self.B, self.B)).astype(np.uint8)
        return np.clip(np.round(128 + sigma * self.rng.standard_normal((self.B, self.B))), 0, 255).astype(np.uint8)

    def group(self, k, spread):
        """k free window centres within `spread` of the first, their windows apart."""
        h = self.half
        for _ in range(200):
            pts = [self.spot()]
            for _ in range(50 * k):
                p = self.spot(near=pts[0], spread=spread, tries=1)
                if p and all(max(abs(p[0] - q[0]), abs(p[1] - q[1])) > 2 * h for q in pts):
                    pts.append(p)
                    if len(pts) == k:
                        return pts
        raise RuntimeError("no free group")

    def spot(self, near=None, spread=30, tries=4000):
        """A free window centre (near a point when given)."""
        for _ in range(tries):
            if near is None:
                u, v = int(self.rng.integers(self.half, W - self.half)), int(self.rng.integers(self.half, H - self.half))
            else:
                u = int(near[0] + self.rng.integers(-spread, spread + 1))
                v = int(near[1] + self.rng.integers(-spread, spread + 1))
            if self.free(u, v):
                return u, v
        if tries == 1:
            return None
        raise RuntimeError("no free spot")


def _copy_family(b):
    """Copies at kernel-geometry positions of every radius of SWEEP, found in whole-image boxes (box column / row 0 at
    image u / v = HALF), and a local ellipse around each pair."""
    B, half = b.B, b.half
    CW, CH = W - B + 1, H - B + 1
    V = filter_strip(B)

    def place(label, options):
        """The first option whose copies all fit; options yield lists of box positions, the last one the winner."""
        for pos in options:
            uv = [(half + cu, half + cv) for cu, cv in pos]
            if all(0 <= cu < CW and 0 <= cv < CH for cu, cv in pos) and all(b.free(u, v) for u, v in uv):
                t = b.random_template()
                f = b.template(t)
                for u, v in uv:
                    b.paste(t, u, v)
                b.copies[f] = uv
                return f, uv
        raise RuntimeError("copy family: no room for " + label)

    def shuffled(xs):
        xs = list(xs)
        b.rng.shuffle(xs)
        return xs

    # the box's first and last candidates (image corners), the last one wins
    made = [("box-corners", place("corners", [[(0, 0), (CW - 1, 0), (0, CH - 1), (CW - 1, CH - 1)]]))]
    for r in sorted(SWEEP, reverse=True):        # the widest tiles have the fewest boundaries: placed first
        TCW, TCH, _ = search_layout(B, r)
        kxs, kys = range(1, (CW - 1) // TCW + 1), range(1, (CH - 1) // TCH + 1)
        jhi = min(V, TCH) - 1                      # last strip slot a tile row can hold
        # X in the first column of tile (kx, ky - 1) and the last row of its tile; Y in the last column of tile
        # (kx - 1, ky): visited after X, but X has the larger scan index
        made.append(("tile-corner r=%d" % r, place("corner", (
            [(kx * TCW - 1, ky * TCH + B), (kx * TCW, ky * TCH - 1)] for kx in shuffled(kxs) for ky in shuffled(kys)))))
        # one column, both sides of a tile row boundary: the lower copy wins
        made.append(("tile-v r=%d" % r, place("v", (
            [(c, ky * TCH - 1), (c, ky * TCH - 1 + B)] for ky in shuffled(kys) for c in shuffled(range(CW))))))
        if len(kxs):
            # one row, both sides of a tile column boundary, windows side by side: the right copy wins
            made.append(("tile-u r=%d" % r, place("u", (
                [(kx * TCW - 1 - (B - 1) // 2, v), (kx * TCW + B // 2, v)] for kx in shuffled(kxs)
                for v in shuffled(range(CH))))))
        # strip slot 0 and the strip's last slot in neighbouring lanes (columns B apart), each of them the winner once
        tys = [ky * TCH for ky in range((CH - 1) // TCH + 1)]
        for name, a, z in (("slot0-wins", jhi, 0), ("slotV-1-wins", 0, jhi)):
            opts = []
            for ty in shuffled(tys):
                tch = min(TCH, CH - ty)
                for st in shuffled(range((tch - 1 - jhi) // V + 1) if tch > jhi else []):
                    for c in shuffled(range(CW - B))[:8]:
                        opts.append([(c, ty + st * V + a), (c + B, ty + st * V + z)])
            made.append(("%s r=%d" % (name, r), place(name, opts)))

    whole = [(circle(WHOLE), "1e6"), (circle(3000.0), "3000"), (pu_from(900.0, 700.0, 0.4), "rot900"),
             (circle(600.0), "600")]
    for i, (label, (f, uv)) in enumerate(made):
        pu, ext = whole[i % len(whole)]
        c = (float(b.rng.uniform(20, W - 20)), float(b.rng.uniform(20, H - 20)))
        j = b.job(f, c, pu, "copy/%s/whole-%s" % (label, ext))
        b.winner[j] = copy_winner(B, c, pu, uv)
        assert b.winner[j] == uv[-1], (label, b.winner[j], uv)
        # local ellipse around the pair, slightly rotated: its own box and tile grid
        (u0, v0), (u1, v1) = uv[0], uv[-1]
        mid = ((u0 + u1) / 2 + 0.3, (v0 + v1) / 2 - 0.2)
        d = max(abs(u1 - u0), abs(v1 - v0)) / 2 + 3
        pu2 = pu_from(d / 2.2, d / 2.2, 0.2 * (-1) ** i)
        w2 = copy_winner(B, mid, pu2, uv)
        if w2 is not None:
            j = b.job(f, mid, pu2, "copy/%s/local" % label)
            b.winner[j] = w2


def _moved(b, t, k):
    """t with k distinct pixels moved by +-1 (no clipping)."""
    w = t.astype(np.int64).ravel().copy()
    idx = b.rng.permutation(w.size)
    done = 0
    for i in idx:
        s = 1 if b.rng.random() < 0.5 else -1
        if 0 <= w[i] + s <= 255:
            w[i] += s
            done += 1
            if done == k:
                break
    return w.reshape(t.shape).astype(np.uint8)


def _straddle_family(b):
    B = b.B
    sigmas = (10.5, 12, 15, 20, 26, 33, 45, 60, 80, 120)
    pairs = ((1, 2), (2, 3), (1, 3), (1, 12), (3, 3), (2, 2), (4, 5))
    for si, sg in enumerate(sigmas):
        t = b.random_template(sigma=sg)
        f = b.template(t)
        for pi in range(2):
            ka, kb = pairs[(si + 2 * pi) % len(pairs)]
            pa, pb = b.group(2, B + 8)
            b.paste(_moved(b, t, ka), *pa)
            b.paste(_moved(b, t, kb), *pb)
            mid = ((pa[0] + pb[0]) / 2 + 0.21, (pa[1] + pb[1]) / 2 + 0.37)
            d = max(abs(pa[0] - pb[0]), abs(pa[1] - pb[1])) / 2 + 2
            j = b.job(f, mid, pu_from(d / 2.0, d / 2.4, 0.3 * (-1) ** pi), "straddle/sigma%g/k%d-%d" % (sg, ka, kb))
            b.straddle_jobs.append(j)
    # sigma chosen so that the expected gap |ka - kb| / (n sigma^2) is 0.6x, 1x and 1.6x the filter window
    for dk, m in ((1, 0.6), (1, 1.0), (1, 1.6), (2, 0.8), (2, 1.3)):
        sg = math.sqrt(dk / (B * B * 1e-5 * m))
        t = b.random_template(sigma=sg)
        f = b.template(t)
        pa, pb = b.group(2, B + 8)
        b.paste(_moved(b, t, 1), *pa)
        b.paste(_moved(b, t, 1 + dk), *pb)
        mid = ((pa[0] + pb[0]) / 2 - 0.13, (pa[1] + pb[1]) / 2 + 0.29)
        d = max(abs(pa[0] - pb[0]), abs(pa[1] - pb[1])) / 2 + 2
        j = b.job(f, mid, pu_from(d / 2.0, d / 2.0, 0.1), "straddle/window sigma%.1f/k1-%d" % (sg, 1 + dk))
        b.straddle_jobs.append(j)
    # affine copies a g + b (no clipping): exact ties up to the FP64 rounding of the score
    for ai, (lo, hi, maps) in enumerate(((40, 150, ((2, -70), (1, 60))), (60, 120, ((3, -170), (2, -110))),
                                         (90, 160, ((1, -80), (1, 90))), (30, 110, ((2, 0), (3, -80))))):
        t = b.random_template(lo=lo, hi=hi)
        f = b.template(t)
        pts = b.group(1 + len(maps), 2 * B)
        b.paste(t, *pts[0])
        for (a, c), p in zip(maps, pts[1:]):
            g = t.astype(np.int64) * a + c
            assert g.min() >= 0 and g.max() <= 255
            b.paste(g.astype(np.uint8), *p)
        us, vs = [p[0] for p in pts], [p[1] for p in pts]
        mid = ((min(us) + max(us)) / 2 + 0.1, (min(vs) + max(vs)) / 2 - 0.4)
        d = max(max(us) - min(us), max(vs) - min(vs)) / 2 + 3
        j = b.job(f, mid, pu_from(d / 2.0, d / 2.0, 0.0), "straddle/affine%d" % ai)
        b.straddle_jobs.append(j)


def knife_window(rng, B, d, sigma=10.0):
    """A B x B window (int64) with n S2 - S1^2 = 100 n^2 + d exactly (d one of 0 and knife_steps(B))."""
    n = B * B
    target = 100 * n * n + d
    for _ in range(50):
        w = np.clip(np.round(120 + sigma * rng.standard_normal(n)), 20, 235).astype(np.int64)
        # S1 to a residue with S1^2 = -d (mod n): V = n S2 - S1^2 = -S1^2 (mod n)
        while (w.sum() ** 2 + d) % n:
            w[rng.integers(n)] += 1
        # then pairs (+1 on a, -1 on b) keep S1 and move V by 2 n (g_a - g_b + 1)
        for _ in range(400):
            D = target - (n * int((w * w).sum()) - int(w.sum()) ** 2)
            if D == 0:
                return w.reshape(B, B)
            assert D % (2 * n) == 0
            k = D // (2 * n)
            want = max(-60, min(60, k)) - 1            # g_a - g_b
            a = rng.integers(n)
            cand = np.flatnonzero(w == w[a] - want)
            cand = cand[cand != a]
            if len(cand) and w[a] < 255 and w[cand[0]] > 0:
                w[a] += 1
                w[cand[0]] -= 1
    raise RuntimeError("knife window not reached")


def _knife_family(b):
    B, n = b.B, b.B * b.B
    lo, hi = knife_steps(B)
    wins = []
    for d in (lo, 0, hi):
        w = knife_window(b.rng, B, d)
        outcomes = {}
        for c in range(-19, 20):                  # a constant shift keeps n S2 - S1^2: only the FP64 rounding moves
            g = w + c
            s = sigma_fp64(int(g.sum()), int((g * g).sum()), n)
            outcomes.setdefault(s >= 10.0, (g, s))
        if d == 0:
            assert len(outcomes) == 2, "both FP64 outcomes of the knife edge"
            wins += [(d, g, s) for g, s in outcomes.values()]
        else:
            wins += [(d, g, s) for g, s in list(outcomes.values())[:1]]
        if d == 0:                                # a second knife window of each outcome with other sums
            w2 = knife_window(b.rng, B, 0, sigma=10.0)
            for c in range(-19, 20):
                g = w2 + c
                s = sigma_fp64(int(g.sum()), int((g * g).sum()), n)
                if (s >= 10.0) != (wins[-1][2] >= 10.0):
                    wins.append((0, g, s))
                    break
    for d, g, s in wins:
        # the window in the image; its template a few +-1 moves away, moved away from the mean so sigma0 > 10
        t = g.copy().ravel()
        dev = t - t.mean()
        for i in np.argsort(-np.abs(dev))[:3]:
            t[i] += 1 if dev[i] > 0 else -1
        f = b.template(t.reshape(B, B))
        p = b.spot()
        b.paste(g.astype(np.uint8), *p)
        b.knife.append((p[0], p[1], d, s, f))
        for k, (c, pu) in enumerate((((p[0] + 0.4, p[1] - 0.3), circle(6.0)),
                                    ((p[0] - 3.2, p[1] + 2.6), pu_from(3.0, 2.5, 0.6)))):
            b.knife_jobs.append(b.job(f, c, pu, "knife/window d=%d sigma=%r/%d" % (d, s, k)))
    # templates on the knife edge (the template gate): pasted as they are, so the copy is the only match
    for want in (True, False):
        g = None
        while g is None:
            w = knife_window(b.rng, B, 0)
            for c in range(-19, 20):
                s = sigma_fp64(int((w + c).sum()), int(((w + c) ** 2).sum()), n)
                if (s >= 10.0) == want:
                    g = w + c
                    break
        f = b.template(g.astype(np.uint8))
        p = b.spot()
        b.paste(g.astype(np.uint8), *p)
        b.knife.append((p[0], p[1], 0, s, f))
        b.knife_jobs.append(b.job(f, (p[0] - 0.2, p[1] + 0.1), circle(5.0), "knife/template sigma0=%r" % s))


def _geometry_family(b):
    B, half = b.B, b.half
    # templates cut from the background: one natural, unique match each
    pts = []
    for _ in range(8):
        u, v = b.spot()
        b.occ[v - half:v + half + 1, u - half:u + half + 1] = True
        pts.append((u, v))
    fs = [b.template(b.img[v - half:v + half + 1, u - half:u + half + 1].copy()) for u, v in pts]

    def at(i, du=0.0, dv=0.0):
        return (pts[i][0] + du, pts[i][1] + dv)

    lo, hi = 1e-7, 1e7
    for k, P11 in enumerate((lo, np.nextafter(lo, 0), np.nextafter(lo, 1), 2e-7, 5e-8)):
        b.job(fs[0], at(0, 0.3, -0.2), [0.04, 0.0, P11], "geometry/P11 %r" % P11)
        P01 = 0.6 * math.sqrt(0.04 * P11)
        b.job(fs[1], at(1, -0.4, 0.1), [0.04, P01 * (-1) ** k, P11], "geometry/P11 %r rotated" % P11)
    for P11 in (hi, np.nextafter(hi, 0), np.nextafter(hi, np.inf), 2e7, 5e6):
        b.job(fs[2], at(2, 0.2, 0.4), [0.03, 0.0, P11], "geometry/P11 %r" % P11)
        b.job(fs[2], at(2, -0.1, -0.3), [0.03, 0.5 * math.sqrt(0.03 * P11), P11], "geometry/P11 %r rotated" % P11)
    for rho in (0.9, -0.99, 0.995, 0.999, -0.999):
        for sx, sy in ((6.0, 8.0), (20.0, 4.0), (3.0, 25.0)):
            b.job(fs[3], at(3, 0.45, -0.35), pu_from(sx, sy, rho), "geometry/rho %g %gx%g" % (rho, sx, sy))
    for kk in (3, 5, 7, 10, 13):                  # column minimum P00 k k, 9 up to rounding, at the vertex row 0
        for P00 in (9.0 / (kk * kk), np.nextafter(9.0 / (kk * kk), 0), np.nextafter(9.0 / (kk * kk), 1)):
            b.job(fs[4], at(4, 0.2, 0.1), [P00, 0.0, 0.02], "geometry/vertex9 k=%d %r" % (kk, P00))
    for ext, rho in ((1e6, 0.0), (1e6, 0.7), (2.0e5, -0.3), (1e4, 0.0), (400.0, 0.5)):
        b.job(fs[5], at(5, 0.1, 0.2), pu_from(ext / 3, ext / 3, rho), "geometry/whole %g rho %g" % (ext, rho))
    for i, c, pu, label in ((5, (-50.2, 100.0), circle(20.0), "outside left"),
                            (5, (W + 40.0, H + 60.0), circle(30.0), "outside"),
                            (5, (100.0, -45.0), circle(25.0), "outside top"), (5, (-0.5, 30.5), circle(40.0), "negative"),
                            (5, (-3.2, -1.5), circle(60.0), "negative corner"),
                            (5, (W - 0.5, H - 0.5), circle(25.0), "far corner"),
                            (6, at(6, 0.5, 0.5), circle(4.0), "on .5"), (6, at(6, -0.5, 0.5), circle(3.0), "on -.5"),
                            (7, at(7, 0.5, -0.5), pu_from(1.0, 1.5, 0.3), "on .5 rotated"),
                            (7, at(7, 1.5, 2.5), circle(2.0), "on .5 small")):
        b.job(fs[i], c, pu, "geometry/centre %s" % label)


def _gated_family(b):
    B = b.B
    low = np.clip(np.round(120 + 5 * b.rng.standard_normal((B, B))), 0, 255).astype(np.uint8)
    f = b.template(low)
    p = b.spot()
    b.paste(low, *p)
    b.job(f, (p[0] + 0.2, p[1]), circle(8.0), "gated/template sigma<10")
    f2 = b.template(b.random_template())
    cu = (FLAT[1].start + FLAT[1].stop) / 2
    cv = (FLAT[0].start + FLAT[0].stop) / 2
    b.job(f2, (cu - 8, cv), circle(6.0), "gated/windows flat")
    b.job(f2, (cu + 12, cv + 3), circle(5.0), "gated/windows low contrast")


@functools.lru_cache(maxsize=None)
def cases(B):
    b = _Builder(B, 5000 + B)
    _copy_family(b)
    _knife_family(b)
    _straddle_family(b)
    _geometry_family(b)
    _gated_family(b)
    c = Cases(B, b.img, np.stack(b.patches), np.array(b.feat, np.int32), np.stack(b.centres), np.stack(b.pu),
              b.labels, b.copies, b.winner, b.knife, b.knife_jobs, b.straddle_jobs)
    # copies and knife windows are what they were pasted as
    for f, uv in c.copies.items():
        for u, v in uv:
            assert (window(c, u, v) == c.patches[f]).all()
    return c


def window(c, u, v):
    h = (c.B - 1) // 2
    return c.image[v - h:v + h + 1, u - h:u + h + 1]


@functools.lru_cache(maxsize=None)
def smoe_cases(B):
    """[(label, template, PuInv (K, 3), centres (K, 2))]: K <= 256 overlapping ellipses per call on cases(B).image."""
    c = cases(B)
    rng = np.random.default_rng(7000 + B)
    out = []

    def centres_near(p, K, spread):
        xy = np.column_stack([p[0] + rng.normal(0, spread, K), p[1] + rng.normal(0, spread, K)])
        frac = rng.choice([0.0, 0.5, 0.99, 0.49999999, 0.25], (K, 2))
        return np.floor(xy) + frac                # x.5 / x.99: truncation and rounding disagree

    def pus(K, lo, hi):
        return np.stack([pu_from(rng.uniform(lo, hi), rng.uniform(lo, hi), rng.uniform(-0.9, 0.9)) for _ in range(K)])

    # copy ties: the pair of a copy-family template, many ellipses around it
    for f in list(c.copies)[:: max(1, len(c.copies) // 3)][:3]:
        (u0, v0), (u1, v1) = c.copies[f][0], c.copies[f][-1]
        p = ((u0 + u1) / 2, (v0 + v1) / 2)
        out.append(("smoe/copy %d" % f, c.patches[f], pus(256, 1.0, 12.0), centres_near(p, 256, 6.0)))
    # knife windows: every window below sigma 10 gets +5, so the penalty decides these searches
    for u, v, d, s, f in c.knife:
        out.append(("smoe/knife d=%d sigma=%r" % (d, s), c.patches[f], pus(64, 0.8, 4.0), centres_near((u, v), 64, 2.0)))
    # the flat corner: a window of sigma 0 scores 1 (+5), below every textured window without the penalty
    cu, cv = FLAT[1].start, FLAT[0].start
    K = 128
    out.append(("smoe/flat border", c.patches[c.feat[c.jobs("straddle")[0]]], pus(K, 0.8, 5.0),
                centres_near((cu, cv), K, 8.0)))
    # every border and corner: boxes clipped, truncated and negative centres
    K = 256
    xy = np.column_stack([rng.choice([-3.7, -0.5, 0.5, 3.99, 160.5, W - 4.5, W - 0.01, W + 2.5], K),
                          rng.choice([-2.5, -0.99, 0.5, 4.5, 120.5, H - 5.5, H - 0.5, H + 1.7], K)])
    xy += rng.choice([0.0, 0.0, 1.0, 7.0], (K, 2))
    f = c.jobs("geometry")[0]
    out.append(("smoe/borders", c.patches[c.feat[f]], pus(K, 2.0, 20.0), xy))
    return out
