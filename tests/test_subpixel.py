"""The sub-pixel refinement's restatement (tests/subpixel_ref.py) on the CPU: the score against the oracle's
correlate2_warning, the fit against exact rational arithmetic, its fallbacks and knife edges, broken copies that must
be caught, and the recovery of textures shifted by known fractions of a pixel."""
import math
from fractions import Fraction as Q

import numpy as np
import pytest

import subpixel_ref as ref

F = np.float64


def rnd(x):
    """The double nearest the exact rational x (one correctly rounded operation)."""
    return F(float(x))


def fit_rational(c):
    """The fit with every operation formed exactly and then rounded once, in the header's order: an independent
    statement of what fit() must return bit for bit."""
    q = [[Q(float(c[i][j])) for j in range(3)] for i in range(3)]
    R = lambda x: Q(float(x))  # noqa: E731
    gu = R(R(q[2][1] - q[0][1]) * Q(1, 2))
    gv = R(R(q[1][2] - q[1][0]) * Q(1, 2))
    huu = R(R(q[2][1] + q[0][1]) - R(2 * q[1][1]))
    hvv = R(R(q[1][2] + q[1][0]) - R(2 * q[1][1]))
    huv = R(R(R(q[2][2] - q[2][0]) - R(q[0][2] - q[0][0])) * Q(1, 4))
    det = R(R(huu * hvv) - R(huv * huv))
    if not (huu > 0 and det > 0):
        return None
    du = R(R(R(huv * gv) - R(hvv * gu)) / det)
    dv = R(R(R(huv * gu) - R(huu * gv)) / det)
    return float(du), float(dv)


def quadratic(c0, huu, huv, hvv, du, dv):
    """c(a, b) = c0 + huu/2 (a - du)^2 + huv (a - du)(b - dv) + hvv/2 (b - dv)^2, exactly, as doubles."""
    out = np.zeros((3, 3))
    for a in (-1, 0, 1):
        for b in (-1, 0, 1):
            x, y = Q(a) - Q(du), Q(b) - Q(dv)
            v = Q(c0) + Q(huu) / 2 * x * x + Q(huv) * x * y + Q(hvv) / 2 * y * y
            assert Q(float(v)) == v, "the test surface must be exact in doubles"
            out[a + 1, b + 1] = float(v)
    return out


def dyadic(rng, bits, lo, hi):
    return float(Q(int(rng.integers(round(lo * 2 ** bits), round(hi * 2 ** bits) + 1)), 2 ** bits))


# ---- the score --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [11, 15])
def test_score_equals_the_oracle(oracle, B):
    rng = np.random.default_rng(B)
    img = rng.integers(0, 256, (60, 80), dtype=np.uint8)
    for k in range(40):
        patch = rng.integers(0, 256, (B, B), dtype=np.uint8)
        if k % 4 == 0:  # low-contrast windows, near the sigma gate
            img2 = (img // 16 + 100).astype(np.uint8)
        else:
            img2 = img
        u, v = int(rng.integers(B, 80 - B)), int(rng.integers(B, 60 - B))
        h = (B - 1) // 2
        want = oracle.correlate2_warning(patch, img2, u - h, v - h)
        got, sg1 = ref.window_score(img2, patch, u, v)
        w = want[0] if isinstance(want, tuple) else want
        assert F(w).tobytes() == got.tobytes()


# ---- the fit against exact arithmetic -----------------------------------------------------------------------------
def test_an_exact_quadratic_returns_its_minimum():
    rng = np.random.default_rng(1)
    for _ in range(400):
        huu, hvv = dyadic(rng, 4, 0.25, 4.0), dyadic(rng, 4, 0.25, 4.0)
        huv = dyadic(rng, 4, -0.9, 0.9) * math.sqrt(huu * hvv)
        huv = float(Q(round(huv * 16), 16))
        if huu * hvv - huv * huv <= 0:
            continue
        du, dv = dyadic(rng, 6, -0.5, 0.5), dyadic(rng, 6, -0.5, 0.5)
        c = quadratic(dyadic(rng, 4, 0.0, 2.0), huu, huv, hvv, du, dv)
        gdu, gdv, ok = ref.fit(c)
        assert ok and gdu == du and gdv == dv


def test_the_fit_equals_exact_rounding_of_each_operation():
    rng = np.random.default_rng(2)
    for _ in range(2000):
        c = rng.uniform(0.0, 2.0, (3, 3))
        c[1, 1] = c.min() - rng.uniform(0.0, 0.5)
        want = fit_rational(c)
        du, dv, ok = ref.fit(c)
        if want is None:
            assert not ok
        else:
            assert (du, dv) == want
            assert ok == (abs(want[0]) <= 0.5 and abs(want[1]) <= 0.5)


def test_a_symmetric_surface_gives_zero():
    rng = np.random.default_rng(3)
    for _ in range(100):
        c = rng.uniform(0.5, 2.0, (3, 3))
        c = np.where(np.arange(9).reshape(3, 3) > 4, c[::-1, ::-1], c)  # c(a, b) = c(-a, -b)
        c[1, 1] = 0.1
        du, dv, ok = ref.fit(c)
        if ok:
            assert du == 0.0 and dv == 0.0


def test_the_offset_knife_edge():
    # huv = 0, hvv = 1, c(0,0) = 0, c(-1,0) = 1: du = -g_u / h_uu with c(1,0) = t
    def surface(t):
        c = np.array([[2.0, 1.0, 2.0], [0.5, 0.0, 0.5], [2.0, t, 2.0]])
        c[0, 0] = c[0, 2] = c[2, 0] = c[2, 2] = 2.0
        return c
    du, dv, ok = ref.fit(surface(0.0))
    assert du == 0.5 and ok  # exactly 0.5 is accepted
    above = np.nextafter(0.5, 1.0)
    du, dv, ok = ref.fit(surface(-2.0 ** -53))
    assert du == above and fit_rational(surface(-2.0 ** -53))[0] == above
    assert not ok  # the next double above 0.5 is refused
    du, dv, ok = ref.fit(surface(0.0)[::-1])  # mirrored: du = -0.5
    assert du == -0.5 and ok


@pytest.mark.parametrize("case", ["huu_zero", "det_zero", "det_negative", "nan"])
def test_degenerate_surfaces_fall_back(case):
    c = np.array([[1.0, 1.0, 1.0], [1.0, 0.0, 1.0], [1.0, 1.0, 1.0]])
    if case == "huu_zero":
        c[0, 1] = c[2, 1] = 0.0
    elif case == "det_zero":  # huu = hvv = 2, huv = 2
        c[2, 2] = c[0, 0] = 1.0 + 4.0
    elif case == "det_negative":  # a saddle
        c[1, 0] = c[1, 2] = -1.0
    else:
        c[2, 2] = np.nan
    if case == "det_zero":
        huu = (c[2, 1] + c[0, 1]) - 2 * c[1, 1]
        huv = ((c[2, 2] - c[2, 0]) - (c[0, 2] - c[0, 0])) * 0.25
        assert huu > 0 and huu * huu - huv * huv == 0.0
    assert not ref.fit(c)[2]


def textured(rng, H, W, sigma=2.0, contrast=60.0):
    """A smooth random texture, evaluated at any real position: a sum of sinusoids of wavelength >= 2 pi sigma."""
    k = rng.normal(0.0, 1.0 / sigma, (24, 2))
    ph = rng.uniform(0, 2 * np.pi, 24)
    amp = rng.uniform(0.5, 1.0, 24)

    def at(x, y):
        s = np.zeros(np.broadcast(x, y).shape)
        for i in range(24):
            s += amp[i] * np.cos(k[i, 0] * x + k[i, 1] * y + ph[i])
        return np.clip(np.rint(128.0 + contrast * s / np.sqrt((amp ** 2).sum() / 2)), 0, 255).astype(np.uint8)
    return at


def test_the_sigma_gate_and_the_image_edge_fall_back():
    rng = np.random.default_rng(5)
    at = textured(rng, 60, 60)
    ys, xs = np.mgrid[0:60, 0:60]
    img = at(xs.astype(float), ys.astype(float))
    B, h = 11, 5
    patch = img[30 - h:30 + h + 1, 31 - h:31 + h + 1].copy()
    zu, zv, ok = ref.refine(img, 60, 60, patch, 31, 30)
    assert ok
    # a window of the nine leaves the image: u - 1 - h < 0 or u + 1 + h > W - 1
    assert not ref.refine(img, 60, 60, patch, h, 30)[2]
    assert not ref.refine(img, 60, 60, patch, 31, 60 - 1 - h)[2]
    assert not ref.refine(img, 37 + h, 60, patch, 37, 30)[2]  # the stream's own width
    # one window flat enough to have sigma_g1 < 10
    flat = img.copy()
    flat[30 - h - 1:30 + h, 31 - h - 1:31 + h] = (flat[30 - h - 1:30 + h, 31 - h - 1:31 + h] // 16 + 120)
    c, sg = ref.scores(flat, patch, 31, 30)
    assert (sg < 10).any()
    assert not ref.refine(flat, 60, 60, patch, 31, 30)[2]


# ---- broken copies ------------------------------------------------------------------------------------------------
def fit_broken(c, flip_huv=False, fma_det=False):
    """fit() with h_uv's sign swapped, or det formed with one fused multiply-add."""
    c = [[F(c[i][j]) for j in range(3)] for i in range(3)]
    gu = (c[2][1] - c[0][1]) * F(0.5)
    gv = (c[1][2] - c[1][0]) * F(0.5)
    huu = (c[2][1] + c[0][1]) - F(2.0) * c[1][1]
    hvv = (c[1][2] + c[1][0]) - F(2.0) * c[1][1]
    huv = ((c[2][2] - c[2][0]) - (c[0][2] - c[0][0])) * F(0.25)
    if flip_huv:
        huv = -huv
    det = rnd(Q(float(huu)) * Q(float(hvv)) - Q(float(huv * huv))) if fma_det else huu * hvv - huv * huv
    if not (huu > 0.0 and det > 0.0):
        return F(0.0), F(0.0), False
    du = (huv * gv - hvv * gu) / det
    dv = (huv * gu - huu * gv) / det
    return du, dv, bool(-0.5 <= du <= 0.5 and -0.5 <= dv <= 0.5)


def refine_gate_le(image, width, height, patch, u, v):
    """sigma_g1 <= 10 refused instead of < 10."""
    c, sg = ref.scores(image, patch, u, v)
    if (sg <= 10.0).any():
        return F(u), F(v), False
    return ref.refine(image, width, height, patch, u, v)


def test_broken_fits_are_caught():
    rng = np.random.default_rng(7)
    cases = []
    for _ in range(300):
        c = rng.uniform(0.0, 2.0, (3, 3))
        c[1, 1] = c.min() - rng.uniform(0.0, 0.5)
        cases.append(c)

    def caught(broken):
        for c in cases:
            a, b = ref.fit(c), broken(c)
            if a[2] != b[2] or (a[2] and (a[0].tobytes(), a[1].tobytes()) != (F(b[0]).tobytes(), F(b[1]).tobytes())):
                return True
        return False
    for c in cases:  # the restatement itself is the exact rounding of each operation
        want, got = fit_rational(c), ref.fit(c)
        assert (want is None and not got[2]) or (want is not None and (got[0], got[1]) == want)
    assert not caught(ref.fit)
    assert not caught(fit_broken)
    assert caught(lambda c: fit_broken(c, flip_huv=True))
    assert caught(lambda c: fit_broken(c, fma_det=True))


def test_a_wrong_sigma_gate_is_caught():
    # a window with sigma_g1 exactly 10: the search accepts it, so the refinement must too
    B, h = 11, 5
    n = B * B
    vals = np.full(n, 100, np.int64)
    # sigma^2 = S2/n - (S1/n)^2 = 100 exactly: 100 pixels at 100 +- 11 and 21 at 100 gives var = 100 * 121 / 121
    vals[:50] = 111
    vals[50:100] = 89
    S1, S2 = int(vals.sum()), int((vals * vals).sum())
    assert ref.exact_score(ref.patch_const(B, 5000, 300000), S1, S2, 0)[1] == 10.0
    rng = np.random.default_rng(9)
    win = vals.reshape(B, B)
    img = rng.integers(0, 256, (40, 40), dtype=np.uint8)
    img[20 - h:20 + h + 1, 20 - h:20 + h + 1] = win
    patch = img[20 - h:20 + h + 1, 21 - h:21 + h + 1].copy()
    c, sg = ref.scores(img, patch, 21, 20)
    assert sg[0, 1] == 10.0 and (sg >= 10.0).all()
    assert ref.refine(img, 40, 40, patch, 21, 20)[2]  # the search's gate: sigma_g1 = 10 passes
    assert not refine_gate_le(img, 40, 40, patch, 21, 20)[2]


# ---- capability on shifted textures --------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [11, 15])
def test_fractional_shifts_are_recovered(B):
    rng = np.random.default_rng(20 + B)
    H = W = 48
    h = (B - 1) // 2
    ys, xs = np.mgrid[0:H, 0:W].astype(float)
    err_int, err_sub, refined = [], [], []
    for _ in range(60):
        at = textured(rng, H, W)
        patch = at(xs, ys)[24 - h:24 + h + 1, 24 - h:24 + h + 1]
        dx, dy = rng.uniform(-0.5, 0.5, 2)
        img = at(xs - dx, ys - dy)  # the patch's centre is now at (24 + dx, 24 + dy)
        best, bu, bv = np.inf, 0, 0
        for u in range(20, 29):
            for v in range(20, 29):
                s, sg = ref.window_score(img, patch, u, v)
                if s <= best:
                    best, bu, bv = s, u, v
        zu, zv, ok = ref.refine(img, W, H, patch, bu, bv)
        refined.append(ok)
        err_int.append(np.hypot(bu - 24 - dx, bv - 24 - dy))
        err_sub.append(np.hypot(zu - 24 - dx, zv - 24 - dy))
    err_int, err_sub, refined = np.array(err_int), np.array(err_sub), np.array(refined)
    # the fits that land beyond half a pixel (true offsets near +-0.5) keep the integer match
    assert refined.mean() >= 0.85
    assert err_sub[refined].max() < 0.3
    assert np.sqrt((err_sub ** 2).mean()) <= 0.6 * np.sqrt((err_int ** 2).mean())


# ---- the oracle's refinement ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [11, 15])
def test_the_oracle_refines_like_the_restatement(B):
    import subpixel_oracle as so
    rng = np.random.default_rng(40 + B)
    H = W = 48
    h = (B - 1) // 2
    ys, xs = np.mgrid[0:H, 0:W].astype(float)
    refined = 0
    for k in range(40):
        at = textured(rng, H, W)
        patch = at(xs, ys)[24 - h:24 + h + 1, 24 - h:24 + h + 1]
        dx, dy = rng.uniform(-0.5, 0.5, 2)
        img = at(xs - dx, ys - dy)
        for u, v in ((24, 24), (25, 24), (h + 1, 24), (24, W - 2 - h)):
            want = ref.refine(img, W, H, patch, u, v)
            got = so.refine(img, W, H, patch, u, v)
            assert got[2] == want[2] and F(got[0]).tobytes() == want[0].tobytes() and F(got[1]).tobytes() == want[1].tobytes()
            refined += got[2]
    assert refined >= 40
