"""NumPy restatement of the sub-pixel refinement (csrc/subpixel.cu subpixel_kernel, include/sl2b200.h
sl2_set_stream_subpixel): the search's exact score of the 3 x 3 windows around an integer match (improc.cpp:99-133 as
sl2_score.cuh states it) and the quadratic fit, one correctly rounded float64 operation at a time in the device's
order."""
import numpy as np

F = np.float64
SIGMA_GATE = 10.0  # kCorrelationSigmaThreshold: the search's gate on sigma_g1


def patch_const(B, Sg0, Sg0sq):
    """sl2_score.cuh patch_const: the template's constants from its integer sums."""
    with np.errstate(all="ignore"):
        n = F(B * B)
        Sg0d, Sg0sqd = F(Sg0), F(Sg0sq)
        g0bar = Sg0d / n
        varg0 = Sg0sqd / n - g0bar * g0bar
        sigmag0 = np.sqrt(varg0)
        return dict(n=n, sigmag0=sigmag0, A0=Sg0sqd / varg0, g0s=g0bar / sigmag0, Sg0x2=Sg0d * F(2.0))


def exact_score(pc, Sg1, Sg1sq, Sg0g1):
    """sl2_score.cuh exact_score_fn -> (score, sigma_g1)."""
    with np.errstate(all="ignore"):
        n = pc["n"]
        Sg1d, Sg1sqd, Sg0g1d = F(Sg1), F(Sg1sq), F(Sg0g1)
        g1bar = Sg1d / n
        varg1 = Sg1sqd / n - g1bar * g1bar
        sigmag1 = np.sqrt(varg1)
        if pc["sigmag0"] == 0.0:
            return (F(0.0) if sigmag1 == 0.0 else F(1.0)), sigmag1
        if sigmag1 == 0.0:
            return F(1.0), sigmag1
        k = pc["g0s"] - g1bar / sigmag1
        C = pc["A0"] + Sg1sqd / varg1
        C = C + n * (k * k)
        C = C - (Sg0g1d * F(2.0)) / (pc["sigmag0"] * sigmag1)
        C = C - (pc["Sg0x2"] * k) / pc["sigmag0"]
        C = C + ((Sg1d * F(2.0)) * k) / sigmag1
        return C / n, sigmag1


def window_score(image, patch, uc, vc):
    """The exact score and sigma_g1 of the window of `image` centred at (uc, vc) against `patch` (B x B u8)."""
    B = patch.shape[0]
    h = (B - 1) // 2
    T = patch.astype(np.int64)
    g = image[vc - h:vc + h + 1, uc - h:uc + h + 1].astype(np.int64)
    pc = patch_const(B, int(T.sum()), int((T * T).sum()))
    return exact_score(pc, int(g.sum()), int((g * g).sum()), int((T * g).sum()))


def fit(c):
    """The fit of the 3 x 3 scores c[a + 1][b + 1] = c(a, b) -> (du, dv, ok); ok = False: keep the integer match."""
    c = [[F(c[i][j]) for j in range(3)] for i in range(3)]
    with np.errstate(all="ignore"):
        gu = (c[2][1] - c[0][1]) * F(0.5)
        gv = (c[1][2] - c[1][0]) * F(0.5)
        huu = (c[2][1] + c[0][1]) - F(2.0) * c[1][1]
        hvv = (c[1][2] + c[1][0]) - F(2.0) * c[1][1]
        huv = ((c[2][2] - c[2][0]) - (c[0][2] - c[0][0])) * F(0.25)
        det = huu * hvv - huv * huv
        if not (huu > 0.0 and det > 0.0):
            return F(0.0), F(0.0), False
        du = (huv * gv - hvv * gu) / det
        dv = (huv * gu - huu * gv) / det
    ok = bool(-0.5 <= du <= 0.5 and -0.5 <= dv <= 0.5)
    return du, dv, ok


def scores(image, patch, u, v):
    """c[a + 1][b + 1] and sigma_g1 of the nine windows around (u, v) (all inside the image)."""
    c = np.zeros((3, 3))
    sg = np.zeros((3, 3))
    for a in (-1, 0, 1):
        for b in (-1, 0, 1):
            c[a + 1, b + 1], sg[a + 1, b + 1] = window_score(image, patch, u + a, v + b)
    return c, sg


def refine(image, width, height, patch, u, v):
    """The refinement of a successful match (u, v) of `patch` in the stream's width x height `image` -> (zu, zv,
    refined)."""
    h = (patch.shape[0] - 1) // 2
    if u - 1 - h < 0 or u + 1 + h > width - 1 or v - 1 - h < 0 or v + 1 + h > height - 1:
        return F(u), F(v), False
    c, sg = scores(image, patch, u, v)
    if (sg < SIGMA_GATE).any():
        return F(u), F(v), False
    du, dv, ok = fit(c)
    if not ok:
        return F(u), F(v), False
    return F(u) + du, F(v) + dv, True
