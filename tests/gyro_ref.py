"""The gyroscope update restated op for op (include/sl2b200.h, sl2_set_stream_gyro; csrc/gyro.cu): Python floats for the
3 x 3 part and NumPy elementwise float64 operations, each one correctly rounded and never fused, for the rows of W and
the n x n downdate.  x and P are the stream's state of size n (P column-major as sl2_get_state returns it, which is the
same array as row-major since P is symmetric)."""
import math

import numpy as np


def rc_of(R, C):
    """Rc = R^T C R as sl2_set_stream_gyro forms it: M = C R, then the upper triangle of R^T M, mirrored."""
    R = [[float(v) for v in row] for row in np.asarray(R, np.float64).reshape(3, 3)]
    C = [[float(v) for v in row] for row in np.asarray(C, np.float64).reshape(3, 3)]
    M = [[(C[k][0] * R[0][j] + C[k][1] * R[1][j]) + C[k][2] * R[2][j] for j in range(3)] for k in range(3)]
    Rc = [[0.0] * 3 for _ in range(3)]
    for i in range(3):
        for j in range(i, 3):
            Rc[i][j] = Rc[j][i] = (R[0][i] * M[0][j] + R[1][i] * M[1][j]) + R[2][i] * M[2][j]
    return Rc


def zc_of(R, b, z):
    """zc = R^T (z - b)"""
    R = np.asarray(R, np.float64).reshape(3, 3)
    d = [float(z[k]) - float(b[k]) for k in range(3)]
    return [(float(R[0, i]) * d[0] + float(R[1, i]) * d[1]) + float(R[2, i]) * d[2] for i in range(3)]


def prep(x, P, Rc, zc, nis_terms=3, bad_W=False):
    """gyro_prep_kernel on copies: -> (status, nis, W (n x 3) or None, x').  nis_terms / bad_W make the broken copies
    the tests must catch (a missing NIS term; W formed from rows of P that the downdate already changed)."""
    x = np.array(x, np.float64)
    n = x.size
    Pw = lambda i, j: float(P[10 + i, 10 + j])  # noqa: E731
    S00, S10, S20 = Pw(0, 0) + Rc[0][0], Pw(1, 0) + Rc[1][0], Pw(2, 0) + Rc[2][0]
    S11, S21, S22 = Pw(1, 1) + Rc[1][1], Pw(2, 1) + Rc[2][1], Pw(2, 2) + Rc[2][2]
    sq = lambda v: math.sqrt(v) if v >= 0 else math.nan  # noqa: E731  (NaN: the device's sqrt of a negative)
    l00 = sq(S00)
    l10, l20 = _div(S10, l00), _div(S20, l00)
    a11 = S11 - l10 * l10
    l11 = sq(a11)
    l21 = _div(S21 - l20 * l10, l11)
    a22 = (S22 - l20 * l20) - l21 * l21
    l22 = sq(a22)
    nu = [zc[i] - float(x[10 + i]) for i in range(3)]
    w0 = _div(nu[0], l00)
    w1 = _div(nu[1] - l10 * w0, l11)
    w2 = _div((nu[2] - l20 * w0) - l21 * w1, l22)
    q = (w0 * w0 + w1 * w1) + (w2 * w2 if nis_terms == 3 else 0.0)
    vals = (S00, S10, S20, S11, S21, S22, l00, l10, l20, l11, l21, l22, *nu, w0, w1, w2, q)
    if not (S00 > 0 and a11 > 0 and a22 > 0 and all(math.isfinite(v) for v in vals)):
        return 2, 0.0, None, x
    p0, p1, p2 = (np.array(P[:n, 10 + c], np.float64) for c in range(3))
    W0 = p0 / l00
    W1 = (p1 - W0 * l10) / l11
    W2 = ((p2 - W0 * l20) - W1 * l21) / l22
    if bad_W:  # the rows 10..12 of P already downdated by the earlier rows' W
        Wg = np.stack([W0, W1, W2], 1)
        Pd = downdate(P, Wg)
        p0, p1, p2 = (Pd[:n, 10 + c] for c in range(3))
        W0 = p0 / l00
        W1 = (p1 - W0 * l10) / l11
        W2 = ((p2 - W0 * l20) - W1 * l21) / l22
    x = x + ((W0 * w0 + W1 * w1) + W2 * w2)
    return 1, q, np.stack([W0, W1, W2], 1), x


def _div(a, b):
    return a / b if b != 0.0 else math.nan  # a zero divisor is a pivot argument that is not > 0: skipped either way


def downdate(P, W):
    """gyro_downdate_kernel: P(i, j) - ((W[i][0] W[j][0] + W[i][1] W[j][1]) + W[i][2] W[j][2]) over the n x n block."""
    P = np.array(P, np.float64)
    n = W.shape[0]
    a, b = W[:, None, :], W[None, :, :]
    P[:n, :n] = P[:n, :n] - ((a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2])
    return P


def update(x, P, R, bias, cov, z, transpose_R=False, flip_bias=False, nis_terms=3, bad_W=False):
    """The whole update of one sample z: -> (x', P', nis, status).  The keyword arguments make broken copies."""
    R = np.asarray(R, np.float64).reshape(3, 3)
    Rk = R.T if transpose_R else R
    b = -np.asarray(bias, np.float64) if flip_bias else np.asarray(bias, np.float64)
    st, q, W, x2 = prep(x, P, rc_of(Rk, cov), zc_of(Rk, b, z), nis_terms, bad_W)
    if st != 1:
        return np.array(x, np.float64), np.array(P, np.float64), 0.0, st
    return x2, downdate(P, W), q, st
