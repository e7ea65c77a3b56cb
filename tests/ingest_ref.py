"""NumPy restatement of the raw-frame conversions of sl2_set_stream_source (csrc/ingest.cu): the cvtColor + resize of
the reference's camera grabber (framegrabber/usbcamgrabber.cpp:75-113).  Needs NumPy only; tests/test_ingest.py
checks it against cv2 where cv2 is installed."""
import numpy as np

SRC_GRAY8, SRC_RGB24, SRC_UYVY = 1, 2, 3
BPP = {SRC_GRAY8: 1, SRC_RGB24: 3, SRC_UYVY: 2}


def rgb_to_gray(rgb):
    """OpenCV 2.4's RGB2Gray<uchar> (yuv_shift 14): what the reference's pinned OpenCV 2.4.2 computes."""
    r, g, b = (rgb[..., i].astype(np.int64) for i in range(3))
    return ((4899 * r + 9617 * g + 1868 * b + 8192) >> 14).astype(np.uint8)


def rgb_to_gray_cv4(rgb):
    """OpenCV 4's form (shift 15), for the comparison with an installed cv2 only."""
    r, g, b = (rgb[..., i].astype(np.int64) for i in range(3))
    return ((9798 * r + 19235 * g + 3735 * b + 16384) >> 15).astype(np.uint8)


def uyvy_to_gray(uyvy):
    """(H, 2W) or (H, W, 2) bytes U Y0 V Y1 ...: byte 1 of every 2-byte pixel."""
    return np.ascontiguousarray(np.asarray(uyvy).reshape(uyvy.shape[0], -1)[:, 1::2])


def _taps(d, s, clamp):
    scale = 1.0 / (d / s)
    f = ((np.arange(d) + 0.5) * scale - 0.5).astype(np.float32)
    i = np.floor(f).astype(np.int64)
    f = (f - i.astype(np.float32)).astype(np.float32)
    if clamp:
        lo = i < 0
        f[lo], i[lo] = 0, 0
        hi = i >= s - 1
        f[hi], i[hi] = 0, s - 1
    w1 = np.rint(f * np.float32(2048)).astype(np.int64)
    w0 = np.rint((np.float32(1) - f) * np.float32(2048)).astype(np.int64)
    return i, w0, w1


def resize_linear(src, dw, dh):
    """OpenCV's 8-bit INTER_LINEAR resize of a gray image to dw x dh (pinned to cv2 4.13; the 2x case is the same in
    every OpenCV version).  Columns clamp their index and weight at both borders, rows only their index."""
    sh, sw = src.shape
    s = src.astype(np.int64)
    if (dw, dh) == (sw, sh):
        return src.copy()
    if (2 * dw, 2 * dh) == (sw, sh):  # INTER_AREA's fast path
        return ((s[0::2, 0::2] + s[0::2, 1::2] + s[1::2, 0::2] + s[1::2, 1::2] + 2) >> 2).astype(np.uint8)
    xi, a0, a1 = _taps(dw, sw, True)
    S = s[:, xi] * a0 + s[:, np.minimum(xi + 1, sw - 1)] * a1
    yi, b0, b1 = _taps(dh, sh, False)
    r0, r1 = np.clip(yi, 0, sh - 1), np.clip(yi + 1, 0, sh - 1)
    out = (((b0[:, None] * (S[r0] >> 4)) >> 16) + ((b1[:, None] * (S[r1] >> 4)) >> 16) + 2) >> 2
    return out.astype(np.uint8)


def to_gray(fmt, raw, width, height):
    """A packed raw frame (bytes in any shape) of format fmt and size width x height -> its gray image."""
    raw = np.ascontiguousarray(raw, np.uint8).reshape(height, width * BPP[fmt])
    if fmt == SRC_RGB24:
        return rgb_to_gray(raw.reshape(height, width, 3))
    if fmt == SRC_UYVY:
        return uyvy_to_gray(raw)
    return raw.copy()


def ingest(fmt, raw, width, height, dw, dh):
    """What the device writes into a stream's ring block: gray conversion, then the resize to dw x dh."""
    return resize_linear(to_gray(fmt, raw, width, height), dw, dh)


def raw_like(fmt, gray, rng, noise=6):
    """A raw frame of format fmt whose gray image is close to `gray` (same size): colour channels or chroma bytes
    around it, so that a tracker still sees the scene after the conversion."""
    h, w = gray.shape
    g = gray.astype(np.int64)
    if fmt == SRC_RGB24:
        out = g[..., None] + rng.integers(-noise, noise + 1, (h, w, 3))
        return np.clip(out, 0, 255).astype(np.uint8)
    if fmt == SRC_UYVY:
        out = rng.integers(0, 256, (h, w, 2), dtype=np.uint8)
        out[..., 1] = gray
        return out
    return gray.copy()


def upsample2(gray):
    return np.repeat(np.repeat(gray, 2, axis=0), 2, axis=1)
