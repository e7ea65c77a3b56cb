"""CPU checks of the raw-frame sources (sl2_set_stream_source): the NumPy restatement of the device's conversions
(tests/ingest_ref.py) against OpenCV where cv2 is installed, and the golden fixtures the GPU tests read against the
restatement."""
import glob
import os

import numpy as np
import pytest

import ingest_ref as ir

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _size_pairs(rng):
    """(sw, sh, dw, dh): every class at least ~60 times: downscales, upscales, identity, exact 2x, 1-pixel and odd
    sizes, mixed (up in one direction, down in the other), and camera sizes to the reference's 320 x 240."""
    pairs = [(640, 480, 320, 240), (1280, 720, 320, 240), (352, 288, 320, 240), (160, 120, 320, 240),
             (320, 240, 320, 240), (1, 1, 7, 5), (7, 5, 1, 1), (1, 9, 1, 4), (9, 1, 4, 1)]
    for k in range(540):
        cls = k % 9
        a, b = (int(v) for v in rng.integers(1, 160, 2))
        c, d = (int(v) for v in rng.integers(1, 160, 2))
        if cls == 0:
            pairs.append((max(a, c) + 1, max(b, d) + 1, min(a, c), min(b, d)))  # down
        elif cls == 1:
            pairs.append((min(a, c), min(b, d), max(a, c) + 1, max(b, d) + 1))  # up
        elif cls == 2:
            pairs.append((a, b, a, b))
        elif cls == 3:
            pairs.append((2 * a, 2 * b, a, b))
        elif cls == 4:
            pairs.append((1, b, c, d) if k % 2 else (a, 1, c, d))
        elif cls == 5:
            pairs.append((a, b, 1, d) if k % 2 else (a, b, c, 1))
        elif cls == 6:
            pairs.append((a | 1, b | 1, c | 1, d | 1))
        elif cls == 7:
            pairs.append((a, min(b, d), c, max(b, d) + 3))
        else:
            pairs.append((int(rng.integers(321, 1400)), int(rng.integers(241, 1000)), 320, 240))
    return pairs


def test_resize_matches_cv2_on_random_size_pairs():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(20261016)
    pairs = _size_pairs(rng)
    assert len(pairs) >= 500
    for sw, sh, dw, dh in pairs:
        src = rng.integers(0, 256, (sh, sw), dtype=np.uint8)
        ref = cv2.resize(src, (dw, dh), interpolation=cv2.INTER_LINEAR)
        assert np.array_equal(ir.resize_linear(src, dw, dh), ref), (sw, sh, dw, dh)


def test_rows_keep_their_weights_at_the_border():
    """The rule that tells the vertical pass from the horizontal one: clamping the row weights as the columns' are
    would differ from cv2 on upscales."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(3)
    src = rng.integers(0, 256, (5, 40), dtype=np.uint8)
    ref = cv2.resize(src, (40, 17), interpolation=cv2.INTER_LINEAR)
    assert np.array_equal(ir.resize_linear(src, 40, 17), ref)
    # the top output row lies above source row 0 (f < 0): its weights are not (2048, 0) and rounding shows it
    i, w0, w1 = ir._taps(17, 5, False)
    assert i[0] < 0 and w1[0] > 0


def test_uyvy_matches_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(4)
    for h, w in ((1, 2), (37, 46), (240, 320), (3, 1000)):
        raw = rng.integers(0, 256, (h, w, 2), dtype=np.uint8)
        assert np.array_equal(ir.uyvy_to_gray(raw), cv2.cvtColor(raw, cv2.COLOR_YUV2GRAY_UYVY))
        assert np.array_equal(ir.to_gray(ir.SRC_UYVY, raw, w, h), raw[..., 1])
    assert cv2.COLOR_YUV2GRAY_Y422 == cv2.COLOR_YUV2GRAY_UYVY


def test_rgb_over_every_colour():
    """All 2^24 colours: the restatement is OpenCV 2.4's 14-bit formula, an installed cv2 (OpenCV 4) is exactly the
    15-bit one, and the two versions differ by one grey level on the colours where their roundings part."""
    c = np.arange(1 << 24, dtype=np.uint32)
    rgb = np.stack([(c >> 16) & 255, (c >> 8) & 255, c & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
    r, g, b = (rgb[..., i].astype(np.int64) for i in range(3))
    g14 = ir.rgb_to_gray(rgb)
    assert np.array_equal(g14, (4899 * r + 9617 * g + 1868 * b + 8192) >> 14)
    g15 = ir.rgb_to_gray_cv4(rgb)
    diff = g14.astype(np.int16) - g15.astype(np.int16)
    assert np.abs(diff).max() == 1 and 0 < np.count_nonzero(diff) < (1 << 24) // 100
    try:
        import cv2
    except ImportError:
        return
    assert np.array_equal(cv2.cvtColor(rgb, cv2.COLOR_RGB2GRAY), g15)


def test_golden_fixtures_match_the_restatement():
    files = sorted(glob.glob(os.path.join(GOLDEN, "ingest_*.npz")))
    assert files
    n = 0
    for p in files:
        z = np.load(p)
        for k in range(int(z["count"])):
            fmt, sw, sh, dw, dh = (int(v) for v in z["case_%d" % k])
            assert np.array_equal(ir.ingest(fmt, z["raw_%d" % k], sw, sh, dw, dh), z["gray_%d" % k]), (p, k)
            n += 1
    assert n >= 15
