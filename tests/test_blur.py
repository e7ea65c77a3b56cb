"""The exposure blur on the CPU: the op-for-op restatement (tests/blur_ref.py) against the extended-precision truth
(tests/blur_truth.py) on every decided byte, exact constructions, the fallback, the quadratic's departure from exact
per-sample mapping, broken copies the comparison must catch, and the sl2_stream_blur layout."""
import numpy as np
import pytest

import blur_ref as br
import blur_truth as bt
import warp_cases as wc
import warp_ref
from test_abi import AbiCase, _c_layout
from scenelib2_b200 import lib as mirror

EXPOSURE = 1.0 / 60.0
RATES = (0.0, 0.4, 1.5, 3.0, 6.0, 15.0)  # rad/s: streaks from 0 to beyond the 32-sample cap at 1/60 s


def blur_cases(seed=23):
    """[(name, cam8, B, y, xo, x (13), exposure, offset, warp)] over the warp's random cases (every camera, |q| != 1
    included), at rates from rest to beyond the cap, with offsets 0, -exposure/2 and a positive one, warp on and off."""
    rng = np.random.default_rng(seed)
    out = []
    for i, (name, cam8, B, y, xo, xp, T) in enumerate(wc.random_cases(per=1, seed=5)):
        rate = RATES[i % len(RATES)]
        axis = rng.standard_normal(3)
        om = axis / np.linalg.norm(axis) * rate
        v = rng.standard_normal(3) * 0.3 * (rate > 0)
        x = np.concatenate([xp, v, om])
        offset = (0.0, -EXPOSURE / 2, 0.004)[i % 3]
        out.append((name, cam8, B, y, xo, x, EXPOSURE, offset, bool(i % 2), T))
    return out


CASES = blur_cases()


def test_restatement_equals_the_truth_on_every_decided_byte():
    ks, decided_bytes, blurred = set(), 0, 0
    for name, cam8, B, y, xo, x, ex, off, warp, T in CASES:
        out, valid, K = br.blur_template(cam8, T, y, xo, x, ex, off, warp)
        t = bt.blur_truth(cam8, T, y, xo, x, ex, off, warp)
        case_ok, mask = bt.decided(t)
        if not case_ok:
            continue
        if t.v is None:
            assert valid != 2, name
            continue
        assert valid == 2 and K == t.K, (name, K, t.K, t.L)
        ks.add(K)
        blurred += 1
        decided_bytes += int(mask.sum())
        assert (out[mask] == t.byte[mask]).all(), (name, np.argwhere(out != t.byte))
    assert blurred >= 0.6 * len(CASES), blurred
    assert 1 in ks and 32 in ks and any(1 < k < 32 for k in ks), ks
    assert decided_bytes >= 0.99 * 121 * blurred


def test_seeded_normals_equal_the_truth():
    """The warp's plane through an estimated tilt nW(theta) (normals on), with the warp on and off."""
    rng = np.random.default_rng(41)
    checked = 0
    for name, cam8, B, y, xo, x, ex, off, warp, T in CASES[::2]:
        theta = tuple(rng.uniform(-0.3, 0.3, 2))
        out, valid, K = br.blur_template(cam8, T, y, xo, x, ex, off, warp, theta=theta)
        t = bt.blur_truth(cam8, T, y, xo, x, ex, off, warp, theta=theta)
        case_ok, mask = bt.decided(t)
        if not case_ok or t.v is None:
            continue
        assert valid == 2 and K == t.K, name
        assert (out[mask] == t.byte[mask]).all(), name
        checked += 1
    assert checked >= 0.5 * len(CASES[::2]), checked


def test_longdouble_truth_agrees_with_50_digits():
    name, cam8, B, y, xo, x, ex, off, warp, T = next(
        c for c in CASES if c[2] == 11 and 1 < br.blur_template(c[1], c[9], *c[3:9])[2] <= 8)
    ld = bt.blur_truth(cam8, T, y, xo, x, ex, off, warp, prec="ld", theta=(0.2, -0.1))
    mp = bt.blur_truth(cam8, T, y, xo, x, ex, off, warp, prec="mp", theta=(0.2, -0.1))
    assert ld.K == mp.K and ld.valid == mp.valid and ld.K > 1
    assert abs(ld.L - mp.L) <= 1e-12 * max(1.0, mp.L)
    assert np.nanmax(np.abs(ld.src - mp.src)) <= 1e-12
    assert np.abs(ld.v - mp.v).max() <= 1e-9 and (ld.byte == mp.byte).all()


@pytest.mark.parametrize("warp", [False, True])
def test_exposure_zero_is_the_warp_or_the_stored_template(warp):
    for name, cam8, B, y, xo, x, ex, off, _, T in CASES[:30]:
        out, valid, K = br.blur_template(cam8, T, y, xo, x, 0.0, 0.0, warp)
        want, wv = warp_ref.warp_template(cam8, T, y, xo, x[:7]) if warp else (np.asarray(T, np.uint8), 0)
        if warp and not wv:
            assert valid == 1 or valid == 0
            continue
        assert valid == 2 and K == 1, name
        assert out.tobytes() == want.tobytes(), name


@pytest.mark.parametrize("B", [11, 15])
@pytest.mark.parametrize("K", [3, 5, 7])
def test_translation_along_a_fronto_parallel_plane_averages_shifted_columns(B, K):
    """kd1 = 0, fku = 256, the plane z = 2 faced by a camera at the origin moving along x with a 1/64 s exposure: the
    sources move by 128 v s px, so v = K / 2 gives a streak of exactly K px and K samples on integer columns."""
    rng = np.random.default_rng(K + B)
    cam8 = wc.CAM_EXACT
    T = rng.integers(0, 256, (B, B)).astype(np.uint8)
    x = np.array([0, 0, 0, 1, 0, 0, 0, K / 2.0, 0, 0, 0, 0, 0], np.float64)
    out, valid, k = br.blur_template(cam8, T, wc.Y_AXIS, wc.XO_AXIS, x, 1.0 / 64, 0.0, False)
    assert valid == 2 and k == K
    h = K // 2
    cols = np.stack([T[:, h + j: B - h + j].astype(np.int64) for j in range(-h, h + 1)])
    want = np.floor(cols.sum(0) / K + 0.5).astype(np.uint8)
    assert (out[:, h:B - h] == want).all()
    t = bt.blur_truth(cam8, T, wc.Y_AXIS, wc.XO_AXIS, x, 1.0 / 64, 0.0, False)
    assert t.K == K and (t.byte == out).all()


@pytest.mark.parametrize("warp", [False, True])
def test_an_invalid_end_pose_falls_back(warp):
    """The camera at the origin facing the plane z = 2 moves along z at 300 m/s: at s+ = 1/120 s it is behind the
    plane, so the blur falls back to the warp's template (warp on) or the stored one."""
    B = 11
    T = np.random.default_rng(3).integers(0, 256, (B, B)).astype(np.uint8)
    x = np.array([0, 0, 0, 1, 0, 0, 0, 0, 0, 300.0, 0, 0, 0], np.float64)
    xo = np.array([0.0, 0.0, 0.25, 1, 0, 0, 0])
    out, valid, K = br.blur_template(wc.CAM_EXACT, T, wc.Y_AXIS, xo, x, EXPOSURE, 0.0, warp)
    want, wv = warp_ref.warp_template(wc.CAM_EXACT, T, wc.Y_AXIS, xo, x[:7]) if warp else (T, 0)
    assert K == 0 and valid == wv and out.tobytes() == want.tobytes()
    assert not bt.blur_truth(wc.CAM_EXACT, T, wc.Y_AXIS, xo, x, EXPOSURE, 0.0, warp).valid


def test_quadratic_departs_from_exact_per_sample_mapping_by_little():
    """At the tested rates, with streaks up to the 32-px cap, the quadratic through the three exact sources stays
    within 0.05 template px of the exact source at every sample's own time (0.041 px at a 30 px streak)."""
    worst, streak = 0.0, 0.0
    for name, cam8, B, y, xo, x, ex, off, warp, T in CASES:
        J = br.setup(cam8, B, y, xo, x, ex, off, warp)
        L, K, ok = br.sample_count(cam8, B, J)
        if not ok or K == 1 or L > 32:
            continue
        s = [br.sources(cam8, B, J, k) for k in range(3)]
        if not all(v.all() for _, v in s):
            continue
        pts = br.quadratic_points(s[0][0], s[1][0], s[2][0], K)
        for m in range(K):
            u = (m + 0.5) / K - 0.5
            Jm = br.setup(cam8, B, y, xo, x, 0.0, off + u * ex, warp)
            exact, v = br.sources(cam8, B, Jm, 1)
            worst = max(worst, float(np.abs(pts[m] - exact)[v].max()))
        streak = max(streak, L)
    print("quadratic departure", worst, "px over streaks up to", streak, "px")
    assert streak > 10 and worst <= 0.05, (worst, streak)


BROKEN = {"swap_order": dict(swap_order=True), "centre_at_s": dict(centre_at_s=True),
          "round_samples": dict(round_samples=True), "half_step": dict(half_step=True)}


@pytest.mark.parametrize("which", sorted(BROKEN))
def test_broken_copies_are_caught(which):
    caught = 0
    for name, cam8, B, y, xo, x, ex, off, warp, T in CASES:
        t = bt.blur_truth(cam8, T, y, xo, x, ex, off, warp)
        case_ok, mask = bt.decided(t)
        if not case_ok or t.v is None or t.K == 1:
            continue
        out, valid, K = br.blur_template(cam8, T, y, xo, x, ex, off, warp, **BROKEN[which])
        if valid != 2 or K != t.K or (out[mask] != t.byte[mask]).any():
            caught += 1
    assert caught >= 3, (which, caught)


def test_blur_struct_matches_header(tmp_path):
    case = AbiCase("sl2_stream_blur", mirror.Sl2StreamBlur, ("on", "reserved", "exposure", "offset"), size=24)
    out = _c_layout(tmp_path, case)
    import ctypes as C
    assert out["sizeof"] == (C.sizeof(mirror.Sl2StreamBlur),) == (24,)
    for f, t in mirror.Sl2StreamBlur._fields_:
        assert out[f] == (getattr(mirror.Sl2StreamBlur, f).offset, C.sizeof(t)), f
