"""The planar patch warp's restatement (tests/warp_ref.py) against exact constructions, and the C ABI of its entry
points.  CPU only: the device is held to the restatement byte for byte by tests/test_gpu_warp.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import scenelib2_b200.lib as mirror
import warp_ref
from scenelib2_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# kd1 = 0, fku = fkv, an integer principal point: the constructions below are exact up to rounding
CAM0 = np.array([320.0, 240.0, 200.0, 200.0, 160.0, 120.0, 0.0, 1.0])
C45, S45 = np.cos(np.pi / 4), np.sin(np.pi / 4)
ON_AXIS = dict(y=[0.0, 0.0, 2.0], xo=[0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0])  # fronto-parallel plane z = 2


def random_pose(rng):
    q = rng.standard_normal(4)
    return np.concatenate([rng.uniform(-1, 1, 3), q / np.linalg.norm(q)])


def point_seen_from(cam8, xo, rng, margin=30):
    """A world point that the camera at xo sees at a random pixel at least `margin` inside its image."""
    u, v = rng.uniform(margin, cam8[0] - 1 - margin), rng.uniform(margin, cam8[1] - 1 - margin)
    c0, c1 = warp_ref.unproject_point(cam8, u, v)
    zc = np.array([float(c0), float(c1), 1.0]) * rng.uniform(0.5, 3.0)
    return xo[:3] + np.array(warp_ref.rrw(xo)).T @ zc


@pytest.mark.parametrize("name", ["C1", "C3"])
def test_identity_returns_the_stored_template(name):
    """At xp = xp_org every pixel maps to itself (within rounding, which the bilinear weights absorb): the warp
    returns the stored bytes, valid, for the scene's features and for random features seen from random poses."""
    sc = synth.make_scene(name, n_frames=1)
    assert sc.cam8[6] != 0.0
    B = sc.boxsize
    rng = np.random.default_rng(7)
    y = sc.x0[13:].reshape(-1, 3)
    T = rng.integers(0, 256, (len(y), B, B), dtype=np.uint8)
    out, valid = warp_ref.warp_templates(sc.cam8, T, y, sc.xp_org, sc.xp_org[0])
    assert valid.all() and (out == T).all()
    for _ in range(40):
        xo = random_pose(rng)
        yk = point_seen_from(sc.cam8, xo, rng)
        Tk = rng.integers(0, 256, (B, B), dtype=np.uint8)
        o, v = warp_ref.warp_template(sc.cam8, Tk, yk, xo, xo)
        assert v == 1 and (o == Tk).all()


@pytest.mark.parametrize("B", [11, 15])
def test_roll_of_90_degrees_rotates_the_template(B):
    """A roll of exactly +-90 degrees about the optical axis, feature on the axis: np.rot90 of the template."""
    rng = np.random.default_rng(B)
    T = rng.integers(0, 256, (B, B), dtype=np.uint8)
    for sign, k in ((1, 1), (-1, -1)):
        out, valid = warp_ref.warp_template(CAM0, T, ON_AXIS["y"], ON_AXIS["xo"], [0, 0, 0, C45, 0, 0, sign * S45])
        assert valid == 1 and (out == np.rot90(T, k)).all(), sign


@pytest.mark.parametrize("B", [11, 15])
def test_half_the_distance_magnifies_twice(B):
    """The camera halfway to the plane along the axis sees the template twice as large: output offset d samples
    source offset d / 2, the average of two (or four) pixels where d is odd.  Multiples of 4 keep every average an
    integer, so no sample lies on a .5 tie."""
    half = (B - 1) // 2
    rng = np.random.default_rng(100 + B)
    T = (rng.integers(0, 64, (B, B)) * 4).astype(np.uint8)
    out, valid = warp_ref.warp_template(CAM0, T, ON_AXIS["y"], ON_AXIS["xo"], [0, 0, 1.0, 1, 0, 0, 0])
    assert valid == 1
    Ti = T.astype(np.int64)
    want = np.zeros((B, B), np.int64)
    for a in range(B):
        for b in range(B):
            ys = sorted({half + (a - half) // 2, half + (a - half + 1) // 2})
            xs = sorted({half + (b - half) // 2, half + (b - half + 1) // 2})
            want[a, b] = sum(Ti[r, c] for r in ys for c in xs) // (len(ys) * len(xs))
    assert (out == want).all()


@pytest.mark.parametrize("xp, why", [
    ([0, 0, 0, 0, 0, 1.0, 0], "plane behind the camera (t < 0)"),
    ([-1.0, 0, 2.0, C45, 0, S45, 0], "camera in the plane: rays parallel to it or meeting it at t = 0"),
])
def test_invalid_pixels_keep_the_stored_template(xp, why):
    rng = np.random.default_rng(3)
    T = rng.integers(0, 256, (11, 11), dtype=np.uint8)
    src, ok, _ = warp_ref.warp_source(CAM0, 11, ON_AXIS["y"], ON_AXIS["xo"], xp)
    assert not ok.all(), why
    out, valid = warp_ref.warp_template(CAM0, T, ON_AXIS["y"], ON_AXIS["xo"], xp)
    assert valid == 0 and (out == T).all(), why


def test_sampling_repeats_edge_pixels():
    """Source positions outside the template are clamped to its border (the edge repeat of a shrinking warp)."""
    T = np.arange(121, dtype=np.uint8).reshape(11, 11)
    src = np.array([[-3.0, -7.0], [14.0, 2.0], [4.0, 30.0], [10.0, 10.0]])
    assert warp_ref.sample(T, src).tolist() == [T[0, 0], T[2, 10], T[10, 4], T[10, 10]]


def test_entry_points_match_the_header(tmp_path):
    """The header's prototypes compile against the function-pointer types the ctypes mirror assumes, and lib.py
    exports and declares all three."""
    src = tmp_path / "warp_abi.c"
    src.write_text("\n".join([
        '#include "sl2b200.h"',
        "int (*set_warp)(sl2_ctx *, int32_t, int32_t) = sl2_set_stream_warp;",
        "int (*get_warp)(sl2_ctx *, int32_t, int32_t *) = sl2_get_stream_warp;",
        "int (*warp)(sl2_ctx *, int32_t, int32_t, const int32_t *, const double *, uint8_t *, uint8_t *) = "
        "sl2_warp_templates;",
        "int main(void) { return set_warp == 0 || get_warp == 0 || warp == 0; }", ""]))
    subprocess.check_call([os.environ.get("CC", "cc"), "-std=c99", "-Werror", "-Wall", "-c", "-I",
                           os.path.join(ROOT, "include"), "-o", str(tmp_path / "warp_abi.o"), str(src)])
    for name in ("sl2_set_stream_warp", "sl2_get_stream_warp", "sl2_warp_templates"):
        assert name in mirror.EXPORTS
    L = mirror.load()
    assert L.sl2_set_stream_warp.argtypes == [C.c_void_p, C.c_int32, C.c_int32]
    assert L.sl2_get_stream_warp.argtypes == [C.c_void_p, C.c_int32, mirror.i32p]
    assert len(L.sl2_warp_templates.argtypes) == 7 and L.sl2_warp_templates.argtypes[1:3] == [C.c_int32, C.c_int32]
