"""The patch normal alignment on the CPU: the restatement (tests/normals_ref.py) against the model from its definition
(tests/normals_truth.py), theta = 0 against the plain warp, convergence toward a rendered plane's true tilt, broken
copies of the restatement each caught by a named check, and the setting's layout."""
import ctypes as C

import mpmath as mp
import numpy as np
import pytest

import normals_ref
import normals_scene
import normals_truth
import warp_ref
from camera_ref import camera_points, project_point
from scenelib2_b200 import lib

EPS = np.finfo(np.float64).eps
PRM = (8, 0.5, 8.0, 0.02)


@pytest.fixture(scope="module")
def scene():
    return normals_scene.make_slanted_scene(steps=20, end_deg=20.0, n_features=12)


def cam_kd0():
    c = normals_scene.warp_scene.CAM.copy()
    c[6] = 0.0
    return c


def rel_err(a, b):
    return float(abs(mp.mpf(float(a)) - b) / max(abs(b), 1))


# ---- the model ------------------------------------------------------------------------------------------------------
def test_theta_zero_is_nw0_and_warps_as_the_plain_warp(scene):
    for k in range(len(scene.y)):
        b = normals_ref.basis(scene.xp_org[k], scene.y[k])
        assert normals_ref.normal(b, 0.0, 0.0) == b[0]
        # the basis is orthogonal, E1 and E2 as long as nW0
        n0, E1, E2 = (np.array(v) for v in b)
        L = np.linalg.norm(n0)
        assert abs(n0 @ E1) < 1e-14 * L * L and abs(n0 @ E2) < 1e-14 * L * L and abs(E1 @ E2) < 1e-14 * L * L
        assert abs(np.linalg.norm(E1) - L) < 1e-14 * L and abs(np.linalg.norm(E2) - L) < 1e-14 * L
        for t in (5, 10, 20):
            a = normals_ref.warp_template(scene.cam8, scene.patches[k], scene.y[k], scene.xp_org[k], scene.poses[t],
                                          (0.0, 0.0))
            w = warp_ref.warp_template(scene.cam8, scene.patches[k], scene.y[k], scene.xp_org[k], scene.poses[t])
            assert a[1] == w[1] and a[0].tobytes() == w[0].tobytes()


@pytest.mark.parametrize("kd0", [True, False])
def test_forward_map_equals_the_plane_induced_map(scene, kd0):
    """kd1 = 0: the homography K (R + t n^T / d) K^-1; kd1 != 0 (the C1 camera, and C3's): ray casting."""
    rng = np.random.default_rng(5)
    cams = [cam_kd0()] if kd0 else [scene.cam8, normals_scene.synth.camera_params(640, 480)]
    worst = 0.0
    for cam8 in cams:
        for k in range(4):
            th = rng.uniform(-0.8, 0.8, 2)
            x = scene.poses[5 * (k + 1) % len(scene.poses)].copy()
            x[:3] += rng.normal(0, 0.02, 3)
            fw = normals_ref.forward(cam8, 11, scene.y[k], scene.xp_org[k], x, th)
            want = (normals_truth.forward_homography if kd0 else normals_truth.forward_rays)(
                cam8, 11, scene.y[k], scene.xp_org[k], x, th)
            assert fw["valid"].all()
            for i in range(0, 121, 7):
                for j in range(2):
                    worst = max(worst, rel_err(fw["g"][j][i], want[i][j]))
    # a few hundred correctly rounded operations on values of a few hundred pixels
    assert worst < 400 * EPS, worst


def test_warp_source_through_the_true_normal_equals_the_plane_to_plane_view(scene):
    """The warp's direction (frame -> template) at the rendered plane's true theta, against casting each output pixel
    onto that plane at 50 digits."""
    n = normals_scene.plane_normal(normals_scene.TILT)
    worst = 0.0
    for k in range(4):
        th = normals_scene.true_theta(scene.y[k], scene.xp_org[k], n)
        for t in (4, 12, 20):
            src, valid = normals_ref.warp_source(scene.cam8, 11, scene.y[k], scene.xp_org[k], scene.poses[t], th)
            want = normals_truth.warp_source(scene.cam8, 11, scene.y[k], scene.xp_org[k], scene.poses[t], th)
            assert valid.all()
            for i in range(121):
                for j in range(2):
                    worst = max(worst, float(abs(mp.mpf(float(src.reshape(-1, 2)[i, j])) - want[i][j])))
    # positions of about 10 px, a few hundred correctly rounded operations
    assert worst < 1e-11, worst


def test_dg_dtheta_equals_mpmath_differentiation(scene):
    rng = np.random.default_rng(7)
    for cam8 in (scene.cam8, cam_kd0()):
        for k in range(3):
            th = rng.uniform(-0.5, 0.5, 2)
            x = scene.poses[12]
            fw = normals_ref.forward(cam8, 11, scene.y[k], scene.xp_org[k], x, th)
            for i in (0, 60, 120):
                d = normals_truth.dg_dtheta(cam8, 11, scene.y[k], scene.xp_org[k], x, th, i)
                for w, t in ((0, fw["ta"]), (1, fw["tb"])):
                    for j in range(2):
                        got = fw["Jw"][j][i] * t[i]
                        assert abs(mp.mpf(float(got)) - d[w][j]) <= 1e-11 * max(1.0, abs(d[w][j])), (k, i, w, j)


# ---- the alignment --------------------------------------------------------------------------------------------------
def run_sequence(scene, k, variant=None, steps=range(2, 21, 2), offset=(0.3, -0.2)):
    """Feature k aligned on the views `steps` at the true poses, its match offset from the projection: per view the
    restatement's result and system."""
    th, cov = [0.0, 0.0], [PRM[1] ** 2, 0.0, PRM[1] ** 2]
    out = []
    for t in steps:
        x = scene.poses[t]
        z = project_point(scene.cam8, camera_points(x, scene.y[k]))[0] + np.array(offset)
        (th, cov, acc, st), info = normals_ref.align(scene.cam8, scene.frames[t], scene.patches[k], scene.y[k],
                                                     scene.xp_org[k], x, z, th, cov, PRM, variant)
        out.append((t, list(th), list(cov), st, info))
    return out


def check_converges(scene, variant=None):
    """Named check: the median angle to the plane's normal falls from its start to below 5 degrees."""
    n = normals_scene.plane_normal(normals_scene.TILT)
    start, end = [], []
    for k in range(6):
        seq = run_sequence(scene, k, variant)
        start.append(normals_scene.normal_angle_deg(scene.y[k], scene.xp_org[k], (0.0, 0.0), n))
        end.append(normals_scene.normal_angle_deg(scene.y[k], scene.xp_org[k], seq[-1][1], n))
    return np.median(end) < 5.0 and np.median(end) < 0.2 * np.median(start)


def check_posterior(scene, variant=None):
    """Named check: Sigma+ is the theta block of the inverted Hessian (the marginal), to 1e-10 relative."""
    for k in range(3):
        for t, th, cov, st, info in run_sequence(scene, k, variant, steps=(4, 8)):
            if info is None:
                continue
            H = list(info["H"])
            if variant == "no_prior":  # the system the definition asks for has the prior in it
                H[0], H[1], H[6] = H[0] + info["Li"][0], H[1] + info["Li"][1], H[6] + info["Li"][2]
            want = normals_truth.marginal(H)
            for a, b in zip(cov, want):
                if abs(mp.mpf(a) - b) > 1e-10 * abs(want[0]):
                    return False
    return True


def check_stationary(scene, variant=None):
    """Named check: at the accepted iterate, the Gauss-Newton step of the system from its definition is below 0.2
    posterior sigma in every unknown.  Not zero: the iteration stops at the first step that does not lower the cost,
    and the cost of a bilinear image is only piecewise smooth (0.12 sigma at most on this scene)."""
    for k in range(3):
        for t, th, cov, st, info in run_sequence(scene, k, variant, steps=(6, 12)):
            if info is None:
                return False
            step = normals_truth.gauss_newton_step(scene.cam8, scene.frames[t], scene.patches[k], scene.y[k],
                                                   scene.xp_org[k], scene.poses[t], info["phi"], info["th0"],
                                                   info["Li"], info["w2"])
            if not np.abs(step).max() < 0.2:
                return False
    return True


def test_restatement_converges_to_the_rendered_planes_tilt(scene):
    assert check_converges(scene)


def test_posterior_is_the_marginal_of_the_inverted_hessian(scene):
    assert check_posterior(scene)


def test_accepted_iterate_is_stationary(scene):
    assert check_stationary(scene)


@pytest.mark.parametrize("variant,check", [("no_prior", check_posterior), ("theta_block", check_posterior),
                                           ("tau_sign", check_stationary), ("template_gradient", check_stationary)])
def test_broken_copies_are_caught(scene, variant, check):
    assert check(scene)
    assert not check(scene, variant)


def test_status_of_an_invalid_start_and_of_no_step(scene):
    k, t = 0, 6
    x = scene.poses[t]
    z = project_point(scene.cam8, camera_points(x, scene.y[k]))[0]
    cov = [0.25, 0.0, 0.25]
    # the match far outside the image: the start is invalid, nothing changes
    r, info = normals_ref.align(scene.cam8, scene.frames[t], scene.patches[k], scene.y[k], scene.xp_org[k], x,
                                z + 1000.0, [0.1, 0.0], cov, PRM)
    assert r == ([0.1, 0.0], cov, 0, 3) and info is None
    # no iteration allowed: no step accepted
    r, info = normals_ref.align(scene.cam8, scene.frames[t], scene.patches[k], scene.y[k], scene.xp_org[k], x, z,
                                [0.1, 0.0], cov, (0, 0.5, 8.0, 0.0))
    assert r == ([0.1, 0.0], cov, 0, 2) and info is None


def test_the_reduction_is_the_lane_sums_then_the_xor_tree():
    v = np.random.default_rng(3).normal(size=225) * 10.0 ** np.random.default_rng(4).integers(-8, 8, 225)
    P = np.zeros(32)
    for k in range(225):
        P[k % 32] = P[k % 32] + v[k]
    for off in (16, 8, 4, 2, 1):
        P = np.array([P[l] + P[l ^ off] for l in range(32)])
    assert normals_ref.warp_sum(v) == P[0]


def test_the_settings_layout_matches_the_header():
    assert C.sizeof(lib.Sl2StreamNormals) == 32
    offs = [getattr(lib.Sl2StreamNormals, f).offset for f, _ in lib.Sl2StreamNormals._fields_]
    assert offs == [0, 4, 8, 16, 24]
    assert lib.SL2_MAX_NORMAL_ITERATIONS == 8
    for name in ("sl2_set_stream_normals", "sl2_get_stream_normals", "sl2_get_patch_normals", "sl2_set_patch_normals",
                 "sl2_align_normals"):
        assert name in lib.EXPORTS
