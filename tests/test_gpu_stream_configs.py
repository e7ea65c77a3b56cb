"""Per-stream cameras (sl2_set_stream_config): the camera streams of one context with different calibrations, image
sizes, frame periods and selection counts, each checked against its own oracle and against a context of its own.
The frame ring keeps the context's size; the ring bytes outside a smaller stream image hold noise that changes every
frame, so any read past the stream's image would show up in the results."""
import ctypes as C
import hashlib

import numpy as np
import pytest

from gpu_util import (CAMS_320, assert_same_bytes, assert_state_close, camera, check_streams_against_oracle,
                      ctx_from_scenes, oracle_slam_from_scene, ring_block, sl2, step_frames, stream_result, synth)

STREAM_FIELDS = ("width", "height", "fku", "fkv", "u0", "v0", "kd1", "sd", "delta_t", "number_of_features_to_select")
# the four calibrations of the mixed-camera tests: a full 640x480 camera, two 320x240 ones (the second with a shifted
# principal point, 1.3x the focal length and 3x the radial distortion) and a 400x300 one with twice the pixel noise
CAMS_640 = [camera(640, 480), camera(320, 240), camera(320, 240, focal=1.3, shift=(9.0, -7.0), kd1=3.0),
            camera(400, 300, sd=2.0)]
DTS = (1.0 / 60, 1.0 / 30, 1.0 / 15)
NSEL = (10, 50, 100)


def _stream_cfg(ctx, s):
    sc = ctx.stream_config(s)
    return tuple(getattr(sc, k) for k in STREAM_FIELDS)


def _cfg_tuple(sc):
    return tuple(getattr(sc, k) for k in STREAM_FIELDS)


def _mixed_scenes(n_frames=6):
    """8 streams of 24-feature C2 scenes over the four CAMS_640 calibrations, three frame periods and three selection
    counts, ellipses from S (no fixed search override)."""
    scenes = []
    for s in range(8):
        sc = synth.make_scene("C2", stream_id=s, n_frames=n_frames, n_features=24, override=False,
                              camera=CAMS_640[s % 4], delta_t=DTS[s % 3])
        sc.n_select = NSEL[(s + s // 4) % 3]
        scenes.append(sc)
    return scenes


def _mixed_context(scenes, W, H, frame_slots=1, groups=1, **kw):
    """One context of W x H frames (box and search settings of scenes[0]) holding every scene on its own camera."""
    big = scenes[0]
    cfg = sl2.config_for_scene(big, num_streams=len(scenes), frame_slots=frame_slots,
                               max_features=max(sc.n_features for sc in scenes), **kw)
    cfg.width, cfg.height = W, H
    ctx = sl2.Context(cfg)
    ctx.set_step_groups(groups)
    for s, sc in enumerate(scenes):
        ctx.set_stream_config(s, sl2.stream_config_for_scene(sc))
        sl2.load_scene(ctx, s, sc)
    return ctx


# ---- CPU ------------------------------------------------------------------------------------------------------------
# sha256 (first 32 hex digits) of every output of make_scene(name, stream_id=s, n_frames=3) before the camera and
# delta_t arguments existed: the default scenes, and so every recorded result that uses them, must not move
DEFAULT_SCENE_DIGESTS = {
    ("C1", 0): "8c253a6429d230e25f48bd637cad9d05",
    ("C1", 3): "563b87ec30b82fa3ad965694feab8b93",
    ("C2", 0): "5359053952228c7fe943515354698bf0",
    ("C2", 1): "03c8e7ea56bf90ce8926ce4db42740e1",
    ("C3", 0): "7843889c3ecebf3cec29fc3217051d5d",
    ("C4", 0): "cadda14f037d3dc7bd0f81d210d08da1",
    ("C4", 7): "8e5d27089b5f3266979cdbd6659e1c69",
    ("C4", 131): "bf9e51023765e1f8dfa32f7e38342564",
}


def _scene_digest(sc):
    h = hashlib.sha256()
    for a in (sc.cam8, sc.x0, sc.P0, sc.xp_org, sc.patches, sc.pix, sc.frames, sc.shifts,
              np.array([sc.delta_t, sc.n_select, sc.boxsize], np.float64), np.array(sc.search_override, np.float64)):
        a = np.ascontiguousarray(a)
        h.update(str(a.dtype).encode() + str(a.shape).encode() + a.tobytes())
    return h.hexdigest()[:32]


@pytest.mark.parametrize("name,stream_id", sorted(DEFAULT_SCENE_DIGESTS))
def test_make_scene_defaults_are_unchanged(name, stream_id):
    sc = synth.make_scene(name, stream_id=stream_id, n_frames=3)
    assert _scene_digest(sc) == DEFAULT_SCENE_DIGESTS[(name, stream_id)]
    # naming the default camera and frame period explicitly is the same scene
    same = synth.make_scene(name, stream_id=stream_id, n_frames=3, camera=sc.cam8, delta_t=sc.delta_t)
    assert _scene_digest(same) == DEFAULT_SCENE_DIGESTS[(name, stream_id)]


def test_make_scene_renders_for_the_given_camera():
    cam = CAMS_640[3]
    sc = synth.make_scene("C2", stream_id=2, n_frames=2, n_features=24, camera=cam, delta_t=1.0 / 15)
    assert (sc.width, sc.height) == (400, 300) and sc.frames.shape == (2, 300, 400)
    assert (sc.cam8 == cam).all() and sc.delta_t == 1.0 / 15
    # the features' 3-D points project onto their template centres through this camera
    h = synth.project(cam, sc.x0[13:].reshape(-1, 3) - sc.x0[:3])
    assert np.abs(h - sc.pix).max() < 1e-9
    ssc = sl2.stream_config_for_scene(sc)
    assert _cfg_tuple(ssc) == (400, 300, *[float(v) for v in cam[2:8]], 1.0 / 15, sc.n_select)


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _run_mixed(scenes, W, H, steps, groups=1, oracles=None, picks=(), seed=0, snap=True):
    """Fused steps of the scenes in one W x H context; the ring outside each stream's image is fresh noise every
    frame.  Returns the context and (with `snap`) the snapshots of every stream after every step."""
    ctx = _mixed_context(scenes, W, H, frame_slots=2, groups=groups)
    rng = np.random.default_rng(seed)
    snaps = []
    for t in range(steps):
        step_frames(ctx, np.stack([ring_block(sc.frames[t], H, W, rng) for sc in scenes]), t % 2)
        if oracles is not None:
            check_streams_against_oracle(ctx, oracles, picks, lambda s: scenes[s], t)
        if snap:
            snaps.append([stream_result(ctx, s) for s in range(len(scenes))])
    return ctx, snaps


def _run_alone(sc, steps):
    ctx = ctx_from_scenes([sc], frame_slots=2)
    snaps = []
    for t in range(steps):
        step_frames(ctx, sc.frames[t][None], t % 2)
        snaps.append(stream_result(ctx, 0))
    ctx.close()
    return snaps


@pytest.mark.gpu
def test_mixed_cameras_fused_step_against_oracle_and_dedicated_contexts(oracle):
    """8 streams, four calibrations (640x480, 320x240, a re-calibrated 320x240, 400x300 with sd = 2), frame periods
    1/60, 1/30, 1/15 and selection counts 10, 50, 100 in one 640x480 context, 6 fused steps: every stream matches its
    own oracle (built from its own camera and image) at the tolerances of check_streams_against_oracle, and is
    bit-identical -- x, P, h, S, z, flags, ranks, counters -- to the same scene run alone in a context created with
    that camera and image size."""
    scenes = _mixed_scenes()
    assert {sc.width for sc in scenes} == {640, 320, 400} and {sc.n_select for sc in scenes} == set(NSEL)
    oracles = {s: oracle_slam_from_scene(oracle, sc) for s, sc in enumerate(scenes)}
    ctx, snaps = _run_mixed(scenes, 640, 480, 6, oracles=oracles, picks=range(8))
    for s in range(8):  # the run tracked: features were found on every camera
        assert (ctx.features(s)["flags"] & 2).any(), s
    ctx.close()
    for s, sc in enumerate(scenes):
        alone = _run_alone(sc, 6)
        for t in range(6):
            assert_same_bytes(snaps[t][s], alone[t], (s, t))


@pytest.mark.gpu
def test_noop_setter_and_getter():
    """After sl2_create every stream reports the sl2_config values; the getter returns what the setter set; setting a
    stream's current values again changes no bit of a run."""
    scenes = _mixed_scenes(n_frames=4)
    cfg = sl2.config_for_scene(scenes[0], num_streams=3, max_features=24)
    cfg.width, cfg.height = 640, 480
    ctx = sl2.Context(cfg)
    want = (640, 480, cfg.fku, cfg.fkv, cfg.u0, cfg.v0, cfg.kd1, cfg.sd, cfg.delta_t,
            cfg.number_of_features_to_select)
    assert all(_stream_cfg(ctx, s) == want for s in range(3))
    for s in range(3):
        ctx.set_stream_config(s, sl2.stream_config_for_scene(scenes[s]))
        assert _stream_cfg(ctx, s) == _cfg_tuple(sl2.stream_config_for_scene(scenes[s]))
    ctx.close()
    a, sa = _run_mixed(scenes, 640, 480, 4, seed=3)
    b = _mixed_context(scenes, 640, 480, frame_slots=2)
    rng = np.random.default_rng(3)
    for t in range(4):
        for s in range(8):  # before every step, and between the upload and the step
            b.set_stream_config(s, b.stream_config(s))
        b.set_frames(t % 2, np.stack([ring_block(sc.frames[t], 480, 640, rng) for sc in scenes]))
        b.set_stream_config(t % 8, sl2.stream_config_for_scene(scenes[t % 8]))
        b.step(t % 2)
        for s in range(8):
            assert_same_bytes(sa[t][s], stream_result(b, s), (s, t))
    a.close()
    b.close()


def _switch_scene():
    """A 24-feature C2 scene on the default 320x240 camera, and a second camera B: a smaller 288x224 image, another
    calibration, frame period and selection count."""
    sc = synth.make_scene("C2", stream_id=5, n_frames=7, n_features=24, override=False)
    cam_b = camera(288, 224, focal=1.1, shift=(-6.0, 4.0), kd1=2.0, sd=1.5)
    b = sl2.Sl2StreamConfig()
    b.width, b.height = 288, 224
    b.fku, b.fkv, b.u0, b.v0, b.kd1, b.sd = [float(v) for v in cam_b[2:8]]
    b.delta_t = 1.0 / 15
    b.number_of_features_to_select = 7
    return sc, b


def _ctx_for_camera(sc, b, x, P):
    """A context created with camera b, holding sc's map at the state (x, P)."""
    cfg = sl2.config_for_scene(sc, frame_slots=2)
    cfg.width, cfg.height = b.width, b.height
    cfg.fku, cfg.fkv, cfg.u0, cfg.v0, cfg.kd1, cfg.sd = b.fku, b.fkv, b.u0, b.v0, b.kd1, b.sd
    cfg.delta_t = b.delta_t
    cfg.number_of_features_to_select = b.number_of_features_to_select
    ctx = sl2.Context(cfg)
    ctx.set_features(0, sc.x0[13:].reshape(-1, 3), sc.xp_org, sc.patches)
    ctx.set_state(0, x, P)
    return ctx


def _assert_switch_matches(a, b, where):
    """x, P, h, S, the selection and the matches of the selected features: bit-identical (counters and the flags of
    unselected features carry the history before the switch)."""
    assert_same_bytes(a, b, where, keys=("x", "P", "h", "S", "select_rank"))
    sel = b["select_rank"] >= 0
    assert sel.any(), where
    assert a["z"][sel].tobytes() == b["z"][sel].tobytes() and (a["flags"][sel] == b["flags"][sel]).all(), where


@pytest.mark.gpu
def test_camera_change_mid_run():
    """3 steps with camera A, then camera B (smaller image, new calibration, frame period and selection count) for 4
    steps == a context created with B that starts from the state after step 3.  Repeated with the switch between two
    sl2_step_host_async calls on different slots, with no synchronisation around it.  7 steps stay below the cull
    threshold (10 attempts)."""
    import torch
    sc, cam_b = _switch_scene()
    rng = np.random.default_rng(11)
    frames = np.stack([ring_block(sc.frames[t], 240, 320, rng) for t in range(7)])
    a = ctx_from_scenes([sc], frame_slots=2)
    for t in range(3):
        a.set_frames(t % 2, frames[t][None])
        a.step(t % 2)
    x3, P3 = a.get_state(0)
    a.set_stream_config(0, cam_b)
    assert _cfg_tuple(a.stream_config(0)) == _cfg_tuple(cam_b)
    ref = _ctx_for_camera(sc, cam_b, x3, P3)
    for t in range(3, 7):
        a.set_frames(t % 2, frames[t][None])
        a.step(t % 2)
        ref.set_frames(t % 2, np.ascontiguousarray(sc.frames[t][:224, :288])[None])
        ref.step(t % 2)
        _assert_switch_matches(stream_result(a, 0), stream_result(ref, 0), t)
    assert ref.features(0)["attempted"].max() < 10
    final = stream_result(ref, 0)
    a.close()
    ref.close()
    # the same switch between two asynchronous steps
    host = torch.empty((7, 1, 240, 320), dtype=torch.uint8, pin_memory=True)
    host.numpy()[:] = frames[:, None]
    xv = torch.zeros((7, 1, 13), dtype=torch.float64, pin_memory=True)
    c = ctx_from_scenes([sc], frame_slots=2)
    for t in range(7):
        if t == 3:
            c.set_stream_config(0, cam_b)
        c.step_host_async(t % 2, host[t].data_ptr(), xv[t].data_ptr())
    c.sync()
    _assert_switch_matches(stream_result(c, 0), final, "async")
    assert xv[6].numpy().tobytes() == final["x"][:13].tobytes()
    c.close()


@pytest.mark.gpu
def test_staged_path_and_score_map_on_a_smaller_stream(oracle):
    """sl2_ekf_predict -> sl2_predict_measurements -> sl2_make_measurements -> sl2_ekf_update_measured on a
    re-calibrated 320x240 stream of a 640x480 context agrees with the oracle; sl2_score_map near the smaller image's
    right and bottom edges equals the oracle's search_box / score_map on that image."""
    scenes = _mixed_scenes(n_frames=3)
    s = 2
    sc = scenes[s]
    assert (sc.width, sc.height) == (320, 240) and sc.cam8[2] != synth.camera_params(320, 240)[2]
    ctx = _mixed_context(scenes, 640, 480)
    o = oracle_slam_from_scene(oracle, sc)
    rng = np.random.default_rng(5)
    for t in range(3):
        ctx.set_frames(0, np.stack([ring_block(scn.frames[t], 480, 640, rng) for scn in scenes]))
        ctx.set_frame(s, 0, sc.frames[t])  # copies the stream's 320 x 240 image only
        ctx.ekf_predict(s)
        ctx.predict_measurements(s)
        cnt = ctx.make_measurements(s, 0)
        ctx.ekf_update_measured(s)
        o.predict()
        o.select()
        assert cnt == o.measure(sc.frames[t])
        o.update()
        o.normalise()
        o.finish()
        fg, fo = ctx.features(s), o.features()
        assert (fg["z"] == fo["z"]).all() and (fg["flags"] == fo["flags"]).all()
        assert (fg["select_rank"] == fo["select_rank"]).all()
        assert (fg["attempted"] == fo["attempted"]).all() and (fg["successful"] == fo["successful"]).all()
        assert_state_close(*ctx.get_state(s), *o.get_state())
    img = sc.frames[2]
    for feat, c, p in [(0, [315.2, 120.0], [0.02, 0.0, 0.02]), (1, [160.0, 236.7], [0.01, 0.003, 0.02]),
                       (2, [318.9, 238.4], [0.03, -0.01, 0.02]), (3, [300.0, 229.0], [0.004, 0.0, 0.004])]:
        box, corr, sd, inside = ctx.score_map(s, 0, feat, c, p)
        obox, ocorr, osd, oinside = oracle.score_map(img, sc.patches[feat], c, p)
        assert (box == obox).all() and (box == oracle.search_box(320, 240, 11, c, p)).all()
        assert corr.size and (inside == oinside).all()
        assert corr.tobytes() == ocorr.tobytes() and sd.tobytes() == osd.tobytes()
    ctx.close()


@pytest.mark.gpu
def test_partial_features_and_detector_on_a_smaller_stream(oracle):
    """sl2_measure_partial_features on a re-calibrated 320x240 stream of a 640x480 context: h, S^-1 and det S
    bit-identical to predict_particles with that camera; matches, survivors and probabilities against smoe_search /
    particle_update on the stream's own image, with ellipses clipped by its right and bottom edges.
    sl2_find_best_patch with regions that run past the smaller image equals find_best_patch on that image."""
    rng = np.random.default_rng(78)
    img = synth.make_texture(rng, 240, 320)
    B = 11
    cam8 = CAMS_640[2]
    cfg = sl2.default_config()
    cfg.width, cfg.height, cfg.num_streams, cfg.max_features = 640, 480, 3, 1
    ctx = sl2.Context(cfg)
    for s in range(3):
        ctx.set_features(s, np.zeros((1, 3)), np.array([[0, 0, 0, 1, 0, 0, 0.0]]), np.zeros((1, B, B), np.uint8))
    s = 1
    sc = sl2.Sl2StreamConfig()
    sc.width, sc.height = 320, 240
    sc.fku, sc.fkv, sc.u0, sc.v0, sc.kd1, sc.sd = [float(v) for v in cam8[2:8]]
    sc.delta_t, sc.number_of_features_to_select = 1.0 / 30, 10
    ctx.set_stream_config(s, sc)
    ring = np.stack([ring_block(img, 480, 640, rng) for _ in range(3)])
    ctx.set_frames(0, ring)
    xv = np.zeros(13)
    xv[:3] = [0.02, -0.01, 0.01]
    q = np.array([1.0, 0.01, -0.02, 0.015])
    xv[3:7] = q / np.linalg.norm(q)
    A = rng.normal(0, 1, (16, 16))
    P = A @ A.T * 2e-6 + 1e-8 * np.eye(16)
    ctx.set_state(s, np.concatenate([xv, [0.1, 0.1, 2.0]]), P)
    # rays towards an interior pixel and towards the right and bottom edges of the smaller image (boxes clipped there;
    # this camera's strong distortion reaches only pixels within 1 / sqrt(2 kd1) = 136 px of its principal point, so
    # the two rays near the right edge get wide ellipses)
    pix = [(150.0, 110.0), (300.0, 115.0), (171.0, 236.0), (240.0, 225.0)]
    grow = [1.0, 100.0, 1.0, 100.0]  # scale of the ray's own covariance Pyy
    F, Kmax = len(pix), 48
    K = np.array([Kmax, Kmax - 5, 30, 17], np.int32)
    ypi, Pxy, Pyy = np.zeros((F, 6)), np.zeros((F, 13, 6)), np.zeros((F, 6, 6))
    lam, prob = np.zeros((F, Kmax)), np.zeros((F, Kmax))
    patches = np.zeros((F, B, B), np.uint8)
    for f, (u, v) in enumerate(pix):
        hh = synth.unproject(cam8, np.array([u, v]), 1.0)
        ypi[f] = np.concatenate([[0.0, 0.0, 0.0], hh / np.linalg.norm(hh)])
        Af = rng.normal(0, 1, (19, 19))
        Pf = Af @ Af.T * 2e-6 + 1e-8 * np.eye(19)
        Pf[:13, :13] = P[:13, :13]
        Pxy[f], Pyy[f] = Pf[:13, 13:], Pf[13:, 13:] * grow[f]
        lam[f] = np.linspace(0.4, 6.0, Kmax)
        p0 = rng.uniform(0.2, 1.0, Kmax)
        p0[K[f]:] = 0.0
        prob[f] = p0 / p0.sum()
        h_mid = oracle.predict_particles(cam8, xv, ypi[f], lam[f, K[f] // 2:K[f] // 2 + 1], P[:13, :13], Pxy[f],
                                         Pyy[f])[0][0]
        cu = int(np.clip(round(h_mid[0]), 5, 314))
        cv = int(np.clip(round(h_mid[1]), 5, 234))
        patches[f] = img[cv - 5:cv + 6, cu - 5:cu + 6]
    out = ctx.measure_partial_features(s, 0, patches, ypi, Pxy, Pyy, lam, 0.05, prob, K=K)
    any_found = clipped = False
    for f in range(F):
        k = K[f]
        oh, oS, osi, odet = oracle.predict_particles(cam8, xv, ypi[f], lam[f, :k], P[:13, :13], Pxy[f], Pyy[f])
        assert out["h"][f, :k].tobytes() == oh.tobytes(), f
        assert out["Sinv3"][f, :k].tobytes() == osi.tobytes(), f
        assert out["detS"][f, :k].tobytes() == odet.tobytes(), f
        for j in range(k):
            bx = oracle.search_box(320, 240, B, oh[j], osi[j])
            full = oracle.search_box(640, 480, B, oh[j], osi[j])
            clipped |= bool((bx != full).any())
        ou, ov, of, _ = oracle.smoe_search(img, patches[f], osi, oh)
        assert (out["found"][f, :k] == of).all(), f
        z = out["z"][f, :k]
        assert (z[of > 0, 0] == ou[of > 0]).all() and (z[of > 0, 1] == ov[of > 0]).all(), f
        any_found |= bool(of.any())
        oleft, oprob, okeep, ocum, omv = oracle.particle_update(oh, osi, odet, lam[f, :k], np.column_stack([ou, ov]),
                                                                of, 0.05, prob[f, :k])
        assert out["left"][f] == oleft and (out["keep"][f, :k] == okeep).all(), f
        np.testing.assert_allclose(out["prob"][f, :k], oprob, rtol=1e-13, atol=1e-300)
        np.testing.assert_allclose(out["cumulative"][f, :k], ocum, rtol=1e-13, atol=1e-300)
        np.testing.assert_allclose(out["mean_var"][f], omv, rtol=1e-12, atol=1e-15)
    assert any_found and clipped
    regions = np.array([[250, 180, 400, 300], [-5, 200, 500, 479], [300, -3, 639, 100], [0, 0, 640, 480],
                        [310, 230, 330, 250], [100, 50, 200, 150], [330, 10, 400, 100]], np.int32)
    u, v, ev = ctx.find_best_patch(s, 0, regions, ubest=-7, vbest=-9)
    for i, reg in enumerate(regions):
        ou, ov, oev = oracle.find_best_patch(img, B, reg, ubest=-7, vbest=-9)
        assert (u[i], v[i]) == (ou, ov), (i, reg)
        assert np.float64(ev[i]).tobytes() == np.float64(oev).tobytes(), (i, reg)
    assert ev[0] > 0 and ev[6] == 0.0
    ctx.close()


@pytest.mark.gpu
def test_bench_shape_264_streams_mixed_cameras(oracle):
    """The benchmark's shape (264 C4 streams in one 320x240 context) cycling through four calibrations (one with a
    288x224 image) and selection counts 100, 50, 10, 3 frames: streams 0, 131, 132 and 263 match the oracle, every
    two streams with the same scene and config are bit-identical in x and P, and the run with two step groups is
    bit-identical to the serial one."""
    nS, T = 264, 3
    scene_cache = {}

    def key(s):  # (scene, calibration, selection count): streams 0, 131, 132, 263 use all four calibrations
        return ((s * 5) % 8, (s // 2) % 4, s % 3)

    def scene_of(s):
        u, k, j = key(s)
        if (u, k, j) not in scene_cache:
            sc = synth.make_scene("C4", stream_id=u, n_frames=T, camera=CAMS_320[k])
            sc.n_select = (100, 50, 10)[j]
            scene_cache[(u, k, j)] = sc
        return scene_cache[(u, k, j)]

    scenes = [scene_of(s) for s in range(nS)]
    picks = (0, 131, 132, 263)
    assert len({key(s)[1] for s in picks}) == 4
    oracles = {s: oracle_slam_from_scene(oracle, scenes[s]) for s in picks}
    ctx, _ = _run_mixed(scenes, 320, 240, T, oracles=oracles, picks=picks, seed=264, snap=False)
    two, _ = _run_mixed(scenes, 320, 240, T, groups=2, seed=264, snap=False)
    first = {}
    for s in range(nS):
        x, P = ctx.get_state(s)
        x2, P2 = two.get_state(s)
        assert x.tobytes() == x2.tobytes() and P.tobytes() == P2.tobytes(), s
        if key(s) in first:
            assert x.tobytes() == first[key(s)][0].tobytes() and P.tobytes() == first[key(s)][1].tobytes(), s
        else:
            first[key(s)] = (x, P)
    assert len(first) == 24
    ctx.close()
    two.close()


@pytest.mark.gpu
def test_capacity_256_per_stream_selection(oracle):
    """A context of capacity 256 with 200-feature maps selecting 128 and 10 features per step: 4 steps against the
    oracle.  The setter rejects number_of_features_to_select = 129 there and accepts it at capacity 128."""
    scenes = []
    for s, ns in enumerate((128, 10)):
        sc = synth.make_scene("C4", stream_id=s, n_frames=4, n_features=200)
        sc.n_select = ns
        scenes.append(sc)
    cfg = sl2.config_for_scene(scenes[0], num_streams=2, frame_slots=2, max_features=256)
    ctx = sl2.Context(cfg)
    for s, sc in enumerate(scenes):
        ctx.set_stream_config(s, sl2.stream_config_for_scene(sc))
        sl2.load_scene(ctx, s, sc)
    oracles = {s: oracle_slam_from_scene(oracle, sc) for s, sc in enumerate(scenes)}
    for t in range(4):
        step_frames(ctx, np.stack([sc.frames[t] for sc in scenes]), t % 2)
        check_streams_against_oracle(ctx, oracles, (0, 1), lambda s: scenes[s], t)
    assert (ctx.features(0)["select_rank"] >= 0).sum() == 128 and (ctx.features(1)["select_rank"] >= 0).sum() == 10
    before = _stream_cfg(ctx, 0)
    with pytest.raises(sl2.Sl2Error):
        ctx.set_stream_config(0, number_of_features_to_select=129)
    assert _stream_cfg(ctx, 0) == before
    ctx.close()
    cfg.max_features = 128
    small = sl2.Context(cfg)
    small.set_stream_config(1, number_of_features_to_select=129)
    assert small.stream_config(1).number_of_features_to_select == 129
    small.close()


@pytest.mark.gpu
def test_setter_argument_checks():
    """Every rejected argument returns SL2_ERR_ARG and leaves the stream's config as it was."""
    cfg = sl2.default_config()
    cfg.width, cfg.height, cfg.num_streams, cfg.boxsize = 320, 240, 2, 15
    ctx = sl2.Context(cfg)
    L, h = ctx.L, ctx.h
    good = ctx.stream_config(1)
    good.width, good.height, good.fku, good.delta_t = 200, 150, 230.0, 0.05
    assert L.sl2_set_stream_config(h, 1, C.byref(good)) == 0
    want = _stream_cfg(ctx, 1)
    assert want == _cfg_tuple(good)
    assert L.sl2_set_stream_config(h, -1, C.byref(good)) == -1
    assert L.sl2_set_stream_config(h, 2, C.byref(good)) == -1
    assert L.sl2_set_stream_config(h, 1, None) == -1
    assert L.sl2_get_stream_config(h, 2, C.byref(sl2.Sl2StreamConfig())) == -1
    assert L.sl2_get_stream_config(h, 1, None) == -1
    bad = []
    for f in ("fku", "fkv", "u0", "v0", "kd1", "sd", "delta_t"):
        bad += [(f, float("nan")), (f, float("inf")), (f, -float("inf"))]
    bad += [("fku", 0.0), ("fku", -1.0), ("fkv", 0.0), ("fkv", -195.0), ("delta_t", 0.0), ("delta_t", -0.03)]
    bad += [("width", 15), ("width", 14), ("height", 15), ("width", 321), ("height", 241), ("width", 0),
            ("height", -240), ("number_of_features_to_select", -1)]
    for f, v in bad:
        sc = sl2.Sl2StreamConfig.from_buffer_copy(good)
        setattr(sc, f, v)
        assert L.sl2_set_stream_config(h, 1, C.byref(sc)) == -1, (f, v)
        assert _stream_cfg(ctx, 1) == want, (f, v)
    # the bounds themselves are accepted: 16 at box 15 (max(16, boxsize)), the context's size, no selection
    for f, v in (("width", 16), ("height", 16), ("width", 320), ("height", 240), ("number_of_features_to_select", 0)):
        sc = sl2.Sl2StreamConfig.from_buffer_copy(good)
        setattr(sc, f, v)
        assert L.sl2_set_stream_config(h, 1, C.byref(sc)) == 0, (f, v)
        assert getattr(ctx.stream_config(1), f) == v
    assert _stream_cfg(ctx, 0) == (320, 240, cfg.fku, cfg.fkv, cfg.u0, cfg.v0, cfg.kd1, cfg.sd, cfg.delta_t,
                                   cfg.number_of_features_to_select)
    ctx.close()
