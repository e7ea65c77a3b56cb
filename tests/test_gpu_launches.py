"""Kernel launches of every entry point, as sl2_launch_count reports them: a call adds exactly the launches of the
kernels it runs, a zero-size call and a call the host refuses add none.  The fused step runs 8 kernels per step group
(predict, search, the update's five, cull) and one more with records on."""
import ctypes as C

import numpy as np
import pytest

from gpu_util import ctx_from_scenes, patch_snapshot_field, random_measurements, sl2, synth

ERR_ARG, ERR_STATE = -1, -3
STEP = 8  # kernels of one step group


def _launches(ctx, fn):
    """(what fn returned, launches it added)."""
    n0 = ctx.launch_count()
    r = fn()
    return r, ctx.launch_count() - n0


def _refused(ctx, fn, code=ERR_ARG):
    rc, n = _launches(ctx, fn)
    assert rc == code
    return n


def _scene_ctx(num_streams=2, n_features=24, frame_slots=2):
    scenes = [synth.make_scene("C2", stream_id=s, n_frames=2, n_features=n_features) for s in range(num_streams)]
    ctx = ctx_from_scenes(scenes, frame_slots=frame_slots, max_features=n_features + 8)  # room to append
    for slot in range(frame_slots):
        ctx.set_frames(slot, np.stack([sc.frames[0] for sc in scenes]))
    return ctx, scenes


def _ray_ctx():
    """One stream at the origin with the identity orientation and a small covariance: depth particles along the ray
    through the image centre project into the image."""
    cfg = sl2.default_config()
    cfg.max_features = 1
    ctx = sl2.Context(cfg)
    B = cfg.boxsize
    ctx.set_features(0, np.zeros((1, 3)), np.array([[0, 0, 0, 1, 0, 0, 0.0]]), np.zeros((1, B, B), np.uint8))
    rng = np.random.default_rng(5)
    ctx.set_frame(0, 0, synth.make_texture(rng, 240, 320))
    x = np.zeros(16)
    x[3], x[15] = 1.0, 2.0
    ctx.set_state(0, x, 1e-6 * np.eye(16))
    return ctx


@pytest.mark.gpu
def test_staged_entry_points():
    """Launches of each synchronous entry point, with sizes above zero."""
    ctx, scenes = _scene_ctx()
    ctx.step(0)
    ctx.sync()
    L, h = ctx.L, ctx.h
    B = ctx.cfg.boxsize
    feat = np.array([0, 3, 5], np.int32)
    centres = np.array([[100.0, 80.0], [160.0, 120.0], [200.0, 150.0]])
    puinv = np.tile([0.02, 0.0, 0.02], (3, 1))
    assert _launches(ctx, lambda: ctx.set_stream_config(1))[1] == 1
    assert _launches(ctx, lambda: ctx.patch_search(0, 0, feat, centres, puinv))[1] == 1
    assert _launches(ctx, lambda: ctx.score_map(0, 0, 3, centres[1], puinv[1]))[1] == 1
    assert _launches(ctx, lambda: ctx.smoe_search(0, 0, 3, puinv, centres))[1] == 2
    assert _launches(ctx, lambda: ctx.smoe_search_patch(0, 0, scenes[0].patches[3], puinv, centres))[1] == 2
    K = 3
    args = (centres, puinv, np.ones(K), np.linspace(1.0, 2.0, K), 0.05, np.full(K, 1.0 / K))
    assert _launches(ctx, lambda: ctx.measure_particles(0, 0, 3, *args))[1] == 3
    assert _launches(ctx, lambda: ctx.measure_particles(0, 0, 0, *args, patch=scenes[0].patches[3]))[1] == 3
    regions = np.array([[10, 10, 100, 80], [150, 100, 300, 220]], np.int32)
    assert _launches(ctx, lambda: ctx.find_best_patch(0, 0, regions))[1] == 2
    assert _launches(ctx, lambda: ctx.ekf_predict(0))[1] == 1
    assert _launches(ctx, lambda: ctx.ekf_predict(0, [0.01, 0.0, 0.0]))[1] == 1
    assert _launches(ctx, lambda: ctx.predict_measurements(0))[1] == 1
    assert _launches(ctx, lambda: ctx.make_measurements(0, 0))[1] == 1
    n = ctx.state_size(0)
    fi, Hxv, Hy, R, nu, _, _ = random_measurements(np.random.default_rng(3), n, (n - 13) // 3, 4)
    assert _launches(ctx, lambda: ctx.ekf_update(0, fi, Hxv, Hy, R, nu))[1] == 5
    assert _launches(ctx, lambda: ctx.ekf_update_measured(0))[1] == 5
    assert _launches(ctx, lambda: ctx.normalise_state(0))[1] == 1
    assert _launches(ctx, lambda: ctx.delete_feature(1, 7))[1] == 1
    sc = scenes[1]
    assert _launches(ctx, lambda: ctx.append_feature(1, sc.x0[13:16], sc.xp_org[0], sc.patches[0]))[1] == 1
    Pcol = np.zeros((ctx.state_size(1) + 3, 3))
    assert _launches(ctx, lambda: ctx.append_feature(1, sc.x0[13:16], sc.xp_org[0], sc.patches[0], Pcol))[1] == 1
    # sl2_measure_particles_patch through the C ABI (no feature index at all)
    z, found, keep, cum, mv = (np.zeros(2 * K, np.int32), np.zeros(K, np.uint8), np.zeros(K, np.uint8), np.zeros(K),
                               np.zeros(2))
    c, p, d, lam, prob = (np.ascontiguousarray(a, np.float64) for a in (centres, puinv, args[2], args[3], args[5]))
    f64 = C.POINTER(C.c_double)
    patch = np.ascontiguousarray(scenes[0].patches[3])
    rc, nl = _launches(ctx, lambda: L.sl2_measure_particles_patch(
        h, 0, 0, patch.ctypes.data, K, c.ctypes.data_as(f64), p.ctypes.data_as(f64), d.ctypes.data_as(f64),
        lam.ctypes.data_as(f64), 0.05, prob.ctypes.data_as(f64), z.ctypes.data_as(C.POINTER(C.c_int32)),
        found.ctypes.data_as(C.POINTER(C.c_uint8)), keep.ctypes.data_as(C.POINTER(C.c_uint8)),
        cum.ctypes.data_as(f64), mv.ctypes.data_as(f64)))
    assert rc >= 0 and nl == 3
    ctx.close()
    ray = _ray_ctx()
    F, Kmax = 2, 6
    ray_dir = synth.unproject(np.array([320, 240, 195, 195, 162, 125, 9e-06, 1.0]), np.array([160.0, 120.0]), 1.0)
    ypi = np.tile(np.concatenate([[0.0, 0.0, 0.0], ray_dir / np.linalg.norm(ray_dir)]), (F, 1))
    out, nl = _launches(ray, lambda: ray.measure_partial_features(
        0, 0, np.zeros((F, B, B), np.uint8), ypi, np.zeros((F, 13, 6)), np.tile(1e-6 * np.eye(6), (F, 1, 1)),
        np.tile(np.linspace(0.5, 5.0, Kmax), (F, 1)), 0.05, np.full((F, Kmax), 1.0 / Kmax)))
    assert nl == 4 and np.isfinite(out["h"]).all()
    ray.close()


@pytest.mark.gpu
def test_zero_size_and_refused_calls_launch_nothing():
    """Calls with nothing to do (n = 0, m = 0, F = 0, K = 0, cnt = 0) and calls the host's argument checks refuse."""
    import torch
    ctx, scenes = _scene_ctx()
    ctx.step(0)
    ctx.sync()
    L, h = ctx.L, ctx.h
    B = ctx.cfg.boxsize
    e2, e3, e0 = np.zeros((0, 2)), np.zeros((0, 3)), np.zeros(0)
    none = np.zeros(0, np.int32)
    sb = ctx.snapshot_bytes()
    dev = torch.zeros(2 * sb, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    zero = [lambda: ctx.patch_search(0, 0, none, e2, e3),
            lambda: ctx.smoe_search(0, 0, 3, e3, e2),
            lambda: ctx.smoe_search_patch(0, 0, scenes[0].patches[3], e3, e2),
            lambda: ctx.measure_particles(0, 0, 3, e2, e3, e0, e0, 0.05, e0),
            lambda: L.sl2_measure_partial_features(h, 0, 0, 0, 4, *[None] * 6, C.c_double(0.05), *[None] * 10),
            lambda: L.sl2_measure_partial_features(h, 0, 0, 2, 0, *[None] * 6, C.c_double(0.05), *[None] * 10),
            lambda: ctx.find_best_patch(0, 0, np.zeros((0, 4), np.int32)),
            lambda: ctx.ekf_update(0, none, np.zeros((0, 13)), np.zeros((0, 3)), np.zeros((0, 2, 2)), e0),
            lambda: ctx.save_streams(0, 0),
            lambda: ctx.load_streams([], 0),
            lambda: ctx.save_streams_dev(0, 0, dev.data_ptr(), sb),
            lambda: ctx.load_streams_dev(0, 0, dev.data_ptr(), sb)]
    for i, fn in enumerate(zero):
        assert _launches(ctx, fn)[1] == 0, i
    feat = np.array([0, 3], np.int32)
    c2, p2 = np.array([[100.0, 80.0], [160.0, 120.0]]), np.tile([0.02, 0.0, 0.02], (2, 1))
    f64, i32 = C.POINTER(C.c_double), C.POINTER(C.c_int32)
    sc = sl2.Sl2StreamConfig.from_buffer_copy(ctx.stream_config(0))
    bad_sc = sl2.Sl2StreamConfig.from_buffer_copy(sc)
    bad_sc.fku = 0.0
    far = np.array([0, 99], np.int32)
    refused = [lambda: L.sl2_set_stream_config(h, 2, C.byref(sc)),
               lambda: L.sl2_set_stream_config(h, 0, C.byref(bad_sc)),
               lambda: L.sl2_delete_feature(h, 0, 24),
               lambda: L.sl2_patch_search(h, 0, 0, 2, far.ctypes.data_as(i32), c2.ctypes.data_as(f64),
                                          p2.ctypes.data_as(f64), None, None, None, None),
               lambda: L.sl2_patch_search(h, 0, 2, 2, feat.ctypes.data_as(i32), c2.ctypes.data_as(f64),
                                          p2.ctypes.data_as(f64), None, None, None, None),
               lambda: L.sl2_score_map(h, 0, 0, 24, c2.ctypes.data_as(f64), p2.ctypes.data_as(f64),
                                       np.zeros(6, np.int32).ctypes.data_as(i32), None, None, None, 16),
               lambda: L.sl2_smoe_search(h, 0, 0, 24, 2, p2.ctypes.data_as(f64), c2.ctypes.data_as(f64), None,
                                         None, None),
               lambda: L.sl2_find_best_patch(h, 0, 0, 1, None, None, None, None),
               lambda: L.sl2_ekf_predict(h, 2, None),
               lambda: L.sl2_predict_measurements(h, -1),
               lambda: L.sl2_make_measurements(h, 0, 2),
               lambda: L.sl2_ekf_update(h, 0, 3, None, None, None, None, None),
               lambda: L.sl2_ekf_update_measured(h, 2),
               lambda: L.sl2_normalise_state(h, 2),
               lambda: L.sl2_step(h, 2),
               lambda: L.sl2_save_streams_dev(h, 0, 3, dev.data_ptr(), sb),
               lambda: L.sl2_load_streams_dev(h, 0, 1, dev.data_ptr(), 64)]
    for i, fn in enumerate(refused):
        assert _refused(ctx, fn) == 0, i
    full = ctx_from_scenes([synth.make_scene("C2", n_frames=1, n_features=24)], max_features=24)
    sc0 = scenes[0]
    assert _refused(full, lambda: L.sl2_append_feature(
        full.h, 0, np.ascontiguousarray(sc0.x0[13:16]).ctypes.data_as(f64),
        np.ascontiguousarray(sc0.xp_org[0]).ctypes.data_as(f64), C.c_void_p(np.ascontiguousarray(sc0.patches[0]).ctypes.data),
        None), ERR_STATE) == 0
    full.close()
    ctx.close()


@pytest.mark.gpu
def test_option_setters_launch_nothing():
    """Every per-stream option setter writes its device copies with ordered copies, no kernel: the first turn-on (which
    sizes the feature's buffer), a turn-off and a repeat each add 0 launches.  sl2_set_stream_config launches one."""
    ctx, _ = _scene_ctx()
    setters = {"consensus": (lambda on: ctx.set_stream_consensus(1, 2.0 * on)),
               "rescue": (lambda on: ctx.set_stream_rescue(1, 5.991 * on)),
               "warp": (lambda on: ctx.set_stream_warp(1, on)),
               "blur": (lambda on: ctx.set_stream_blur(1, on, exposure=0.01)),
               "subpixel": (lambda on: ctx.set_stream_subpixel(1, on)),
               "selection": (lambda on: ctx.set_stream_selection(1, on, min_bits=0.5 * on)),
               "gyro": (lambda on: ctx.set_stream_gyro(1, on)),
               "accel": (lambda on: ctx.set_stream_accel(1, on)),
               "iterated": (lambda on: ctx.set_stream_iterated(1, 2 * on)),
               "recovery": (lambda on: ctx.set_stream_recovery(1, 3 * on, Pxx=1e-6 * np.eye(13))),
               "normals": (lambda on: ctx.set_stream_normals(1, 2 * on))}
    for name, set_on in setters.items():
        for on in (1, 0, 1, 1, 0):
            assert _launches(ctx, lambda: set_on(on))[1] == 0, (name, on)
    assert _launches(ctx, lambda: ctx.set_stream_config(1))[1] == 1
    ctx.close()


@pytest.mark.gpu
def test_snapshots():
    """The device save is one launch and the device load two (check, unpack); a device blob the check kernel refuses
    costs that one launch.  The host forms launch once per staging group of streams."""
    import torch
    ctx, _ = _scene_ctx()
    ctx.step(0)
    ctx.sync()
    sb = ctx.snapshot_bytes()
    dev = torch.zeros(2 * sb, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    assert _launches(ctx, lambda: ctx.save_streams_dev(0, 2, dev.data_ptr(), sb))[1] == 1
    assert _launches(ctx, lambda: ctx.load_streams_dev(0, 2, dev.data_ptr(), sb))[1] == 2
    good = ctx.save_streams()
    nf = sl2.read_snapshot(good[0])["nfeat"]
    bad = np.frombuffer(patch_snapshot_field(good[0], "job_feat", 0, nf), np.uint8)
    ctx.sync()
    dev[:bad.size] = torch.from_numpy(bad.copy()).cuda()
    torch.cuda.synchronize()
    assert _refused(ctx, lambda: ctx.L.sl2_load_streams_dev(ctx.h, 0, 1, dev.data_ptr(), sb)) == 1
    assert _launches(ctx, lambda: ctx.save_streams(0, 2))[1] == 1
    assert _launches(ctx, lambda: ctx.load_streams(good, 0))[1] == 1
    ctx.close()
    # staging groups of at most 64 MB: 256-feature maps make a group of a dozen or so streams
    cfg = sl2.default_config()
    cfg.max_features, cfg.number_of_features_to_select = 256, 10
    g = max(1, (64 << 20) // sl2.lib.snapshot_layout(256, cfg.boxsize)[1])
    cfg.num_streams = 2 * g + 1
    big = sl2.Context(cfg)
    blobs, n = _launches(big, lambda: big.save_streams())
    assert n == 3 and len(blobs) == cfg.num_streams
    assert _launches(big, lambda: big.save_streams(1, g))[1] == 1
    assert _launches(big, lambda: big.save_streams(0, g + 1))[1] == 2
    assert _launches(big, lambda: big.load_streams(blobs))[1] == 3
    assert _launches(big, lambda: big.load_streams(blobs[:g]))[1] == 1
    big.close()


@pytest.mark.gpu
@pytest.mark.parametrize("records", [False, True])
@pytest.mark.parametrize("groups", [1, 2])
def test_fused_step(groups, records):
    """sl2_step and sl2_step_host_async: 8 launches per step group, plus one per group with records on;
    sl2_step_host always runs as one group."""
    ctx, scenes = _scene_ctx(num_streams=3)
    if records:
        ctx.enable_records(4)
    ctx.set_step_groups(groups)
    per_step = groups * (STEP + records)

    def step():
        ctx.step(0)
        ctx.sync()
    assert _launches(ctx, step)[1] == per_step
    frames = np.ascontiguousarray(np.stack([sc.frames[1] for sc in scenes]))
    xv = np.zeros((3, 13))

    def step_async():
        ctx.step_host_async(1, frames.ctypes.data, xv.ctypes.data)
        ctx.wait_slot(1)
        ctx.sync()
    assert _launches(ctx, step_async)[1] == per_step
    assert _launches(ctx, lambda: ctx.step_host(0, frames.ctypes.data, xv.ctypes.data))[1] == STEP + records
    assert np.isfinite(xv).all()
    ctx.close()
