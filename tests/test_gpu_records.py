"""Step records (sl2_enable_records / sl2_get_records[_dev]): one record per camera stream per fused step, with the
trajectory point, the map counts, NIS = nu^T S^-1 nu and log det S of the step's update, and the camera block of x and
P.  Records are off by default and never change what the step computes; their values are checked against an
independent NumPy computation of S from the staged path, against the oracle's counts and against the getters."""
import os

import numpy as np
import pytest

from gpu_util import (CAMS_320, assert_same_bytes, ctx_from_scenes, large_variant, oracle_slam_from_scene,
                      random_measurements, ring_block, sl2, step_frames, stream_result, synth, update_variant)

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ERR_ARG, ERR_STATE = -1, -3
# NIS relative and log det S absolute, record vs NumPy on the staged path's S (m up to 256)
NIS_RTOL, LOGDET_ATOL = 1e-9, 1e-9
WORST = {"nis": 0.0, "logdet": 0.0}


# ---- helpers --------------------------------------------------------------------------------------------------------
def _twin(sc, max_features):
    """A one-stream context that runs the staged path on a copy of a stream."""
    return sl2.Context(sl2.config_for_scene(sc, num_streams=1, max_features=max_features))


def _expected(ctx, s, twin, frame):
    """The stream's state before its next fused step, copied into `twin` and run through the staged path
    (sl2_ekf_predict, sl2_predict_measurements, sl2_make_measurements): the predicted P and the H, R, nu of every
    measured feature give S = H P H^T + R, NIS and log det S in NumPy."""
    twin.load_stream(0, ctx.save_stream(s))
    twin.set_frame(0, 0, frame)
    twin.ekf_predict(0)
    nv = twin.predict_measurements(0)
    cnt = twin.make_measurements(0, 0)
    _, P = twin.get_state(0)
    f = twin.features(0)
    J, Jy, R, nu = twin.feature_jacobians(0)
    meas = [i for i in np.argsort(f["select_rank"]) if f["select_rank"][i] >= 0 and f["flags"][i] & 2]
    assert len(meas) == cnt
    n, m = P.shape[0], 2 * cnt
    H, Rm, v = np.zeros((m, n)), np.zeros((m, m)), np.zeros(m)
    for k, i in enumerate(meas):
        H[2 * k:2 * k + 2, :13] = J[i].reshape(13, 2).T
        H[2 * k:2 * k + 2, 13 + 3 * i:16 + 3 * i] = Jy[i].reshape(3, 2).T
        Rm[2 * k:2 * k + 2, 2 * k:2 * k + 2] = R[i].reshape(2, 2).T
        v[2 * k:2 * k + 2] = nu[i]
    if m == 0:
        return dict(m=0, nvisible=nv, nmeas=0, nis=0.0, logdet=0.0)
    S = H @ P @ H.T + Rm
    sign, logdet = np.linalg.slogdet(S)
    assert sign > 0
    return dict(m=m, nvisible=nv, nmeas=cnt, nis=float(v @ np.linalg.solve(S, v)), logdet=float(logdet))


def _check_values(rec, want, where):
    assert (rec["m"], rec["nvisible"], rec["nmeas"]) == (want["m"], want["nvisible"], want["nmeas"]), where
    if want["m"] == 0:
        assert rec["nis"] == 0.0 and rec["logdet_s"] == 0.0, where
        return
    e_nis = abs(rec["nis"] - want["nis"]) / want["nis"]
    e_ld = abs(rec["logdet_s"] - want["logdet"])
    WORST["nis"], WORST["logdet"] = max(WORST["nis"], e_nis), max(WORST["logdet"], e_ld)
    assert e_nis <= NIS_RTOL and e_ld <= LOGDET_ATOL, (where, e_nis, e_ld)


def _check_getters(ctx, s, rec, where):
    x, P = ctx.get_state(s)
    assert rec["xv"].tobytes() == x[:13].tobytes(), where
    assert rec["pxx_diag"].tobytes() == np.ascontiguousarray(np.diag(P)[:13]).tobytes(), where
    assert rec["nfeat"] == ctx.num_features(s), where


def _oracle_step(o, frame):
    """One GoOneStep of the oracle in its stages: (nvisible, nmeas, nsel, nculled, nfeat) as the record counts them."""
    o.predict()
    nv = o.select()
    nm = o.measure(frame)
    o.update()
    o.normalise()
    nf = o.num_features
    o.finish()
    return dict(nvisible=nv, nmeas=nm, nsel=int((o.features()["select_rank"] >= 0).sum()),
                nculled=nf - o.num_features, nfeat=o.num_features)


def _run_checked(oracle, scenes, steps, cap=None, slots=2, depth=64):
    """Fused steps of the scenes with records on; every stream's record of every step checked against the staged twin,
    the oracle's counts and the getters.  Returns the records of stream 0 (the last step's ring)."""
    cap = cap or max(sc.n_features for sc in scenes)
    ctx = ctx_from_scenes(scenes, frame_slots=slots, max_features=cap)
    ctx.enable_records(depth)
    twin = _twin(scenes[0], cap)
    oracles = [oracle_slam_from_scene(oracle, sc) for sc in scenes]
    try:
        for t in range(steps):
            k = t % scenes[0].frames.shape[0]
            want = [_expected(ctx, s, twin, sc.frames[k]) for s, sc in enumerate(scenes)]
            step_frames(ctx, np.stack([sc.frames[k] for sc in scenes]), t % slots)
            recs = ctx.records(max=1)
            for s, sc in enumerate(scenes):
                rec = recs[s, 0]
                assert rec["step"] == t
                _check_values(rec, want[s], (t, s))
                _check_getters(ctx, s, rec, (t, s))
                counts = _oracle_step(oracles[s], sc.frames[k])
                assert {c: int(rec[c]) for c in counts} == counts, (t, s)
        return ctx.records()
    finally:
        ctx.close()
        twin.close()


# ---- GPU: off by default, and the step unchanged ---------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 264])
def test_records_off_by_default_and_the_step_unchanged(B):
    """Without sl2_enable_records a step launches what it always did and a get is refused with SL2_ERR_STATE; with
    records on, each step launches exactly one kernel more (one CTA per stream after the cull) and x, P and every
    feature getter after 10 C4 steps are byte-identical to the context without records.  B = 1 runs the PDL chain."""
    cache = {}
    scenes = [cache.setdefault(s % 8, synth.make_scene("C4", stream_id=s % 8, n_frames=10)) for s in range(B)]
    off = ctx_from_scenes(scenes, frame_slots=2)
    on = ctx_from_scenes(scenes, frame_slots=2)
    on.enable_records(16)
    rec = np.zeros(1, sl2.STEP_RECORD_DTYPE)
    assert off.L.sl2_get_records(off.h, 0, 1, 1, rec.ctypes.data) == ERR_STATE
    for t in range(10):
        frames = np.stack([sc.frames[t] for sc in scenes])
        l0, l1 = off.launch_count(), on.launch_count()
        step_frames(off, frames, t % 2)
        step_frames(on, frames, t % 2)
        assert on.launch_count() - l1 == off.launch_count() - l0 + 1, t
    for s in range(B):
        assert_same_bytes(stream_result(on, s, jacobians=True), stream_result(off, s, jacobians=True), s)
    got = on.records()
    assert got.shape == (B, 10) and (got["step"] == np.arange(10)).all()
    assert off.L.sl2_get_records(off.h, 0, 1, 1, rec.ctypes.data) == ERR_STATE
    off.close()
    on.close()


# ---- GPU: values ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_values_c1_and_c4_against_numpy_and_oracle(oracle):
    """20 steps of a C1 scene (the reference's configuration) and of two C4 streams: NIS and log det S of every record
    against S = H P H^T + R formed in NumPy from the staged path of a copy of the stream, the counts against the
    oracle, xv and the Pxx diagonal bit-identical to sl2_get_state."""
    kp = np.load(os.path.join(G, "known_patches.npy"))
    _run_checked(oracle, [synth.make_scene("C1", n_frames=20, known_patches=kp)], 20)
    _run_checked(oracle, [synth.make_scene("C4", stream_id=s, n_frames=20) for s in range(2)], 20)
    print("\nworst NIS relative error %.2e, worst log det S error %.2e" % (WORST["nis"], WORST["logdet"]))


@pytest.mark.gpu
def test_cull_step_records(oracle):
    """A map with 20 features that never match (culled at the 10th step) beside a healthy one: nculled and nfeat are
    right at the cull step, and NIS / log det S stay right there too (the cull reuses the update's scratch)."""
    scenes = [update_variant(100, 100, bad=20, stream_id=0, n_frames=12), update_variant(100, 100, stream_id=1,
                                                                                         n_frames=12)]
    recs = _run_checked(oracle, scenes, 12)
    culled = recs[0]["nculled"]
    assert culled.sum() == 20 and culled[9] == 20 and recs[0]["nfeat"][9] == 80 and recs[0]["nfeat"][8] == 100
    assert (recs[1]["nculled"] == 0).all() and (recs[1]["nfeat"] == 100).all()


@pytest.mark.gpu
def test_capacity_256_with_m_256(oracle):
    """A 256-feature map measuring 128 features (m = 256, n = 781) and a 256-feature map with nothing in view
    (m = 0: nis = logdet_s = 0, nothing of the update scratch is read)."""
    scenes = [large_variant(256, 128, stream_id=3, n_frames=3), large_variant(256, 0, stream_id=4, n_frames=3)]
    recs = _run_checked(oracle, scenes, 3, cap=256)
    assert (recs[0]["m"] == 256).all() and (recs[1]["m"] == 0).all()
    assert (recs[1]["nis"] == 0).all() and (recs[1]["logdet_s"] == 0).all()


@pytest.mark.gpu
def test_staged_update_between_fused_steps_does_not_leak():
    """A staged sl2_ekf_update (host rows, another m) between two fused steps writes no record, and the next record
    describes the fused step's own update; on a stream whose features are all out of view the staged update fills
    the update scratch and the next fused step still records m = 0, nis = logdet_s = 0."""
    scenes = [synth.make_scene("C4", n_frames=3), update_variant(100, 100, out_of_view=True, stream_id=1, n_frames=3)]
    ctx = ctx_from_scenes(scenes, frame_slots=2)
    ctx.enable_records(8)
    twin = _twin(scenes[0], 100)
    step_frames(ctx, np.stack([sc.frames[0] for sc in scenes]))
    before = ctx.records()
    rng = np.random.default_rng(7)
    for s in (0, 1):
        feats, Hxv, Hy, R, nu, _, _ = random_measurements(rng, 313, 100, 5)
        ctx.ekf_update(s, feats, Hxv, Hy, R, nu)
    for s in (0, 1):  # the other staged entry points write no record either
        ctx.ekf_predict(s)
        ctx.predict_measurements(s)
        ctx.make_measurements(s, 0)
    after = ctx.records()
    assert after.shape == (2, 1) and after.tobytes() == before.tobytes()
    want = [_expected(ctx, s, twin, scenes[s].frames[1]) for s in (0, 1)]
    step_frames(ctx, np.stack([sc.frames[1] for sc in scenes]), 1)
    recs = ctx.records(max=1)
    for s in (0, 1):
        assert recs[s, 0]["step"] == 1
        _check_values(recs[s, 0], want[s], s)
    assert recs[0, 0]["m"] not in (0, 10) and recs[1, 0]["m"] == 0  # the staged update had m = 10
    ctx.close()
    twin.close()


# ---- GPU: the ring --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_ring_order_wrap_max_and_reenable():
    """depth 8 over 20 steps keeps exactly steps 12..19, oldest first (the copy wraps around the ring's end); max below
    and above what is available; the device form equals the host form byte for byte for every (lo, cnt, max);
    re-enabling, also at the same depth, clears the ring and restarts step at 0."""
    import torch
    scenes = [synth.make_scene("C2", stream_id=s, n_frames=20, n_features=24) for s in range(3)]
    ctx = ctx_from_scenes(scenes, frame_slots=2)
    ctx.enable_records(8)
    hist = []
    for t in range(20):
        step_frames(ctx, np.stack([sc.frames[t] for sc in scenes]), t % 2)
        hist.append(ctx.records(max=1)[:, 0].copy())
        if t == 4:  # not wrapped yet: everything so far
            early = ctx.records()
            assert early.shape == (3, 5) and (early["step"] == np.arange(5)).all()
    hist = np.stack(hist, axis=1)  # [stream][step]
    got = ctx.records()
    assert got.shape == (3, 8) and (got["step"] == np.arange(12, 20)).all()
    assert got.tobytes() == np.ascontiguousarray(hist[:, 12:]).tobytes()
    assert ctx.records(max=3).tobytes() == np.ascontiguousarray(hist[:, 17:]).tobytes()
    assert ctx.records(max=100).shape == (3, 8)
    assert ctx.records(1, 1, 5).tobytes() == np.ascontiguousarray(hist[1:2, 15:]).tobytes()
    R = sl2.STEP_RECORD_DTYPE.itemsize
    for lo, cnt, mx in ((0, 3, 8), (0, 3, 3), (1, 2, 11), (2, 1, 1), (0, 3, 5)):
        buf = torch.full((cnt * mx * R,), 0xAB, dtype=torch.uint8, device="cuda")
        k = ctx.records_dev(lo, cnt, mx, buf.data_ptr())
        ctx.sync()
        dev = buf.cpu().numpy().reshape(cnt, mx, R)
        assert k == min(mx, 8)
        assert dev[:, :k].tobytes() == ctx.records(lo, cnt, mx).tobytes(), (lo, cnt, mx)
        assert (dev[:, k:] == 0xAB).all(), (lo, cnt, mx)
    ctx.enable_records(8)
    assert ctx.records().shape == (3, 0)
    step_frames(ctx, np.stack([sc.frames[0] for sc in scenes]))
    assert ctx.records().shape == (3, 1) and (ctx.records()["step"] == 0).all()
    ctx.enable_records(3)
    for t in range(4):
        step_frames(ctx, np.stack([sc.frames[t] for sc in scenes]), t % 2)
    assert (ctx.records()["step"] == np.array([1, 2, 3])).all()
    ctx.enable_records(0)
    with pytest.raises(sl2.Sl2Error):
        ctx.records()
    ctx.close()


# ---- GPU: batch independence ----------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_bench_shape_records_do_not_depend_on_the_batch():
    """264 C4 streams in one 320x240 context over four calibrations and three selection counts: the serial step, two
    step groups and sl2_step_host_async over two slots give byte-identical records, every two streams of the same
    scene and camera give byte-identical records, and records add exactly one launch per step group."""
    import torch
    nS, T = 264, 3
    cache = {}

    def key(s):
        return ((s * 5) % 8, (s // 2) % 4, s % 3)

    def scene_of(s):
        if key(s) not in cache:
            u, k, j = key(s)
            sc = synth.make_scene("C4", stream_id=u, n_frames=T, camera=CAMS_320[k])
            sc.n_select = (100, 50, 10)[j]
            cache[key(s)] = sc
        return cache[key(s)]

    scenes = [scene_of(s) for s in range(nS)]
    rng = np.random.default_rng(264)
    frames = [np.stack([ring_block(sc.frames[t], 240, 320, rng) for sc in scenes]) for t in range(T)]

    def context(groups):
        ctx = ctx_from_scenes(scenes, frame_slots=2)
        ctx.set_step_groups(groups)
        for s, sc in enumerate(scenes):
            ctx.set_stream_config(s, sl2.stream_config_for_scene(sc))
        ctx.enable_records(4)
        return ctx

    runs = {}
    for name, groups in (("serial", 1), ("groups", 2)):
        ctx = context(groups)
        for t in range(T):
            step_frames(ctx, frames[t], t % 2)
        runs[name] = ctx
    ctx = context(2)
    host = torch.empty((T, nS, 240, 320), dtype=torch.uint8, pin_memory=True)
    host.numpy()[:] = np.stack(frames)
    xv = torch.zeros((T, nS, 13), dtype=torch.float64, pin_memory=True)
    for t in range(T):
        ctx.step_host_async(t % 2, host[t].data_ptr(), xv[t].data_ptr())
    ctx.wait_slot((T - 1) % 2)
    ctx.sync()
    runs["async"] = ctx
    ref = runs["serial"].records()
    assert ref.shape == (nS, T) and (ref["step"] == np.arange(T)).all() and (ref["m"] > 0).all()
    for name in ("groups", "async"):
        assert runs[name].records().tobytes() == ref.tobytes(), name
    assert (xv.numpy()[T - 1] == ref[:, -1]["xv"]).all()
    first = {}
    for s in range(nS):
        first.setdefault(key(s), s)
        assert ref[s].tobytes() == ref[first[key(s)]].tobytes(), s
    assert len(first) == 24
    for name, groups in (("serial", 1), ("groups", 2)):
        c = runs[name]
        l0 = c.launch_count()
        step_frames(c, frames[0])
        with_rec = c.launch_count() - l0
        c.enable_records(0)
        l0 = c.launch_count()
        step_frames(c, frames[0])
        assert with_rec == c.launch_count() - l0 + groups, name
    for c in runs.values():
        c.close()


# ---- GPU: rejections ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_rejections_and_entry_points_that_write_no_record():
    """Every bad argument returns its code and leaves the ring and the streams unchanged; snapshot saves and loads,
    sl2_set_state and sl2_append_feature / sl2_delete_feature write no record and alter none, and the next fused step
    continues the step count."""
    import torch
    scenes = [synth.make_scene("C2", stream_id=s, n_frames=4, n_features=24) for s in range(2)]
    ctx = ctx_from_scenes(scenes, frame_slots=2, max_features=32)
    ctx.enable_records(4)
    for t in range(3):
        step_frames(ctx, np.stack([sc.frames[t] for sc in scenes]), t % 2)
    L, h = ctx.L, ctx.h
    recs, blobs = ctx.records(), ctx.save_streams()
    out = np.zeros((2, 4), sl2.STEP_RECORD_DTYPE)
    buf = torch.zeros(2 * 4 * 256 + 8, dtype=torch.uint8, device="cuda")
    for lo, cnt, mx, ptr in ((-1, 1, 4, out.ctypes.data), (0, 3, 4, out.ctypes.data), (1, 2, 4, out.ctypes.data),
                             (0, -1, 4, out.ctypes.data), (0, 2, 0, out.ctypes.data), (0, 2, -3, out.ctypes.data),
                             (0, 2, 4, None)):
        assert L.sl2_get_records(h, lo, cnt, mx, ptr) == ERR_ARG, (lo, cnt, mx)
        dptr = buf.data_ptr() if ptr else None
        assert L.sl2_get_records_dev(h, lo, cnt, mx, dptr) == ERR_ARG, (lo, cnt, mx)
    assert L.sl2_get_records_dev(h, 0, 2, 4, buf.data_ptr() + 4) == ERR_ARG  # not 8-byte aligned
    assert (buf.cpu().numpy() == 0).all() and (out["step"] == 0).all() and (out["m"] == 0).all()
    for depth in (-1, 4097, 1 << 30):
        assert L.sl2_enable_records(h, depth) == ERR_ARG, depth
    assert L.sl2_enable_records(None, 4) == ERR_ARG
    # entry points that are not the fused step
    ctx.load_streams(blobs[::-1])
    ctx.save_streams()
    ctx.load_streams(blobs)
    x, P = ctx.get_state(0)
    ctx.set_state(0, x, P)
    idx = ctx.append_feature(1, scenes[1].x0[13:16], scenes[1].xp_org[0], scenes[1].patches[0])
    ctx.delete_feature(1, idx)
    assert ctx.records().tobytes() == recs.tobytes()
    assert ctx.save_streams(0, 1) == blobs[:1]
    step_frames(ctx, np.stack([sc.frames[3] for sc in scenes]), 1)
    assert (ctx.records()["step"] == np.arange(4)).all()
    assert ctx.records()[:, :3].tobytes() == recs.tobytes()
    ctx.enable_records(0)
    assert L.sl2_get_records(h, 0, 2, 4, out.ctypes.data) == ERR_STATE
    assert L.sl2_get_records_dev(h, 0, 2, 4, buf.data_ptr()) == ERR_STATE
    ctx.close()
