"""Stream snapshots (sl2_save_streams / sl2_load_streams and their device forms): a stream saved from one context and
loaded into any stream id of another (other stream count, capacity, frame size, device) continues bit for bit, the
blob round-trips byte for byte, and every malformed blob is refused before anything is written."""
import ctypes as C
import functools
import os
import subprocess

import numpy as np
import pytest

from gpu_util import (assert_same_bytes, check_streams_against_oracle, ctx_from_scenes, oracle_slam_from_scene,
                      patch_snapshot_field, ring_block, sl2, step_frames, stream_result, synth, update_variant)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "scenelib2_b200", "host")
ERR_ARG, ERR_STATE = -1, -3
# everything of a stream that a snapshot carries, as the getters show it
_carried = functools.partial(stream_result, jacobians=True, camera=True)


# ---- helpers --------------------------------------------------------------------------------------------------------
def _blank_ctx(sc, num_streams, **kw):
    return sl2.Context(sl2.config_for_scene(sc, num_streams=num_streams, frame_slots=2, **kw))


def _patch_header(blob, **fields):
    """The blob with header fields replaced."""
    h = sl2.Sl2SnapshotHeader.from_buffer_copy(blob[:C.sizeof(sl2.Sl2SnapshotHeader)])
    for k, v in fields.items():
        if k.startswith("cam."):
            setattr(h.cam, k[4:], v)
        else:
            setattr(h, k, v)
    return bytes(h) + blob[C.sizeof(h):]


# ---- CPU ------------------------------------------------------------------------------------------------------------
def _hand_blob(nfeat=5, box=11, seed=0):
    """A blob of the documented format built field by field in NumPy, and the arrays that went into it."""
    rng = np.random.default_rng(seed)
    n = 13 + 3 * nfeat
    want = {"x": rng.normal(size=n), "P": np.asfortranarray(rng.normal(size=(n, n)))}
    for name, shape, dt in sl2.lib.SNAPSHOT_FIELDS:
        want[name] = (rng.normal(size=(nfeat,) + shape) if dt == np.float64
                      else rng.integers(-1, 100, (nfeat,) + shape).astype(dt))
    want["templates"] = rng.integers(0, 256, (nfeat, box, box), dtype=np.uint8)
    parts = [want["x"].tobytes(), want["P"].tobytes(order="F")]
    parts += [want[name].tobytes() for name, _, _ in sl2.lib.SNAPSHOT_FIELDS] + [want["templates"].tobytes()]
    body = b"".join(p + b"\0" * ((-len(p)) % 8) for p in parts)
    h = sl2.Sl2SnapshotHeader()
    h.magic, h.version, h.header_bytes = sl2.lib.SL2_SNAPSHOT_MAGIC, 1, 128
    h.total_bytes = 128 + len(body)
    h.boxsize, h.nfeat, h.n = box, nfeat, n
    h.cam.width, h.cam.height, h.cam.fku, h.cam.delta_t, h.cam.number_of_features_to_select = 320, 240, 195.0, 0.03, 7
    h.nsel, h.nvisible, h.nmeas, h.ncull = 3, 4, 2, 1
    return bytes(h) + body, want


def test_read_snapshot_parses_a_hand_built_blob():
    for nfeat in (0, 1, 5, 8):  # odd and even n, sections that need padding and ones that do not
        blob, want = _hand_blob(nfeat)
        got = sl2.read_snapshot(blob)
        assert got["nfeat"] == nfeat and got["n"] == 13 + 3 * nfeat and got["total_bytes"] == len(blob)
        assert (got["nsel"], got["nvisible"], got["nmeas"], got["ncull"]) == (3, 4, 2, 1)
        assert got["cam"]["width"] == 320 and got["cam"]["number_of_features_to_select"] == 7
        for k, a in want.items():
            assert got[k].shape == a.shape and got[k].tobytes() == np.ascontiguousarray(a).tobytes(), (nfeat, k)
        assert np.array_equal(got["P"], want["P"])
        assert sl2.lib.snapshot_layout(nfeat, 11)[1] == len(blob)


def test_read_snapshot_rejects_malformed_blobs():
    blob, _ = _hand_blob(6)
    for cut in (0, 64, 127, 128, len(blob) // 2, len(blob) - 1):
        with pytest.raises(ValueError):
            sl2.read_snapshot(blob[:cut])
    for fields in ({"magic": 0x534C3253}, {"version": 2}, {"header_bytes": 120}, {"reserved0": 1}, {"reserved1": 2},
                   {"n": 30}, {"nfeat": -1},
                   {"total_bytes": len(blob) + 8}):
        with pytest.raises(ValueError):
            sl2.read_snapshot(_patch_header(blob, **fields))


def test_c_layout_matches_the_python_parser():
    """sl2_snapshot_layout (the offsets the kernels and the C++ shim use) equals lib.snapshot_layout, the one
    read_snapshot parses with, for odd and even n and both template sizes; out-of-range arguments are refused."""
    L = sl2.load()
    for box in (11, 15):
        for nfeat in (0, 1, 2, 7, 100, 255, 256):
            got = sl2.lib.Sl2SnapshotSections()
            assert L.sl2_snapshot_layout(nfeat, box, C.byref(got)) == 0
            want, total = sl2.lib.snapshot_layout(nfeat, box)
            names = [nm for nm, _, _ in sl2.lib.SNAPSHOT_FIELDS]
            assert (got.x, got.P, got.templates, got.total) == (want["x"][0], want["P"][0], want["templates"][0], total)
            assert list(got.field) == [want[nm][0] for nm in names], (box, nfeat)
    for nfeat, box in ((-1, 11), (257, 11), (5, 0)):
        assert L.sl2_snapshot_layout(nfeat, box, C.byref(sl2.lib.Sl2SnapshotSections())) == ERR_ARG


# ---- GPU: round trip ------------------------------------------------------------------------------------------------
def _c4_scenes(count, n_frames, first=0):
    return [synth.make_scene("C4", stream_id=first + s, n_frames=n_frames) for s in range(count)]


@pytest.mark.gpu
def test_round_trip_eight_c4_streams():
    """8 C4 streams, 3 steps, all saved and loaded into a fresh context of the same config: every getter is
    bit-identical; every section of the blob agrees with the getters or, for the job list and the search results,
    with a staged search of the last frame; 5 more steps on both stay bit-identical and the blobs saved then are
    byte-identical."""
    scenes = _c4_scenes(8, 8)
    a = ctx_from_scenes(scenes, frame_slots=2)
    for t in range(3):
        step_frames(a, np.stack([sc.frames[t] for sc in scenes]), t % 2)
    blobs = a.save_streams()
    assert len(blobs) == 8 and all(len(b) <= a.snapshot_bytes() for b in blobs)
    assert a.save_streams(2, 3) == blobs[2:5] and a.save_stream(7) == blobs[7]
    for s, (sc, blob) in enumerate(zip(scenes, blobs)):
        r, snap = _carried(a, s), sl2.read_snapshot(blob)
        assert snap["x"].tobytes() == r["x"].tobytes() and snap["P"].tobytes() == r["P"].tobytes()
        for k in ("attempted", "successful"):
            assert (snap[k] == r[k]).all()
        assert (snap["sel_rank"] == r["select_rank"]).all() and (snap["h"] == r["h"]).all()
        assert (snap["S"] == r["S"]).all() and (snap["z_uv"] == r["z"]).all()
        assert (snap["xp_org"] == sc.xp_org).all() and (snap["templates"] == sc.patches).all()
        assert snap["nsel"] == (r["select_rank"] >= 0).sum() > 0 and snap["nfeat"] == sc.n_features
        nf, nsel = snap["nfeat"], snap["nsel"]
        J = r["dh_dxv"].reshape(nf, 13, 2).transpose(0, 2, 1)  # each feature's column-major 2 x 13
        assert (snap["dh_dxp"] == J[:, :, :7]).all() and (J[:, :, 7:] == 0).all()
        assert (snap["dh_dy"] == r["dh_dy"].reshape(nf, 3, 2).transpose(0, 2, 1)).all()
        assert (snap["Rvar"] == r["R"][:, 0]).all() and (snap["Rvar"] == r["R"][:, 3]).all()
        assert (snap["found"] == ((r["flags"] & 2) >> 1)).all()
        jobs = np.full(nf, -1, np.int32)
        sel = np.flatnonzero(r["select_rank"] >= 0)
        jobs[r["select_rank"][sel]] = sel
        assert (snap["job_feat"] == jobs).all()
        # no cull in these steps (nfeat is the scene's), so the job list is the one the last step searched: the staged
        # search of its frame (slot 0) with that list reproduces the matches
        feat = snap["job_feat"][:nsel]
        u, v, found, best = a.patch_search(s, 0, feat, snap["job_centre"][:nsel], snap["job_puinv"][:nsel])
        assert (found == snap["found"][feat]).all() and best.tobytes() == snap["best"][feat].tobytes()
        assert (np.stack([u, v], 1) == snap["z_uv"][feat]).all()
    b = _blank_ctx(scenes[0], 8)
    b.load_streams(blobs)
    for s in range(8):
        assert_same_bytes(_carried(b, s), _carried(a, s), ("loaded", s))
    for t in range(3, 8):
        for c in (a, b):
            step_frames(c, np.stack([sc.frames[t] for sc in scenes]), t % 2)
        for s in range(8):
            assert_same_bytes(_carried(b, s), _carried(a, s), ("step", t, s))
    assert b.save_streams() == a.save_streams()
    b.load_streams(b.save_streams())  # loading a context's own blobs changes nothing
    assert b.save_streams() == a.save_streams()
    a.close()
    b.close()


# ---- GPU: migration across shapes -----------------------------------------------------------------------------------
@pytest.mark.gpu
def test_migration_from_the_bench_shape(oracle):
    """Streams of the 264-stream C4 context (the benchmark's shape) after 3 steps go into a 3-stream context at other
    stream ids, a capacity-256 context, a context of capacity exactly nf and a 640x480 context; each continues for 3
    steps bit-identically to its source stream, and against the oracle at every step."""
    B, T0, T1, U = 264, 3, 3, 8
    uniq = _c4_scenes(U, T0 + T1)
    scene_of = lambda s: uniq[(s * 5) % U]
    src = ctx_from_scenes([scene_of(s) for s in range(B)], frame_slots=2)
    picks = (0, 131, 132, 263)
    for t in range(T0):
        step_frames(src, np.stack([scene_of(s).frames[t] for s in range(B)]), t % 2)
    blobs = {s: src.save_stream(s) for s in picks}
    sc0 = uniq[0]
    nf = sc0.n_features
    rng = np.random.default_rng(7)
    # (name, context, {destination stream: source stream}, frame size)
    # the kernels' shared-memory opt-in is set per process by the context created last: the largest capacity goes last
    dests = [("3 streams", _blank_ctx(sc0, 3), {2: 0, 0: 263, 1: 132}, (240, 320)),
             ("capacity nf", _blank_ctx(sc0, 5, max_features=nf), {4: 131, 1: 263}, (240, 320))]
    cfg = sl2.config_for_scene(sc0, num_streams=2, frame_slots=2)
    cfg.width, cfg.height = 640, 480
    dests.append(("640x480", sl2.Context(cfg), {1: 131, 0: 0}, (480, 640)))
    dests.append(("capacity 256", _blank_ctx(sc0, 4, max_features=256), dict(zip((3, 1, 0, 2), picks)), (240, 320)))
    for name, ctx, m, _ in dests:
        for d, s in m.items():
            ctx.load_stream(d, blobs[s])
            assert ctx.save_stream(d) == blobs[s], (name, d)
    oracles = {}
    for name, ctx, m, _ in dests:
        oracles[name] = {}
        for d, s in m.items():
            o = oracle_slam_from_scene(oracle, scene_of(s))
            for t in range(T0):
                o.step(scene_of(s).frames[t])
            oracles[name][d] = o
    for t in range(T0, T0 + T1):
        step_frames(src, np.stack([scene_of(s).frames[t] for s in range(B)]), t % 2)
        for name, ctx, m, (H, W) in dests:
            frames = np.zeros((ctx.cfg.num_streams, H, W), np.uint8)
            for d in range(ctx.cfg.num_streams):
                img = scene_of(m[d]).frames[t] if d in m else uniq[0].frames[t]
                frames[d] = ring_block(img, H, W, rng)
            step_frames(ctx, frames, t % 2)
            check_streams_against_oracle(ctx, oracles[name], sorted(m), lambda d: scene_of(m[d]), t)
            for d, s in m.items():
                assert_same_bytes(_carried(ctx, d), _carried(src, s), (name, t, d, s))
    for _, ctx, _, _ in dests:
        ctx.close()
    src.close()


# ---- GPU: counters ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_counters_survive_and_the_cull_happens_on_time(oracle):
    """A scene whose bad features are culled at step 10: saved after step 7 and loaded into stream 1 of another
    context, the run to step 12 equals the uninterrupted run and the oracle, cull included.  Rebuilding the stream
    with sl2_set_features + sl2_set_state from the same x and P does not: its counters start at zero, so the cull
    does not happen at step 10."""
    cap, nf, bad = 40, 40, 4
    sc = update_variant(cap, nf, bad=bad, n_frames=12)
    a = ctx_from_scenes([sc], frame_slots=2)
    o_a = {0: oracle_slam_from_scene(oracle, sc)}
    for t in range(7):
        step_frames(a, sc.frames[t][None], t % 2)
        check_streams_against_oracle(a, o_a, (0,), lambda s: sc, t)
    blob = a.save_stream(0)
    x7, P7 = a.get_state(0)
    snap = sl2.read_snapshot(blob)
    assert snap["attempted"].max() == 7
    b = _blank_ctx(sc, 2, max_features=cap)
    b.load_stream(1, blob)
    r = _blank_ctx(sc, 1, max_features=cap)  # the map rebuilt from its parts: counters reset
    r.set_features(0, x7[13:].reshape(-1, 3), snap["xp_org"], snap["templates"])
    r.set_state(0, x7, P7)
    for t in range(7, 12):
        step_frames(a, sc.frames[t][None], t % 2)
        check_streams_against_oracle(a, o_a, (0,), lambda s: sc, t)
        step_frames(b, np.stack([sc.frames[t]] * 2), t % 2)
        step_frames(r, sc.frames[t][None], t % 2)
        assert_same_bytes(_carried(b, 1), _carried(a, 0), ("step", t))
        if t + 1 == 10:
            assert a.num_features(0) == nf - bad
    assert b.num_features(1) == nf - bad
    assert r.num_features(0) == nf and r.features(0)["attempted"].max() == 5
    for c in (a, b, r):
        c.close()


def _save_load_continue(src, s, frame_of, steps, where):
    """Stream s of src saved (host and device form) and loaded into streams 2 and 0 of a fresh 3-stream context of
    src's configuration: both continue bit-identically with src for `steps` steps, frame_of(t) giving the frame."""
    import torch
    blob = src.save_stream(s)
    cfg = sl2.Sl2Config.from_buffer_copy(src.cfg)
    cfg.num_streams = 3
    dst = sl2.Context(cfg)
    dst.load_stream(2, blob)
    buf = torch.zeros(src.snapshot_bytes(), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    src.save_streams_dev(s, 1, buf.data_ptr(), src.snapshot_bytes())
    dst.load_streams_dev(0, 1, buf.data_ptr(), src.snapshot_bytes())
    assert dst.save_stream(2) == dst.save_stream(0) == blob, where
    for t in range(steps):
        fr = frame_of(t)
        step_frames(src, np.stack([fr] * src.cfg.num_streams), t % 2)
        step_frames(dst, np.stack([fr] * 3), t % 2)
        for d in (2, 0):
            assert_same_bytes(_carried(dst, d), _carried(src, s), (where, t, d))
    assert dst.save_stream(2) == src.save_stream(s), where
    dst.close()
    return blob


@pytest.mark.gpu
def test_states_left_by_a_cull_a_delete_and_a_rebuild():
    """The counts of the header describe the last prediction / update and are not renewed when the map changes: right
    after the step that culls 24 of 40 features, nvisible (40) and ncull (24) exceed nfeat (16); after
    sl2_delete_feature nvisible exceeds nfeat; after sl2_set_features on a stream that has stepped, nsel exceeds the new
    map and its job slots are empty.  Each of these states is saved, loaded by both forms and continues
    bit-identically."""
    cap, nf, bad = 40, 40, 24
    sc = update_variant(cap, nf, bad=bad, n_frames=13)
    a = ctx_from_scenes([sc], frame_slots=2)
    for t in range(10):
        step_frames(a, sc.frames[t][None], t % 2)
    h = sl2.read_snapshot(a.save_stream(0))
    assert h["nfeat"] == nf - bad and h["nvisible"] == nf and h["ncull"] == bad, (h["nfeat"], h["nvisible"], h["ncull"])
    _save_load_continue(a, 0, lambda t: sc.frames[10 + t], 3, "cull")
    a.close()
    # sl2_delete_feature after a step
    scenes = _c4_scenes(1, 5, first=3)
    b = ctx_from_scenes(scenes, frame_slots=2)
    for t in range(2):
        step_frames(b, scenes[0].frames[t][None], t % 2)
    b.delete_feature(0, 5)
    h = sl2.read_snapshot(b.save_stream(0))
    assert h["nvisible"] > h["nfeat"] == scenes[0].n_features - 1
    _save_load_continue(b, 0, lambda t: scenes[0].frames[2 + t], 3, "delete")
    b.close()
    # sl2_set_features with a smaller map on a stream that has stepped
    c2 = synth.make_scene("C2", stream_id=4, n_frames=5, n_features=24)
    c = ctx_from_scenes([c2], frame_slots=2)
    for t in range(2):
        step_frames(c, c2.frames[t][None], t % 2)
    x, P = c.get_state(0)
    k = 10
    c.set_features(0, x[13:13 + 3 * k].reshape(k, 3), c2.xp_org[:k], c2.patches[:k])
    c.set_state(0, x[:13 + 3 * k], P[:13 + 3 * k, :13 + 3 * k])
    h = sl2.read_snapshot(c.save_stream(0))
    assert h["nsel"] > h["nfeat"] == k and (h["job_feat"] == -1).all()
    _save_load_continue(c, 0, lambda t: c2.frames[2 + t], 3, "rebuild")
    c.close()


# ---- GPU: device form: rollback, clone, reset -----------------------------------------------------------------------
def _dev_buf(ctx, cnt):
    import torch
    buf = torch.zeros(cnt * ctx.snapshot_bytes(), dtype=torch.uint8, device="cuda:%d" % ctx.cfg.device)
    torch.cuda.synchronize()  # the context works on its own stream
    return buf


@pytest.mark.gpu
def test_device_rollback_clone_and_reset():
    """save_streams_dev at step 2, 3 steps, load_streams_dev, the same 3 steps again: bit-identical.  Stream 1 cloned
    onto stream 3 inside a context: the two stay bit-identical, and every other stream equals a run without the clone.
    A blob loaded into a slot that held a larger map gives what it gives in a fresh context."""
    scenes = _c4_scenes(4, 8)
    frames = lambda t, clone=False: np.stack([scenes[1 if clone and s == 3 else s].frames[t] for s in range(4)])
    a = ctx_from_scenes(scenes, frame_slots=2)
    for t in range(2):
        step_frames(a, frames(t), t % 2)
    buf, stride = _dev_buf(a, 4), a.snapshot_bytes()
    a.save_streams_dev(0, 4, buf.data_ptr(), stride)
    first = []
    for t in range(2, 5):
        step_frames(a, frames(t), t % 2)
        first.append([_carried(a, s) for s in range(4)])
    a.load_streams_dev(0, 4, buf.data_ptr(), stride)
    for j, t in enumerate(range(2, 5)):
        step_frames(a, frames(t), t % 2)
        for s in range(4):
            assert_same_bytes(_carried(a, s), first[j][s], ("rollback", t, s))
    # clone 1 -> 3, then step on; the reference context never clones
    ref = ctx_from_scenes(scenes, frame_slots=2)
    for t in range(5):
        step_frames(ref, frames(t), t % 2)
    a.save_streams_dev(1, 1, buf.data_ptr(), stride)
    a.load_streams_dev(3, 1, buf.data_ptr(), stride)
    for t in range(5, 8):
        step_frames(a, frames(t, clone=True), t % 2)
        step_frames(ref, frames(t), t % 2)
        assert_same_bytes(_carried(a, 3), _carried(a, 1), ("clone", t))
        for s in range(3):
            assert_same_bytes(_carried(a, s), _carried(ref, s), ("others", t, s))
    # a 30-feature blob into a slot that held a 100-feature map == into a fresh context
    small = synth.make_scene("C4", stream_id=9, n_frames=3, n_features=30)
    c = ctx_from_scenes([small], frame_slots=2, max_features=100)
    step_frames(c, small.frames[0][None])
    blob = c.save_stream(0)
    fresh = _blank_ctx(small, 4, max_features=100)
    a.load_stream(2, blob)
    fresh.load_stream(2, blob)
    for t in (1, 2):
        fr = np.stack([small.frames[t]] * 4)
        step_frames(a, fr, t % 2)
        step_frames(fresh, fr, t % 2)
        assert_same_bytes(_carried(a, 2), _carried(fresh, 2), ("reset", t))
    assert a.save_stream(2) == fresh.save_stream(2)
    for x in (a, ref, c, fresh):
        x.close()


# ---- GPU: staged sequence and ordering ------------------------------------------------------------------------------
@pytest.mark.gpu
def test_save_between_staged_calls():
    """A save between sl2_predict_measurements and sl2_make_measurements carries the job list: the staged sequence
    finished in the saving and in the receiving context gives identical results."""
    sc = synth.make_scene("C2", stream_id=3, n_frames=3, n_features=24)
    a = ctx_from_scenes([sc], frame_slots=1)
    step_frames(a, sc.frames[0][None])
    a.ekf_predict(0)
    nv = a.predict_measurements(0)
    assert nv > 0
    blob = a.save_stream(0)
    assert sl2.read_snapshot(blob)["nsel"] > 0
    b = _blank_ctx(sc, 2)
    b.load_stream(1, blob)
    a.set_frames(0, sc.frames[1][None])
    b.set_frames(0, np.stack([sc.frames[1]] * 2))
    assert b.make_measurements(1, 0) == a.make_measurements(0, 0) > 0
    a.ekf_update_measured(0)
    b.ekf_update_measured(1)
    assert_same_bytes(_carried(b, 1), _carried(a, 0), "staged")
    assert b.save_stream(1) == a.save_stream(0)
    a.close()
    b.close()


@pytest.mark.gpu
def test_ordering_with_two_step_groups():
    """With two step groups: a save queued right after sl2_step_host_async (no wait) captures that step; a load
    between two sl2_step_host_async calls is seen by the second."""
    import torch
    scenes = [synth.make_scene("C2", stream_id=s, n_frames=3, n_features=24) for s in range(6)]
    host = torch.empty((3, 6, 240, 320), dtype=torch.uint8, pin_memory=True)
    host.numpy()[:] = np.stack([np.stack([sc.frames[t] for sc in scenes]) for t in range(3)])
    xv = torch.zeros((3, 6, 13), dtype=torch.float64, pin_memory=True)
    ref = ctx_from_scenes(scenes, frame_slots=2)
    after = []
    for t in range(2):
        step_frames(ref, host[t].numpy(), t % 2)
        after.append(ref.save_streams())
    a = ctx_from_scenes(scenes, frame_slots=2)
    a.set_step_groups(2)
    a.step_host_async(0, host[0].data_ptr(), xv[0].data_ptr())
    assert a.save_streams() == after[0]
    a.step_host_async(1, host[1].data_ptr(), xv[1].data_ptr())
    a.load_streams(after[0])  # back to the state after step 1 ...
    a.step_host_async(0, host[1].data_ptr(), xv[2].data_ptr())  # ... so this step is step 2 again
    a.sync()
    assert a.save_streams() == after[1]
    assert xv[2].numpy().tobytes() == np.stack([sl2.read_snapshot(b)["x"][:13] for b in after[1]]).tobytes()
    a.close()
    ref.close()


# ---- GPU: large maps ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_large_maps_round_trip_and_move():
    """Capacity 256 with 256-feature maps (n = 781): round trip into a context of the same config, and a move into a
    capacity-256 context of another stream count, each continuing bit-identically for 3 steps."""
    scenes = []
    for s in range(2):
        sc = synth.make_scene("C4", stream_id=s, n_frames=6, n_features=256)
        sc.n_select = 128
        scenes.append(sc)
    a = ctx_from_scenes(scenes, frame_slots=2, max_features=256)
    for s, sc in enumerate(scenes):
        a.set_stream_config(s, sl2.stream_config_for_scene(sc))
    for t in range(3):
        step_frames(a, np.stack([sc.frames[t] for sc in scenes]), t % 2)
    blobs = a.save_streams()
    assert [sl2.read_snapshot(b)["n"] for b in blobs] == [781, 781]
    assert len(blobs[0]) == a.snapshot_bytes()
    same = _blank_ctx(scenes[0], 2, max_features=256)
    same.load_streams(blobs)
    other = _blank_ctx(scenes[0], 5, max_features=256)
    other.load_streams(blobs, lo=3)
    for t in range(3, 6):
        fr = np.stack([sc.frames[t] for sc in scenes])
        step_frames(a, fr, t % 2)
        step_frames(same, fr, t % 2)
        step_frames(other, np.concatenate([fr[:1]] * 3 + [fr]), t % 2)
        for s in range(2):
            assert_same_bytes(_carried(same, s), _carried(a, s), ("same", t, s))
            assert_same_bytes(_carried(other, 3 + s), _carried(a, s), ("other", t, s))
    assert same.save_streams() == a.save_streams() == other.save_streams(3, 2)
    for c in (a, same, other):
        c.close()


# ---- GPU: rejections ------------------------------------------------------------------------------------------------
def _bad_blobs(good, nsel):
    """(description, blob, expected code) of every malformed variant of `good` (a blob with 0 < nsel < nfeat)."""
    h = sl2.read_snapshot(good)
    nf, n = h["nfeat"], h["n"]
    job = int(np.nonzero(h["sel_rank"] < 0)[0][0])
    out = [("magic", _patch_header(good, magic=0x12345678)),
           ("byte order", _patch_header(good, magic=0x534C3253)),
           ("version", _patch_header(good, version=2)),
           ("header size", _patch_header(good, header_bytes=120)),
           ("total above stride", _patch_header(good, total_bytes=(1 << 40))),
           ("total mismatch", _patch_header(good, total_bytes=len(good) - 8)),
           ("n", _patch_header(good, n=n + 3)),
           ("negative nfeat", _patch_header(good, nfeat=-1, n=10)),
           ("negative nsel", _patch_header(good, nsel=-1)),
           ("negative nvisible", _patch_header(good, nvisible=-1)),
           ("negative nmeas", _patch_header(good, nmeas=-1)),
           ("negative ncull", _patch_header(good, ncull=-1)),
           ("reserved0", _patch_header(good, reserved0=1)),
           ("reserved1", _patch_header(good, reserved1=-1)),
           ("nsel above 128", _patch_header(good, nsel=129)),
           ("nmeas above 128", _patch_header(good, nmeas=129)),
           ("nvisible above 256", _patch_header(good, nvisible=257)),
           ("ncull above 256", _patch_header(good, ncull=257)),
           ("boxsize", _patch_header(good, boxsize=15)),
           ("job_feat past the map", patch_snapshot_field(good, "job_feat", 0, nf)),
           ("job_feat below -1", patch_snapshot_field(good, "job_feat", 0, -2)),
           ("job_feat after nsel", patch_snapshot_field(good, "job_feat", nsel, 0)),
           ("sel_rank at nsel", patch_snapshot_field(good, "sel_rank", job, nsel)),
           ("sel_rank at nfeat below nsel",
            patch_snapshot_field(_patch_header(good, nsel=nf + 5), "sel_rank", job, nf)),
           ("sel_rank below -1", patch_snapshot_field(good, "sel_rank", job, -2)),
           ("image wider than the frame", _patch_header(good, **{"cam.width": 321})),
           ("image below the box", _patch_header(good, **{"cam.height": 15})),
           ("fku", _patch_header(good, **{"cam.fku": 0.0})),
           ("delta_t", _patch_header(good, **{"cam.delta_t": float("nan")})),
           ("selection", _patch_header(good, **{"cam.number_of_features_to_select": -1}))]
    return [(d, b, ERR_ARG) for d, b in out]


@pytest.mark.gpu
def test_rejections_leave_every_stream_unchanged():
    """Every malformed blob, range, pointer and stride is refused by the host and the device form with the documented
    code, also as the last blob of a batch of good ones, and no stream of the batch changes."""
    import torch
    scenes = [synth.make_scene("C2", stream_id=s, n_frames=2, n_features=24) for s in range(3)]
    for sc in scenes:
        sc.n_select = 10
    ctx = ctx_from_scenes(scenes)
    step_frames(ctx, np.stack([sc.frames[0] for sc in scenes]))
    good = ctx.save_streams()
    nsel = sl2.read_snapshot(good[0])["nsel"]
    assert 0 < nsel < 24
    big_sc = synth.make_scene("C2", stream_id=5, n_frames=1, n_features=30)
    big = ctx_from_scenes([big_sc])
    cases = _bad_blobs(good[0], nsel) + [("map above max_features", big.save_stream(0), ERR_STATE)]
    big.close()
    L, h = ctx.L, ctx.h
    sb = ctx.snapshot_bytes()
    S = (max([sb] + [len(b) for _, b, _ in cases]) + 7) & ~7  # one stride for every case
    dev = torch.zeros(3 * S, dtype=torch.uint8, device="cuda")

    def unchanged(what):
        assert ctx.save_streams() == good, what

    def to_dev(blobs, stride):
        dev.zero_()
        for i, b in enumerate(blobs):
            dev[i * stride:i * stride + len(b)] = torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda()
        torch.cuda.synchronize()

    for what, blob, code in cases:
        for batch, lo in (([blob], 1), (good[:2] + [blob], 0)):
            buf = np.zeros(len(batch) * S, np.uint8)
            for i, b in enumerate(batch):
                buf[i * S:i * S + len(b)] = np.frombuffer(b, np.uint8)
            assert L.sl2_load_streams(h, lo, len(batch), buf.ctypes.data, S) == code, (what, "host", len(batch))
            unchanged((what, "host", len(batch)))
            to_dev(batch, S)
            assert L.sl2_load_streams_dev(h, lo, len(batch), dev.data_ptr(), S) == code, (what, "dev", len(batch))
            unchanged((what, "dev", len(batch)))
    # ranges, pointers and strides
    buf = np.zeros(3 * sb, np.uint8)
    sizes = (C.c_size_t * 3)()
    to_dev(good, sb)
    for lo, cnt in ((-1, 1), (0, 4), (3, 1), (2, 2), (0, -1)):
        assert L.sl2_load_streams(h, lo, cnt, buf.ctypes.data, sb) == ERR_ARG
        assert L.sl2_load_streams_dev(h, lo, cnt, dev.data_ptr(), sb) == ERR_ARG
        assert L.sl2_save_streams(h, lo, cnt, buf.ctypes.data, sb, sizes) == ERR_ARG
        assert L.sl2_save_streams_dev(h, lo, cnt, dev.data_ptr(), sb) == ERR_ARG
    assert L.sl2_load_streams(h, 0, 1, None, sb) == ERR_ARG and L.sl2_load_streams_dev(h, 0, 1, None, sb) == ERR_ARG
    assert L.sl2_save_streams(h, 0, 1, None, sb, sizes) == ERR_ARG
    assert L.sl2_save_streams_dev(h, 0, 1, None, sb) == ERR_ARG
    assert L.sl2_load_streams(h, 0, 1, buf.ctypes.data, 64) == ERR_ARG
    assert L.sl2_load_streams_dev(h, 0, 1, dev.data_ptr(), 64) == ERR_ARG
    assert L.sl2_save_streams(h, 0, 2, buf.ctypes.data, sb - 8, sizes) == ERR_ARG
    assert L.sl2_save_streams_dev(h, 0, 2, dev.data_ptr(), sb - 8) == ERR_ARG
    assert L.sl2_save_streams_dev(h, 0, 1, dev.data_ptr() + 4, sb) == ERR_ARG
    assert L.sl2_load_streams_dev(h, 0, 1, dev.data_ptr(), sb + 4) == ERR_ARG
    unchanged("ranges")
    # the dev buffer still holds the good blobs: a valid device load of them is accepted
    assert L.sl2_load_streams_dev(h, 0, 3, dev.data_ptr(), sb) == 0
    unchanged("good device load")
    ctx.close()
    # a selection above 128 is refused in a context above 128 features, accepted in a small one
    blob129 = _patch_header(good[0], **{"cam.number_of_features_to_select": 129})
    large = ctx_from_scenes(scenes[:1], max_features=256)
    before = large.save_stream(0)
    with pytest.raises(sl2.Sl2Error):
        large.load_stream(0, blob129)
    assert large.save_stream(0) == before
    large.close()
    small = ctx_from_scenes(scenes[:1])
    small.load_stream(0, blob129)
    assert small.stream_config(0).number_of_features_to_select == 129
    small.close()


# ---- GPU: the C++ shim ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_headless_save_and_load_state(tmp_path):
    """sl2_headless on C1 raw frames: 3 frames with SL2_HEADLESS_SAVE_STATE, then the remaining 5 with
    SL2_HEADLESS_LOAD_STATE, against one run of all 8: the per-frame lines of the second run equal lines 3.. of the
    straight run, and the final state files are byte-identical."""
    kp = np.load(os.path.join(ROOT, "tests", "golden", "known_patches.npy"))
    T, k = 8, 3
    sc = synth.make_scene("C1", n_frames=T, known_patches=kp)
    Pxx = np.diag([4e-4] * 3 + [2e-5] * 4 + [1e-3] * 3 + [1e-3] * 3)
    sc.P0 = np.zeros_like(sc.P0)
    sc.P0[:13, :13] = Pxx
    synth.write_reference_case(str(tmp_path), sc, Pxx)
    (tmp_path / "head.raw").write_bytes(sc.frames[:k].tobytes())
    (tmp_path / "tail.raw").write_bytes(sc.frames[k:].tobytes())
    exe = os.path.join(HOST, "sl2_headless")
    cfg = str(tmp_path / "case.cfg")

    def run(raw, frames, **env):
        r = subprocess.run([exe, cfg, str(tmp_path / raw), "320", "240", str(frames)], capture_output=True, text=True,
                           env=dict(os.environ, **env))
        assert r.returncode == 0, r.stderr
        return [ln.split(None, 2)[2] for ln in r.stdout.splitlines() if ln.startswith("frame ")]

    straight = run("frames.raw", T, SL2_HEADLESS_SAVE_STATE=str(tmp_path / "straight.bin"))
    head = run("head.raw", k, SL2_HEADLESS_SAVE_STATE=str(tmp_path / "mid.bin"))
    tail = run("tail.raw", T - k, SL2_HEADLESS_LOAD_STATE=str(tmp_path / "mid.bin"),
               SL2_HEADLESS_SAVE_STATE=str(tmp_path / "end.bin"))
    assert len(straight) == T and head == straight[:k] and tail == straight[k:]
    assert "measured 0" not in " ".join(straight)
    end, ref = (tmp_path / "end.bin").read_bytes(), (tmp_path / "straight.bin").read_bytes()
    assert end == ref


# ---- GPU: two devices -----------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_move_between_devices():
    """Saved on device 0, loaded on device 1 (host form): the continuation is bit-identical."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two visible GPUs")
    scenes = _c4_scenes(3, 5)
    a = ctx_from_scenes(scenes, frame_slots=2, device=0)
    for t in range(2):
        step_frames(a, np.stack([sc.frames[t] for sc in scenes]), t % 2)
    b = sl2.Context(sl2.config_for_scene(scenes[0], num_streams=3, frame_slots=2, device=1))
    b.load_streams(a.save_streams())
    for t in range(2, 5):
        for c in (a, b):
            step_frames(c, np.stack([sc.frames[t] for sc in scenes]), t % 2)
        for s in range(3):
            assert_same_bytes(_carried(b, s), _carried(a, s), ("device 1", t, s))
    a.close()
    b.close()
