"""Raw camera frames converted on the device (sl2_set_stream_source, csrc/ingest.cu): every result equals that of a
context fed the gray images of the NumPy restatement (tests/ingest_ref.py) through the default path."""
import os

import numpy as np
import pytest

import ingest_ref as ir
from gpu_util import assert_same_bytes, ctx_from_scenes, ring_block, sl2, stream_result, synth

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
G8, RGB, UYVY = ir.SRC_GRAY8, ir.SRC_RGB24, ir.SRC_UYVY


def _frame_set(blocks):
    return np.concatenate([np.ascontiguousarray(b, np.uint8).ravel() for b in blocks])


def _fixture_contexts(rng):
    z = np.load(GOLDEN + "/ingest_cases.npz")
    W, H = (int(v) for v in z["context"])
    cases = [tuple(int(v) for v in z["case_%d" % k]) for k in range(int(z["count"]))]
    cfg = sl2.default_config()
    cfg.width, cfg.height, cfg.num_streams, cfg.frame_slots, cfg.max_features = W, H, len(cases), 2, 1
    cfg.search_tile_radius = 5  # a window tile within the small frame
    patch = rng.integers(0, 256, (1, 11, 11), dtype=np.uint8)
    ctxs = []
    for _ in range(2):
        c = sl2.Context(cfg)
        for s, (fmt, sw, sh, dw, dh) in enumerate(cases):
            c.set_stream_config(s, width=dw, height=dh)
            c.set_features(s, np.zeros((1, 3)), np.array([[0, 0, 0, 1, 0, 0, 0.0]]), patch)
        ctxs.append(c)
    return z, cases, (W, H), ctxs


def _compare_ring(a, b, cases, slot, rng):
    """sl2_score_map with one ellipse over every stream's whole image (corr and sd_image of every candidate depend on
    every pixel of its window) and sl2_find_best_patch over regions that tile it."""
    for s, (_, _, _, dw, dh) in enumerate(cases):
        if dw * dh <= 40000:
            ellipses = [([dw / 2.0, dh / 2.0], [1e-5, 0.0, 1e-5])]
        else:  # 3-sigma radius 60 px around centres 80 px apart, each within the score map's capacity
            ellipses = [([min(u, dw - 1.0), min(v, dh - 1.0)], [0.0025, 0.0, 0.0025])
                        for u in range(40, dw + 40, 80) for v in range(40, dh + 40, 80)]
        for c, p in ellipses:
            ra, rb = a.score_map(s, slot, 0, c, p), b.score_map(s, slot, 0, c, p)
            assert ra[1].size > 0
            for x, y in zip(ra, rb):
                assert x.tobytes() == y.tobytes(), (s, c)
        regions = [[u, v, min(u + 15, dw - 1), min(v + 11, dh - 1)] for u in range(0, dw, 16) for v in range(0, dh, 12)]
        regions.append([0, 0, dw - 1, dh - 1])
        for x, y in zip(a.find_best_patch(s, slot, regions), b.find_best_patch(s, slot, regions)):
            assert x.tobytes() == y.tobytes(), s


@pytest.mark.gpu
def test_fixture_frames_give_the_restatements_ring_bytes():
    """Every format and size class of the golden fixtures, through sl2_set_frames and through sl2_set_frame with
    padded raw rows, against the fixtures' gray images in a context without sources; the ring of the raw context held
    noise before, the gray one gets fresh noise around every smaller image."""
    rng = np.random.default_rng(1)
    z, cases, (W, H), (a, b) = _fixture_contexts(rng)
    n = len(cases)
    for slot in (0, 1):
        a.set_frames(slot, rng.integers(0, 256, (n, H, W), dtype=np.uint8))
    for s, (fmt, sw, sh, _, _) in enumerate(cases):
        a.set_stream_source(s, fmt, sw, sh)
        assert (a.stream_source(s).format, a.stream_source(s).width, a.stream_source(s).height) == (fmt, sw, sh)
    lay = a.frame_set_layout()
    assert lay == [0] + list(np.cumsum([sw * sh * ir.BPP[f] for f, sw, sh, _, _ in cases]))
    raws = [z["raw_%d" % k] for k in range(n)]
    grays = [z["gray_%d" % k] for k in range(n)]
    a.set_frames(0, _frame_set(raws))
    b.set_frames(0, np.stack([ring_block(g, H, W, rng) for g in grays]))
    _compare_ring(a, b, cases, 0, rng)
    for s in range(n):  # one stream at a time, raw rows 7 bytes apart more than their length
        r = raws[s]
        padded = np.zeros((r.shape[0], r.shape[1] + 7), np.uint8)
        padded[:, :r.shape[1]] = r
        assert a.L.sl2_set_frame(a.h, s, 1, padded.ctypes.data, padded.strides[0]) == 0
    a.sync()
    b.set_frames(1, np.stack([ring_block(g, H, W, rng) for g in grays]))
    _compare_ring(a, b, cases, 1, rng)
    a.close()
    b.close()


@pytest.mark.gpu
def test_camera_sizes_and_the_widest_rows():
    """The general INTER_LINEAR path at camera sizes (1280 x 720, 352 x 288 and 640 x 360 to 320 x 240) and raw rows
    of SL2_MAX_SOURCE_DIM pixels (RGB24 4096 x 60, which also upscales vertically, and UYVY 4096 x 4096 to a
    288 x 224 image): the ring equals the restatement's gray in a context without sources."""
    rng = np.random.default_rng(12)
    cases = [(RGB, 1280, 720, 320, 240), (G8, 352, 288, 320, 240), (UYVY, 640, 360, 320, 240),
             (RGB, 4096, 60, 320, 240), (UYVY, 4096, 4096, 288, 224)]
    cfg = sl2.default_config()
    cfg.num_streams, cfg.max_features = len(cases), 1
    patch = rng.integers(0, 256, (1, 11, 11), dtype=np.uint8)
    a, b = sl2.Context(cfg), sl2.Context(cfg)
    for c in (a, b):
        for s, (_, _, _, dw, dh) in enumerate(cases):
            c.set_stream_config(s, width=dw, height=dh)
            c.set_features(s, np.zeros((1, 3)), np.array([[0, 0, 0, 1, 0, 0, 0.0]]), patch)
    a.set_frames(0, rng.integers(0, 256, (len(cases), 240, 320), dtype=np.uint8))
    raws, grays = [], []
    for s, (fmt, sw, sh, dw, dh) in enumerate(cases):
        a.set_stream_source(s, fmt, sw, sh)
        raws.append(synth.make_texture(rng, sh, sw * ir.BPP[fmt]) if sh <= 720 else
                    rng.integers(0, 256, (sh, sw * ir.BPP[fmt]), dtype=np.uint8))
        grays.append(ir.ingest(fmt, raws[-1], sw, sh, dw, dh))
    a.set_frames(0, _frame_set(raws))
    b.set_frames(0, np.stack([ring_block(g, 240, 320, rng) for g in grays]))
    _compare_ring(a, b, cases, 0, rng)
    a.close()
    b.close()


@pytest.mark.gpu
def test_a_load_changes_the_resize_target():
    """A blob of a stream with a 288 x 224 image loaded (host and device form) into a slot whose source is an RGB24
    640 x 480 camera and whose stream had a 320 x 240 image: the next frames are resized to 288 x 224, like a
    context without sources fed the restatement's gray at that size."""
    import torch
    sc = _c2_scenes(4)[0]
    rng = np.random.default_rng(13)
    x = ctx_from_scenes([sc])
    x.set_stream_config(0, width=288, height=224)
    blob = x.save_stream(0)
    x.close()
    host, dev, ref = ctx_from_scenes([sc]), ctx_from_scenes([sc]), ctx_from_scenes([sc])
    for c in (host, dev):
        c.set_stream_source(0, RGB, 640, 480)
        c.set_frames(0, ir.raw_like(RGB, ir.upsample2(sc.frames[0]), rng))  # converted at 320 x 240
    host.load_stream(0, blob)
    stride = (len(blob) + 7) & ~7
    buf = torch.zeros(stride, dtype=torch.uint8, device="cuda")
    buf[:len(blob)] = torch.frombuffer(bytearray(blob), dtype=torch.uint8).cuda()
    torch.cuda.synchronize()
    dev.load_streams_dev(0, 1, buf.data_ptr(), stride)
    ref.load_stream(0, blob)
    for c in (host, dev, ref):
        assert (c.stream_config(0).width, c.stream_config(0).height) == (288, 224)
    for t in range(1, 4):
        raw = ir.raw_like(RGB, ir.upsample2(sc.frames[t]), rng)
        for c in (host, dev):
            c.set_frames(0, raw)
            c.step(0)
        ref.set_frames(0, ring_block(ir.ingest(RGB, raw, 640, 480, 288, 224), 240, 320, rng)[None])
        if t == 1:  # the ring itself, whether or not the tracker finds its features in the resized image
            for c in (host, dev):
                _compare_ring(c, ref, [(RGB, 640, 480, 288, 224)], 0, rng)
        ref.step(0)
        want = stream_result(ref, 0)
        assert_same_bytes(stream_result(host, 0), want, ("host", t))
        assert_same_bytes(stream_result(dev, 0), want, ("dev", t))
    for c in (host, dev, ref):
        c.close()


# the mixed sources of the whole-step test, by stream: (format, width, height); stream images are C4's 320 x 240
FORMS = [(0, 0, 0), (G8, 640, 480), (RGB, 640, 480), (UYVY, 640, 480), (RGB, 320, 240)]


def _raw_and_gray(form, g, rng):
    """A stream's frame-set block and the gray image the device makes of it."""
    fmt, w, h = form
    if fmt == 0:
        return g, g
    base = ir.upsample2(g) if (w, h) == (640, 480) else g
    raw = ir.raw_like(fmt, base, rng)
    return raw, ir.ingest(fmt, raw, w, h, 320, 240)


@pytest.mark.gpu
def test_whole_step_with_mixed_sources_equals_the_gray_path():
    """264 C4 streams with mixed sources, 10 steps, serially, with two step groups, through sl2_step_host_async over
    a 3-slot ring and through sl2_set_frames_dev + sl2_step: x, P, the feature getters and every step record are
    byte-identical to a context fed the restatement's gray frames through the default path."""
    import torch
    nS, T = 264, 10
    scenes = {u: synth.make_scene("C4", stream_id=u, n_frames=T) for u in range(8)}
    sc_of = [scenes[s % 8] for s in range(nS)]
    forms = [FORMS[(s // 8 + s) % 5] for s in range(nS)]
    ref = ctx_from_scenes(sc_of)
    runs = {k: ctx_from_scenes(sc_of, frame_slots=3) for k in ("serial", "groups", "async", "dev")}
    runs["groups"].set_step_groups(2)
    for c in [ref] + list(runs.values()):
        c.enable_records(16)
    for c in runs.values():
        for s, (fmt, w, h) in enumerate(forms):
            if fmt:
                c.set_stream_source(s, fmt, w, h)
    total = runs["serial"].frame_set_layout()[-1]
    pinned = [torch.empty(total, dtype=torch.uint8, pin_memory=True) for _ in range(3)]
    xv = torch.zeros((3, nS, 13), dtype=torch.float64, pin_memory=True)
    dev = torch.empty(total, dtype=torch.uint8, device="cuda")
    rng = np.random.default_rng(264)
    for t in range(T):
        blocks, grays = zip(*[_raw_and_gray(forms[s], sc_of[s].frames[t], rng) for s in range(nS)])
        fs = _frame_set(blocks)
        assert fs.size == total
        ref.set_frames(0, np.stack(grays))
        ref.step(0)
        for k in ("serial", "groups"):
            runs[k].set_frames(t % 3, fs)
            runs[k].step(t % 3)
        runs["async"].wait_slot(t % 3)
        pinned[t % 3].numpy()[:] = fs
        runs["async"].step_host_async(t % 3, pinned[t % 3].data_ptr(), xv[t % 3].data_ptr())
        torch.cuda.synchronize()
        dev.copy_(torch.from_numpy(fs))
        torch.cuda.synchronize()
        runs["dev"].set_frames_dev(t % 3, dev.data_ptr())
        runs["dev"].step(t % 3)
        runs["dev"].sync()
    for c in runs.values():
        c.sync()
    rec = ref.records()
    assert rec.shape == (nS, T)
    for s in range(nS):
        want = stream_result(ref, s)
        for k, c in runs.items():
            assert_same_bytes(stream_result(c, s), want, (k, s))
    for k, c in runs.items():
        assert c.records().tobytes() == rec.tobytes(), k
    assert xv[(T - 1) % 3].numpy().tobytes() == np.stack([ref.get_state(s)[0][:13] for s in range(nS)]).tobytes()
    assert (ref.features(0)["flags"] & 2).any()  # the converted frames still track
    for c in [ref] + list(runs.values()):
        c.close()


def _c2_scenes(n_frames):
    return [synth.make_scene("C2", stream_id=s, n_frames=n_frames, n_features=24) for s in range(2)]


@pytest.mark.gpu
def test_source_change_mid_run_and_resize_target_change():
    """Stream 0 switches from RGB24 to UYVY (both 640 x 480) between two sl2_step_host_async calls, unsynchronised:
    the result equals a context created with UYVY that loads the state after step 3.  Then sl2_set_stream_config
    shrinking the image to 288 x 224 makes the next copy resize to it."""
    import torch
    T = 7
    scs = _c2_scenes(T)
    rng = np.random.default_rng(7)
    forms_t = [(RGB, 640, 480) if t < 3 else (UYVY, 640, 480) for t in range(T)]
    sets = []
    for t in range(T):
        raw0, _ = _raw_and_gray(forms_t[t], scs[0].frames[t], rng)
        sets.append(_frame_set([raw0, scs[1].frames[t]]))
    a = ctx_from_scenes(scs, frame_slots=2)
    a.set_stream_source(0, *forms_t[0])
    host = [torch.empty(max(f.size for f in sets), dtype=torch.uint8, pin_memory=True) for _ in range(T)]
    xv = torch.zeros((T, 2, 13), dtype=torch.float64, pin_memory=True)
    for t in range(T):
        if t == 3:
            a.set_stream_source(0, *forms_t[3])
        host[t].numpy()[:sets[t].size] = sets[t]
        a.step_host_async(t % 2, host[t].data_ptr(), xv[t].data_ptr())
    a.sync()
    r = ctx_from_scenes(scs)
    r.set_stream_source(0, *forms_t[0])
    for t in range(3):
        r.set_frames(0, sets[t])
        r.step(0)
    blobs = r.save_streams()
    c = ctx_from_scenes(scs)
    c.set_stream_source(0, *forms_t[3])
    c.load_streams(blobs)
    for t in range(3, T):
        c.set_frames(0, sets[t])
        c.step(0)
    for s in range(2):
        assert_same_bytes(stream_result(a, s), stream_result(c, s), s)
    for x in (a, r, c):
        x.close()
    # the resize target follows sl2_set_stream_config
    sc = scs[0]
    d = ctx_from_scenes([sc])
    e = ctx_from_scenes([sc])
    d.set_stream_source(0, RGB, 640, 480)
    for t in range(4):
        if t == 2:
            for x in (d, e):
                x.set_stream_config(0, width=288, height=224)
        raw = ir.raw_like(RGB, ir.upsample2(sc.frames[t]), rng)
        dw, dh = (320, 240) if t < 2 else (288, 224)
        d.set_frames(0, raw)
        e.set_frames(0, ring_block(ir.ingest(RGB, raw, 640, 480, dw, dh), 240, 320, rng)[None])
        d.step(0)
        e.step(0)
        assert_same_bytes(stream_result(d, 0), stream_result(e, 0), t)
    d.close()
    e.close()


@pytest.mark.gpu
def test_launch_counts():
    """One conversion launch per frame copy that involves a stream with a source, none otherwise; a source table
    write is one launch per 64 streams with a source."""
    import torch
    cfg = sl2.default_config()
    cfg.num_streams, cfg.frame_slots = 3, 2
    c = sl2.Context(cfg)
    n0 = c.launch_count()

    def delta(f):
        before = c.launch_count()
        f()
        c.sync()
        return c.launch_count() - before

    gray = np.zeros((3, 240, 320), np.uint8)
    assert delta(lambda: c.set_frames(0, gray)) == 0
    assert delta(lambda: c.set_frame(1, 0, gray[1])) == 0
    assert c.launch_count() == n0
    assert delta(lambda: c.set_stream_source(1, RGB, 100, 60)) == 1
    assert delta(lambda: c.set_stream_source(2, UYVY, 64, 48)) == 1
    fs = np.zeros(c.frame_set_layout()[-1], np.uint8)
    assert fs.size == 240 * 320 + 100 * 60 * 3 + 64 * 48 * 2
    assert delta(lambda: c.set_frames(0, fs)) == 1
    assert delta(lambda: c.set_frame(1, 0, np.zeros((60, 300), np.uint8))) == 1
    assert delta(lambda: c.set_frame(0, 0, gray[0])) == 0
    pin = torch.zeros(fs.size, dtype=torch.uint8, pin_memory=True)
    assert delta(lambda: c.step_host_async(1, pin.data_ptr(), None)) == 8 + 1
    dev = torch.zeros(fs.size, dtype=torch.uint8, device="cuda")
    assert delta(lambda: c.set_frames_dev(0, dev.data_ptr())) == 1
    assert delta(lambda: c.set_stream_source(1, 0)) == 1
    assert delta(lambda: c.set_stream_source(2, 0)) == 0
    assert delta(lambda: c.set_frames(0, gray)) == 0
    pin_gray = torch.zeros(gray.size, dtype=torch.uint8, pin_memory=True)
    assert delta(lambda: c.step_host_async(1, pin_gray.data_ptr(), None)) == 8
    c.close()


@pytest.mark.gpu
def test_snapshots_leave_the_source_with_the_slot():
    """A blob saved from a stream with a source is byte-identical to one from the same stream fed gray; loading a
    blob leaves the receiving slot's source as it was."""
    scs = _c2_scenes(2)
    rng = np.random.default_rng(9)
    a, b = ctx_from_scenes(scs), ctx_from_scenes(scs)
    a.set_stream_source(0, UYVY, 640, 480)
    for t in range(2):
        raw, g = _raw_and_gray((UYVY, 640, 480), scs[0].frames[t], rng)
        a.set_frames(0, _frame_set([raw, scs[1].frames[t]]))
        b.set_frames(0, np.stack([g, scs[1].frames[t]]))
        a.step(0)
        b.step(0)
    ba, bb = a.save_streams(), b.save_streams()
    assert ba == bb
    b.load_streams(ba)
    a.load_streams(bb)
    assert a.stream_source(0).format == UYVY and (a.stream_source(0).width, a.stream_source(0).height) == (640, 480)
    assert b.stream_source(0).format == 0 and b.frame_set_layout()[-1] == 2 * 240 * 320
    a.close()
    b.close()


@pytest.mark.gpu
def test_rejected_sources_change_nothing():
    import ctypes as C
    from scenelib2_b200.lib import Sl2StreamSource
    scs = _c2_scenes(1)
    c = ctx_from_scenes(scs)
    c.set_stream_source(1, RGB, 100, 80)
    rng = np.random.default_rng(2)
    raw = rng.integers(0, 256, (80, 300), dtype=np.uint8)
    c.set_frames(0, _frame_set([scs[0].frames[0], raw]))
    region = [[0, 0, 319, 239]]

    def look():
        return ([(c.stream_source(s).format, c.stream_source(s).width, c.stream_source(s).height,
                  c.stream_source(s).reserved) for s in range(2)], c.frame_set_layout(),
                [tuple(getattr(c.stream_config(s), k) for k in ("width", "height", "fku")) for s in range(2)],
                [x.tobytes() for s in range(2) for x in c.find_best_patch(s, 0, region)], c.get_state(0)[0].tobytes())

    before = look()
    bad = [(4, 10, 10, 0), (-1, 10, 10, 0), (RGB, 10, 10, 1), (0, 320, 240, 0), (0, 0, 1, 0), (RGB, 0, 10, 0),
           (RGB, 10, 0, 0), (RGB, 4097, 10, 0), (G8, 10, 4097, 0), (UYVY, 641, 480, 0), (UYVY, -2, 480, 0)]
    for s in (0, 1):
        for f in bad:
            src = Sl2StreamSource(*f)
            assert c.L.sl2_set_stream_source(c.h, s, C.byref(src)) == -1, (s, f)
            assert look() == before, (s, f)
    for s in (-1, 2):
        assert c.L.sl2_set_stream_source(c.h, s, C.byref(Sl2StreamSource(G8, 10, 10, 0))) == -1
    assert c.L.sl2_set_stream_source(c.h, 0, None) == -1
    assert look() == before
    # the bounds themselves are accepted
    for f in ((G8, 1, 1, 0), (UYVY, 4096, 4096, 0), (RGB, 4096, 1, 0), (0, 0, 0, 0)):
        assert c.L.sl2_set_stream_source(c.h, 0, C.byref(Sl2StreamSource(*f))) == 0, f
    c.close()
