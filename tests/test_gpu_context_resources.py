"""A staged call whose staging cannot be allocated returns SL2_ERR_CUDA and leaves the context usable: the staging
buffers are released and left empty, and the next staged call allocates them again."""
import ctypes as C

import numpy as np
import pytest

from gpu_util import ctx_from_scenes, synth

ERR_CUDA = -2


def _scenes():
    return [synth.make_scene("C2", stream_id=s, n_frames=2, n_features=24) for s in range(2)]


def _context(scenes):
    ctx = ctx_from_scenes(scenes)
    ctx.set_frames(0, np.stack([sc.frames[0] for sc in scenes]))
    return ctx


def _staged_results(ctx):
    """Bytes of a score map, a patch search and a snapshot of stream 0."""
    feat = np.array([0, 3, 5], np.int32)
    centres = np.array([[100.0, 80.0], [160.0, 120.0], [200.0, 150.0]])
    puinv = np.tile([0.02, 0.0, 0.02], (3, 1))
    score = ctx.score_map(0, 0, 3, centres[1], puinv[1])
    search = ctx.patch_search(0, 0, feat, centres, puinv)
    return [a.tobytes() for a in score + search] + [ctx.save_stream(0)]


@pytest.mark.gpu
def test_failed_staging_grow_leaves_the_context_usable():
    scenes = _scenes()
    ctx = _context(scenes)
    before = _staged_results(ctx)
    # 17 bytes of staging per entry: about 2 TiB, beyond device memory, so the device allocation fails and nothing is
    # pinned; NULL outputs, as the call never gets to copy them
    f64, i32 = C.POINTER(C.c_double), C.POINTER(C.c_int32)
    centre, puinv, box = np.array([160.0, 120.0]), np.array([0.02, 0.0, 0.02]), np.zeros(6, np.int32)
    rc = ctx.L.sl2_score_map(ctx.h, 0, 0, 3, centre.ctypes.data_as(f64), puinv.ctypes.data_as(f64),
                             box.ctypes.data_as(i32), None, None, None, 1 << 37)
    msg = ctx.L.sl2_last_error(ctx.h).decode()
    assert rc == ERR_CUDA, (rc, msg)
    assert "cuda_malloc(" in msg and "out of memory" in msg, msg
    assert _staged_results(ctx) == before
    # and the fused step runs as in a context that never failed
    twin = _context(scenes)
    for x in (ctx, twin):
        x.step(0)
        x.sync()
    assert ctx.save_streams() == twin.save_streams()
    ctx.close()
    twin.close()
