"""Whole fused steps with the iterated update against the CPU oracle's step with its first update replaced by the
iterated one (tests/iterate_oracle.cpp, on top of the sub-pixel, consensus and rescue oracles): 20 steps of two
culling streams with N = 2 relinearisations at tol = 0, the refinement, the consensus and the rescue on, each stream
with 8 uncertain new features and two distractor templates that the cull deletes.  Selection, flags, matches,
counters and iteration counts exactly; h and S at the suite's step tolerances; state at 1e-8 (gpu_util)."""
import numpy as np
import pytest

import iterate_oracle as io
from gpu_util import check_streams_against_oracle, ctx_from_scenes, step_frames
from rescue_scene import rescue_scene

TAU = 2.5
CHI2 = 5.991
N, TOL = 2, 0.0


@pytest.mark.gpu
def test_twenty_fused_steps_of_two_culling_streams_match_the_oracle():
    T = 20
    scs = [rescue_scene("C2", stream_id=s, n_frames=T, n_features=50, new=range(42, 50), sigma=0.03, wrong=[3, 25])
           for s in range(2)]
    ctx = ctx_from_scenes(scs)
    oracles = [io.slam_from_scene(sc, TAU, CHI2, N, TOL) for sc in scs]
    for s in range(2):
        ctx.set_stream_subpixel(s, 1)
        ctx.set_stream_consensus(s, TAU)
        ctx.set_stream_rescue(s, CHI2)
        ctx.set_stream_iterated(s, N, TOL)
    relinearised = 0
    for t in range(T):
        step_frames(ctx, np.stack([sc.frames[t] for sc in scs]))
        check_streams_against_oracle(ctx, oracles, [0, 1], lambda s: scs[s], t)
        it, st, _ = ctx.iterated_results()
        for s in range(2):
            oi, ost, _ = oracles[s].results()
            assert (int(it[s]), int(st[s])) == (oi, ost), (t, s)
            relinearised += oi
    assert relinearised == 2 * T * N  # every step of both streams ran out its relinearisations
    for s in range(2):
        assert oracles[s].num_features < scs[s].n_features  # through a cull
