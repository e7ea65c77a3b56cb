"""Cost of the iterated EKF update (sl2_set_stream_iterated) with every stream on: 264 camera streams of the
benchmark's C4 shape, the iteration off and then on with N = 1, 2, 3 relinearisations at tol = 0 (every pass runs: the
worst case) and at --tol, alternated --rounds times in one process so that every setting sees the same card and clocks.
Prints one JSON line: per setting the host-clock time of a fused step (ms, over --steps steps ending in a synchronise),
the launches per step, the mean relinearisations per stream and step, the cost per iteration pass ((step - off) / N_g)
the kernels' own device time per step at N = 1 from a separate torch.profiler run, and the card's name and
power limit read in the same run.

  python tools/iterate_bench.py [--streams 264] [--steps 30] [--warmup 5] [--rounds 3] [--tol 1e-3]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from consensus_bench import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C4", choices=["C3", "C4"])
    ap.add_argument("--streams", type=int, default=264)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--tol", type=float, default=1e-3)
    ap.add_argument("--unique", type=int, default=16, help="distinct synthetic scenes, tiled over the streams")
    ap.add_argument("--ring", type=int, default=4, help="distinct frames per stream")
    args = ap.parse_args()

    import scenelib2_b200 as sl2
    from scenelib2_b200 import synth

    B, R = args.streams, args.ring
    scenes = [synth.make_scene(args.config, stream_id=u, n_frames=R) for u in range(min(args.unique, B))]
    ctx = sl2.Context(sl2.config_for_scene(scenes[0], num_streams=B, frame_slots=R))
    for s in range(B):
        sl2.load_scene(ctx, s, scenes[s % len(scenes)])
    for k in range(R):
        ctx.set_frames(k, np.stack([scenes[s % len(scenes)].frames[k] for s in range(B)]))
    ctx.sync()
    snaps = ctx.save_streams()  # every setting starts from the same maps

    def run(N, tol):
        ctx.load_streams(snaps, 0)
        for s in range(B):
            ctx.set_stream_iterated(s, N, tol)
        ctx.sync()
        for k in range(args.warmup):
            ctx.step(k % R)
        ctx.sync()
        l0 = ctx.launch_count()
        iters = 0.0
        t0 = time.perf_counter()
        for k in range(args.steps):
            ctx.step(k % R)
        ctx.sync()
        ms = (time.perf_counter() - t0) * 1e3 / args.steps
        launches = (ctx.launch_count() - l0) / args.steps
        if N:
            it, st, _ = ctx.iterated_results()
            iters = float(it.mean())
        return ms, launches, iters

    settings = [("off", 0, 0.0)] + [("N%d_tol0" % N, N, 0.0) for N in (1, 2, 3)] + \
               [("N%d_tol%g" % (N, args.tol), N, args.tol) for N in (1, 2, 3)]
    res = {name: [] for name, _, _ in settings}
    for _ in range(args.rounds):
        for name, N, tol in settings:
            res[name].append(run(N, tol))

    # the kernels' own device time per step at N = 1, tol = 0, in a run of its own: upd_hp / upd_hp2 and upd_chol run
    # twice per step (the pass and the final update), iterate_kernel once
    from torch.profiler import ProfilerActivity, profile
    run(1, 0.0)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for k in range(args.steps):
            ctx.step(k % R)
        ctx.sync()
    kern = {}
    for e in prof.key_averages():
        for key in ("upd_hp", "upd_chol", "upd_solve", "upd_syrk", "upd_finish", "iterate_kernel"):
            if key in e.key:
                kern[key] = kern.get(key, 0.0) + e.device_time_total / args.steps / 1e3
    gpu, power = card()
    out = {"tool": "iterate_bench", "streams": B, "config": args.config, "steps": args.steps, "rounds": args.rounds,
           "gpu": gpu, "power_limit": power,
           "kernel_ms_per_step_N1": {k: round(v, 4) for k, v in sorted(kern.items())}}
    off = float(np.median(np.array(res["off"])[:, 0]))
    for name, N, tol in settings:
        a = np.array(res[name])
        med = float(np.median(a[:, 0]))
        out[name] = {"ms_per_step": [round(v, 4) for v in a[:, 0]], "launches_per_step": float(a[0, 1]),
                     "mean_iterations_last_step": round(float(a[-1, 2]), 3)}
        if N:
            out[name]["ms_per_pass"] = round((med - off) / N, 4)
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
