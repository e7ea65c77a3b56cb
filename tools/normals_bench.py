"""Cost of the patch normals (sl2_set_stream_normals) with every stream on: 264 camera streams of the benchmark's C4
shape (or --config C3), all with the planar patch warp on, the normals off and then on for all of them, alternated
--rounds times in one process so that both settings see the same card and clocks.  Prints one JSON line: per setting
the host-clock time of a fused step (ms, over --steps steps ending in a synchronise), sl2_last_step_times()[2] (the
update interval, the alignment included, between the context's CUDA events) and the launches per step; the alignment
kernel's time per step as the difference of the medians of that event interval with the normals on and off (the
alignment is the only launch the setting adds to it); and the card's name and power limit read in the same run.

  python tools/normals_bench.py [--config C4] [--streams 264] [--steps 40] [--warmup 5] [--rounds 3]
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
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
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

    for s in range(B):
        ctx.set_stream_warp(s, 1)

    def set_all(on):
        for s in range(B):
            ctx.set_stream_normals(s, 8 if on else 0, sigma0=0.5, sigma_i=8.0, sigma_step=0.02)
        ctx.sync()

    def run(on):
        set_all(on)
        for k in range(args.warmup):
            ctx.step(k % R)
        ctx.sync()
        l0 = ctx.launch_count()
        t0 = time.perf_counter()
        for k in range(args.steps):
            ctx.step(k % R)
        ctx.sync()
        ms = (time.perf_counter() - t0) * 1e3 / args.steps
        launches = (ctx.launch_count() - l0) / args.steps
        ctx.enable_timing(True)
        t1 = []
        for k in range(args.steps):
            ctx.step(k % R)
            t1.append(ctx.last_step_times())
        ctx.enable_timing(False)
        t1 = np.array(t1)
        return ms, float(t1[:, 2].mean()), launches

    res = {"off": [], "on": []}
    for _ in range(args.rounds):
        for name, on in (("off", 0), ("on", 1)):
            res[name].append(run(on))

    upd = {k: float(np.median(np.array(v)[:, 1])) for k, v in res.items()}

    gpu, power = card()
    out = {"tool": "normals_bench", "streams": B, "config": args.config, "steps": args.steps, "rounds": args.rounds,
           "gpu": gpu, "power_limit": power,
           "normals_kernel_ms_per_step_events": round(upd["on"] - upd["off"], 4)}
    for name, rows in res.items():
        a = np.array(rows)
        out[name] = {"ms_per_step": [round(v, 4) for v in a[:, 0]],
                     "update_ms": [round(v, 4) for v in a[:, 1]],
                     "launches_per_step": float(a[0, 2]),
                     "frames_per_s": round(float(B / (np.median(a[:, 0]) * 1e-3)), 1)}
    out["step_cost_pct"] = round(100.0 * (np.median(np.array(res["on"])[:, 0]) /
                                          np.median(np.array(res["off"])[:, 0]) - 1.0), 2)
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
