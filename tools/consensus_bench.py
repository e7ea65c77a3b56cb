"""Cost of the match consensus (sl2_set_stream_consensus) on the benchmark's C4 shape: 264 camera streams of 100
features, every stream with the consensus off and then on (inlier radius --tau), alternated --rounds times in one
process so that both settings see the same card and clocks.  Prints one JSON line: per setting the device time of a
fused step (ms), sl2_last_step_times()[1] (patch search + consensus, ms) and frames/s, with the card's name and power
limit read in the same run.

  python tools/consensus_bench.py [--streams 264] [--steps 40] [--warmup 5] [--rounds 3] [--tau 2.5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=264)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--tau", type=float, default=2.5)
    ap.add_argument("--unique", type=int, default=16, help="distinct synthetic scenes, tiled over the streams")
    ap.add_argument("--ring", type=int, default=4, help="distinct frames per stream")
    args = ap.parse_args()

    import scenelib2_b200 as sl2
    from scenelib2_b200 import synth

    B, R = args.streams, args.ring
    scenes = [synth.make_scene("C4", stream_id=u, n_frames=R) for u in range(min(args.unique, B))]
    ctx = sl2.Context(sl2.config_for_scene(scenes[0], num_streams=B, frame_slots=R))
    for s in range(B):
        sl2.load_scene(ctx, s, scenes[s % len(scenes)])
    for k in range(R):
        ctx.set_frames(k, np.stack([scenes[s % len(scenes)].frames[k] for s in range(B)]))
    ctx.sync()

    def set_all(tau):
        for s in range(B):
            ctx.set_stream_consensus(s, tau)
        ctx.sync()

    def run(tau):
        set_all(tau)
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
        return ms, float(t1[:, 1].mean()), float(t1.sum(axis=1).mean()), launches

    res = {"off": [], "on": []}
    for _ in range(args.rounds):
        for name, tau in (("off", 0.0), ("on", args.tau)):
            res[name].append(run(tau))
    gpu, power = card()
    out = {"tool": "consensus_bench", "streams": B, "config": "C4", "steps": args.steps, "rounds": args.rounds,
           "tau_px": args.tau, "gpu": gpu, "power_limit": power}
    for name, rows in res.items():
        a = np.array(rows)
        out[name] = {"ms_per_step": [round(v, 4) for v in a[:, 0]],
                     "search_ms": [round(v, 4) for v in a[:, 1]],
                     "timed_step_ms": [round(v, 4) for v in a[:, 2]],
                     "launches_per_step": float(a[0, 3]),
                     "frames_per_s": round(float(B / (np.median(a[:, 0]) * 1e-3)), 1)}
    out["step_cost_pct"] = round(100.0 * (np.median(np.array(res["on"])[:, 0]) /
                                          np.median(np.array(res["off"])[:, 0]) - 1.0), 2)
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
