"""Cost of the consensus rescue (sl2_set_stream_rescue) on the benchmark's C4 shape: 264 camera streams of 100
features, 8 of them new (position sigma 3 cm, tests/rescue_scene.py), every stream with the match consensus on, the
rescue off and then on (chi2 --chi2), alternated --rounds times in one process so that both settings see the same card
and clocks.  Every timed step starts from the same saved state (sl2_load_streams, outside the timed window), so every
timed step is the one in which the new features' matches are rejected and, with the rescue on, taken back: the cost of
a step that rescues, on every stream.  Device time per step from sl2_last_step_times (timing mode: serial kernel order).
Prints one JSON line with the card's name and power limit read in the same run.

  python tools/rescue_bench.py [--streams 264] [--steps 20] [--warmup 3] [--rounds 3] [--tau 2.5] [--chi2 5.991]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=264)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--tau", type=float, default=2.5)
    ap.add_argument("--chi2", type=float, default=5.991)
    ap.add_argument("--unique", type=int, default=8, help="distinct synthetic scenes, tiled over the streams")
    args = ap.parse_args()

    import scenelib2_b200 as sl2
    from rescue_scene import rescue_scene

    B = args.streams
    scenes = [rescue_scene("C4", stream_id=u, n_frames=1, n_features=100, new=range(92, 100), sigma=0.03,
                           wrong=[5, 50]) for u in range(min(args.unique, B))]
    ctx = sl2.Context(sl2.config_for_scene(scenes[0], num_streams=B, frame_slots=1))
    for s in range(B):
        sl2.load_scene(ctx, s, scenes[s % len(scenes)])
        ctx.set_stream_consensus(s, args.tau)
    ctx.set_frames(0, np.stack([scenes[s % len(scenes)].frames[0] for s in range(B)]))
    ctx.enable_records(1)
    ctx.sync()
    blob = ctx.save_streams()

    def run(chi2):
        for s in range(B):
            ctx.set_stream_rescue(s, chi2)
        ctx.enable_timing(True)
        rows, launches, m = [], [], []
        for k in range(args.warmup + args.steps):
            ctx.load_streams(blob)
            ctx.sync()
            l0 = ctx.launch_count()
            ctx.step(0)
            t = ctx.last_step_times()
            ctx.sync()
            if k >= args.warmup:
                rows.append(t)
                launches.append(ctx.launch_count() - l0)
                m.append(float(ctx.records()["m"][:, -1].mean()))
        ctx.enable_timing(False)
        a = np.array(rows)
        return float(a.sum(axis=1).mean()), float(a[:, 2].mean()), float(np.mean(launches)), float(np.mean(m))

    res = {"consensus": [], "rescue": []}
    for _ in range(args.rounds):
        for name, chi2 in (("consensus", 0.0), ("rescue", args.chi2)):
            res[name].append(run(chi2))
    gpu, power = card()
    out = {"tool": "rescue_bench", "streams": B, "config": "C4 + 8 new features (sigma 3 cm)", "steps": args.steps,
           "rounds": args.rounds, "tau_px": args.tau, "chi2": args.chi2, "gpu": gpu,
           "power_limit_and_max_sm_clock": power}
    for name, rows in res.items():
        a = np.array(rows)
        out[name] = {"timed_step_ms": [round(v, 4) for v in a[:, 0]],
                     "update_ms": [round(v, 4) for v in a[:, 1]],
                     "launches_per_step": float(a[0, 2]),
                     "mean_rows_m": round(float(a[0, 3]), 2)}
    on, off = np.median(np.array(res["rescue"])[:, 0]), np.median(np.array(res["consensus"])[:, 0])
    out["step_cost_pct"] = round(100.0 * (on / off - 1.0), 2)
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
