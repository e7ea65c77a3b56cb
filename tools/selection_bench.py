"""Cost and effect of the mutual-information selection (sl2_set_stream_selection): 264 camera streams at capacity 256
in the "ref" (40 features in view, n_select 10) and "stress" (256 in view, n_select 128) regimes of
map_capacity_bench.py, every stream on the trace rule, then on the information rule with min_bits 0, 0.5 and 1,
alternated --rounds times in one process so that every setting sees the same card and clocks.  Each run reloads the
same maps first.  Prints one JSON line: per regime and setting the step time (CUDA events over --steps steps), the
timing mode's predict+select, search, update and cull intervals (sl2_last_step_times), the mean measurement rows m
that entered the update and the mean selection count; the select kernel's own device time per step from a separate
torch.profiler run; and the card's name and power limit read in the same run.

  python tools/selection_bench.py [--streams 264] [--steps 30] [--warmup 5] [--rounds 3] [--regimes ref,stress]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from map_capacity_bench import RING, UNIQUE, card, scenes_for  # noqa: E402

CAP = 256
REGIMES = {"ref": (40, 10), "stress": (CAP, 128)}
SETTINGS = (("trace", 0, 0.0), ("info", 1, 0.0), ("info_0.5", 1, 0.5), ("info_1", 1, 1.0))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=264)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--regimes", default="ref,stress")
    args = ap.parse_args()

    import torch
    import scenelib2_b200 as sl2
    from torch.profiler import ProfilerActivity, profile

    B = args.streams
    out = {"tool": "selection_bench", "streams": B, "capacity": CAP, "steps": args.steps, "rounds": args.rounds,
           "card": card(), "regimes": {}}
    for regime in args.regimes.split(","):
        in_view, n_select = REGIMES[regime]
        scenes = scenes_for(CAP, in_view, n_select)
        stream = torch.cuda.Stream()
        ctx = sl2.Context(sl2.config_for_scene(scenes[0], num_streams=B, frame_slots=RING, max_features=CAP,
                                               cuda_stream=stream.cuda_stream))
        for k in range(RING):
            ctx.set_frames(k, np.stack([scenes[s % UNIQUE].frames[k] for s in range(B)]))

        def reset(mode, bits):
            for s in range(B):
                sl2.load_scene(ctx, s, scenes[s % UNIQUE])
                ctx.set_stream_selection(s, mode, bits)
            ctx.sync()

        def run(mode, bits):
            reset(mode, bits)
            for k in range(args.warmup):
                ctx.step(k % RING)
            ctx.sync()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record(stream)
            for k in range(args.steps):
                ctx.step(k % RING)
            ctx.join()
            e1.record(stream)
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / args.steps
            ctx.enable_timing(True)
            kt, rows, nsel = np.zeros(4), [], []
            for k in range(args.steps):
                ctx.step(k % RING)
                kt += ctx.last_step_times()
                if k == args.steps - 1:
                    for s in range(B):
                        f = ctx.features(s)
                        rows.append(2 * int(((f["flags"] & 3) == 3).sum()))
                        nsel.append(int((f["select_rank"] >= 0).sum()))
            ctx.enable_timing(False)
            return ms, kt / args.steps, float(np.mean(rows)), float(np.mean(nsel))

        res = {name: [] for name, _, _ in SETTINGS}
        for _ in range(args.rounds):
            for name, mode, bits in SETTINGS:
                res[name].append(run(mode, bits))
        reg = {"in_view": in_view, "n_select": n_select}
        for name, mode, bits in SETTINGS:
            rows = res[name]
            kt = np.mean([r[1] for r in rows], axis=0)
            reg[name] = {"ms_per_step": [round(r[0], 4) for r in rows],
                         "predict_select_ms": round(float(kt[0]), 4), "search_ms": round(float(kt[1]), 4),
                         "update_ms": round(float(kt[2]), 4), "cull_ms": round(float(kt[3]), 4),
                         "mean_m": round(float(np.mean([r[2] for r in rows])), 2),
                         "mean_nsel": round(float(np.mean([r[3] for r in rows])), 2)}
            if mode:  # the select kernel's own time, in a run of its own
                reset(mode, bits)
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for k in range(args.steps):
                        ctx.step(k % RING)
                    ctx.sync()
                us = sum(e.device_time_total for e in prof.key_averages() if "select_kernel" in e.key) / args.steps
                reg[name]["select_kernel_us_per_step"] = round(us, 2)
        out["regimes"][regime] = reg
        ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
