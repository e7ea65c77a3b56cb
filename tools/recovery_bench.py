"""Cost of stream recovery inside the fused step (sl2_set_stream_recovery) on the benchmark's C4 shape (320x240, 100
features, 11x11) and at C3 (640x480, 100 features, 15x15), 264 streams, serial step order:
  off            no stream has recovery on (the step without the feature)
  on             every stream on, none ever failing: the cost of the three extra launches
  try_1/16/264   that many streams try a relocalisation in every step (their min_matches can never be met, so each
                 step declares them lost and tries, on a frame that shows their map: every try is accepted)
  lost_r1/r10    every stream lost on a frame without its map, retry_period 1 and 10 (steady loss: tries fail)
The step time is a host clock around sl2_step and a synchronise (median of --steps after --warmup); the device time
split by kernel comes from torch.profiler's CUDA activity in a separate pass (the search that follows recover_kernel
is the recovery's).  Prints one JSON line, with the card's name and power limit read in the same run.

  python tools/recovery_bench.py [--steps 20] [--warmup 5]
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

PXX = np.diag([1e-4] * 7 + [2.5e-3] * 6)
RELOC = dict(inlier_px=2.0, min_inliers=6, v=(0.0, 0.0, 0.0), omega=(0.0, 0.0, 1e-3), Pxx=PXX)
NEVER = 1 << 30  # a min_matches no step meets


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def kernel_split(prof, nsteps):
    """ms per step of each kernel family; the search_kernel launched right after recover_kernel is the recovery's"""
    evs = [e for e in prof.events() if e.device_type.name == "CUDA" and e.time_range.elapsed_us() >= 0]
    evs.sort(key=lambda e: e.time_range.start)
    fam = {}
    prev = ""
    for e in evs:
        n = e.name
        if "recover_kernel" in n:
            k = "recover"
        elif "search_kernel" in n:
            k = "recovery_search" if prev == "recover" else "search"
        elif "reloc_kernel" in n:
            k = "pose"
        elif "predict_kernel" in n:
            k = "predict"
        elif "cull_kernel" in n:
            k = "cull"
        elif "records" in n:
            k = "records"
        elif "upd_" in n:
            k = "update"
        else:
            k = "other"
        fam[k] = fam.get(k, 0.0) + e.time_range.elapsed_us() / 1e3 / nsteps
        prev = k
    return {k: round(v, 4) for k, v in sorted(fam.items())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=264)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--unique", type=int, default=8)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    import scenelib2_b200 as sl2
    from scenelib2_b200 import synth

    B = args.streams
    out = {"card": None, "power_limit": None, "streams": B, "configs": {}}
    out["card"], out["power_limit"] = card()
    for name in ("C4", "C3"):
        scenes = [synth.make_scene(name, stream_id=u, n_frames=1) for u in range(args.unique)]
        rng = np.random.default_rng(7)
        shown = np.stack([scenes[s % len(scenes)].frames[0] for s in range(B)])
        hidden = np.stack([synth.make_texture(rng, scenes[0].height, scenes[0].width) for _ in range(B)])
        cases = {"off": ({}, shown), "on": ({s: dict(lost_after=NEVER, min_matches=1) for s in range(B)}, shown)}
        for cnt in (1, 16, B):
            ids = set(range(0, B, max(1, B // cnt))[:cnt])
            cases["try_%d" % cnt] = ({s: dict(lost_after=1, min_matches=NEVER) if s in ids else
                                      dict(lost_after=NEVER, min_matches=1) for s in range(B)}, shown)
        for r in (1, 10):
            cases["lost_r%d" % r] = ({s: dict(lost_after=1, min_matches=NEVER, retry_period=r) for s in range(B)},
                                     hidden)
        res = {}
        for case, (settings, frames) in cases.items():
            ctx = sl2.Context(sl2.config_for_scene(scenes[0], num_streams=B, frame_slots=1))
            for s in range(B):
                sl2.load_scene(ctx, s, scenes[s % len(scenes)])
                if s in settings:
                    ctx.set_stream_recovery(s, **dict(dict(retry_period=1), **settings[s]), **RELOC)
            ctx.set_frames(0, frames)
            l0 = ctx.launch_count()
            ctx.step(0)
            ctx.sync()
            launches = ctx.launch_count() - l0
            for _ in range(args.warmup):
                ctx.step(0)
            ctx.sync()
            ts = []
            for _ in range(args.steps):
                t0 = time.perf_counter()
                ctx.step(0)
                ctx.sync()
                ts.append((time.perf_counter() - t0) * 1e3)
            tries0 = ctx.recovery_results()["attempted"].sum() if settings else 0
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    ctx.step(0)
                ctx.sync()
            r = ctx.recovery_results()
            res[case] = dict(step_ms=round(float(np.median(ts)), 4), launches=int(launches),
                             tries_last_step=int(tries0), recoveries=int(r["recoveries"].sum()),
                             kernels_ms=kernel_split(prof, 5))
            ctx.close()
            torch.cuda.synchronize()
        out["configs"][name] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
