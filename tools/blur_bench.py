"""Cost of the exposure blur (sl2_set_stream_blur) with every stream on: 264 camera streams of the benchmark's C4 shape
(or --config C3), alternated --rounds times in one process so that every setting sees the same card and clocks:
  warp      the planar patch warp on, the blur off;
  rest      warp + blur at a 1/60 s exposure with each stream's v and omega set to 0 (one sample per pixel, K = 1);
  streak    warp + blur with each stream's omega set to --rate rad/s about its y axis and v to 0 before the run,
            an exposure chosen so that the image centre's streak is about --streak px (fku |omega| exposure).
Prints one JSON line: per setting the host-clock time of a fused step (ms, over --steps steps ending in a synchronise),
sl2_last_step_times()[1] (the search interval, the warp kernel included) and the launches per step, and the K the
stream-0 templates get at the start of the timed steps; the warp kernel's own device time per step from a separate
torch.profiler run per setting; and the card's name and power limit read in the same run.  The filter moves omega
during the steps (the synthetic frames do not show that motion), so the streak setting's K is reported, not assumed.

  python tools/blur_bench.py [--config C4] [--streams 264] [--steps 40] [--warmup 5] [--rounds 3]
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
    ap.add_argument("--streak", type=float, default=8.0)
    ap.add_argument("--rate", type=float, default=3.0)
    ap.add_argument("--unique", type=int, default=16, help="distinct synthetic scenes, tiled over the streams")
    ap.add_argument("--ring", type=int, default=4, help="distinct frames per stream")
    args = ap.parse_args()

    import torch  # noqa: F401
    import scenelib2_b200 as sl2
    from scenelib2_b200 import synth
    from torch.profiler import ProfilerActivity, profile

    B, R = args.streams, args.ring
    scenes = [synth.make_scene(args.config, stream_id=u, n_frames=R) for u in range(min(args.unique, B))]
    ctx = sl2.Context(sl2.config_for_scene(scenes[0], num_streams=B, frame_slots=R))
    for k in range(R):
        ctx.set_frames(k, np.stack([scenes[s % len(scenes)].frames[k] for s in range(B)]))
    fku = float(scenes[0].cam8[2])
    exposure = args.streak / (fku * args.rate)

    def load(setting):
        """Reload every stream's scene, with the setting's v and omega, then warm up."""
        for s in range(B):
            sc = scenes[s % len(scenes)]
            x0 = np.array(sc.x0, np.float64)
            x0[7:13] = 0.0
            if setting == "streak":
                x0[11] = args.rate
            sl2.load_scene(ctx, s, sc)
            ctx.set_state(s, x0, sc.P0)
            ctx.set_stream_warp(s, 1)
            ctx.set_stream_blur(s, int(setting != "warp"), exposure if setting == "streak" else 1.0 / 60.0, 0.0)
        ctx.sync()
        x = ctx.get_state(0)[0]
        n = ctx.num_features(0)
        _, valid, K = ctx.blur_templates(0, np.arange(n), x)
        return K

    def run(setting):
        K = load(setting)
        l0 = ctx.launch_count()
        t0 = time.perf_counter()
        for k in range(args.steps):
            ctx.step(k % R)
        ctx.sync()
        ms = (time.perf_counter() - t0) * 1e3 / args.steps
        launches = (ctx.launch_count() - l0) / args.steps
        load(setting)
        ctx.enable_timing(True)
        t1 = []
        for k in range(args.steps):
            ctx.step(k % R)
            t1.append(ctx.last_step_times())
        ctx.enable_timing(False)
        return ms, float(np.array(t1)[:, 1].mean()), launches, K

    names = ("warp", "rest", "streak")
    res = {n: [] for n in names}
    Ks = {}
    for _ in range(args.rounds):
        for n in names:
            ms, search, launches, K = run(n)
            res[n].append((ms, search, launches))
            Ks[n] = K

    kernel_us = {}
    for n in names:  # the warp kernel's own time, in runs of their own
        load(n)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for k in range(args.steps):
                ctx.step(k % R)
            ctx.sync()
        kernel_us[n] = round(sum(e.device_time_total for e in prof.key_averages() if "warp_kernel" in e.key)
                             / args.steps, 2)

    gpu, power = card()
    out = {"tool": "blur_bench", "streams": B, "config": args.config, "steps": args.steps, "rounds": args.rounds,
           "gpu": gpu, "power_limit": power, "streak_exposure_s": exposure, "warp_kernel_us_per_step": kernel_us}
    for n in names:
        a = np.array(res[n])
        K = Ks[n]
        out[n] = {"ms_per_step": [round(v, 4) for v in a[:, 0]], "search_ms": [round(v, 4) for v in a[:, 1]],
                  "launches_per_step": float(a[0, 2]),
                  "K_stream0": {"min": int(K.min()), "median": float(np.median(K)), "max": int(K.max())}}
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
