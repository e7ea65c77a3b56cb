"""Cost of the accelerometer (sl2_set_stream_accel) on the benchmark's shapes: 264 camera streams at C4 (100 features,
n = 313) and at capacity 256 (256 features, n = 781), the accelerometer off and then on for every stream, alternated
--rounds times in one process so that both settings see the same card and clocks.  Every timed step starts from the
same saved state (sl2_load_streams, outside the timed window) with a fresh sample per stream.  Device time per step and
of its predict interval (motion prediction, measurement prediction and selection) from sl2_last_step_times (timing
mode: serial kernel order); launches per step from sl2_launch_count.  Prints one JSON line per shape with the card's
name and power limit read in the same run.

  python tools/accel_bench.py [--streams 264] [--steps 20] [--warmup 3] [--rounds 3]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from gyro_bench import card  # noqa: E402


def bench(args, shape):
    import scenelib2_b200 as sl2
    from gpu_util import large_variant
    from scenelib2_b200 import synth

    B = args.streams
    if shape == "C4":
        scenes = [synth.make_scene("C4", stream_id=u, n_frames=1) for u in range(min(args.unique, B))]
        cap = None
    else:
        scenes = [large_variant(256, 128, stream_id=u, n_frames=1) for u in range(min(args.unique, B))]
        cap = 256
    ctx = sl2.Context(sl2.config_for_scene(scenes[0], num_streams=B, frame_slots=1, max_features=cap))
    for s in range(B):
        sl2.load_scene(ctx, s, scenes[s % len(scenes)])
    ctx.set_frames(0, np.stack([scenes[s % len(scenes)].frames[0] for s in range(B)]))
    ctx.sync()
    blob = ctx.save_streams()
    n = ctx.state_size(0)
    rng = np.random.default_rng(0)
    cov = np.diag([4e-4, 4e-4, 4e-4])
    g = np.array([0.0, -9.81, 0.0])

    def one_step(on, timed):
        ctx.load_streams(blob)
        if on:
            ctx.set_accel_samples(0, rng.normal(0, 3.0, (B, 3)) - g)
        ctx.sync()
        l0 = ctx.launch_count()
        ctx.step(0)
        t = ctx.last_step_times() if timed else None
        ctx.sync()
        return t, ctx.launch_count() - l0

    def run(on):
        for s in range(B):
            ctx.set_stream_accel(s, int(on), cov=cov, gravity=g, sd_a=1.0)
        ctx.enable_timing(True)
        rows, launches = [], []
        for k in range(args.warmup + args.steps):
            t, nl = one_step(on, True)
            if k >= args.warmup:
                rows.append(t)
                launches.append(nl)
        ctx.enable_timing(False)
        a = np.array(rows)
        return float(a.sum(axis=1).mean()), float(a[:, 0].mean()), float(np.mean(launches))

    res = {"off": [], "on": []}
    for _ in range(args.rounds):
        for name in ("off", "on"):
            res[name].append(run(name == "on"))
    _, status = ctx.accel_results()
    gpu, power = card()
    out = {"tool": "accel_bench", "streams": B, "shape": shape, "n": n, "steps": args.steps, "rounds": args.rounds,
           "gpu": gpu, "power_limit_and_max_sm_clock": power}
    for name, rows in res.items():
        a = np.array(rows)
        out[name] = {"timed_step_ms": [round(v, 4) for v in a[:, 0]], "predict_ms": [round(v, 4) for v in a[:, 1]],
                     "launches_per_step": float(a[0, 2])}
    on, off = np.median(np.array(res["on"])[:, 0]), np.median(np.array(res["off"])[:, 0])
    out["step_cost_pct"] = round(100.0 * (on / off - 1.0), 2)
    pon, poff = np.median(np.array(res["on"])[:, 1]), np.median(np.array(res["off"])[:, 1])
    out["predict_cost_ms"] = round(float(pon - poff), 4)
    out["applied_streams"] = int((status == 1).sum())
    print(json.dumps(out))
    ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=264)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--unique", type=int, default=8, help="distinct synthetic scenes, tiled over the streams")
    args = ap.parse_args()
    for shape in ("C4", "cap256"):
        bench(args, shape)


if __name__ == "__main__":
    main()
