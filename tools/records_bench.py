"""Cost of step records: the fused step of the 264-stream C4 context with records off and on, alternating in one run.

  python tools/records_bench.py [--streams 264] [--depth 1000] [--steps 200] [--rounds 8] [--out DIR]

The context is bench.py's C4 shape (capacity 100, 100-feature maps, n = 313, 16 distinct scenes over the streams).
Each round times --steps fused steps (sl2_step, frames alternating between two slots) with CUDA events on the context's
stream, once with records off and once with a ring of --depth records per stream, the order of the two swapped every
round so that drift of the card's clock falls on both.  Reported: median and spread of the per-step time of each mode
over the rounds, their difference, and the time of one read-back of the whole ring (device form into device memory,
and the host form).  The card's name and power limit are read in the same run.  One JSON line on stdout; with --out,
a markdown table in DIR/records_bench.md.  Needs an H100: there is no CPU path.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from snapshot_bench import card, event_ms  # noqa: E402


def make_context(B, stream):
    import scenelib2_b200 as sl2
    from scenelib2_b200 import synth
    U = 16
    uniq = [synth.make_scene("C4", stream_id=u, n_frames=2) for u in range(U)]
    scenes = [uniq[(s * 5) % U] for s in range(B)]
    cfg = sl2.config_for_scene(scenes[0], num_streams=B, frame_slots=2, max_features=100, cuda_stream=stream)
    ctx = sl2.Context(cfg)
    for s, sc in enumerate(scenes):
        sl2.load_scene(ctx, s, sc)
    for t in range(2):
        ctx.set_frames(t, np.stack([sc.frames[t] for sc in scenes]))
    ctx.sync()
    return ctx


def bench(B, depth, steps, rounds):
    import torch
    stream = torch.cuda.current_stream()  # the context queues its work here, so the events bracket it
    ctx = make_context(B, stream.cuda_stream)
    state = {"t": 0}

    def run():
        for _ in range(steps):
            ctx.step(state["t"] % 2)
            state["t"] += 1

    ms = {0: [], depth: []}
    launches = {}
    for r in range(rounds + 1):  # round 0 warms both modes up and is not kept
        for d in ((0, depth) if r % 2 else (depth, 0)):
            ctx.enable_records(d)
            run()  # warm-up of this mode
            l0 = ctx.launch_count()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run()
            e1.record()
            e1.synchronize()
            launches[d] = (ctx.launch_count() - l0) // steps
            if r:
                ms[d].append(e0.elapsed_time(e1) / steps)
    off, on = np.array(ms[0]), np.array(ms[depth])
    out = {"streams": B, "depth": depth, "steps_per_window": steps, "rounds": rounds,
           "step_ms_off": float(np.median(off)), "step_ms_off_spread": [float(off.min()), float(off.max())],
           "step_ms_on": float(np.median(on)), "step_ms_on_spread": [float(on.min()), float(on.max())],
           "launches_per_step_off": launches[0], "launches_per_step_on": launches[depth]}
    out["overhead_ms"] = out["step_ms_on"] - out["step_ms_off"]
    out["overhead_fraction"] = out["overhead_ms"] / out["step_ms_off"]
    # reading the whole ring back: device form into device memory, host form into host memory
    ctx.enable_records(depth)
    for _ in range(depth):
        ctx.step(state["t"] % 2)
        state["t"] += 1
    ctx.sync()
    buf = torch.empty(B * depth * 256, dtype=torch.uint8, device="cuda")
    out["ring_bytes"] = B * depth * 256
    out["read_dev_ms"], out["read_dev_ms_spread"], _ = event_ms(lambda: ctx.records_dev(0, B, depth, buf.data_ptr()),
                                                                0.5)
    t = []
    for _ in range(4):
        t0 = time.perf_counter()
        rec = ctx.records()
        t.append((time.perf_counter() - t0) * 1e3)
    assert rec.shape == (B, depth)
    out["read_host_ms"] = float(np.median(t[1:]))
    ctx.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=264)
    ap.add_argument("--depth", type=int, default=1000)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--out")
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    c = card()
    r = bench(args.streams, args.depth, args.steps, args.rounds)
    r.update(card=c["name"], power_limit=c["power_limit"])
    print(json.dumps(r), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "records_bench.md"), "w") as f:
            f.write("%s, power limit %s; %d streams, depth %d, %d rounds of %d steps\n\n" % (
                c["name"], c["power_limit"], r["streams"], r["depth"], r["rounds"], r["steps_per_window"]))
            f.write("| records | step ms (median) | min .. max | launches / step |\n|---|---|---|---|\n")
            for k, name in (("off", "off"), ("on", "on")):
                f.write("| %s | %.4f | %.4f .. %.4f | %d |\n" % (name, r["step_ms_" + k], *r["step_ms_%s_spread" % k],
                                                                 r["launches_per_step_" + k]))
            f.write("\nOverhead %.4f ms per step (%.2f %%); whole ring (%.1f MB) read back: device form %.3f ms, host "
                    "form %.1f ms\n" % (r["overhead_ms"], 100 * r["overhead_fraction"], r["ring_bytes"] / 1e6,
                                        r["read_dev_ms"], r["read_host_ms"]))


if __name__ == "__main__":
    main()
