"""Cost of relocalisation (sl2_relocalise) on the benchmark's C4 shape (320x240, 100 features, 11x11) and at C3
(640x480, 100 features, 15x15): calls that relocalise 1, 16 and 264 streams of a 264-stream context, each stream on
its scene's own frame.  The call time is a host clock around the synchronous call (median of --reps after --warmup);
the split into the full-image search and the pose kernel comes from torch.profiler's CUDA activity in a separate
pass.  Prints one JSON line, with the card's name and power limit read in the same run.

  python tools/relocalise_bench.py [--reps 10] [--warmup 2]
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
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--unique", type=int, default=8)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    import scenelib2_b200 as sl2
    from scenelib2_b200 import synth

    B = args.streams
    out = {"card": None, "power_limit": None, "configs": {}}
    out["card"], out["power_limit"] = card()
    for name in ("C4", "C3"):
        scenes = [synth.make_scene(name, stream_id=u, n_frames=1) for u in range(args.unique)]
        ctx = sl2.Context(sl2.config_for_scene(scenes[0], num_streams=B, frame_slots=1))
        for s in range(B):
            sl2.load_scene(ctx, s, scenes[s % len(scenes)])
        ctx.set_frames(0, np.stack([scenes[s % len(scenes)].frames[0] for s in range(B)]))
        res = {}
        for cnt in (1, 16, B):
            ids = list(range(0, B, max(1, B // cnt)))[:cnt]
            call = lambda: ctx.relocalise(ids, 0, 2.0, 6, (0, 0, 0), (0, 0, 1e-3), PXX)  # noqa: E731
            for _ in range(args.warmup):
                r, _, _ = call()
            ts = []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                r, _, _ = call()
                ts.append((time.perf_counter() - t0) * 1e3)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(3):
                    call()
            k = {"search": 0.0, "pose": 0.0}
            for e in prof.key_averages():
                if "search_kernel" in e.key:
                    k["search"] += e.device_time_total / 3 / 1e3
                elif "reloc_kernel" in e.key:
                    k["pose"] += e.device_time_total / 3 / 1e3
            res[cnt] = dict(call_ms=float(np.median(ts)), search_ms=k["search"], pose_ms=k["pose"],
                            accepted=int(r["status"].sum()), mean_matches=float(r["matches"].mean()))
        ctx.close()
        out["configs"][name] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
