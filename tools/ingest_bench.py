"""Raw camera frames converted on the device (sl2_set_stream_source) at the benchmark's shape: 264 C4 streams with
320 x 240 images, fed through sl2_step_host_async over a 3-slot pinned ring.

  python tools/ingest_bench.py [--streams 264] [--steps 200] [--out DIR]

Legs: (a) default gray frames (bench.py's e2e leg), (b) RGB24 640 x 480, (c) UYVY 640 x 480, (d) RGB24 640 x 480
already on the device, through sl2_set_frames_dev + sl2_step.  Reported per leg: frames/s (camera frames per second
of wall time over --steps steps, ending in a synchronise), the bytes one step copies host -> device, and the ingest
kernel's device time per frame set with its achieved bytes/s (raw bytes read + gray bytes written) against the H100 SXM
data-sheet 3.35 TB/s.  The kernel time comes from CUDA events on the context's stream: sl2_set_frames_dev of a frame
set whose streams all have a source is one device-to-device copy of the raw bytes into the staging plus the ingest
kernel; the same copy alone is timed the same way and subtracted (both are reported).  As the host alternative,
cv2.cvtColor + cv2.resize of one frame on one core of this machine.  The card's name and power limit are read in the
same run.  One JSON line on stdout; with --out, a markdown table in DIR/ingest_bench.md.  Needs an H100.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from snapshot_bench import card, event_ms  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
LEGS = {"a_gray": (0, 0, 0, False), "b_rgb24_640": (2, 640, 480, False), "c_uyvy_640": (3, 640, 480, False),
        "d_rgb24_640_dev": (2, 640, 480, True)}


def frame_sets(ctx, scenes, fmt, w, h):
    import ingest_ref as ir
    rng = np.random.default_rng(5)
    out = []
    for t in range(2):
        blocks = []
        for sc in scenes:
            g = sc.frames[t]
            blocks.append(g if fmt == 0 else ir.raw_like(fmt, ir.upsample2(g), rng))
        fs = np.concatenate([b.ravel() for b in blocks])
        assert fs.size == ctx.frame_set_layout()[-1]
        out.append(fs)
    return out


def ingest_ms(ctx, dev_sets, min_seconds=0.5):
    """ms per frame set of (copy + ingest kernel) and of the copy alone, from CUDA events on the context's stream (the
    torch stream the context was created on)."""
    import torch
    k = {"i": 0}

    def convert():
        ctx.set_frames_dev(k["i"] % 2, dev_sets[k["i"] % 2].data_ptr())
        k["i"] += 1

    stage = torch.empty_like(dev_sets[0])

    def copy():
        stage.copy_(dev_sets[k["i"] % 2])
        k["i"] += 1

    both, both_spread, _ = event_ms(convert, min_seconds)
    alone, alone_spread, _ = event_ms(copy, min_seconds)
    return both, both_spread, alone, alone_spread


def host_alternative(fmt, w, h, reps=200):
    try:
        import cv2
    except ImportError:
        return None
    cv2.setNumThreads(1)
    rng = np.random.default_rng(1)
    raw = rng.integers(0, 256, (h, w, 3 if fmt == 2 else 2), dtype=np.uint8)
    code = cv2.COLOR_RGB2GRAY if fmt == 2 else cv2.COLOR_YUV2GRAY_UYVY
    t0 = time.perf_counter()
    for _ in range(reps):
        cv2.resize(cv2.cvtColor(raw, code), (320, 240), interpolation=cv2.INTER_LINEAR)
    return (time.perf_counter() - t0) / reps * 1e3


def run_leg(name, B, steps):
    import torch
    import scenelib2_b200 as sl2
    from scenelib2_b200 import synth
    fmt, w, h, on_dev = LEGS[name]
    uniq = [synth.make_scene("C4", stream_id=u, n_frames=2) for u in range(16)]
    scenes = [uniq[(s * 5) % 16] for s in range(B)]
    stream = torch.cuda.Stream()  # the context queues its work here, so the events of ingest_ms bracket it
    cfg = sl2.config_for_scene(scenes[0], num_streams=B, frame_slots=3, max_features=100,
                               cuda_stream=stream.cuda_stream)
    ctx = sl2.Context(cfg)
    for s, sc in enumerate(scenes):
        sl2.load_scene(ctx, s, sc)
        if fmt:
            ctx.set_stream_source(s, fmt, w, h)
    sets = frame_sets(ctx, scenes, fmt, w, h)
    total = sets[0].size
    pinned = [torch.from_numpy(sets[t % 2]).pin_memory() for t in range(3)]
    dev = [torch.from_numpy(s).cuda() for s in sets]
    xv = torch.zeros((3, B, 13), dtype=torch.float64, pin_memory=True)
    torch.cuda.synchronize()

    def run(n):
        for t in range(n):
            if on_dev:
                ctx.set_frames_dev(t % 3, dev[t % 2].data_ptr())
                ctx.step(t % 3)
            else:
                ctx.step_host_async(t % 3, pinned[t % 3].data_ptr(), xv[t % 3].data_ptr())
        ctx.sync()

    run(20)  # warm-up
    t0 = time.perf_counter()
    run(steps)
    wall = time.perf_counter() - t0
    res = {"frames_per_s": steps * B / wall, "step_ms": wall / steps * 1e3, "frame_set_bytes": total,
           "h2d_bytes_per_step": 0 if on_dev else total, "d2d_bytes_per_step": total if on_dev else 0}
    if fmt:
        with torch.cuda.stream(stream):
            both, both_spread, alone, alone_spread = ingest_ms(ctx, dev)
        ms = both - alone
        moved = total + B * 320 * 240
        res.update({"copy_and_ingest_ms": both, "copy_and_ingest_ms_spread": both_spread, "copy_alone_ms": alone,
                    "copy_alone_ms_spread": alone_spread, "ingest_ms": ms, "ingest_bytes": moved,
                    "ingest_GB_per_s": moved / (ms * 1e-3) / 1e9,
                    "ingest_share_of_3_35_TB_per_s": moved / (ms * 1e-3) / HBM_BYTES_PER_S})
        host = host_alternative(fmt, w, h)
        res["host_cv2_ms_per_frame_one_core"] = host
        res["host_cv2_frames_per_s_one_core"] = (1e3 / host) if host else None
    ctx.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=264)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("ingest_bench needs a GPU: there is no CPU path")
    out = {"card": card(), "streams": a.streams, "steps": a.steps, "cpu_cores": os.cpu_count()}
    for name in LEGS:
        out[name] = run_leg(name, a.streams, a.steps)
    print(json.dumps(out))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "ingest_bench.md"), "w") as f:
            f.write("card: %s, power limit %s\n\n" % (out["card"]["name"], out["card"]["power_limit"]))
            f.write("| leg | frames/s | H2D bytes/step | copy + ingest ms | copy ms | ingest ms | ingest GB/s | "
                    "share of 3.35 TB/s | cv2 ms/frame/core |\n")
            f.write("|---|---|---|---|---|---|---|---|---|\n")
            for name in LEGS:
                r = out[name]
                f.write("| %s | %.0f | %d | %s | %s | %s | %s | %s | %s |\n" % (
                    name, r["frames_per_s"], r["h2d_bytes_per_step"],
                    "%.4f" % r["copy_and_ingest_ms"] if "ingest_ms" in r else "-",
                    "%.4f" % r["copy_alone_ms"] if "ingest_ms" in r else "-",
                    "%.4f" % r["ingest_ms"] if "ingest_ms" in r else "-",
                    "%.0f" % r["ingest_GB_per_s"] if "ingest_ms" in r else "-",
                    "%.2f" % r["ingest_share_of_3_35_TB_per_s"] if "ingest_ms" in r else "-",
                    "%.3f" % r["host_cv2_ms_per_frame_one_core"] if r.get("host_cv2_ms_per_frame_one_core") else "-"))


if __name__ == "__main__":
    main()
