"""Cost of stream snapshots: save and load every stream of a 264-stream context, device and host forms.

  python tools/snapshot_bench.py [--streams 264] [--min-seconds 1.0] [--out DIR]

Contexts:
  c4        the C4 context of bench.py: capacity 100, 100-feature maps (n = 313)
  cap256    capacity 256 with 256-feature maps (n = 781), n_select 128
Timing: CUDA events on the context's stream around runs of sl2_save_streams_dev / sl2_load_streams_dev of all streams,
after warm-up, with enough calls per run for a window of at least --min-seconds (a load's window includes its host-side
validation, which it has to wait for); the host forms (sl2_save_streams / sl2_load_streams of the whole context,
through pinned staging) are timed on the host clock.  Reported: bytes moved, computed from the blob sizes (a save
reads the stream's state and writes the blob; a load reads the blob and writes the whole ld x ld block of P, x and
every per-feature slot up to the capacity, which it resets beyond the map), the GB/s that makes and its fraction of
the H100 SXM data sheet's 3.35 TB/s, for comparison a plain device-to-device copy of the blob bytes, and the time of
one fused step (sl2_step) of the same context in the same run.  The card's name and power limit are read in the same
run.  One JSON line per context on stdout; with --out, a markdown table in DIR/snapshot_bench.md.  Needs an H100: there is no CPU path.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_GBS = 3350.0   # H100 SXM data sheet, HBM3


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        name, power = [c.strip() for c in out.split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:  # the numbers are still measured; the card is then unknown
        return {"name": "unknown (%s)" % e, "power_limit": "unknown"}


def make_context(kind, B, stream):
    import scenelib2_b200 as sl2
    from scenelib2_b200 import synth
    U = 16
    uniq = []
    for u in range(U):
        if kind == "c4":
            sc = synth.make_scene("C4", stream_id=u, n_frames=2)
        else:
            sc = synth.make_scene("C4", stream_id=u, n_frames=2, n_features=256)
            sc.n_select = 128
        uniq.append(sc)
    scenes = [uniq[(s * 5) % U] for s in range(B)]
    cfg = sl2.config_for_scene(scenes[0], num_streams=B, frame_slots=1, max_features=100 if kind == "c4" else 256,
                               cuda_stream=stream)
    ctx = sl2.Context(cfg)
    for s, sc in enumerate(scenes):
        sl2.load_scene(ctx, s, sc)
    ctx.set_frames(0, np.stack([sc.frames[0] for sc in scenes]))
    ctx.step(0)  # every per-step array holds a real step's results
    ctx.sync()
    return ctx


def event_ms(fn, min_seconds):
    """ms per call of fn, from CUDA events on the context's stream around a run of calls that lasts at least
    min_seconds (the number of calls doubles until it does); median and spread of three such windows."""
    import torch
    reps = 1
    while True:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        windows = []
        for _ in range(3):
            e0.record()
            for _ in range(reps):
                fn()
            e1.record()
            e1.synchronize()
            windows.append(e0.elapsed_time(e1) / reps)
        if min(windows) * reps >= 1e3 * min_seconds:
            return float(np.median(windows)), [float(min(windows)), float(max(windows))], reps
        reps *= 2


def bench(kind, B, min_seconds):
    import torch
    import scenelib2_b200 as sl2
    stream = torch.cuda.current_stream()  # the context queues its work here, so the events bracket it
    ctx = make_context(kind, B, stream.cuda_stream)
    cfg = ctx.cfg
    sb = ctx.snapshot_bytes()
    buf = torch.zeros(B * sb, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    ptr = buf.data_ptr()
    blobs = ctx.save_streams()
    sizes = [len(b) for b in blobs]
    blob_bytes = int(np.sum(sizes))
    # a load also resets everything up to the capacity: P's ld x ld block, x, every per-feature slot and template
    ld = ((13 + 3 * cfg.max_features) + 7) & ~7
    per_slot = sum(int(np.prod(sh, dtype=np.int64)) * np.dtype(dt).itemsize
                   for _, sh, dt in sl2.lib.SNAPSHOT_FIELDS) + cfg.boxsize * 16
    load_write = B * (8 * ld * ld + 8 * ld + cfg.max_features * per_slot)
    out = {"context": kind, "streams": B, "capacity": cfg.max_features, "n": int(sl2.read_snapshot(blobs[0])["n"]),
           "blob_bytes_per_stream": sizes[0], "blob_bytes_total": blob_bytes,
           "save_hbm_bytes": 2 * blob_bytes, "load_hbm_bytes": blob_bytes + load_write}
    for name, fn, nbytes in (("save_dev", lambda: ctx.save_streams_dev(0, B, ptr, sb), out["save_hbm_bytes"]),
                             ("load_dev", lambda: ctx.load_streams_dev(0, B, ptr, sb), out["load_hbm_bytes"])):
        for _ in range(3):  # warm-up
            fn()
        ms, spread, reps = event_ms(fn, min_seconds)
        out[name + "_ms"], out[name + "_ms_spread"], out[name + "_calls_per_window"] = ms, spread, reps
        out[name + "_GBps"] = nbytes / ms / 1e6
        out[name + "_fraction_of_3350GBps"] = out[name + "_GBps"] / HBM_GBS
    assert ctx.save_streams() == blobs  # saving and loading the context's own blobs changed nothing
    # the achievable copy rate for comparison: one device-to-device copy of the blob bytes (reads and writes them)
    src = torch.empty(blob_bytes, dtype=torch.uint8, device="cuda")
    dst = torch.empty_like(src)
    for _ in range(3):
        dst.copy_(src)
    ms, spread, _ = event_ms(lambda: dst.copy_(src), min_seconds)
    out["d2d_copy_ms"], out["d2d_copy_GBps"] = ms, 2 * blob_bytes / ms / 1e6
    del src, dst
    for name, fn in (("save_host", lambda: ctx.save_streams()), ("load_host", lambda: ctx.load_streams(blobs))):
        fn()
        t = []
        for _ in range(3):
            t0 = time.perf_counter()
            fn()
            t.append((time.perf_counter() - t0) * 1e3)
        out[name + "_ms"] = float(np.median(t))
        out[name + "_GBps"] = blob_bytes / out[name + "_ms"] / 1e6
    # one fused step of the same context in the same run: the yardstick a device snapshot is compared with
    for _ in range(3):
        ctx.step(0)
    out["step_ms"], out["step_ms_spread"], _ = event_ms(lambda: ctx.step(0), min_seconds)
    out["save_dev_fraction_of_step"] = out["save_dev_ms"] / out["step_ms"]
    ctx.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=264)
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--out")
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    c = card()
    rows = []
    for kind in ("c4", "cap256"):
        r = bench(kind, args.streams, args.min_seconds)
        r.update(card=c["name"], power_limit=c["power_limit"])
        print(json.dumps(r), flush=True)
        rows.append(r)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "snapshot_bench.md"), "w") as f:
            f.write("%s, power limit %s\n\n" % (c["name"], c["power_limit"]))
            f.write("| context | blob MB/stream | save_dev ms | GB/s | load_dev ms | GB/s | d2d copy GB/s | save_host ms | "
                    "load_host ms | step ms |\n")
            f.write("|---|---|---|---|---|---|---|---|---|---|\n")
            for r in rows:
                f.write("| %s | %.3f | %.3f | %.0f | %.3f | %.0f | %.0f | %.1f | %.1f | %.3f |\n" % (
                    r["context"], r["blob_bytes_per_stream"] / 1e6, r["save_dev_ms"], r["save_dev_GBps"],
                    r["load_dev_ms"], r["load_dev_GBps"], r["d2d_copy_GBps"], r["save_host_ms"], r["load_host_ms"],
                    r["step_ms"]))


if __name__ == "__main__":
    main()
