"""Fused-step throughput of large maps: C4 frames at 264 camera streams with map capacities above 128 features.

  python tools/map_capacity_bench.py [--streams 264] [--steps 40] [--warmup 10] [--reps 3] [--out DIR]

Cases (every one a context of its own):
  anchor      capacity 100, 100 features in view, n_select 100: the C4 workload of bench.py
  cap/stress  capacity 128 / 192 / 256, every feature in view, n_select 128: m = 256 every step
  cap/ref     capacity 128 / 192 / 256, 40 features in view (the rest moved out of the view), n_select 10: the
              reference's regime, a large map with few features measured
Reported per case: frames/s and ms per step (device-resident sl2_step, CUDA events, median and spread of the
repetitions), sl2_last_step_times / sl2_last_update_times averaged over the timed steps, the EKF update's HBM bytes
computed from the shapes (update_hbm_bytes) and the GB/s they make over the five update kernels' time.  The card's
name, power limit and maximum SM clock are read in the same run.  Writes one JSON line per case to stdout and, with
--out, a markdown table to DIR/map_capacity.md.  Needs an H100: there is no CPU path.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_GBS = 3350.0   # H100 SXM data sheet, HBM3
UNIQUE, RING = 16, 4


def update_hbm_bytes(n, K):
    """Bytes the EKF update of one stream moves through HBM, from the shapes (n state size, K measured features,
    m = 2 K; FP64).  upd_hp reads the 7 dense rows of P and 3 rows per measured feature and writes G = [S | H P | nu];
    upd_chol reads and writes the S block; upd_solve reads H P | nu and writes Y over it; upd_syrk reads Y, reads the
    upper 64 x 64 tiles of P and writes them and their mirrors."""
    if K == 0:
        return {"hp_P_read": 0, "G_write": 0, "G_read": 0, "syrk_P_read": 0, "syrk_P_write": 0, "total": 0}
    m = 2 * K
    nt = (n + 1 + 63) // 64
    tiles = nt * (nt + 1) // 2
    cols = n + 1
    hp_P_read = (7 + 3 * K) * n * 8
    G_write = m * (m + cols) * 8 + m * m * 8 + m * cols * 8              # upd_hp, upd_chol (U), upd_solve (Y)
    G_read = m * m * 8 + m * cols * 8 + m * cols * 8                      # upd_chol, upd_solve, upd_syrk
    p_tile = min(64 * 64, n * n)
    syrk_P_read = tiles * p_tile * 8
    syrk_P_write = n * n * 8
    total = hp_P_read + G_write + G_read + syrk_P_read + syrk_P_write
    return {"hp_P_read": hp_P_read, "G_write": G_write, "G_read": G_read, "syrk_P_read": syrk_P_read,
            "syrk_P_write": syrk_P_write, "total": total}


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        name, power, clock = [c.strip() for c in out.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # the numbers are still measured; the card is then unknown
        return {"name": "unknown (%s)" % e, "power_limit": "unknown", "max_sm_clock": "unknown"}


def scenes_for(cap, in_view, n_select):
    from scenelib2_b200 import synth
    out = []
    for i in range(UNIQUE):
        sc = synth.make_scene("C4", stream_id=i, n_frames=RING, n_features=cap)
        sc.n_select = n_select
        if in_view < cap:
            sc.x0 = sc.x0.copy()
            sc.x0[13 + 3 * in_view:] += np.tile([3.0, 0.0, 0.0], cap - in_view)
        out.append(sc)
    return out


def run_case(name, cap, in_view, n_select, B, steps, warmup, reps):
    import torch
    import scenelib2_b200 as sl2
    scenes = scenes_for(cap, in_view, n_select)
    stream = torch.cuda.Stream()
    cfg = sl2.config_for_scene(scenes[0], num_streams=B, frame_slots=RING, max_features=cap,
                               cuda_stream=stream.cuda_stream)
    ctx = sl2.Context(cfg)
    try:
        for s in range(B):
            sl2.load_scene(ctx, s, scenes[s % UNIQUE])
        for k in range(RING):
            ctx.set_frames(k, np.stack([scenes[s % UNIQUE].frames[k] for s in range(B)]))
        for k in range(warmup):
            ctx.step(k % RING)
        ctx.sync()
        ms = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record(stream)
            for k in range(steps):
                ctx.step(k % RING)
            ctx.join()
            e1.record(stream)
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1) / steps)
        ctx.enable_timing(True)
        kt, ku = np.zeros(4), np.zeros(5)
        for k in range(steps):
            ctx.step(k % RING)
            kt += ctx.last_step_times()
            ku += ctx.last_update_times()
        ctx.enable_timing(False)
        kt /= steps
        ku /= steps
        K = [int(((ctx.features(s)["flags"] & 3) == 3).sum()) for s in range(B)]
        nf = [ctx.num_features(s) for s in range(B)]
    finally:
        ctx.close()
    nbytes = sum(update_hbm_bytes(13 + 3 * f, k)["total"] for f, k in zip(nf, K))
    upd_ms = float(ku.sum())
    med = float(np.median(ms))
    return {"case": name, "capacity": cap, "in_view": in_view, "n_select": n_select, "streams": B,
            "measured_mean": float(np.mean(K)), "n": 13 + 3 * cap,
            "frames_per_s": B / (med * 1e-3), "ms_per_step": med, "ms_per_step_reps": ms,
            "step_times_ms": dict(zip(("predict_select", "patch_search", "ekf_update", "cull"), kt.tolist())),
            "update_times_ms": dict(zip(("hp", "chol", "solve", "syrk", "finish"), ku.tolist())),
            "update_hbm_bytes": nbytes, "update_gbs": nbytes / (upd_ms * 1e-3) / 1e9,
            "update_hbm_frac": nbytes / (upd_ms * 1e-3) / 1e9 / HBM_GBS}


def table(rows, c):
    lines = ["Card: %s, power limit %s, max SM clock %s; %d camera streams, C4 frames (320 x 240)."
             % (c["name"], c["power_limit"], c["max_sm_clock"], rows[0]["streams"]), "",
             "| case | capacity | in view / n_select | K (mean) | frames/s | ms/step (spread) | predict | search | "
             "update | cull | hp | chol | solve | syrk | finish | update HBM MB | GB/s (of 3350) |",
             "|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|"]
    for r in rows:
        st, up = r["step_times_ms"], r["update_times_ms"]
        lines.append("| %s | %d | %d / %d | %.1f | %.0f | %.3f (%.3f-%.3f) | %.3f | %.3f | %.3f | %.3f | %.3f | %.3f | "
                     "%.3f | %.3f | %.3f | %.0f | %.0f (%.0f %%) |"
                     % (r["case"], r["capacity"], r["in_view"], r["n_select"], r["measured_mean"], r["frames_per_s"],
                        r["ms_per_step"], min(r["ms_per_step_reps"]), max(r["ms_per_step_reps"]),
                        st["predict_select"], st["patch_search"], st["ekf_update"], st["cull"], up["hp"], up["chol"],
                        up["solve"], up["syrk"], up["finish"], r["update_hbm_bytes"] / 1e6, r["update_gbs"],
                        100 * r["update_hbm_frac"]))
    return "\n".join(lines) + "\n"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=264)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", help="directory for map_capacity.md")
    a = ap.parse_args()
    import scenelib2_b200  # noqa: F401  (the library as build() left it)
    c = card()
    print(json.dumps({"card": c}), flush=True)
    cases = [("anchor", 100, 100, 100)]
    for cap in (128, 192, 256):
        cases += [("%d/stress" % cap, cap, cap, 128), ("%d/ref" % cap, cap, 40, 10)]
    rows = []
    for name, cap, vis, nsel in cases:
        r = run_case(name, cap, vis, nsel, a.streams, a.steps, a.warmup, a.reps)
        r["card"] = c
        print(json.dumps(r), flush=True)
        rows.append(r)
    md = table(rows, c)
    print(md)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        open(os.path.join(a.out, "map_capacity.md"), "w").write(md)


if __name__ == "__main__":
    main()
