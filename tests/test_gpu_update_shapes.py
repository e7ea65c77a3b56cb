"""The batched EKF update (sl2_launch_update, update.cu) with maps of different sizes in one context.

sl2_launch_update picks its launch shapes from the number of camera streams in the launch and the SM count: one CTA
per stream for H P (and the software-pipelined upd_hp2 when a state column fits one thread) from 2 streams per SM on,
upd_solve walking the column groups of a stream in one CTA from 1 stream per SM on, the upd_solve instantiation from
the capacity.  Inside a launch the per-stream bounds (m, n, the FULL switch of upd_solve, the ragged row blocks of
upd_hp / upd_hp2 / upd_chol, the syrk tile that carries the nu column) differ from CTA to CTA.  Every capacity below is
run with a set of stream variants whose measurement count K and map size nf put those bounds on their edges, in
every launch regime, and compared with the CPU oracle at every step; results must not depend on the launch shape.
"""
import math

import pytest

from gpu_util import record_oracle, run_regimes, update_variant

T = 12              # frames per run; the bad features are culled by the 10th step
SNAP_STEPS = (8, T - 1)   # compared across regimes: the last step before the cull, and the last step

# capacity -> variants (nf, bad, out_of_view, the edge the variant exists for); m = 2 K, n = 13 + 3 nf, K = nf - bad
VARIANTS = {
    32: [(32, 0, False, "m = 64 = 16 NP"),
         (25, 0, False, "m8 = 56 = 16 NP - 8: FULL with a ragged last tile"),
         (24, 0, False, "m8 = 48: just below FULL"),
         (17, 0, False, "n = 64: nu alone in the second syrk tile"),
         (1, 0, False, "K = 1"),
         (3, 3, False, "K = 0, culled to an empty map"),
         (32, 7, False, "cull: n 109 -> 88"),
         (20, 0, True, "out of view: K = 0 with nf > 0"),
         (30, 0, False, "K mod 4 = 2"),
         (31, 0, False, "K mod 4 = 3"),
         (11, 0, False, "two panels, one syrk tile")],
    56: [(56, 0, False, "m = 112 = 16 NP"),
         (49, 0, False, "m8 = 104: FULL edge"),
         (48, 0, False, "m8 = 96: just below FULL"),
         (38, 0, False, "n + 1 = 128: nu is the last column of a tile"),
         (41, 0, False, "K mod 4 = 1, non-FULL"),
         (56, 9, False, "cull, K mod 4 = 3")],
    80: [(80, 0, False, "m = 160 = 16 NP"),
         (73, 0, False, "m8 = 152: FULL edge"),
         (72, 0, False, "m8 = 144: just below FULL"),
         (59, 0, False, "K mod 4 = 3"),
         (38, 0, False, "K mod 4 = 2, n + 1 = 128"),
         (80, 11, False, "cull, K mod 4 = 1"),
         (3, 3, False, "K = 0, culled to an empty map")],
    102: [(102, 0, False, "n + 1 = 320: one state column per hp2 thread, all threads"),
          (97, 0, False, "m8 = 200: FULL with a ragged last tile"),
          (96, 0, False, "m8 = 192: walk, non-FULL"),
          (81, 0, False, "n = 256"),
          (99, 0, False, "m mod 8 = 6: ragged hp2 block"),
          (101, 0, False, "m mod 8 = 2: ragged hp2 block"),
          (102, 5, False, "cull"),
          (1, 0, False, "K = 1")],
    104: [(104, 0, False, "m = 208 = 16 NP, two column chunks"),
          (103, 0, False, "n = 322: two column chunks"),
          (97, 0, False, "one column chunk"),
          (104, 7, False, "cull: n 325 -> 304 crosses 320")],
    128: [(128, 0, False, "m = 256: 16 panels"),
          (127, 0, False, "ragged last panel"),
          (105, 0, False, "14 panels"),
          (49, 0, False, "reaches panel 6: second staging generation"),
          (40, 0, False, "reaches REUSE = 4 only"),
          (128, 31, False, "cull: n 397 -> 304"),
          (3, 3, False, "K = 0, culled to an empty map")],
}


def designed(v):
    """(K, nf before the cull, nf after it) of a variant."""
    nf, bad, out, _ = v
    return (0 if out else nf - bad), nf, nf - bad


def variant_scenes(cap):
    return [update_variant(cap, nf, bad, out, stream_id=i, n_frames=T)
            for i, (nf, bad, out, _) in enumerate(VARIANTS[cap])]


# ---- Python mirror of sl2_launch_update's decisions -----------------------------------------------------------
def launch_shape(cap, cnt, nsm):
    """What sl2_launch_update (update.cu) launches for `cnt` streams of capacity `cap` on `nsm` SMs."""
    keven = (cap + 1) & ~1
    hp_all = (2 * keven + 15) // 16                           # hp_all  (1 up to 8 features)
    hp_one = cnt >= 2 * nsm or hp_all == 1                    # hp_blocks = 1
    piped = hp_one and 13 + 3 * cap <= 320                    # upd_hp2
    panels = (2 * keven + 15) // 16                           # solve_kernel: panels of S at capacity
    NP = next(p for p in (4, 7, 10, 13, 16) if panels <= p)   # solve_kernel: the NP instantiation
    walk = NP <= 13 and cnt >= nsm                            # walk
    return dict(hp_one=hp_one, piped=piped, NP=NP, walk=walk)


def shape_label(L):
    return "hp %s%s, solve NP=%d %s" % ("1 CTA/stream" if L["hp_one"] else "spread",
                                         " hp2" if L["piped"] else "", L["NP"], "walk" if L["walk"] else "slabs")


def stream_edges(L, K, nf):
    """Edges of the update kernels one stream of shape (K, nf) reaches in a launch of shape L."""
    if K == 0:
        return {"K = 0 with nf > 0" if nf else "K = 0, empty map"}
    m, n, NP = 2 * K, 13 + 3 * nf, L["NP"]
    m8 = (m + 7) & ~7
    full = NP <= 13 and m8 >= 16 * NP - 8                     # upd_solve_kernel: full (SPLIT == NP below 16 panels)
    e = {"solve NP=%d" % NP,
         "solve %s %s" % ("walk" if L["walk"] else "slabs", "FULL" if full else "non-FULL"),
         "hp 1 CTA/stream" if L["hp_one"] else "hp spread"}
    if L["piped"]:
        e.add("hp2 K mod 4 = %d" % (K % 4))
        if m % 8:
            e.add("hp2 ragged last block")
    elif L["hp_one"] and n > 320:
        e.add("hp 1 CTA/stream, two column chunks")           # upd_hp_kernel: nch = 2
    if full and m8 == 16 * NP - 8:
        e.add("solve FULL, ragged last tile")
    if NP == 16 and m > 16 * 6:
        e.add("solve NP=16 second staging generation")        # SolveLayout<16>::SPLIT = 6
    elif NP == 16 and m > 16 * 4:
        e.add("solve NP=16 reaches REUSE only")               # SolveLayout<16>::REUSE = 4
    if n % 64 == 0:
        e.add("syrk nu alone in its tile")
    if (n + 1) % 64 == 0:
        e.add("syrk nu last column of a tile")
    return e


def regimes(cap, nsm, U):
    """(name, B, step groups, launches as (stream_lo, count)) for one capacity."""
    return [("small", U, 1, [(0, U)]),
            ("walk", nsm, 1, [(0, nsm)]),
            ("batch", 2 * nsm, 1, [(0, 2 * nsm)]),
            ("groups", 2 * nsm, 2, [(0, nsm), (nsm, nsm)])]


REQUIRED_EDGES = (["hp spread", "hp 1 CTA/stream", "hp2 ragged last block", "hp 1 CTA/stream, two column chunks"] +
                  ["hp2 K mod 4 = %d" % r for r in range(4)] +
                  ["solve NP=%d" % p for p in (4, 7, 10, 13, 16)] +
                  ["solve %s %s" % (w, f) for w in ("walk", "slabs") for f in ("FULL", "non-FULL")] +
                  ["solve FULL, ragged last tile", "solve NP=16 second staging generation",
                   "solve NP=16 reaches REUSE only", "syrk nu alone in its tile", "syrk nu last column of a tile",
                   "K = 0 with nf > 0", "K = 0, empty map", "launch at stream_lo = nsm", "cull shrinks n in the run"])


def coverage(nsm):
    """Rows (cap, regime, B, launch labels, edges reached) and edge -> number of (cap, regime, variant) hits."""
    rows, hits = [], {e: 0 for e in REQUIRED_EDGES}
    for cap, vs in VARIANTS.items():
        U = len(vs)
        for name, B, groups, launches in regimes(cap, nsm, U):
            reached, labels = set(), []
            for lo, cnt in launches:
                L = launch_shape(cap, cnt, nsm)
                labels.append(shape_label(L))
                if lo == nsm:
                    reached.add("launch at stream_lo = nsm")
                for v in vs:
                    K, nf0, nf1 = designed(v)
                    ev = stream_edges(L, K, nf0) | stream_edges(L, K, nf1)
                    if nf1 < nf0:
                        ev.add("cull shrinks n in the run")
                    reached |= ev
                    for e in ev:
                        hits[e] = hits.get(e, 0) + 1
            hits["launch at stream_lo = nsm"] += "launch at stream_lo = nsm" in reached
            rows.append((cap, name, B, sorted(set(labels)), reached))
    return rows, hits


# ---- CPU: the variants still reach their edges ---------------------------------------------------------------
def test_variants_reach_every_update_shape(oracle):
    """Each variant has its designed K at every step and loses exactly its bad features at the 10th step, and the
    capacity x regime list reaches every launch decision and kernel edge of the update (evaluated for the SM counts
    of the H100 SXM5 and PCIe: the regimes are defined relative to the SM count)."""
    for cap, vs in VARIANTS.items():
        assert math.gcd(len(vs), 5) == 1, cap
        assert max(v[0] for v in vs) == cap, cap            # some stream fills the capacity
        if 13 + 3 * cap <= 320:                              # every hp2 ragged-block case
            assert {designed(v)[0] % 4 for v in vs if designed(v)[0]} == {0, 1, 2, 3}, cap
        traj = record_oracle(oracle, variant_scenes(cap), T, states=False)
        for v, rec in zip(vs, traj):
            K, nf0, nf1 = designed(v)
            sel = [int((r["f"]["flags"] & 1).sum()) for r in rec]
            found = [int(((r["f"]["flags"] & 3) == 3).sum()) for r in rec]
            assert found == [K] * T and sel[0] == (0 if v[2] else nf0), (cap, v, sel[0], found)
            assert [r["nf"] for r in rec] == [nf0] * 9 + [nf1] * (T - 9), (cap, v)
    for nsm in (132, 114):
        assert max(len(vs) for vs in VARIANTS.values()) < nsm
        rows, hits = coverage(nsm)
        if nsm == 132:
            for cap, name, B, labels, reached in rows:
                print("\ncap %3d %-11s B = %3d  %s\n    %s" % (cap, name, B, " | ".join(labels),
                                                             ", ".join(sorted(reached))), end="")
            print("\n(capacity, regime, variant) hits per edge at nsm = 132:")
            for e in REQUIRED_EDGES:
                print("  %-42s %4d" % (e, hits[e]))
        missing = [e for e in REQUIRED_EDGES if hits[e] == 0]
        assert not missing, (nsm, missing)




# ---- GPU: every regime against the oracle and against each other ---------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cap", sorted(VARIANTS))
def test_update_shapes_against_oracle(oracle, cap):
    """All regimes of one capacity: every checked stream against the oracle at every step, every stream bit-identical
    to the first stream of its variant, and every variant bit-identical across the regimes (the kernels' per-element
    arithmetic does not depend on the grid: hp vs hp2, spread vs one CTA, slabs vs walk, one launch vs two groups)."""
    import torch

    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    scenes = variant_scenes(cap)
    U = len(scenes)
    assert U < nsm
    traj = record_oracle(oracle, scenes, T)
    for v, rec in zip(VARIANTS[cap], traj):                  # the run is the designed one
        assert int(((rec[0]["f"]["flags"] & 3) == 3).sum()) == designed(v)[0], v
    regs = regimes(cap, nsm, U)
    _, worst = run_regimes(scenes, cap, [r[:3] for r in regs], T, SNAP_STEPS, traj)
    for name, B, _, launches in regs:
        labels = sorted({shape_label(launch_shape(cap, cnt, nsm)) for _, cnt in launches})
        print("\ncap %3d %-11s B = %3d  %-44s worst state %.2e  covariance %.2e"
              % (cap, name, B, " | ".join(labels), *worst[name]))
