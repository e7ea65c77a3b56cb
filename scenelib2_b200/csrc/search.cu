// search.cu — patch-correlation feature search on sm_90a.
//
// Replaces MonoSLAM::elliptical_search (monoslam.cpp:401-477) calling correlate2_warning
// (improc/improc.cpp:55-134).  (SearchMultipleOverlappingEllipses::search lives in smoe.cu.)
//
// Design (one WARP per feature, SL2_SEARCH_WARPS features per CTA):
//   * the feature's search window (bounding box of the 3-sigma ellipse + BOXSIZE-1) is staged
//     from the frame in HBM into shared memory by ONE TMA box load (cp.async.bulk.tensor.3d,
//     tensor = [slot*stream][H][W] u8) that completes on a per-warp mbarrier; windows larger
//     than the tile are walked tile by tile.  The TMA unit needs a 16-byte aligned box start
//     so the box is loaded from x & ~15 and is 15 B wider.
//   * while the TMA is in flight the warp reads the template (the feature's stored one, or the job's warped
//     one from SearchLaunch::job_patches: warp.cu) and forms its constants (first tile only), evaluates the exact FP64 ellipse predicate for every candidate of the tile and
//     compacts the non-empty vertical strips (candidates of one column) into a task list with
//     ballots, so later rounds run with full lanes.
//   * integer phase, per lane = one strip: every image row is read once from shared memory as
//     aligned 32-bit words, byte-aligned with funnel shifts, and feeds all strip candidates that
//     overlap it: Sg0g1 by IDP.4A against the template held in registers, the row's Sg1 / Sg1sq
//     by IDP.4A against 0x01010101 / itself.  All sums are exact int32 like the reference's.
//     The filtered kernel runs strips of filter_strip(BOX) candidates and forms each candidate's
//     Sg1 / Sg1sq as the difference of two running sums over the strip's rows; it scores a
//     candidate as soon as its last row is in, so only the candidates whose rows are still
//     being read hold integer sums.
//   * FP64 phase: the score of improc.cpp:99-133 op-for-op with __d*_rn (no FMA contraction,
//     IEEE div / sqrt) so that scores are bit-identical to the x86-64 SSE2 reference build.
//   * arg-min with the reference's tie-break (`corr <= corrmax` => the LAST candidate in
//     urel-major / vrel-minor scan order wins) carried as (score, scan index) through a
//     warp-shuffle reduction.
// Entry points: sl2_patch_search (the staged search of one stream's jobs) and sl2_score_map (one job's scores).
#include "sl2_context.cuh"
#include "sl2_ptx.cuh"
#include "sl2_score.cuh"

using namespace sl2;

namespace {

__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap *map, uint32_t bar,
                                            int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5}], [%2];" ::"r"(dst),
      "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// Per-warp shared memory of search_kernel: the TMA tile, the task list, the mbarrier and the row table of the ellipse
// test | the column intervals.  TMA needs the box start 16-byte aligned (innermost coordinate * 1 B): the tile is
// loaded from x & ~15 and is 15 bytes wider than the widest window it serves.
struct SearchLayout {
  int tcw, tch;                   // candidate columns / rows one tile serves
  int list, bar, vtab, per_warp;  // byte offsets in a warp's slice; slice size (TMA dst: 128 B aligned)
};
__host__ __device__ inline SearchLayout search_layout(int tile_w, int tile_h, int box) {
  SearchLayout l;
  l.tcw = tile_w - 15 - box + 1;
  l.tch = tile_h - box + 1;
  const int tile_bytes = ((tile_w * tile_h + 16 + 127) / 128) * 128;
  const int max_tasks = l.tcw * ((l.tch + SL2_STRIP - 1) / SL2_STRIP);
  const int list_bytes = ((max_tasks * 4 + 15) / 16) * 16;
  const int col_bytes = ((l.tcw * 4 + 15) / 16) * 16;
  const int vtab_bytes = l.tch * 16 > col_bytes ? l.tch * 16 : col_bytes;
  l.list = tile_bytes;
  l.bar = tile_bytes + list_bytes;
  l.vtab = l.bar + 16;
  l.per_warp = ((l.vtab + vtab_bytes + 127) / 128) * 128;
  return l;
}

// every candidate's score, sigma and ellipse flag by scan index (below cap), and the box: written by <BOX, false> only
struct DumpPtrs {
  double *corr;
  double *sd;
  uint8_t *inside;
  int *box;
  int cap;
};

// One image row of a candidate's window: NW + 1 aligned words from the tile, byte-aligned by `sh` bits, bytes past BOX
// cleared.
template <int BOX>
__device__ __forceinline__ void window_row(const uint32_t *wp, int sh, uint32_t (&sw)[(BOX + 3) / 4]) {
  constexpr int NW = (BOX + 3) / 4;
  constexpr uint32_t LASTMASK = (BOX % 4 == 0) ? 0xffffffffu : ((1u << (8 * (BOX % 4))) - 1u);
  uint32_t w[NW + 1];
#pragma unroll
  for (int k = 0; k <= NW; ++k) w[k] = wp[k];
#pragma unroll
  for (int k = 0; k < NW; ++k) sw[k] = __funnelshift_r(w[k], w[k + 1], sh);
  sw[NW - 1] &= LASTMASK;
}

// The filter's approximate score 2 - 2 rho from the exact integer moments (rho in FP32): +inf when the window's sigma
// is below 10 (never accepted), -3e38 on the knife edge sigma == 10 (the exact chain decides).
template <int BOX>
__device__ __forceinline__ float approx_score(uint32_t ax, uint32_t a1, uint32_t a2, int Sg0, float V0f) {
  constexpr uint32_t NN = BOX * BOX, T100u = 100u * NN * NN;
  const uint32_t V1u = NN * a2 - a1 * a1;
  if (V1u > T100u) {
    float num;
    if constexpr (BOX <= 11) {
      // n^2 var = n Sxx - Sx^2 and n Sxy - Sx0 Sx1 fit 32-bit integers for n <= 121
      // (n^2 255^2 < 2^31): exact in the integer pipe, one conversion each to FP32
      num = (float)((int)NN * (int)ax - Sg0 * (int)a1);
    } else {
      // n = 225: n Sxx, Sx^2 and both terms of n Sxy - Sx0 Sx1 still fit 32 unsigned bits
      // (225 * 225 * 255^2 < 2^32); only the last difference needs 64: exact in the integer pipe
      // (the FP64 pipe runs at half rate and every candidate paid 2 conversions + 2 DFMA + DSETP)
      num = (float)((long long)NN * (long long)ax - (long long)Sg0 * (long long)a1);
    }
    const float rho = num * rsqrtf(V0f * (float)V1u);
    return fmaf(-2.0f, rho, 2.0f);
  }
  return V1u == T100u ? -3.0e38f : __int_as_float(0x7f800000);
}

// Candidates per strip task of the filtered search, per template size, from measurements on an H100 (BASELINE.md §6):
// 8 at 11 x 11 (18 image rows per strip), 16 at 15 x 15 (30 rows: 1.9 instead of 2.75 row reads per candidate).
__host__ __device__ constexpr int filter_strip(int box) { return box <= 11 ? 8 : 16; }

// JOBS: the templates come from L.job_patches by job (the planar patch warp, warp.cu), else from d.patches by feature
template <int BOX, bool FILTER, bool JOBS = false>
__global__ void __launch_bounds__(SL2_SEARCH_WARPS * 32, FILTER ? (BOX <= 11 ? 4 : 3) : 2)
    search_kernel(const __grid_constant__ CUtensorMap tmap, const Sl2Dev d, const SearchLaunch L,
                  const DumpPtrs dump) {
  constexpr int NW = (BOX + 3) / 4;             // 32-bit words per template row
  constexpr int HALF = (BOX - 1) / 2;
  constexpr int V = FILTER ? filter_strip(BOX) : SL2_STRIP;  // candidates per strip
  extern __shared__ __align__(128) uint8_t smem[];
  pdl_prologue();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int groups = (L.jobs_per_stream + SL2_SEARCH_WARPS - 1) / SL2_SEARCH_WARPS;
  const int sl = blockIdx.x / groups;                       // stream, local to the launch
  const int r = (blockIdx.x % groups) * SL2_SEARCH_WARPS + warp;  // job of this warp
  if (r >= L.jobs_per_stream) return;
  const int job = sl * L.jobs_per_stream + r;
  // the job's ellipse is read with its feature index (an empty job's values are never used)
  const int feat = L.job_feat[job];
  const double P00 = L.job_puinv[job * 3 + 0], P01 = L.job_puinv[job * 3 + 1],
               P11 = L.job_puinv[job * 3 + 2];
  const double cx = L.job_centre[job * 2 + 0], cy = L.job_centre[job * 2 + 1];
  if (feat < 0) return;
  const int s = L.stream_lo + sl;

  const int TW = d.tile_w, TH = d.tile_h;
  const SearchLayout lay = search_layout(TW, TH, BOX);
  const int TCW = lay.tcw, TCH = lay.tch;
  uint8_t *tile = smem + (size_t)warp * lay.per_warp;
  uint32_t *list = reinterpret_cast<uint32_t *>(tile + lay.list);
  const uint32_t bar = smem_u32(tile + lay.bar);
  double2 *vtab = reinterpret_cast<double2 *>(tile + lay.vtab);
  short2 *colrange = reinterpret_cast<short2 *>(vtab);  // FILTER path: per-column candidate interval (same bytes)
  const uint32_t tile_s = smem_u32(tile);

  if (lane == 0) {
    mbar_init(bar, 1);
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncwarp();

  // ---- search box around the rounded centre ----------------------------------------------------
  const int uc = __double2int_rz(add_(cx, 0.5));
  const int vc = __double2int_rz(add_(cy, 0.5));
  // clamped to the stream's own image, so no window reads past it (the tile loads may: those bytes feed nothing)
  const SearchBox sb = search_box(P00, P01, P11, uc, vc, stream_width(d.cams[s]), stream_height(d.cams[s]), HALF);
  const Ellipse ell = make_ellipse(P00, P01, P11);
  const int CW = sb.cols(), CH = sb.rows();
  const int x0 = uc + sb.us - HALF, y0 = vc + sb.vs - HALF;
  if (!FILTER && lane == 0) {
    dump.box[0] = sb.us; dump.box[1] = sb.uf; dump.box[2] = sb.vs; dump.box[3] = sb.vf;
    dump.box[4] = uc; dump.box[5] = vc;
  }

  // the first tile's TMA goes out before the template is read and its constants are formed: both overlap the load
  const int img = L.slot * d.B + s;
  const auto stage = [&](int tx0, int ty0) {
    if (lane == 0) {
      mbar_expect_tx(bar, (uint32_t)(TW * TH));
      tma_load_3d(tile_s, &tmap, bar, (x0 + tx0) & ~15, y0 + ty0, img);
    }
  };
  if (CW > 0 && CH > 0) stage(0, 0);

  // ---- template into registers, rows zero-padded to 16 bytes in HBM --------------------------
  uint32_t T[BOX][NW];
  {
    const uint32_t *pp = reinterpret_cast<const uint32_t *>(
        JOBS ? L.job_patches + (size_t)job * (BOX * 16) : d.patches + ((size_t)s * d.Nmax + feat) * (BOX * 16));
#pragma unroll
    for (int rr = 0; rr < BOX; ++rr)
#pragma unroll
      for (int k = 0; k < NW; ++k) T[rr][k] = __ldg(pp + rr * 4 + k);
  }
  int Sg0 = 0, Sg0sq = 0;
#pragma unroll
  for (int rr = 0; rr < BOX; ++rr)
#pragma unroll
    for (int k = 0; k < NW; ++k) {
      Sg0 = __dp4a(T[rr][k], 0x01010101u, (uint32_t)Sg0);
      Sg0sq = __dp4a(T[rr][k], T[rr][k], (uint32_t)Sg0sq);
    }
  const PatchConst pconst = patch_const(BOX, Sg0, Sg0sq);
  // exact integers (< 2^53, so FP64 holds them exactly): n^2 * var = n*Sxx - Sx^2
  const double V0d = fma(pconst.n, (double)Sg0sq, -((double)Sg0 * (double)Sg0));
  const float V0f = (float)V0d;
  const bool patch_ok = !(pconst.sigmag0 < 10.0);  // kCorrelationSigmaThreshold_ gate on the template
  float bmin = 3.0e38f;                            // running minimum of the approximate score

  ScanBest best;
  uint32_t phase = 0;

  if (CW > 0 && CH > 0) {
    for (int ty0 = 0; ty0 < CH; ty0 += TCH) {
      for (int tx0 = 0; tx0 < CW; tx0 += TCW) {
        const int tcw = min(TCW, CW - tx0), tch = min(TCH, CH - ty0);
        const int xoff = (x0 + tx0) & 15;
        if (tx0 != 0 || ty0 != 0) stage(tx0, ty0);
        // ---- task list while the TMA is in flight ------------------------------------------
        const int nstrips = (tch + V - 1) / V;
        const int ntask = tcw * nstrips;
        int nlist = 0;
        if constexpr (FILTER) {
          // The candidates of a column form ONE interval of rows: q(v) = (a + b v) + (P11 v) v is a parabola whose
          // values at consecutive integers differ by >= 2 P11 (>= 2e-4 for a box of <= 255 px) once they are 1.5
          // away from the vertex, eleven orders above the rounding error of the three operations, so the exact
          // FP64 predicate (monoslam.cpp:453-454, same operations, same order) flips exactly once on each side.
          // The ends come from a float estimate of the roots and are then MOVED BY THE EXACT PREDICATE until
          // inside(lo), !inside(lo - 1), inside(hi), !inside(hi + 1) hold (an empty column is confirmed on the
          // three rows around the vertex); a column that does not settle in a few moves is scanned row by row.
          // ~5 exact evaluations per column instead of one per candidate.
          const int vbase = sb.vs + ty0;
          // the estimate's 1 / (2 P11), once per tile instead of one FP64 and one FP32 division per column
          const double r2p11 = 1.0 / (2.0 * P11);
          const float r2p11f = (float)r2p11;
          for (int cu = lane; cu < tcw; cu += 32) {
            const Ellipse::Col col = ell.col((double)(sb.us + tx0 + cu));
            auto inside = [&](int cv) { return ell.inside(col, (double)(vbase + cv)); };
            int lo, hi;
            bool scan = !(P11 > 1e-7) || !(P11 < 1e7);  // degenerate ellipse (or NaN): no shortcut
            if (!scan) {
              const double vx = -col.b * r2p11;                         // vertex (approximate arithmetic from here)
              const double disc = col.b * col.b - 4.0 * P11 * (col.a - 9.0);
              const float r = disc > 0.0 ? __fsqrt_rn((float)disc) * r2p11f : 0.0f;
              const float lo_f = fminf(fmaxf(ceilf((float)vx - r) - (float)vbase, -1.0f), (float)tch);
              const float hi_f = fminf(fmaxf(floorf((float)vx + r) - (float)vbase, -1.0f), (float)tch);
              lo = max(0, min(tch - 1, (int)lo_f));
              hi = max(0, min(tch - 1, (int)hi_f));
              if (hi < lo) hi = lo;
              int it = 0;
              while (lo > 0 && it < 16 && inside(lo - 1)) { --lo; ++it; }
              while (lo <= hi && it < 16 && !inside(lo)) { ++lo; ++it; }
              if (it >= 16) {
                scan = true;
              } else if (lo > hi) {  // nothing found from the estimate: the rows around the vertex decide
                const int v0 = max(0, min(tch - 1, __float2int_rn((float)vx) - vbase));
                const int c0 = max(0, v0 - 1), c1 = min(tch - 1, v0 + 1);
                for (int cv = c0; cv <= c1; ++cv)
                  if (inside(cv)) scan = true;  // (never seen: the estimate is good to a fraction of a row)
              } else {
                while (hi < tch - 1 && it < 16 && inside(hi + 1)) { ++hi; ++it; }
                while (hi > lo && it < 16 && !inside(hi)) { --hi; ++it; }
                if (it >= 16) scan = true;
              }
            }
            if (scan) {
              lo = tch;
              hi = -1;
              for (int cv = 0; cv < tch; ++cv)
                if (inside(cv)) {
                  lo = min(lo, cv);
                  hi = cv;
                }
            }
            colrange[cu] = make_short2((short)lo, (short)hi);
          }
          __syncwarp();
          // task list, strip-major and centre-out (the match is expected near the predicted position, so the running
          // minimum of the filter is tight from the first round on; the arg-min carries its scan index, so the
          // visiting order is free); the lanes of a round read consecutive columns of the same image rows
          for (int sk = 0; sk < nstrips; ++sk) {
            const int st = (sk & 1) ? (nstrips - 1) / 2 + (sk + 1) / 2 : (nstrips - 1) / 2 - sk / 2;
            for (int cu0 = 0; cu0 < tcw; cu0 += 32) {
              const int cu = cu0 + lane;
              uint32_t entry = 0;
              if (cu < tcw) {
                const short2 rg = colrange[cu];
                const int jlo = max((int)rg.x - st * V, 0), jhi = min(min((int)rg.y - st * V, V - 1), tch - 1 - st * V);
                if (jlo <= jhi) {
                  // bits 16..31: the strip's candidates inside the ellipse
                  const uint32_t mask = ((1u << (jhi + 1)) - 1u) & ~((1u << jlo) - 1u);
                  entry = (uint32_t)cu | ((uint32_t)st << 8) | (mask << 16);
                }
              }
              const uint32_t bal = __ballot_sync(0xffffffffu, entry != 0);
              if (entry) list[nlist + __popc(bal & ((1u << lane) - 1u))] = entry;
              nlist += __popc(bal);
            }
          }
        } else {
        // the v-only term of the ellipse test, once per candidate row instead of once per candidate
        for (int cv = lane; cv < tch; cv += 32) {
          const double dv = (double)(sb.vs + ty0 + cv);
          vtab[cv] = make_double2(dv, ell.vterm(dv));
        }
        __syncwarp();
        for (int t0 = 0; t0 < ntask; t0 += 32) {
          const int t = t0 + lane;
          uint32_t entry = 0;
          if (t < ntask) {
            // strip-major order: the lanes of a round mostly share the image rows and read
            // consecutive columns => shared-memory reads are broadcasts / conflict-free
            // strips are visited centre-out (the match is expected near the predicted position, so the
            // running minimum of the filter is tight from the first round on and few candidates need the
            // exact chain); the arg-min carries its scan index, so the visiting order is free
            const int sk = t / tcw, cu = t - sk * tcw;
            const int st = (sk & 1) ? (nstrips - 1) / 2 + (sk + 1) / 2 : (nstrips - 1) / 2 - sk / 2;
            const Ellipse::Col col = ell.col((double)(sb.us + tx0 + cu));
            uint32_t mask = 0;
#pragma unroll
            for (int j = 0; j < V; ++j) {
              const int cv = st * V + j;
              if (cv < tch) {
                const double2 tv = vtab[cv];
                mask |= (ell.inside(col, tv.x, tv.y) ? 1u : 0x100u) << j;
              }
            }
            // bits 0..7: inside ellipse; bits 8..15: outside, scored for the dump
            if (mask) entry = (uint32_t)cu | ((uint32_t)st << 8) | (mask << 16);
          }
          const uint32_t bal = __ballot_sync(0xffffffffu, entry != 0);
          if (entry) list[nlist + __popc(bal & ((1u << lane) - 1u))] = entry;
          nlist += __popc(bal);
        }
        }
        __syncwarp();
        mbar_wait(bar, phase);
        phase ^= 1;

        // ---- strips ------------------------------------------------------------------------
        const int tw4 = TW >> 2;
        if constexpr (FILTER) {
          // The reference's score equals 2 - 2*rho (rho = normalised cross-correlation) up to
          // FP64 rounding (<= 1e-9 for sigma >= 10).  rho is evaluated in FP32 from the EXACT
          // integer moments; only candidates whose approximate score is within kWindow of the
          // running minimum can be the reference's arg-min (or tie with it), and only those go
          // through the exact FP64 chain.  window 1e-5 >= 2 * (FP32 error 1.1e-6 + 1e-9).
          // pass 1: approximate scores of the strip (no FP64 div/sqrt), each candidate scored as
          // soon as its last row is in; pass 2, after the warp has agreed on the running minimum:
          // the survivors' integer sums again from the tile, and the exact chain.
          static_assert(V <= 16, "the task entry holds a 16-bit candidate mask");
          static_assert(V >= SL2_STRIP, "the task list is sized for strips of SL2_STRIP candidates");
          for (int l0 = 0; l0 < nlist; l0 += 32) {
            float cap[V];  // approximate scores of the strip, +inf: not a candidate
#pragma unroll
            for (int j = 0; j < V; ++j) cap[j] = __int_as_float(0x7f800000);
            int cv0 = 0, cand0 = 0;  // strip's first candidate row in the tile, its scan index
            int sh = 0;
            const uint32_t *wbase = nullptr;
            if (l0 + lane < nlist && patch_ok) {
              const uint32_t e = list[l0 + lane];
              const int cu = e & 0xff, st = (e >> 8) & 0xff;
              const uint32_t m_in = e >> 16;
              cv0 = st * V;
              cand0 = (tx0 + cu) * CH + (ty0 + cv0);
              const int cx = cu + xoff;  // byte column of the candidate's window inside the tile
              sh = (cx & 3) * 8;
              wbase = reinterpret_cast<const uint32_t *>(tile) + (cx >> 2);
              // candidate j: Sg1 = s1 - h1[j], Sg1sq = s2 - h2[j], with s the running sums of the rows read so far
              // and h their values before row j (every true sum < 2^31: exact in uint32 arithmetic)
              uint32_t ax[V], h1[V], h2[V], s1 = 0, s2 = 0;
              float lmin = bmin;
#pragma unroll
              for (int j = 0; j < V; ++j) ax[j] = 0;
#pragma unroll
              for (int rr = 0; rr < V + BOX - 1; ++rr) {
                uint32_t sw[NW];
                window_row<BOX>(wbase + min(cv0 + rr, TH - 1) * tw4, sh, sw);
                if (rr < V) {
                  h1[rr] = s1;
                  h2[rr] = s2;
                }
#pragma unroll
                for (int k = 0; k < NW; ++k) {
                  s1 = __dp4a(sw[k], 0x01010101u, s1);
                  s2 = __dp4a(sw[k], sw[k], s2);
                }
#pragma unroll
                for (int j = 0; j < V; ++j) {
                  const int t = rr - j;  // template row seen by candidate j in this image row
                  if (t >= 0 && t < BOX) {
#pragma unroll
                    for (int k = 0; k < NW; ++k) ax[j] = __dp4a(sw[k], T[t][k], ax[j]);
                  }
                }
                const int j = rr - (BOX - 1);  // the candidate whose last row this is
                if (j >= 0 && ((m_in >> j) & 1u)) {
                  cap[j] = approx_score<BOX>(ax[j], s1 - h1[j], s2 - h2[j], Sg0, V0f);
                  if (cap[j] > -1.0e38f) lmin = fminf(lmin, cap[j]);
                }
              }
              bmin = lmin;
            }
            // the warp agrees on the running minimum, then only the survivors take the exact chain
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) bmin = fminf(bmin, __shfl_xor_sync(0xffffffffu, bmin, o));
            const float thr = bmin + 1.0e-5f;  // kWindow, see above
            uint32_t surv = 0;
#pragma unroll
            for (int j = 0; j < V; ++j) surv |= (cap[j] <= thr ? 1u : 0u) << j;
            while (surv) {
              const int j = __ffs(surv) - 1;
              surv &= surv - 1;
              uint32_t ax = 0, a1 = 0, a2 = 0;
#pragma unroll
              for (int t = 0; t < BOX; ++t) {
                uint32_t sw[NW];
                window_row<BOX>(wbase + (cv0 + j + t) * tw4, sh, sw);
#pragma unroll
                for (int k = 0; k < NW; ++k) {
                  ax = __dp4a(sw[k], T[t][k], ax);
                  a1 = __dp4a(sw[k], 0x01010101u, a1);
                  a2 = __dp4a(sw[k], sw[k], a2);
                }
              }
              double sg1;
              const double corr = exact_score_fn(pconst, (double)(int)a1, (double)(int)a2, (double)(int)ax, &sg1);
              if (!(sg1 < 10.0)) best.offer(corr, cand0 + j);
            }
          }
        } else {
          for (int l0 = 0; l0 < nlist; l0 += 32) {
            if (l0 + lane >= nlist) continue;
            uint32_t ax[V], a1[V], a2[V];
#pragma unroll
            for (int j = 0; j < V; ++j) ax[j] = a1[j] = a2[j] = 0;
            const uint32_t e = list[l0 + lane];
            const int cu = e & 0xff, st = (e >> 8) & 0xff;
            const uint32_t m_in = (e >> 16) & 0xff, m_all = m_in | ((e >> 24) & 0xff);
            const int cv0 = st * V;
            const int cx = cu + xoff;  // byte column of the candidate's window inside the tile
            const int sh = (cx & 3) * 8;
            const uint32_t *wbase = reinterpret_cast<const uint32_t *>(tile) + (cx >> 2);
#pragma unroll
            for (int rr = 0; rr < V + BOX - 1; ++rr) {
              uint32_t sw[NW];
              window_row<BOX>(wbase + min(cv0 + rr, TH - 1) * tw4, sh, sw);
              uint32_t rs = 0, rq = 0;
#pragma unroll
              for (int k = 0; k < NW; ++k) {
                rs = __dp4a(sw[k], 0x01010101u, rs);
                rq = __dp4a(sw[k], sw[k], rq);
              }
#pragma unroll
              for (int j = 0; j < V; ++j) {
                const int t = rr - j;  // template row seen by candidate j in this image row
                if (t >= 0 && t < BOX) {
#pragma unroll
                  for (int k = 0; k < NW; ++k) ax[j] = __dp4a(sw[k], T[t][k], ax[j]);
                  a1[j] += rs;
                  a2[j] += rq;
                }
              }
            }
            // ---- FP64 score, improc.cpp:99-133 ------------------------------------------------
#pragma unroll
            for (int j = 0; j < V; ++j) {
              if ((m_all >> j) & 1u) {
                const double Sg1d = (double)(int)a1[j], Sg1sqd = (double)(int)a2[j],
                             Sg0g1d = (double)(int)ax[j];
                double sigmag1;
                const double corr = exact_score_fn(pconst, Sg1d, Sg1sqd, Sg0g1d, &sigmag1);
                const int ui = tx0 + cu, vi = ty0 + cv0 + j;
                const int idx = ui * CH + vi;  // scan index
                const bool inside = (m_in >> j) & 1u;
                if (idx < dump.cap) {
                  dump.corr[idx] = corr;
                  dump.sd[idx] = sigmag1;
                  dump.inside[idx] = inside ? 1 : 0;
                }
                if (inside && patch_ok && !(sigmag1 < 10.0)) best.offer(corr, idx);
              }
            }
          }
        }
        __syncwarp();
        fence_proxy_async();  // the next TMA write reuses the tile the warp has just read
      }
    }
  }

  best.warp_reduce();
  if (lane == 0) {
    const int2 uv = best.idx >= 0 ? scan_position(best.idx, CH, uc + sb.us, vc + sb.vs) : make_int2(-1, -1);
    const int u = uv.x, v = uv.y;
    const uint8_t ok = best.found();
    if (L.out_uv) {
      L.out_uv[job * 2 + 0] = u;
      L.out_uv[job * 2 + 1] = v;
    }
    if (L.out_found) L.out_found[job] = ok;
    if (L.out_best) L.out_best[job] = best.corr;
    if (L.scatter_to_features) {
      const size_t f = (size_t)s * d.Nmax + feat;
      d.z_uv[f * 2 + 0] = u;
      d.z_uv[f * 2 + 1] = v;
      d.found[f] = ok;
      d.best[f] = best.corr;
    }
  }
}

size_t search_smem_bytes(const Sl2Dev &d) {
  return (size_t)SL2_SEARCH_WARPS * search_layout(d.tile_w, d.tile_h, d.box).per_warp;
}

// FILTER = false: every candidate through the exact chain, all of it dumped
template <bool FILTER>
cudaError_t launch(const Sl2Dev &d, const CUtensorMap &tmap, const SearchLaunch &L, const DumpPtrs &dump,
                   Sl2Queue q) {
  return sl2_with_box(d.box, [&](auto box) {
    const int groups = (L.jobs_per_stream + SL2_SEARCH_WARPS - 1) / SL2_SEARCH_WARPS;
    const int grid = groups * L.stream_cnt;
    if (grid <= 0) return cudaSuccess;
    constexpr int BOX = decltype(box)::value;
    auto kern = search_kernel<BOX, FILTER>;
    if constexpr (FILTER)  // the dump path never takes job templates
      if (L.job_patches) kern = search_kernel<BOX, true, true>;
    return sl2_launch_kernel(kern, dim3(grid), dim3(SL2_SEARCH_WARPS * 32), search_smem_bytes(d), q,
                             sl2_use_pdl(L.stream_cnt), tmap, d, L, dump);
  });
}

}  // namespace

// once per context (per device): opt the search kernels in to their dynamic shared memory size
cudaError_t sl2_configure_search(const Sl2Dev &d) {
  const int smem = (int)search_smem_bytes(d);
  return sl2_with_box(d.box, [&](auto box) {
    constexpr int BOX = decltype(box)::value;
    cudaError_t e = cudaFuncSetAttribute(search_kernel<BOX, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(search_kernel<BOX, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(search_kernel<BOX, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    return e;
  });
}

cudaError_t sl2_launch_search(const Sl2Dev &d, const CUtensorMap &tmap, const SearchLaunch &L, Sl2Queue q) {
  return launch<true>(d, tmap, L, DumpPtrs{}, q);
}

// one job (centre, puinv, feature index: device arrays of 2, 3 and 1) with every candidate's score dumped
static cudaError_t sl2_launch_score_map(const Sl2Dev &d, const CUtensorMap &tmap, int stream_id, int slot,
                                        const double *centre_dev, const double *puinv_dev, const int *feat_dev,
                                        int *box_dev, double *corr_dev, double *sd_dev, uint8_t *inside_dev, int cap,
                                        Sl2Queue q) {
  SearchLaunch L = {};
  L.job_centre = centre_dev;
  L.job_puinv = puinv_dev;
  L.job_feat = feat_dev;
  L.jobs_per_stream = 1;
  L.stream_lo = stream_id;
  L.stream_cnt = 1;
  L.slot = slot;
  const DumpPtrs dump = {corr_dev, sd_dev, inside_dev, box_dev, cap};
  return launch<false>(d, tmap, L, dump, q);
}

extern "C" {

int sl2_patch_search(sl2_ctx *c, int32_t s, int32_t slot, int32_t n, const int32_t *feat_index,
                     const double *centre, const double *PuInv3, int32_t *u, int32_t *v,
                     uint8_t *found, double *best) {
  if (n > 0 && !feat_index) return fail(c, SL2_ERR_ARG, "sl2_patch_search: feat_index is null");
  if (bad_stream(c, s) || bad_slot(c, slot) || n < 0 || !centre || !PuInv3)
    return fail(c, SL2_ERR_ARG, "patch search: bad argument");
  if (n == 0) return SL2_OK;
  int rc = check_feature_indices(c, s, feat_index, n, "patch search: feature index out of range");
  if (rc) return rc;
  const size_t N = n;
  Stage ce{STAGE_IN, 16 * N, centre}, pu{STAGE_IN, 24 * N, PuInv3}, fe{STAGE_IN, 4 * N, feat_index},
      uv{STAGE_OUT, 8 * N}, fd{STAGE_OUT, N}, be{STAGE_OUT, 8 * N};
  rc = staged_call(c, {&ce, &pu, &fe, &uv, &fd, &be}, [] {}, [&] {
    SearchLaunch L = {};
    L.job_centre = ce.dev<double>();
    L.job_puinv = pu.dev<double>();
    L.job_feat = fe.dev<int>();
    L.jobs_per_stream = n;
    L.stream_lo = s;
    L.stream_cnt = 1;
    L.slot = slot;
    L.out_uv = uv.dev<int>();
    L.out_found = fd.d;
    L.out_best = be.dev<double>();
    L.scatter_to_features = 0;
    CU_TRY(c, sl2_launch_search(c->d, c->tmap, L, queue(c)));
    return SL2_OK;
  });
  if (rc) return rc;
  for (int i = 0; i < n; ++i) {
    if (u) u[i] = uv.host<int>()[2 * i];
    if (v) v[i] = uv.host<int>()[2 * i + 1];
    if (found) found[i] = fd.h[i];
    if (best) best[i] = be.host<double>()[i];
  }
  return SL2_OK;
}

int sl2_score_map(sl2_ctx *c, int32_t s, int32_t slot, int32_t feat, const double *centre,
                  const double *PuInv3, int32_t *box6, double *corr, double *sd_image,
                  uint8_t *inside, size_t cap) {
  if (bad_stream(c, s) || bad_slot(c, slot) || !centre || !PuInv3 || !box6)
    return fail(c, SL2_ERR_ARG, "sl2_score_map: bad argument");
  int rc = check_feature_indices(c, s, &feat, 1, "sl2_score_map: bad feature index");
  if (rc) return rc;
  Stage ce{STAGE_IN, 16, centre}, pu{STAGE_IN, 24, PuInv3}, fe{STAGE_IN, 4, &feat}, bx{STAGE_OUT, 24},
      co{STAGE_OUT, 8 * cap}, sd{STAGE_OUT, 8 * cap}, in{STAGE_OUT, cap};
  rc = staged_call(c, {&ce, &pu, &fe, &bx, &co, &sd, &in}, [] {}, [&] {
    CU_TRY(c, cudaMemsetAsync(bx.d, 0xff, in.d + cap - bx.d, c->stream));  // NaN / 0xff fill of every output
    CU_TRY(c, sl2_launch_score_map(c->d, c->tmap, s, slot, ce.dev<double>(), pu.dev<double>(), fe.dev<int>(),
                                   bx.dev<int>(), co.dev<double>(), sd.dev<double>(), in.d, (int)cap, queue(c)));
    return SL2_OK;
  });
  if (rc) return rc;
  memcpy(box6, bx.h, 24);
  if (corr) memcpy(corr, co.h, 8 * cap);
  if (sd_image) memcpy(sd_image, sd.h, 8 * cap);
  if (inside) memcpy(inside, in.h, cap);
  return SL2_OK;
}

}  // extern "C"
