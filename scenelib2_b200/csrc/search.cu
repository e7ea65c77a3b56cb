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
//   * while the TMA is in flight the warp evaluates the exact FP64 ellipse predicate for every
//     candidate of the tile and compacts the non-empty vertical strips (SL2_STRIP candidates of
//     one column) into a task list with ballots, so later rounds run with full lanes.
//   * integer phase, per lane = one strip: every image row is read once from shared memory as
//     aligned 32-bit words, byte-aligned with funnel shifts, and feeds all strip candidates that
//     overlap it: Sg0g1 by IDP.4A against the template held in registers, Sg1 / Sg1sq by IDP.4A
//     against 0x01010101 / itself.  All sums are exact int32 like the reference's.
//   * FP64 phase: the score of improc.cpp:99-133 op-for-op with __d*_rn (no FMA contraction,
//     IEEE div / sqrt) so that scores are bit-identical to the x86-64 SSE2 reference build.
//   * arg-min with the reference's tie-break (`corr <= corrmax` => the LAST candidate in
//     urel-major / vrel-minor scan order wins) carried as (score, scan index) through a
//     warp-shuffle reduction.
#include "sl2_common.cuh"
#include "sl2_score.cuh"

namespace {

__device__ __forceinline__ uint32_t smem_u32(const void *p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap *map, uint32_t bar,
                                            int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5}], [%2];" ::"r"(dst),
      "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t phase) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(bar), "r"(phase)
      : "memory");
  return ok != 0;
}

struct Best {
  double corr;
  int idx;
};

// reference acceptance rule folded into an order-independent comparison:
// smaller score wins; equal scores -> the later scan index wins (monoslam.cpp:457, quirk Q3).
__device__ __forceinline__ void consider(Best &b, double corr, int idx) {
  if (corr < b.corr || (corr == b.corr && idx > b.idx)) {
    b.corr = corr;
    b.idx = idx;
  }
}

struct DumpPtrs {
  double *corr;
  double *sd;
  uint8_t *inside;
  int *box;
  int cap;
};

template <int BOX, bool FILTER>
__global__ void __launch_bounds__(SL2_SEARCH_WARPS * 32, FILTER ? (BOX <= 11 ? 4 : 3) : 2)
    search_kernel(const __grid_constant__ CUtensorMap tmap, const Sl2Dev d, const SearchLaunch L,
                  const DumpPtrs dump) {
  constexpr int NW = (BOX + 3) / 4;             // 32-bit words per template row
  constexpr int HALF = (BOX - 1) / 2;
  constexpr int V = SL2_STRIP;
  constexpr uint32_t LASTMASK = (BOX % 4 == 0) ? 0xffffffffu : ((1u << (8 * (BOX % 4))) - 1u);
  extern __shared__ __align__(128) uint8_t smem[];
  pdl_prologue();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int groups = (L.jobs_per_stream + SL2_SEARCH_WARPS - 1) / SL2_SEARCH_WARPS;
  const int sl = blockIdx.x / groups;                       // stream, local to the launch
  const int r = (blockIdx.x % groups) * SL2_SEARCH_WARPS + warp;  // job of this warp
  if (r >= L.jobs_per_stream) return;
  const int job = sl * L.jobs_per_stream + r;
  const int feat = L.job_feat[job];
  if (feat < 0) return;
  const int s = L.stream_lo + sl;

  const int TW = d.tile_w, TH = d.tile_h;
  // TMA needs the box start 16-byte aligned (innermost coordinate * 1 B): the tile is loaded from
  // x & ~15 and is 15 bytes wider than the widest window it serves.
  const int TCW = TW - 15 - BOX + 1, TCH = TH - BOX + 1;
  const int tile_bytes = ((TW * TH + 16 + 127) / 128) * 128;
  const int max_tasks = TCW * ((TCH + V - 1) / V);
  const int list_bytes = ((max_tasks * 4 + 15) / 16) * 16;
  const int vtab_bytes = max(TCH * 16, ((TCW * 4 + 15) / 16) * 16);  // row table of the ellipse test | column intervals
  const int per_warp = ((tile_bytes + list_bytes + 16 + vtab_bytes + 127) / 128) * 128;  // TMA dst: 128 B aligned
  uint8_t *tile = smem + (size_t)warp * per_warp;
  uint32_t *list = reinterpret_cast<uint32_t *>(tile + tile_bytes);
  const uint32_t bar = smem_u32(tile + tile_bytes + list_bytes);
  double2 *vtab = reinterpret_cast<double2 *>(tile + tile_bytes + list_bytes + 16);
  short2 *colrange = reinterpret_cast<short2 *>(vtab);  // FILTER path: per-column candidate interval (same bytes)
  const uint32_t tile_s = smem_u32(tile);

  if (lane == 0) {
    mbar_init(bar, 1);
    fence_barrier_init();
    fence_proxy_async();
  }
  __syncwarp();

  // ---- template into registers, rows zero-padded to 16 bytes in HBM --------------------------
  uint32_t T[BOX][NW];
  {
    const uint32_t *pp =
        reinterpret_cast<const uint32_t *>(d.patches + ((size_t)s * d.Nmax + feat) * (BOX * 16));
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
  // per-feature constants of improc.cpp:99-131
  const double n = (double)(BOX * BOX);
  const double Sg0d = (double)Sg0, Sg0sqd = (double)Sg0sq;
  const double g0bar = div_(Sg0d, n);
  const double varg0 = sub_(div_(Sg0sqd, n), mul_(g0bar, g0bar));
  const double sigmag0 = sqrt_(varg0);
  const double A0 = div_(Sg0sqd, varg0);       // Sg0sqdoub / varg0
  const double g0s = div_(g0bar, sigmag0);     // g0bar / sigmag0
  const double Sg0x2 = mul_(Sg0d, 2.0);        // Sg0doub * 2.0
  // exact integers (< 2^53, so FP64 holds them exactly): n^2 * var = n*Sxx - Sx^2
  const double V0d = fma(n, Sg0sqd, -(Sg0d * Sg0d));
  const float V0f = (float)V0d;
  const bool patch_ok = !(sigmag0 < 10.0);     // kCorrelationSigmaThreshold_ gate on the template
  float bmin = 3.0e38f;                        // running minimum of the approximate score
  const PatchConst pconst = {n, sigmag0, A0, g0s, Sg0x2};

  // ---- search box, monoslam.cpp:416-439 (smoe.cpp:118-147) -----------------------------------
  const double P00 = L.job_puinv[job * 3 + 0], P01 = L.job_puinv[job * 3 + 1],
               P11 = L.job_puinv[job * 3 + 2];
  const double cx = L.job_centre[job * 2 + 0], cy = L.job_centre[job * 2 + 1];
  const int halfwidth =
      __double2int_rz(div_(3.0, sqrt_(sub_(P00, div_(mul_(P01, P01), P11)))));
  const int halfheight =
      __double2int_rz(div_(3.0, sqrt_(sub_(P11, div_(mul_(P01, P01), P00)))));
  const int uc = __double2int_rz(add_(cx, 0.5));
  const int vc = __double2int_rz(add_(cy, 0.5));
  int us = -halfwidth, uf = halfwidth, vs = -halfheight, vf = halfheight;
  if (uc + us - HALF < 0) us = HALF - uc;
  if (uc + uf - HALF > d.W - BOX) uf = d.W - BOX - uc + HALF;
  if (vc + vs - HALF < 0) vs = HALF - vc;
  if (vc + vf - HALF > d.H - BOX) vf = d.H - BOX - vc + HALF;
  const int CW = uf - us + 1, CH = vf - vs + 1;
  const int x0 = uc + us - HALF, y0 = vc + vs - HALF;
  const double twoP01 = mul_(2.0, P01);
  if (dump.box && lane == 0) {
    dump.box[0] = us; dump.box[1] = uf; dump.box[2] = vs; dump.box[3] = vf;
    dump.box[4] = uc; dump.box[5] = vc;
  }

  Best best;
  best.corr = 1000000.0;  // corrmax, monoslam.cpp:444
  best.idx = -1;
  uint32_t phase = 0;
  const int img = L.slot * d.B + s;

  if (CW > 0 && CH > 0) {
    for (int ty0 = 0; ty0 < CH; ty0 += TCH) {
      for (int tx0 = 0; tx0 < CW; tx0 += TCW) {
        const int tcw = min(TCW, CW - tx0), tch = min(TCH, CH - ty0);
        const int xa = (x0 + tx0) & ~15, xoff = (x0 + tx0) & 15;
        if (lane == 0) {
          mbar_expect_tx(bar, (uint32_t)(TW * TH));
          tma_load_3d(tile_s, &tmap, bar, xa, y0 + ty0, img);
        }
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
          const int vbase = vs + ty0;
          for (int cu = lane; cu < tcw; cu += 32) {
            const double du = (double)(us + tx0 + cu);
            const double a = mul_(mul_(P00, du), du);
            const double bcoef = mul_(twoP01, du);
            auto inside = [&](int cv) {
              const double dv = (double)(vbase + cv);
              return add_(add_(a, mul_(bcoef, dv)), mul_(mul_(P11, dv), dv)) < 9.0;
            };
            int lo, hi;
            bool scan = !(P11 > 1e-7) || !(P11 < 1e7);  // degenerate ellipse (or NaN): no shortcut
            if (!scan) {
              const double vx = -bcoef / (2.0 * P11);                   // vertex (approximate arithmetic from here)
              const double disc = bcoef * bcoef - 4.0 * P11 * (a - 9.0);
              const float r = disc > 0.0 ? __fsqrt_rn((float)disc) / (float)(2.0 * P11) : 0.0f;
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
          const double dv = (double)(vs + ty0 + cv);
          vtab[cv] = make_double2(dv, mul_(mul_(P11, dv), dv));
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
            const double du = (double)(us + tx0 + cu);
            const double a = mul_(mul_(P00, du), du);
            const double bcoef = mul_(twoP01, du);
            uint32_t mask = 0;
#pragma unroll
            for (int j = 0; j < V; ++j) {
              const int cv = st * V + j;
              if (cv < tch) {
                const double2 tv = vtab[cv];
                // PuInv(0,0)*u*u + 2*PuInv(0,1)*u*v + PuInv(1,1)*v*v < 9  (monoslam.cpp:453-454)
                const double q = add_(add_(a, mul_(bcoef, tv.x)), tv.y);
                if (q < 9.0 || dump.corr) mask |= (q < 9.0 ? 1u : 0x100u) << j;
              }
            }
            // bits 0..7: inside ellipse; bits 8..15: outside but wanted by the dump mode
            if (mask) entry = (uint32_t)cu | ((uint32_t)st << 8) | (mask << 16);
          }
          const uint32_t bal = __ballot_sync(0xffffffffu, entry != 0);
          if (entry) list[nlist + __popc(bal & ((1u << lane) - 1u))] = entry;
          nlist += __popc(bal);
        }
        }
        __syncwarp();
        while (!mbar_try_wait(bar, phase)) {
        }
        phase ^= 1;

        // ---- strips ------------------------------------------------------------------------
        for (int l0 = 0; l0 < nlist; l0 += 32) {
          const bool has_task = l0 + lane < nlist;
          uint32_t ax[V], a1[V], a2[V];
          float cap[V];           // FILTER: approximate scores of the strip
          int cand0 = 0;          // scan index of candidate j = 0 of the strip
#pragma unroll
          for (int j = 0; j < V; ++j) {
            ax[j] = a1[j] = a2[j] = 0;
            cap[j] = __int_as_float(0x7f800000);  // +inf: not a candidate
          }
          if (has_task) {
            const uint32_t e = list[l0 + lane];
            const int cu = e & 0xff, st = (e >> 8) & 0xff;
            const uint32_t m_in = (e >> 16) & 0xff, m_all = m_in | ((e >> 24) & 0xff);
            const int cv0 = st * V;
            cand0 = (tx0 + cu) * CH + (ty0 + cv0);
            const int cx = cu + xoff;  // byte column of the candidate's window inside the tile
            const int sh = (cx & 3) * 8;
            const uint32_t *wbase = reinterpret_cast<const uint32_t *>(tile) + (cx >> 2);
            const int tw4 = TW >> 2;
#pragma unroll
            for (int rr = 0; rr < V + BOX - 1; ++rr) {
              const int row = min(cv0 + rr, TH - 1);
              const uint32_t *wp = wbase + row * tw4;
              uint32_t w[NW + 1], sw[NW];
#pragma unroll
              for (int k = 0; k <= NW; ++k) w[k] = wp[k];
#pragma unroll
              for (int k = 0; k < NW; ++k) sw[k] = __funnelshift_r(w[k], w[k + 1], sh);
              sw[NW - 1] &= LASTMASK;
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
            auto exact_score = [&](double Sg1d, double Sg1sqd, double Sg0g1d, double &sigmag1) {
              return exact_score_fn(pconst, Sg1d, Sg1sqd, Sg0g1d, &sigmag1);
            };
            if constexpr (FILTER) {
              // The reference's score equals 2 - 2*rho (rho = normalised cross-correlation) up to
              // FP64 rounding (<= 1e-9 for sigma >= 10).  rho is evaluated in FP32 from the EXACT
              // integer moments; only candidates whose approximate score is within kWindow of the
              // running minimum can be the reference's arg-min (or tie with it), and only those go
              // through the exact FP64 chain.  window 1e-5 >= 2 * (FP32 error 1.1e-6 + 1e-9).
              // pass 1: approximate scores of the strip (no FP64 div/sqrt); pass 2, after the warp
              // has agreed on the running minimum: exact chain for the survivors only.
              if (patch_ok) {
                float lmin = bmin;
#pragma unroll
                for (int j = 0; j < V; ++j) {
                  if ((m_in >> j) & 1u) {
                    if constexpr (BOX <= 11) {
                      // n^2 var = n Sxx - Sx^2 and n Sxy - Sx0 Sx1 fit 32-bit integers for n <= 121
                      // (n^2 255^2 < 2^31): exact in the integer pipe, one conversion each to FP32
                      constexpr uint32_t NN = BOX * BOX, T100u = 100u * NN * NN;
                      const uint32_t V1u = NN * a2[j] - a1[j] * a1[j];
                      if (V1u > T100u) {
                        const int N01i = (int)NN * (int)ax[j] - Sg0 * (int)a1[j];
                        const float rho = (float)N01i * rsqrtf(V0f * (float)V1u);
                        cap[j] = fmaf(-2.0f, rho, 2.0f);
                        lmin = fminf(lmin, cap[j]);
                      } else if (V1u == T100u) {
                        cap[j] = -3.0e38f;  // knife edge of sdimage >= 10: the exact chain decides
                      }
                    } else {
                      // n = 225: n Sxx, Sx^2 and both terms of n Sxy - Sx0 Sx1 still fit 32 unsigned bits
                      // (225 * 225 * 255^2 < 2^32); only the last difference needs 64: exact in the integer pipe
                      // (the FP64 pipe runs at half rate and every candidate paid 2 conversions + 2 DFMA + DSETP)
                      constexpr uint32_t NN = BOX * BOX, T100u = 100u * NN * NN;
                      const uint32_t V1u = NN * a2[j] - a1[j] * a1[j];
                      if (V1u > T100u) {
                        const long long N01 = (long long)NN * (long long)ax[j] - (long long)Sg0 * (long long)a1[j];
                        const float rho = (float)N01 * rsqrtf(V0f * (float)V1u);
                        cap[j] = fmaf(-2.0f, rho, 2.0f);
                        lmin = fminf(lmin, cap[j]);
                      } else if (V1u == T100u) {
                        cap[j] = -3.0e38f;  // knife edge of sdimage >= 10: the exact chain decides
                      }
                    }
                  }
                }
                bmin = lmin;
              }
            } else {
#pragma unroll
              for (int j = 0; j < V; ++j) {
                if ((m_all >> j) & 1u) {
                  const double Sg1d = (double)(int)a1[j], Sg1sqd = (double)(int)a2[j],
                               Sg0g1d = (double)(int)ax[j];
                  double sigmag1;
                  double corr = exact_score(Sg1d, Sg1sqd, Sg0g1d, sigmag1);
                  const int ui = tx0 + cu, vi = ty0 + cv0 + j;
                  const int idx = ui * CH + vi;  // urel-major, vrel-minor scan position
                  const bool inside = (m_in >> j) & 1u;
                  if (dump.corr && idx < dump.cap) {
                    dump.corr[idx] = corr;
                    dump.sd[idx] = sigmag1;
                    dump.inside[idx] = inside ? 1 : 0;
                  }
                  if (inside && corr <= 1000000.0 && !(sigmag0 < 10.0) && !(sigmag1 < 10.0))
                    consider(best, corr, idx);  // monoslam.cpp:457-467
                }
              }
            }
          }
          if constexpr (FILTER) {
            // the warp agrees on the running minimum, then only the survivors take the exact chain
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) bmin = fminf(bmin, __shfl_xor_sync(0xffffffffu, bmin, o));
            const float thr = bmin + 1.0e-5f;  // kWindow, see above
#pragma unroll
            for (int j = 0; j < V; ++j) {
              if (cap[j] <= thr) {
                double sg1;
                const double corr = exact_score_fn(pconst, (double)(int)a1[j], (double)(int)a2[j],
                                                   (double)(int)ax[j], &sg1);
                if (corr <= 1000000.0 && !(sg1 < 10.0)) consider(best, corr, cand0 + j);
              }
            }
          }
        }
        __syncwarp();
        fence_proxy_async();  // the next TMA write reuses the tile the warp has just read
      }
    }
  }

  // ---- warp arg-min with the scan-order tie-break -------------------------------------------
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double oc = __shfl_xor_sync(0xffffffffu, best.corr, o);
    const int oi = __shfl_xor_sync(0xffffffffu, best.idx, o);
    consider(best, oc, oi);
  }
  if (lane == 0) {
    int u = -1, v = -1;
    if (best.idx >= 0) {
      u = us + best.idx / CH + uc;
      v = vs + best.idx % CH + vc;
    }
    const uint8_t ok = (best.corr > 0.40) ? 0 : 1;  // monoslam.cpp:472-476
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
  const int TCW = d.tile_w - 15 - d.box + 1, TCH = d.tile_h - d.box + 1;
  const int tile_bytes = ((d.tile_w * d.tile_h + 16 + 127) / 128) * 128;
  const int max_tasks = TCW * ((TCH + SL2_STRIP - 1) / SL2_STRIP);
  const int list_bytes = ((max_tasks * 4 + 15) / 16) * 16;
  const int vtab_bytes = TCH * 16 > ((TCW * 4 + 15) / 16) * 16 ? TCH * 16 : ((TCW * 4 + 15) / 16) * 16;
  return (size_t)SL2_SEARCH_WARPS * (((tile_bytes + list_bytes + 16 + vtab_bytes + 127) / 128) * 128);
}

template <int BOX, bool FILTER>
cudaError_t launch_t(const Sl2Dev &d, const CUtensorMap &tmap, const SearchLaunch &L,
                     const DumpPtrs &dump, cudaStream_t st) {
  const size_t smem = search_smem_bytes(d);
  const int groups = (L.jobs_per_stream + SL2_SEARCH_WARPS - 1) / SL2_SEARCH_WARPS;
  const int grid = groups * L.stream_cnt;
  if (grid <= 0) return cudaSuccess;
  return sl2_launch_kernel(search_kernel<BOX, FILTER>, dim3(grid), dim3(SL2_SEARCH_WARPS * 32), smem, st,
                           sl2_use_pdl(d, L.stream_cnt), tmap, d, L, dump);
}

cudaError_t launch_any(const Sl2Dev &d, const CUtensorMap &tmap, const SearchLaunch &L,
                       const DumpPtrs &dump, cudaStream_t st) {
  const bool exact_all = dump.corr != nullptr;  // score dump: every candidate through the exact chain
  switch (d.box) {
    case 11:
      return exact_all ? launch_t<11, false>(d, tmap, L, dump, st) : launch_t<11, true>(d, tmap, L, dump, st);
    case 15:
      return exact_all ? launch_t<15, false>(d, tmap, L, dump, st) : launch_t<15, true>(d, tmap, L, dump, st);
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace

// once per context (per device): opt the search kernels in to their dynamic shared memory size
cudaError_t sl2_configure_search(const Sl2Dev &d) {
  const int smem = (int)search_smem_bytes(d);
  cudaError_t e = cudaSuccess;
  auto set = [&](const void *f) {
    if (e == cudaSuccess) e = cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  };
  if (d.box == 11) {
    set((const void *)search_kernel<11, true>);
    set((const void *)search_kernel<11, false>);
  } else if (d.box == 15) {
    set((const void *)search_kernel<15, true>);
    set((const void *)search_kernel<15, false>);
  } else {
    e = cudaErrorInvalidValue;
  }
  return e;
}

cudaError_t sl2_launch_search(const Sl2Dev &d, const CUtensorMap &tmap, const SearchLaunch &L,
                              cudaStream_t st) {
  DumpPtrs none = {nullptr, nullptr, nullptr, nullptr, 0};
  return launch_any(d, tmap, L, none, st);
}

cudaError_t sl2_launch_score_map(const Sl2Dev &d, const CUtensorMap &tmap, int stream_id, int slot,
                                 int feat, const double *cp, int *box_dev, double *corr_dev,
                                 double *sd_dev, uint8_t *inside_dev, int cap, cudaStream_t st) {
  // cp = device array: centre(2), puinv(3), then one int job_feat stored after them by the caller
  SearchLaunch L = {};
  L.job_centre = cp;
  L.job_puinv = cp + 2;
  L.job_feat = reinterpret_cast<const int *>(cp + 5);
  L.jobs_per_stream = 1;
  L.stream_lo = stream_id;
  L.stream_cnt = 1;
  L.slot = slot;
  (void)feat;
  DumpPtrs dump = {corr_dev, sd_dev, inside_dev, box_dev, cap};
  return launch_any(d, tmap, L, dump, st);
}
