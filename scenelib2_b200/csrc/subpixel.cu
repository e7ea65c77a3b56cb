// subpixel.cu — the sub-pixel refinement of the patch search's matches on sm_90a, between the search and the match
// consensus of the fused step: a quadratic fit of the search's own correlation score over the 3 x 3 integer positions
// around each match.  One warp per job.  Semantics: include/sl2b200.h, sl2_set_stream_subpixel (which, with
// sl2_get_stream_subpixel, ends this file).
//
// A job of an on stream whose search found a match (found == 1) at (u, v):
//   c(a, b), a, b in {-1, 0, 1}: exact_score_fn (sl2_score.cuh, the search's own chain) of the window centred at
//   (u + a, v + b) against the template the search used (the warped one when the warp is on), with the integer sums
//   the search forms, so c(0, 0) is the search's best bit for bit;
//   every operation one correctly rounded, never-fused op (rd), in this order (tests/subpixel_ref.py restates it):
//     g_u = (c(1,0) - c(-1,0)) * 0.5;  g_v = (c(0,1) - c(0,-1)) * 0.5;
//     h_uu = (c(1,0) + c(-1,0)) - 2 c(0,0);  h_vv = (c(0,1) + c(0,-1)) - 2 c(0,0);
//     h_uv = ((c(1,1) - c(1,-1)) - (c(-1,1) - c(-1,-1))) * 0.25;  det = h_uu h_vv - h_uv h_uv;
//     du = (h_uv g_v - h_vv g_u) / det;  dv = (h_uv g_u - h_uu g_v) / det;
//   refined iff the nine windows lie inside the stream's image, no window has sigma_g1 < 10, h_uu > 0, det > 0 and
//   du, dv are in [-0.5, 0.5] (NaN: never); then z = (u + du, v + dv), else z = (u, v).
// Shape: the warp stages the (B + 2) x (B + 2) image region and the template in shared memory; lane a * 3 + b (< 9)
// forms the sums of window (a - 1, b - 1) and its score; lane 0 fits.
#include <cmath>

#include "sl2_context.cuh"
#include "sl2_score.cuh"

using namespace sl2;

namespace {

constexpr int SUBPIX_WARPS = 4;

template <int BOX>
__global__ void __launch_bounds__(32 * SUBPIX_WARPS) subpixel_kernel(const Sl2Dev d, const SubpixelLaunch L) {
  constexpr int HALF = (BOX - 1) / 2, R = BOX + 2;
  __shared__ uint8_t region[SUBPIX_WARPS][R * R];
  __shared__ uint8_t tpl[SUBPIX_WARPS][BOX * BOX];
  pdl_prologue();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int job = blockIdx.x * SUBPIX_WARPS + warp;  // local to the launch
  if (job >= L.stream_cnt * d.Nmax) return;
  const int s = L.stream_lo + job / d.Nmax;
  if (!L.on[s]) return;
  const int feat = d.job_feat[(size_t)L.stream_lo * d.Nmax + job];
  if (feat < 0) return;
  const size_t f = (size_t)s * d.Nmax + feat;
  const int u = d.z_uv[f * 2 + 0], v = d.z_uv[f * 2 + 1];
  const int W = stream_width(d.cams[s]), H = stream_height(d.cams[s]);
  double zu = (double)u, zv = (double)v;
  bool refined = false;
  // warp-uniform: one job per warp
  if (d.found[f] == 1 && u - 1 - HALF >= 0 && u + 1 + HALF <= W - 1 && v - 1 - HALF >= 0 && v + 1 + HALF <= H - 1) {
    const uint8_t *img = d.frames + (size_t)(L.slot * d.B + s) * d.H * d.pitch;
    const int x0 = u - 1 - HALF, y0 = v - 1 - HALF;
    for (int e = lane; e < R * R; e += 32) region[warp][e] = img[(size_t)(y0 + e / R) * d.pitch + x0 + e % R];
    const uint8_t *tp = L.job_patches ? L.job_patches + (size_t)job * (BOX * 16) : d.patches + f * (BOX * 16);
    for (int e = lane; e < BOX * BOX; e += 32) tpl[warp][e] = tp[(e / BOX) * 16 + e % BOX];
    __syncwarp();
    double c = 0.0, sg1 = 0.0;
    if (lane < 9) {
      const int a = lane / 3, b = lane % 3;  // window centred at (u + a - 1, v + b - 1)
      int Sg0 = 0, Sg0sq = 0, Sg1 = 0, Sg1sq = 0, Sg0g1 = 0;
      for (int r = 0; r < BOX; ++r)
        for (int k = 0; k < BOX; ++k) {
          const int t = tpl[warp][r * BOX + k], g = region[warp][(b + r) * R + a + k];
          Sg0 += t;
          Sg0sq += t * t;
          Sg1 += g;
          Sg1sq += g * g;
          Sg0g1 += t * g;
        }
      const PatchConst pc = patch_const(BOX, Sg0, Sg0sq);
      c = exact_score_fn(pc, (double)Sg1, (double)Sg1sq, (double)Sg0g1, &sg1);
    }
    const bool gated = __ballot_sync(0xffffffffu, lane < 9 && sg1 < 10.0) != 0u;
    double cs[9];
#pragma unroll
    for (int o = 0; o < 9; ++o) cs[o] = __shfl_sync(0xffffffffu, c, o);
    if (!gated) {
      // cs[(a + 1) * 3 + (b + 1)] = c(a, b)
      const rd c00(cs[4]), cp0(cs[7]), cm0(cs[1]), c0p(cs[5]), c0m(cs[3]);
      const rd cpp(cs[8]), cpm(cs[6]), cmp(cs[2]), cmm(cs[0]);
      const rd gu = (cp0 - cm0) * rd(0.5), gv = (c0p - c0m) * rd(0.5);
      const rd huu = (cp0 + cm0) - rd(2.0) * c00, hvv = (c0p + c0m) - rd(2.0) * c00;
      const rd huv = ((cpp - cpm) - (cmp - cmm)) * rd(0.25);
      const rd det = huu * hvv - huv * huv;
      if (huu.v > 0.0 && det.v > 0.0) {
        const rd du = (huv * gv - hvv * gu) / det, dv = (huv * gu - huu * gv) / det;
        if (du.v >= -0.5 && du.v <= 0.5 && dv.v >= -0.5 && dv.v <= 0.5) {
          zu = (rd(zu) + du).v;
          zv = (rd(zv) + dv).v;
          refined = true;
        }
      }
    }
  }
  if (lane == 0) {
    L.out.z[f * 2 + 0] = zu;
    L.out.z[f * 2 + 1] = zv;
    L.out.refined[f] = refined ? 1 : 0;
  }
}

}  // namespace

cudaError_t sl2_launch_subpixel(const Sl2Dev &d, const SubpixelLaunch &L, Sl2Queue q) {
  const int jobs = L.stream_cnt * d.Nmax;
  if (jobs <= 0) return cudaSuccess;
  return sl2_with_box(d.box, [&](auto box) {
    return sl2_launch_kernel(subpixel_kernel<decltype(box)::value>, dim3((jobs + SUBPIX_WARPS - 1) / SUBPIX_WARPS),
                             dim3(32 * SUBPIX_WARPS), 0, q, sl2_use_pdl(L.stream_cnt), d, L);
  });
}

namespace sl2 {

Sl2Subpix subpixel_args(const sl2_ctx *c, int lo, int cnt) {
  if (!c->subpix_buf || !any_stream(c, lo, cnt, [](const StreamOptions &o) { return o.subpixel != 0; })) return {};
  return c->subpix_dev;
}

int subpixel_streams(sl2_ctx *c, int slot, int lo, int cnt, const uint8_t *job_patches, Sl2Queue q) {
  SubpixelLaunch L = {};
  L.stream_lo = lo;
  L.stream_cnt = cnt;
  L.slot = slot;
  L.on = c->subpix_on_dev;
  L.job_patches = job_patches;
  L.out = c->subpix_dev;
  CU_TRY(c, sl2_launch_subpixel(c->d, L, q));
  return SL2_OK;
}

int subpixel_forget(sl2_ctx *c, int lo, int cnt) {
  if (c->subpix_buf && cnt > 0)
    CU_TRY(c, cudaMemsetAsync(c->subpix_dev.refined + (size_t)lo * c->d.Nmax, 0, (size_t)cnt * c->d.Nmax, c->stream));
  return SL2_OK;
}

}  // namespace sl2

extern "C" {

int sl2_set_stream_subpixel(sl2_ctx *c, int32_t s, int32_t on) {
  if (bad_stream(c, s) || (on != 0 && on != 1)) return fail(c, SL2_ERR_ARG, "sl2_set_stream_subpixel: bad argument");
  if (on && !c->subpix_buf) {
    const size_t BN = (size_t)c->d.B * c->d.Nmax;
    Sl2Subpix &sp = c->subpix_dev;
    const int rc = alloc_sections(
        c, c->subpix_buf, {{&sp.z, BN * 2 * sizeof(double)}, {&sp.refined, BN}, {&c->subpix_on_dev, (size_t)c->d.B}});
    if (rc) return rc;
  }
  if (c->subpix_buf) {
    CU_TRY(c, cudaMemsetAsync(c->subpix_on_dev + s, on, 1, c->stream));
    // the refined flags describe steps the stream ran with the refinement on, and an off stream has none
    const int rc = subpixel_forget(c, s, 1);
    if (rc) return rc;
  }
  c->opt[s].subpixel = (uint8_t)on;
  return SL2_OK;
}

int sl2_get_stream_subpixel(sl2_ctx *c, int32_t s, int32_t *on) {
  if (bad_stream(c, s) || !on) return fail(c, SL2_ERR_ARG, "sl2_get_stream_subpixel: bad argument");
  *on = c->opt[s].subpixel;
  return SL2_OK;
}

}  // extern "C"
