// warp.cu — the planar patch warp on sm_90a: each measurement job's template warped to the predicted viewpoint before
// the patch search (Davison, Reid, Molton, Stasse, PAMI 2007; Molton, Davison, Reid, BMVC 2004).  Semantics:
// include/sl2b200.h, sl2_set_stream_warp (which, with sl2_get_stream_warp and sl2_warp_templates, ends this file).
//
// The surface around feature i is taken as planar, through y_i with the world normal nW = xp_org[i][0:3] - y_i.  Output
// pixel (a, b) of the warped template at pose xp is the point of that plane the camera at xp sees at h + (b - HALF,
// a - HALF), projected into the camera at xp_org[i] and sampled bilinearly from the stored template there
// (patch_warp_setup, patch_warp_source, patch_sample in sl2_model.cuh: every operation one correctly rounded,
// never-fused op in the order written; tests/warp_ref.py restates them op for op, tests/warp_truth.py states the
// geometry from its definition).
// Shape: one warp per job, WARP_WARPS jobs per CTA; the lanes take the bytes of the row-padded output (col < BOX is a
// pixel, the rest the zero padding); the stored template is staged in shared memory.  A stream whose setting is off
// gets its stored templates copied, so the search reads every job of the launch from one place.
#include <cmath>

#include "sl2_context.cuh"
#include "sl2_model.cuh"

using namespace sl2;

namespace {

#define WARP_WARPS 4

template <int BOX>
__global__ void __launch_bounds__(32 * WARP_WARPS) warp_kernel(const Sl2Dev d, const WarpLaunch L) {
  pdl_prologue();
  constexpr int HALF = (BOX - 1) / 2, BYTES = BOX * 16, PER = (BYTES + 31) / 32;
  __shared__ __align__(16) uint8_t tpl[WARP_WARPS][BYTES];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int job = blockIdx.x * WARP_WARPS + w;
  if (job >= L.stream_cnt * L.jobs_per_stream) return;
  const int feat = L.job_feat[job];
  if (feat < 0) {
    if (L.valid && lane == 0) L.valid[job] = 0;
    return;
  }
  const int s = L.stream_lo + job / L.jobs_per_stream;
  const size_t g = (size_t)s * d.Nmax + feat;
  const uint32_t *src32 = reinterpret_cast<const uint32_t *>(d.patches + g * BYTES);
  uint32_t *t32 = reinterpret_cast<uint32_t *>(tpl[w]);
  for (int k = lane; k < BYTES / 4; k += 32) t32[k] = src32[k];
  __syncwarp();
  uint8_t *out = L.out + (size_t)job * BYTES;
  bool ok = !L.on || L.on[s];
  uint8_t res[PER];
  if (ok) {
    const double *xp = L.xp ? L.xp : d.x + (size_t)s * d.ld;
    const double *xo = d.xp_org + g * 7;
    const double *cam = d.cams[s].cam;
    const double *yp = d.x + (size_t)s * d.ld + SL2_NXV + 3 * feat;
    const rd y[3] = {rd(yp[0]), rd(yp[1]), rd(yp[2])};
    PatchWarp pw;
    patch_warp_setup(cam, xp, xo, y, pw);
#pragma unroll
    for (int k = 0; k < PER; ++k) {
      const int i = lane + 32 * k, a = i >> 4, b = i & 15;
      res[k] = 0;
      if (i < BYTES && b < BOX) {
        rd sp[2];
        ok = patch_warp_source(cam, pw, xp, xo, b - HALF, a - HALF, HALF, sp) && ok;
        if (ok) res[k] = (uint8_t)patch_sample(tpl[w], 16, BOX, sp);
      }
    }
  }
  // one invalid pixel: the feature keeps its stored template
  const bool warped = __all_sync(0xffffffffu, ok);
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    const int i = lane + 32 * k;
    if (i < BYTES) out[i] = warped ? res[k] : tpl[w][i];
  }
  if (L.valid && lane == 0) L.valid[job] = warped ? 1 : 0;
}

}  // namespace

cudaError_t sl2_launch_warp(const Sl2Dev &d, const WarpLaunch &L, Sl2Queue q) {
  const int jobs = L.stream_cnt * L.jobs_per_stream;
  if (jobs <= 0) return cudaSuccess;
  return sl2_with_box(d.box, [&](auto box) {
    return sl2_launch_kernel(warp_kernel<decltype(box)::value>, dim3((jobs + WARP_WARPS - 1) / WARP_WARPS),
                             dim3(32 * WARP_WARPS), 0, q, sl2_use_pdl(L.stream_cnt), d, L);
  });
}

extern "C" {

int sl2_set_stream_warp(sl2_ctx *c, int32_t s, int32_t on) {
  if (bad_stream(c, s) || (on != 0 && on != 1)) return fail(c, SL2_ERR_ARG, "sl2_set_stream_warp: bad argument");
  const Sl2Dev &d = c->d;
  if (on) {  // the job-indexed templates of every stream, once
    const int rc = grow_scratch(c, (size_t)d.B * d.Nmax * d.box * 16, c->warp_patches_bytes, c->warp_patches);
    if (rc) return rc;
  }
  CU_TRY(c, cudaMemsetAsync(c->warp_on_dev + s, on, 1, c->stream));
  c->warp_on[s] = (uint8_t)on;
  return SL2_OK;
}

int sl2_get_stream_warp(sl2_ctx *c, int32_t s, int32_t *on) {
  if (bad_stream(c, s) || !on) return fail(c, SL2_ERR_ARG, "sl2_get_stream_warp: bad argument");
  *on = c->warp_on[s];
  return SL2_OK;
}

int sl2_warp_templates(sl2_ctx *c, int32_t s, int32_t n, const int32_t *feat_index, const double *xp, uint8_t *out,
                       uint8_t *valid) {
  if (bad_stream(c, s) || n < 0 || n > c->cfg.max_features || (n > 0 && (!feat_index || !xp || !out)))
    return fail(c, SL2_ERR_ARG, "sl2_warp_templates: bad argument");
  if (n == 0) {
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    return SL2_OK;
  }
  for (int i = 0; i < 7; ++i)
    if (!std::isfinite(xp[i])) return fail(c, SL2_ERR_ARG, "sl2_warp_templates: xp must be finite");
  if (xp[3] == 0.0 && xp[4] == 0.0 && xp[5] == 0.0 && xp[6] == 0.0)
    return fail(c, SL2_ERR_ARG, "sl2_warp_templates: the quaternion of xp is zero");
  int rc = check_feature_indices(c, s, feat_index, n, "sl2_warp_templates: feature index out of range");
  if (rc) return rc;
  const int box = c->d.box;
  const size_t N = n;
  Stage fe{STAGE_IN, 4 * N, feat_index}, xs{STAGE_IN, 56, xp}, to{STAGE_OUT, N * box * 16}, va{STAGE_OUT, N};
  rc = staged_call(c, {&fe, &xs, &to, &va}, [] {}, [&] {
    WarpLaunch W = {};
    W.job_feat = fe.dev<int>();
    W.jobs_per_stream = n;
    W.stream_lo = s;
    W.stream_cnt = 1;
    W.xp = xs.dev<double>();
    W.out = to.d;
    W.valid = va.d;
    CU_TRY(c, sl2_launch_warp(c->d, W, queue(c)));
    return SL2_OK;
  });
  if (rc) return rc;
  for (size_t r = 0; r < N * box; ++r) memcpy(out + r * box, to.h + r * 16, box);
  if (valid) memcpy(valid, va.h, N);
  return SL2_OK;
}

}  // extern "C"
