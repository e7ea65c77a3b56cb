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
// The exposure blur (include/sl2b200.h, sl2_set_stream_blur) is the second instantiation, warp_kernel<BOX, true>,
// launched only for launches with a blur-on stream: lane 0 forms the per-job terms of the three exposure poses and the
// reference camera once into shared memory, every lane then forms the same sample count K (warp-uniform) and maps its
// pixels through the three poses, one unproject_point per pixel; each of the K samples is then one bilinear read.
#include <cmath>

#include "sl2_context.cuh"
#include "sl2_model.cuh"

using namespace sl2;

namespace {

#define WARP_WARPS 4
#define BLUR_MAX_SAMPLES 32

// The warp of one job into res (pixel i = lane + 32 k of the row-padded layout); true when every pixel is valid
// (warp-uniform)
template <int BOX, int PER>
__device__ __forceinline__ bool warp_job(const double *cam, const double *xp, const double *xo, const double *yp,
                                         const double *theta, const uint8_t *tpl, int lane, uint8_t res[PER]) {
  constexpr int HALF = (BOX - 1) / 2, BYTES = BOX * 16;
  const rd y[3] = {rd(yp[0]), rd(yp[1]), rd(yp[2])};
  PatchWarp pw;
  patch_warp_setup(cam, xp, xo, y, pw, theta);
  bool ok = true;
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    const int i = lane + 32 * k, a = i >> 4, b = i & 15;
    res[k] = 0;
    if (i < BYTES && b < BOX) {
      rd sp[2];
      ok = patch_warp_source(cam, pw, b - HALF, a - HALF, HALF, sp) && ok;
      if (ok) res[k] = (uint8_t)patch_sample(tpl, 16, BOX, sp);
    }
  }
  return __all_sync(0xffffffffu, ok);
}

// What one job's blur shares over its pixels: the poses at s-, s_c, s+ (ident[k]: the source is the pixel itself, the
// warp off and s = 0), the reference camera, the plane's normal and h0
struct BlurJob {
  PatchPose pose[3];
  PatchRef ref;
  rd nW[3], h0[2];
  int ident[3];
};

// Lane 0's part of blur_job: the per-job terms into J
__device__ __noinline__ void blur_setup(const double *cam, const double *x, const double *xo, const double *yp,
                                        const double *theta, bool warp, const sl2_stream_blur &bl, BlurJob &J) {
  const rd y[3] = {rd(yp[0]), rd(yp[1]), rd(yp[2])};
  PatchWarp pw;
  patch_warp_setup(cam, x, xo, y, pw, theta);
  for (int i = 0; i < 3; ++i) J.nW[i] = pw.nW[i];
  J.h0[0] = pw.h[0];
  J.h0[1] = pw.h[1];
  if (warp) {
    J.ref = pw.ref;
  } else {
    rd d[3], z[3];
    pose_RRW(x, J.ref.RRW);
    zeroed_point(J.ref.RRW, y, x, d, z);
    for (int i = 0; i < 3; ++i) J.ref.r[i] = rd(x[i]);
    J.ref.c[0] = pw.h[0];
    J.ref.c[1] = pw.h[1];
  }
  const rd hx = rd(bl.exposure) * rd(0.5), off(bl.offset);
  const rd times[3] = {off - hx, off, off + hx};
  for (int k = 0; k < 3; ++k) {
    const rd t = times[k];
    J.ident[k] = !warp && t.v == 0.0;
    if (t.v == 0.0) {  // the pose x[0:7] itself
      J.pose[k] = pw.at;
      continue;
    }
    // the motion model's prediction of r and q over dt = t
    double xs[7];
    for (int i = 0; i < 3; ++i) xs[i] = (rd(x[i]) + rd(x[7 + i]) * t).v;
    const rd av[3] = {rd(x[10]) * t, rd(x[11]) * t, rd(x[12]) * t};
    const Quat qs = quat_mul(Quat{rd(x[3]), rd(x[4]), rd(x[5]), rd(x[6])}, quat_from_angular_velocity(av));
    xs[3] = qs.w.v;
    xs[4] = qs.x.v;
    xs[5] = qs.y.v;
    xs[6] = qs.z.v;
    rd RRW[3][3], d[3], z[3];
    pose_RRW(xs, RRW);
    zeroed_point(RRW, y, xs, d, z);
    patch_pose_terms(xs, RRW, d, J.nW, J.pose[k]);
  }
}

// src(s_k) of the ray c through output pixel (b, a)
__device__ __forceinline__ bool blur_source(const double *cam, const BlurJob &J, int k, const rd c[3], int b, int a,
                                            int half, rd src[2]) {
  if (J.ident[k]) {
    src[0] = rd((double)b);
    src[1] = rd((double)a);
    return true;
  }
  return patch_ray_source(cam, J.pose[k], J.ref, J.nW, c, half, src);
}

// The blur of one job into res; returns K, or 0 when a needed source is invalid or L is not finite (warp-uniform)
template <int BOX, int PER>
__device__ __forceinline__ int blur_job(const double *cam, const BlurJob &J, const uint8_t *tpl, int lane,
                                        uint8_t res[PER]) {
  constexpr int HALF = (BOX - 1) / 2, BYTES = BOX * 16;
  // the sample count from the centre pixel's streak, the same on every lane
  rd c0[3], sm[2], sp[2];
  unproject_point(cam, J.h0, c0);
  bool ok = blur_source(cam, J, 0, c0, HALF, HALF, HALF, sm);
  ok = blur_source(cam, J, 2, c0, HALF, HALF, HALF, sp) && ok;
  const rd dx = sp[0] - sm[0], dy = sp[1] - sm[1];
  const rd len = rsqrt_(dx * dx + dy * dy);
  ok = ok && isfinite(len.v);
  const int K = ok ? (int)fmin((double)BLUR_MAX_SAMPLES, fmax(1.0, ceil(len.v))) : 1;
  const rd rK((double)K), half(0.5), two(2.0);
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    const int i = lane + 32 * k, a = i >> 4, b = i & 15;
    res[k] = 0;
    if (i < BYTES && b < BOX && ok) {
      const rd p[2] = {J.h0[0] + rd((double)(b - HALF)), J.h0[1] + rd((double)(a - HALF))};
      rd c[3], s0[2], s1[2], s2[2];
      unproject_point(cam, p, c);
      ok = blur_source(cam, J, 1, c, b, a, HALF, s1);
      if (K > 1) {
        ok = blur_source(cam, J, 0, c, b, a, HALF, s0) && ok;
        ok = blur_source(cam, J, 2, c, b, a, HALF, s2) && ok;
      }
      if (ok) {
        rd v;
        if (K == 1) {
          v = patch_bilinear(tpl, 16, BOX, s1);
        } else {
          rd d1[2], d2[2];
          for (int j = 0; j < 2; ++j) {
            d1[j] = s2[j] - s0[j];
            d2[j] = (s2[j] - two * s1[j]) + s0[j];
          }
          rd sum(0.0);
          for (int m = 0; m < K; ++m) {
            const rd u = ((rd((double)m) + half) / rK) - half;
            const rd w2 = (two * u) * u;
            const rd sk[2] = {(s1[0] + u * d1[0]) + w2 * d2[0], (s1[1] + u * d1[1]) + w2 * d2[1]};
            sum = sum + patch_bilinear(tpl, 16, BOX, sk);
          }
          v = sum / rK;
        }
        res[k] = (uint8_t)(int)(v + half).v;
      }
    }
  }
  return __all_sync(0xffffffffu, ok) ? K : 0;
}

template <int BOX, bool BLUR>
__global__ void __launch_bounds__(32 * WARP_WARPS) warp_kernel(const Sl2Dev d, const WarpLaunch L) {
  pdl_prologue();
  constexpr int BYTES = BOX * 16, PER = (BYTES + 31) / 32;
  __shared__ __align__(16) uint8_t tpl[WARP_WARPS][BYTES];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int job = blockIdx.x * WARP_WARPS + w;
  if (job >= L.stream_cnt * L.jobs_per_stream) return;
  const int feat = L.job_feat[job];
  if (feat < 0) {
    if (L.valid && lane == 0) L.valid[job] = 0;
    if (BLUR && L.samples && lane == 0) L.samples[job] = 0;
    return;
  }
  const int s = L.stream_lo + job / L.jobs_per_stream;
  const size_t g = (size_t)s * d.Nmax + feat;
  const uint32_t *src32 = reinterpret_cast<const uint32_t *>(d.patches + g * BYTES);
  uint32_t *t32 = reinterpret_cast<uint32_t *>(tpl[w]);
  for (int k = lane; k < BYTES / 4; k += 32) t32[k] = src32[k];
  __syncwarp();
  uint8_t *out = L.out + (size_t)job * BYTES;
  const bool warp = !L.on || L.on[s];
  const double *xp = L.xp ? L.xp : d.x + (size_t)s * d.ld;
  const double *xo = d.xp_org + g * 7;
  const double *cam = d.cams[s].cam;
  const double *yp = d.x + (size_t)s * d.ld + SL2_NXV + 3 * feat;
  uint8_t res[PER];
  int mode = 0, K = 0;  // 2 blurred (K samples), 1 warped, 0 the stored template
  if constexpr (BLUR) {
    if (L.blur[s].on) {
      __shared__ __align__(16) unsigned char jobs[WARP_WARPS][sizeof(BlurJob)];
      BlurJob &J = *reinterpret_cast<BlurJob *>(jobs[w]);
      if (lane == 0)
        blur_setup(cam, xp, xo, yp, normals_on(L.nrm, s) ? L.nrm.theta + g * 2 : nullptr, warp, L.blur[s], J);
      __syncwarp();
      K = blur_job<BOX, PER>(cam, J, tpl[w], lane, res);
      mode = K > 0 ? 2 : 0;
    }
  }
  // one invalid pixel: the feature keeps its stored template
  if (mode == 0 && warp)
    mode = warp_job<BOX, PER>(cam, xp, xo, yp, normals_on(L.nrm, s) ? L.nrm.theta + g * 2 : nullptr, tpl[w], lane,
                              res) ? 1 : 0;
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    const int i = lane + 32 * k;
    if (i < BYTES) out[i] = mode ? res[k] : tpl[w][i];
  }
  if (L.valid && lane == 0) L.valid[job] = (uint8_t)mode;
  if (BLUR && L.samples && lane == 0) L.samples[job] = K;
}

}  // namespace

cudaError_t sl2_launch_warp(const Sl2Dev &d, const WarpLaunch &L, Sl2Queue q) {
  const int jobs = L.stream_cnt * L.jobs_per_stream;
  if (jobs <= 0) return cudaSuccess;
  return sl2_with_box(d.box, [&](auto box) {
    constexpr int BOX = decltype(box)::value;
    return sl2_launch_kernel(L.blur ? warp_kernel<BOX, true> : warp_kernel<BOX, false>,
                             dim3((jobs + WARP_WARPS - 1) / WARP_WARPS), dim3(32 * WARP_WARPS), 0, q,
                             sl2_use_pdl(L.stream_cnt), d, L);
  });
}

extern "C" {

namespace {
// the job-indexed templates of every stream, once (the warp and the blur both write them)
int size_job_templates(sl2_ctx *c) {
  const Sl2Dev &d = c->d;
  return grow_scratch(c, (size_t)d.B * d.Nmax * d.box * 16, c->warp_patches_bytes, c->warp_patches);
}
}  // namespace

int sl2_set_stream_warp(sl2_ctx *c, int32_t s, int32_t on) {
  if (bad_stream(c, s) || (on != 0 && on != 1)) return fail(c, SL2_ERR_ARG, "sl2_set_stream_warp: bad argument");
  if (on) {
    const int rc = size_job_templates(c);
    if (rc) return rc;
  }
  CU_TRY(c, cudaMemsetAsync(c->warp_on_dev + s, on, 1, c->stream));
  c->opt[s].warp = (uint8_t)on;
  return SL2_OK;
}

int sl2_get_stream_warp(sl2_ctx *c, int32_t s, int32_t *on) {
  if (bad_stream(c, s) || !on) return fail(c, SL2_ERR_ARG, "sl2_get_stream_warp: bad argument");
  *on = c->opt[s].warp;
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
    W.nrm = normals_args(c, s, 1);
    CU_TRY(c, sl2_launch_warp(c->d, W, queue(c)));
    return SL2_OK;
  });
  if (rc) return rc;
  for (size_t r = 0; r < N * box; ++r) memcpy(out + r * box, to.h + r * 16, box);
  if (valid) memcpy(valid, va.h, N);
  return SL2_OK;
}

int sl2_set_stream_blur(sl2_ctx *c, int32_t s, const sl2_stream_blur *b) {
  if (bad_stream(c, s) || !b || b->reserved != 0 || (b->on != 0 && b->on != 1) || !std::isfinite(b->exposure) ||
      !(b->exposure >= 0.0) || !std::isfinite(b->offset))
    return fail(c, SL2_ERR_ARG, "sl2_set_stream_blur: bad argument");
  if (b->on) {
    const int rc = size_job_templates(c);
    if (rc) return rc;
  }
  const sl2_stream_blur v = *b;  // pageable copies have read their sources when they return; ordered on the stream
  CU_TRY(c, cudaMemcpyAsync(c->blur_dev + s, &v, sizeof v, cudaMemcpyHostToDevice, c->stream));
  c->opt[s].blur = v;
  return SL2_OK;
}

int sl2_get_stream_blur(sl2_ctx *c, int32_t s, sl2_stream_blur *b) {
  if (bad_stream(c, s) || !b) return fail(c, SL2_ERR_ARG, "sl2_get_stream_blur: bad argument");
  *b = c->opt[s].blur;
  return SL2_OK;
}

int sl2_blur_templates(sl2_ctx *c, int32_t s, int32_t n, const int32_t *feat_index, const double *xv, uint8_t *out,
                       uint8_t *valid, int32_t *samples) {
  if (bad_stream(c, s) || n < 0 || n > c->cfg.max_features || (n > 0 && (!feat_index || !xv || !out)))
    return fail(c, SL2_ERR_ARG, "sl2_blur_templates: bad argument");
  if (n == 0) {
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    return SL2_OK;
  }
  for (int i = 0; i < SL2_NXV; ++i)
    if (!std::isfinite(xv[i])) return fail(c, SL2_ERR_ARG, "sl2_blur_templates: xv must be finite");
  if (xv[3] == 0.0 && xv[4] == 0.0 && xv[5] == 0.0 && xv[6] == 0.0)
    return fail(c, SL2_ERR_ARG, "sl2_blur_templates: the quaternion of xv is zero");
  int rc = check_feature_indices(c, s, feat_index, n, "sl2_blur_templates: feature index out of range");
  if (rc) return rc;
  const int box = c->d.box;
  const size_t N = n;
  Stage fe{STAGE_IN, 4 * N, feat_index}, xs{STAGE_IN, 8 * SL2_NXV, xv}, to{STAGE_OUT, N * box * 16},
      va{STAGE_OUT, N}, ks{STAGE_OUT, 4 * N};
  rc = staged_call(c, {&fe, &xs, &to, &va, &ks}, [] {}, [&] {
    WarpLaunch W = {};
    W.job_feat = fe.dev<int>();
    W.jobs_per_stream = n;
    W.stream_lo = s;
    W.stream_cnt = 1;
    W.xp = xs.dev<double>();
    W.on = c->warp_on_dev;
    W.out = to.d;
    W.valid = va.d;
    W.nrm = normals_args(c, s, 1);
    W.blur = c->blur_dev;
    W.samples = ks.dev<int>();
    CU_TRY(c, sl2_launch_warp(c->d, W, queue(c)));
    return SL2_OK;
  });
  if (rc) return rc;
  for (size_t r = 0; r < N * box; ++r) memcpy(out + r * box, to.h + r * 16, box);
  if (valid) memcpy(valid, va.h, N);
  if (samples) memcpy(samples, ks.h, 4 * N);
  return SL2_OK;
}

}  // extern "C"
