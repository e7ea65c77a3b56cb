// normals.cu — the patch normal alignment on sm_90a, after the fused step's last update: each matched feature's stored
// template aligned with the step's frame through the homography its plane induces, with the plane's tilt theta as the
// free parameter (Molton, Davison, Reid, BMVC 2004), and carried as a Gaussian per feature.  Semantics:
// include/sl2b200.h, sl2_set_stream_normals (which, with the other entry points of the feature, ends this file);
// tests/normals_ref.py restates the kernel op for op, tests/normals_truth.py states the model from its definition.
// Shape: one warp per feature slot, NRM_WARPS per CTA.  Every lane evaluates the pixels k = lane + 32 j of the
// template (patch_warp_forward in sl2_model.cuh, bilinear samples of the frame through L2), forms its partial sums of
// the 21 products J_p J_q, the 6 of J_p e and e^2, and the xor-shuffle tree leaves the whole sums on every lane; every
// lane then runs the same 6 x 6 solve, so the control flow stays warp-uniform, and lane 0 writes.
#include <cmath>

#include "sl2_context.cuh"
#include "sl2_model.cuh"

using namespace sl2;

namespace {

constexpr int NRM_WARPS = 4;
constexpr int NRM_SUMS = 28;  // 21 of J^T J (p <= q, row by row), 6 of J^T e, e^2

struct NormalsLaunch {
  int stream_lo, stream_cnt;
  int slot;
  Sl2Subpix sp;
  Sl2Normals nrm;
};

// bilinear sample of the image (row stride pitch) at (u, v), both inside [0, W - 1) x [0, H - 1); not rounded
__device__ __forceinline__ rd frame_sample(const uint8_t *img, int pitch, rd u, rd v) {
  const int x0 = (int)floor(u.v), y0 = (int)floor(v.v);
  const rd fx = u - rd((double)x0), fy = v - rd((double)y0), one(1.0);
  const uint8_t *r0 = img + (size_t)y0 * pitch + x0, *r1 = r0 + pitch;
  const rd top = (one - fx) * rd((double)r0[0]) + fx * rd((double)r0[1]);
  const rd bot = (one - fx) * rd((double)r1[0]) + fx * rd((double)r1[1]);
  return (one - fy) * top + fy * bot;
}

// What one feature's alignment shares over its evaluations
struct AlignSetup {
  const double *cam, *xo, *x;
  const uint8_t *tpl, *img;
  int pitch, W, H;
  rd adjo[3][3], RRW[3][3], ho[2];
  PatchBasis b;
  rd yx[3], ry[3];  // y - xo[0:3], x[0:3] - y
};

// sum[0 .. 21) = J^T J (upper triangle, row by row), sum[21 .. 27) = J^T e, sum[27] = e^T e at phi, over the whole
// warp; returns whether phi is valid (every pixel, and the normal faces both cameras)
template <int BOX>
__device__ __forceinline__ bool align_eval(const AlignSetup &a, const rd phi[6], int lane, rd sum[NRM_SUMS]) {
  constexpr int HALF = (BOX - 1) / 2, NPIX = BOX * BOX;
  rd nW[3];
  patch_normal(a.b, phi[0], phi[1], nW);
  const rd nd = dot3(nW, a.yx), nE1 = dot3(a.b.E1, a.yx), nE2 = dot3(a.b.E2, a.yx);
  bool ok = dot3(nW, a.b.n0).v > 0.0 && dot3(nW, a.ry).v > 0.0;
#pragma unroll
  for (int p = 0; p < NRM_SUMS; ++p) sum[p] = rd(0.0);
  const double wlim = (double)(a.W - 2), hlim = (double)(a.H - 2);
  for (int k = lane; k < NPIX; k += 32) {
    const int r = k / BOX, c = k - r * BOX;
    PatchFwd fw;
    const bool in = patch_warp_forward(a.cam, a.adjo, a.ho, a.xo, a.RRW, a.x, a.b, nW, nd, nE1, nE2, c - HALF, r - HALF,
                                       fw);
    const rd gu = fw.g[0] + phi[2], gv = fw.g[1] + phi[3];
    ok = ok && in && gu.v >= 1.0 && gu.v < wlim && gv.v >= 1.0 && gv.v < hlim;
    if (!ok) break;
    const rd one(1.0), half(0.5);
    const rd I = frame_sample(a.img, a.pitch, gu, gv);
    const rd Iu = (frame_sample(a.img, a.pitch, gu + one, gv) - frame_sample(a.img, a.pitch, gu - one, gv)) * half;
    const rd Iv = (frame_sample(a.img, a.pitch, gu, gv + one) - frame_sample(a.img, a.pitch, gu, gv - one)) * half;
    const rd e = (phi[4] * I + phi[5]) - rd((double)a.tpl[r * 16 + c]);
    const rd ag = phi[4] * (Iu * fw.Jw[0] + Iv * fw.Jw[1]);
    const rd J[6] = {ag * fw.ta, ag * fw.tb, phi[4] * Iu, phi[4] * Iv, I, one};
    int o = 0;
#pragma unroll
    for (int p = 0; p < 6; ++p)
#pragma unroll
      for (int q = p; q < 6; ++q) sum[o] = sum[o] + J[p] * J[q], ++o;
#pragma unroll
    for (int p = 0; p < 6; ++p) sum[21 + p] = sum[21 + p] + J[p] * e;
    sum[27] = sum[27] + e * e;
  }
  ok = __all_sync(0xffffffffu, ok);
  if (!ok) return false;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1)
#pragma unroll
    for (int p = 0; p < NRM_SUMS; ++p) sum[p] = sum[p] + rd(__shfl_xor_sync(0xffffffffu, sum[p].v, off));
  return true;
}

// The Gauss-Newton system at phi: H (upper triangle, 21) = (J^T J) w2 + L on the theta block, G = (J^T e) w2 + L dt on
// theta, and the cost
struct AlignSys {
  rd H[21], G[6], cost;
};
__device__ __forceinline__ void align_system(const rd sum[NRM_SUMS], const rd phi[6], const rd th0[2], const rd L[3],
                                             rd w2, AlignSys &s) {
#pragma unroll
  for (int p = 0; p < 21; ++p) s.H[p] = sum[p] * w2;
#pragma unroll
  for (int p = 0; p < 6; ++p) s.G[p] = sum[21 + p] * w2;
  const rd da = phi[0] - th0[0], db = phi[1] - th0[1];
  const rd pa = L[0] * da + L[1] * db, pb = L[1] * da + L[2] * db;
  s.H[0] = s.H[0] + L[0];  // (0, 0)
  s.H[1] = s.H[1] + L[1];  // (0, 1)
  s.H[6] = s.H[6] + L[2];  // (1, 1)
  s.G[0] = s.G[0] + pa;
  s.G[1] = s.G[1] + pb;
  s.cost = sum[27] * w2 + (da * pa + db * pb);
}

// index of (p, q), p <= q, in the upper triangle stored row by row
__device__ __forceinline__ constexpr int tri(int p, int q) { return p * 6 - p * (p - 1) / 2 + (q - p); }

// H = L L^T (L lower, Lm[i][j] for j <= i); false at a pivot that is not > 0 (NaN included)
__device__ __forceinline__ bool chol6(const rd H[21], rd Lm[6][6]) {
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    rd s = H[tri(j, j)];
#pragma unroll
    for (int k = 0; k < j; ++k) s = s - Lm[j][k] * Lm[j][k];
    if (!(s.v > 0.0)) return false;
    Lm[j][j] = rsqrt_(s);
#pragma unroll
    for (int i = j + 1; i < 6; ++i) {
      rd t = H[tri(j, i)];
#pragma unroll
      for (int k = 0; k < j; ++k) t = t - Lm[i][k] * Lm[j][k];
      Lm[i][j] = t / Lm[j][j];
    }
  }
  return true;
}

template <int BOX>
__global__ void __launch_bounds__(32 * NRM_WARPS) normals_kernel(const Sl2Dev d, const NormalsLaunch L) {
  pdl_prologue();
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int job = blockIdx.x * NRM_WARPS + w;  // one feature slot, local to the launch
  if (job >= L.stream_cnt * d.Nmax) return;
  const int s = L.stream_lo + job / d.Nmax, i = job - (job / d.Nmax) * d.Nmax;
  if (!normals_on(L.nrm, s) || i >= d.nfeat[s]) return;
  const size_t fb = (size_t)s * d.Nmax, f = fb + i;
  const int r = d.sel_rank[f];
  // a feature of this step's job list whose match the update used
  if (!(r >= 0 && r < d.Nmax && d.job_feat[fb + r] == i && d.found[f] == 1)) {
    if (lane == 0) L.nrm.status[f] = 0;
    return;
  }
  const sl2_stream_normals prm = L.nrm.prm[s];
  AlignSetup a;
  a.cam = d.cams[s].cam;
  a.W = stream_width(d.cams[s]);
  a.H = stream_height(d.cams[s]);
  a.xo = d.xp_org + f * 7;
  a.x = d.x + (size_t)s * d.ld;
  a.tpl = d.patches + f * (BOX * 16);
  a.img = d.frames + (size_t)(L.slot * d.B + s) * d.H * d.pitch;
  a.pitch = d.pitch;
  const double *yp = a.x + SL2_NXV + 3 * i;
  const rd y[3] = {rd(yp[0]), rd(yp[1]), rd(yp[2])};
  rd RRWo[3][3], dd[3], zz[3], uc, vc;
  pose_RRW(a.xo, RRWo);
  mat3_adj(RRWo, a.adjo);
  zeroed_point(RRWo, y, a.xo, dd, zz);
  project_point(a.cam, zz, a.ho, uc, vc);
  patch_basis(a.xo, y, RRWo, a.b);
  for (int k = 0; k < 3; ++k) {
    a.yx[k] = y[k] - rd(a.xo[k]);
    a.ry[k] = rd(a.x[k]) - y[k];
  }
  rd hp[2];
  pose_RRW(a.x, a.RRW);
  zeroed_point(a.RRW, y, a.x, dd, zz);
  project_point(a.cam, zz, hp, uc, vc);
  // the prior
  const rd th0[2] = {rd(L.nrm.theta[f * 2]), rd(L.nrm.theta[f * 2 + 1])};
  const rd ss = rd(prm.sigma_step) * rd(prm.sigma_step);
  const rd Saa = rd(L.nrm.cov[f * 3]) + ss, Sab(L.nrm.cov[f * 3 + 1]), Sbb = rd(L.nrm.cov[f * 3 + 2]) + ss;
  const rd det = Saa * Sbb - Sab * Sab;
  const rd Li[3] = {Sbb / det, (-Sab) / det, Saa / det};
  const rd w2 = rd(1.0) / (rd(prm.sigma_i) * rd(prm.sigma_i));
  rd phi[6] = {th0[0], th0[1], rd(match_z(d, L.sp, f, 0)) - hp[0], rd(match_z(d, L.sp, f, 1)) - hp[1], rd(1.0),
               rd(0.0)};
  rd sum[NRM_SUMS];
  AlignSys cur;
  int status = 3, accepted = 0;
  if (align_eval<BOX>(a, phi, lane, sum)) {
    align_system(sum, phi, th0, Li, w2, cur);
    status = 2;
    for (int it = 0; it < prm.max_iterations; ++it) {
      rd Lm[6][6];
      if (!chol6(cur.H, Lm)) break;
      rd u[6], v[6], nphi[6];
#pragma unroll
      for (int p = 0; p < 6; ++p) {
        rd t = cur.G[p];
#pragma unroll
        for (int k = 0; k < p; ++k) t = t - Lm[p][k] * u[k];
        u[p] = t / Lm[p][p];
      }
#pragma unroll
      for (int p = 5; p >= 0; --p) {
        rd t = u[p];
#pragma unroll
        for (int k = p + 1; k < 6; ++k) t = t - Lm[k][p] * v[k];
        v[p] = t / Lm[p][p];
      }
#pragma unroll
      for (int p = 0; p < 6; ++p) nphi[p] = phi[p] - v[p];
      if (!align_eval<BOX>(a, nphi, lane, sum)) break;
      AlignSys nxt;
      align_system(sum, nphi, th0, Li, w2, nxt);
      if (!(nxt.cost.v < cur.cost.v)) break;
#pragma unroll
      for (int p = 0; p < 6; ++p) phi[p] = nphi[p];
      cur = nxt;
      ++accepted;
    }
  }
  rd Lm[6][6];
  if (accepted > 0 && chol6(cur.H, Lm)) {
    // the first two columns of L^-1, then the theta block of H^-1 = L^-T L^-1
    rd c0[6], c1[6];
#pragma unroll
    for (int p = 0; p < 6; ++p) {
      rd t0(p == 0 ? 1.0 : 0.0), t1(p == 1 ? 1.0 : 0.0);
#pragma unroll
      for (int k = 0; k < p; ++k) {
        t0 = t0 - Lm[p][k] * c0[k];
        t1 = t1 - Lm[p][k] * c1[k];
      }
      c0[p] = t0 / Lm[p][p];
      c1[p] = t1 / Lm[p][p];
    }
    rd saa(0.0), sab(0.0), sbb(0.0);
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      saa = saa + c0[k] * c0[k];
      sab = sab + c0[k] * c1[k];
      sbb = sbb + c1[k] * c1[k];
    }
    status = 1;
    if (lane == 0) {
      L.nrm.theta[f * 2] = phi[0].v;
      L.nrm.theta[f * 2 + 1] = phi[1].v;
      L.nrm.cov[f * 3] = saa.v;
      L.nrm.cov[f * 3 + 1] = sab.v;
      L.nrm.cov[f * 3 + 2] = sbb.v;
      L.nrm.count[f] += 1;
    }
  } else if (accepted > 0) {
    status = 2;
  }
  if (lane == 0) L.nrm.status[f] = (uint8_t)status;
}

// the estimates of features idx[0 .. n) of stream s (get), or written from theta / cov in index order (set)
__global__ void normals_io_kernel(const Sl2Dev d, const Sl2Normals N, int s, int n, const int *idx, int set,
                                  const double *theta_in, const double *cov_in, double *theta, double *cov, double *nw,
                                  int *count, uint8_t *status) {
  const size_t fb = (size_t)s * d.Nmax;
  if (set) {
    if (threadIdx.x + blockIdx.x > 0) return;
    for (int j = 0; j < n; ++j) {  // serial: a repeated index keeps its last values
      const size_t f = fb + idx[j];
      for (int e = 0; e < 2; ++e) N.theta[f * 2 + e] = theta_in[j * 2 + e];
      for (int e = 0; e < 3; ++e) N.cov[f * 3 + e] = cov_in[j * 3 + e];
      N.count[f] = 0;
      N.status[f] = 0;
    }
    return;
  }
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const size_t f = fb + idx[j];
  const double *xo = d.xp_org + f * 7, *yp = d.x + (size_t)s * d.ld + SL2_NXV + 3 * idx[j];
  const rd y[3] = {rd(yp[0]), rd(yp[1]), rd(yp[2])};
  rd RRWo[3][3], nW[3];
  pose_RRW(xo, RRWo);
  PatchBasis b;
  patch_basis(xo, y, RRWo, b);
  patch_normal(b, rd(N.theta[f * 2]), rd(N.theta[f * 2 + 1]), nW);
  const rd len = rsqrt_(dot3(nW, nW));
  for (int e = 0; e < 2; ++e) theta[j * 2 + e] = N.theta[f * 2 + e];
  for (int e = 0; e < 3; ++e) cov[j * 3 + e] = N.cov[f * 3 + e];
  for (int e = 0; e < 3; ++e) nw[j * 3 + e] = (nW[e] / len).v;
  count[j] = N.count[f];
  status[j] = N.status[f];
}

bool normals_params_ok(const sl2_stream_normals *v) {
  return v && v->reserved == 0 && v->max_iterations >= 0 && v->max_iterations <= SL2_MAX_NORMAL_ITERATIONS &&
         std::isfinite(v->sigma0) && v->sigma0 > 0.0 && std::isfinite(v->sigma_i) && v->sigma_i > 0.0 &&
         std::isfinite(v->sigma_step) && v->sigma_step >= 0.0;
}

}  // namespace

cudaError_t sl2_launch_normals(const Sl2Dev &d, int stream_lo, int stream_cnt, int slot, const Sl2Subpix &sp,
                               const Sl2Normals &nrm, Sl2Queue q) {
  const int jobs = stream_cnt * d.Nmax;
  if (jobs <= 0) return cudaSuccess;
  const NormalsLaunch L = {stream_lo, stream_cnt, slot, sp, nrm};
  return sl2_with_box(d.box, [&](auto box) {
    return sl2_launch_kernel(normals_kernel<decltype(box)::value>, dim3((jobs + NRM_WARPS - 1) / NRM_WARPS),
                             dim3(32 * NRM_WARPS), 0, q, sl2_use_pdl(stream_cnt), d, L);
  });
}

namespace sl2 {

Sl2Normals normals_args(const sl2_ctx *c, int lo, int cnt) {
  const auto on = [](const StreamOptions &o) { return o.nrm.max_iterations > 0; };
  return c->nrm_buf && any_stream(c, lo, cnt, on) ? c->nrm_dev : Sl2Normals{};
}

int normals_reset(sl2_ctx *c, int s, int f0, int n) {
  const sl2_stream_normals &v = c->opt[s].nrm;
  if (!c->nrm_buf || v.max_iterations == 0 || n <= 0) return SL2_OK;
  const Sl2Normals &N = c->nrm_dev;
  const size_t f = (size_t)s * c->d.Nmax + f0;
  const double v0 = v.sigma0 * v.sigma0;
  std::vector<double> cov((size_t)n * 3);  // pageable: the copy has read it when cudaMemcpyAsync returns
  for (int j = 0; j < n; ++j) {
    cov[j * 3] = v0;
    cov[j * 3 + 1] = 0.0;
    cov[j * 3 + 2] = v0;
  }
  CU_TRY(c, cudaMemsetAsync(N.theta + f * 2, 0, (size_t)n * 2 * sizeof(double), c->stream));
  CU_TRY(c, cudaMemcpyAsync(N.cov + f * 3, cov.data(), cov.size() * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, cudaMemsetAsync(N.count + f, 0, (size_t)n * sizeof(int), c->stream));
  CU_TRY(c, cudaMemsetAsync(N.status + f, 0, (size_t)n, c->stream));
  return SL2_OK;
}

}  // namespace sl2

extern "C" {

int sl2_set_stream_normals(sl2_ctx *c, int32_t s, const sl2_stream_normals *v) {
  if (bad_stream(c, s) || !normals_params_ok(v)) return fail(c, SL2_ERR_ARG, "sl2_set_stream_normals: bad argument");
  if (v->max_iterations > 0 && !c->nrm_buf) {
    const size_t B = c->d.B, BN = (size_t)c->d.B * c->d.Nmax;
    Sl2Normals &N = c->nrm_dev;
    const int rc = alloc_sections(c, c->nrm_buf,
                                  {{&N.prm, B * sizeof(sl2_stream_normals)}, {&N.theta, BN * 2 * sizeof(double)},
                                   {&N.cov, BN * 3 * sizeof(double)}, {&N.count, BN * sizeof(int)}, {&N.status, BN}});
    if (rc) return rc;
  }
  c->opt[s].nrm = *v;
  if (c->nrm_buf) {
    CU_TRY(c, cudaMemcpyAsync(const_cast<sl2_stream_normals *>(c->nrm_dev.prm) + s, &c->opt[s].nrm,
                              sizeof(sl2_stream_normals), cudaMemcpyHostToDevice, c->stream));
    const int rc = normals_reset(c, s, 0, c->d.Nmax);
    if (rc) return rc;
    CU_TRY(c, cudaStreamSynchronize(c->stream));
  }
  return SL2_OK;
}

int sl2_get_stream_normals(sl2_ctx *c, int32_t s, sl2_stream_normals *v) {
  if (bad_stream(c, s) || !v) return fail(c, SL2_ERR_ARG, "sl2_get_stream_normals: bad argument");
  *v = c->opt[s].nrm;
  return SL2_OK;
}

int sl2_get_patch_normals(sl2_ctx *c, int32_t s, int32_t n, const int32_t *feat_index, double *theta, double *cov,
                          double *normal_w, int32_t *count, uint8_t *status) {
  if (bad_stream(c, s) || n < 0 || n > c->cfg.max_features || (n > 0 && !feat_index))
    return fail(c, SL2_ERR_ARG, "sl2_get_patch_normals: bad argument");
  if (c->opt[s].nrm.max_iterations == 0)
    return fail(c, SL2_ERR_STATE, "sl2_get_patch_normals: the stream has normals off");
  int rc = check_feature_indices(c, s, feat_index, n, "sl2_get_patch_normals: feature index out of range");
  if (rc || n == 0) return rc;
  const size_t N = n;
  Stage fe{STAGE_IN, 4 * N, feat_index}, th{STAGE_OUT, 16 * N}, cv{STAGE_OUT, 24 * N}, nw{STAGE_OUT, 24 * N},
      ct{STAGE_OUT, 4 * N}, st{STAGE_OUT, N};
  rc = staged_call(c, {&fe, &th, &cv, &nw, &ct, &st}, [] {}, [&] {
    CU_TRY(c, sl2_launch_kernel(normals_io_kernel, dim3((n + 127) / 128), dim3(128), 0, queue(c), false, c->d,
                                c->nrm_dev, s, n, fe.dev<int>(), 0, nullptr, nullptr, th.dev<double>(),
                                cv.dev<double>(), nw.dev<double>(), ct.dev<int>(), st.d));
    return SL2_OK;
  });
  if (rc) return rc;
  if (theta) memcpy(theta, th.h, 16 * N);
  if (cov) memcpy(cov, cv.h, 24 * N);
  if (normal_w) memcpy(normal_w, nw.h, 24 * N);
  if (count) memcpy(count, ct.h, 4 * N);
  if (status) memcpy(status, st.h, N);
  return SL2_OK;
}

int sl2_set_patch_normals(sl2_ctx *c, int32_t s, int32_t n, const int32_t *feat_index, const double *theta,
                          const double *cov) {
  if (bad_stream(c, s) || n < 0 || n > c->cfg.max_features || (n > 0 && (!feat_index || !theta || !cov)))
    return fail(c, SL2_ERR_ARG, "sl2_set_patch_normals: bad argument");
  if (c->opt[s].nrm.max_iterations == 0)
    return fail(c, SL2_ERR_STATE, "sl2_set_patch_normals: the stream has normals off");
  for (int j = 0; j < n; ++j) {
    const double a = cov[j * 3], b = cov[j * 3 + 1], e = cov[j * 3 + 2];
    if (!std::isfinite(theta[j * 2]) || !std::isfinite(theta[j * 2 + 1]) || !std::isfinite(a) || !std::isfinite(b) ||
        !std::isfinite(e) || !(a > 0.0) || !(a * e - b * b > 0.0))
      return fail(c, SL2_ERR_ARG, "sl2_set_patch_normals: theta must be finite and cov positive definite");
  }
  int rc = check_feature_indices(c, s, feat_index, n, "sl2_set_patch_normals: feature index out of range");
  if (rc || n == 0) return rc;
  const size_t N = n;
  Stage fe{STAGE_IN, 4 * N, feat_index}, th{STAGE_IN, 16 * N, theta}, cv{STAGE_IN, 24 * N, cov};
  return staged_call(c, {&fe, &th, &cv}, [] {}, [&] {
    CU_TRY(c, sl2_launch_kernel(normals_io_kernel, dim3(1), dim3(32), 0, queue(c), false, c->d, c->nrm_dev, s, n,
                                fe.dev<int>(), 1, th.dev<double>(), cv.dev<double>(), nullptr, nullptr, nullptr,
                                nullptr, nullptr));
    return SL2_OK;
  });
}

int sl2_align_normals(sl2_ctx *c, int32_t s, int32_t slot) {
  if (bad_stream(c, s) || bad_slot(c, slot)) return fail(c, SL2_ERR_ARG, "sl2_align_normals: bad stream/slot");
  if (c->opt[s].nrm.max_iterations == 0) return fail(c, SL2_ERR_STATE, "sl2_align_normals: the stream has normals off");
  CU_TRY(c, sl2_launch_normals(c->d, s, 1, slot, subpixel_args(c, s, 1), normals_args(c, s, 1), queue(c)));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return SL2_OK;
}

}  // extern "C"
