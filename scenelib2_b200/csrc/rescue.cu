// rescue.cu — the consensus rescue on sm_90a, between the first EKF update and the cull of the fused step: the
// high-innovation stage of 1-point RANSAC (Civera, Grasa, Davison, Montiel, J. Field Robotics 2010) after the match
// consensus (consensus.cu).  One CTA per camera stream of the launch; streams whose chi2[s] (0 = off) or consensus
// tau2[s] is not > 0 return at once.  Semantics: include/sl2b200.h, sl2_set_stream_rescue (which, with
// sl2_get_stream_rescue, ends this file).
//
// M = the job slots r < nsel whose feature has found == 2 (rejected by the consensus), in rank order (match j,
// k = |M| <= SL2_MAX_MEASURED); x', P' are the state and covariance after the first update (its finish included).
// Per match j, every operation one correctly rounded, never-fused op (rd), in this order (tests/rescue_ref.py and
// tests/rescue_oracle.cpp restate it):
//   predict_feature(x', P', y'_j) (sl2_model.cuh, predict_kernel's own code): h', dh/dxp', dh/dy', R' = var' I,
//   S' = H' P' H'^T + R', depth' = camera-frame depth of y'_j;
//   nu0 = z_u - h'0, nu1 = z_v - h'1 (z: the consensus's match, sub-pixel when refined);  (Si00, Si01, Si11) = sinv_from_S(S'00, S'10, S'11);
//   w0 = Si00 nu0 + Si01 nu1;  w1 = Si01 nu0 + Si11 nu1;  q = nu0 w0 + nu1 w1;
//   rescued iff depth' > 0 and q <= chi2 (NaN: never): found = SL2_FOUND_RESCUED, and h, S, Rvar, dh_dxp, dh_dy take
//   the re-prediction.
// Before the decisions, a stream with k > 0 keeps its first update's NIS and log det S (update_sums over G and Wp, as
// record_kernel forms them) in the rescue scratch: the second update overwrites G and Wp.
// Then sl2_launch_update_rescued runs the five update kernels over the rescued rows (update.cu).
#include <cmath>

#include "sl2_context.cuh"
#include "sl2_model.cuh"

using namespace sl2;

namespace {

constexpr int RESC_THREADS = 256;  // update_sums reduces over 256 slots; the gather needs SL2_MAX_MEASURED threads
static_assert(SL2_MAX_MEASURED <= RESC_THREADS, "one thread per job slot");

__global__ void __launch_bounds__(RESC_THREADS) rescue_kernel(const Sl2Dev d, int stream_lo, const double *chi2,
                                                              const double *tau2, double *nis1, double *logdet1,
                                                              const Sl2Subpix sp) {
  pdl_prologue();
  const int s = stream_lo + blockIdx.x;
  const double c2 = chi2[s];
  if (!(c2 > 0.0) || !(tau2[s] > 0.0)) return;
  const int tid = threadIdx.x;
  const int ld = d.ld;
  const size_t fb = (size_t)s * d.Nmax;
  const double *P = d.P + (size_t)s * ld * ld;
  const double *x = d.x + (size_t)s * ld;

  __shared__ int mf[SL2_MAX_MEASURED];
  __shared__ int wcount[RESC_THREADS / 32];
  __shared__ double s_nis[RESC_THREADS], s_ld[RESC_THREADS];
  __shared__ double Pxx[169], xv[SL2_NXV];
  __shared__ Sl2StreamCam sc;

  // ---- M in rank order (job slots < nsel <= kmax <= SL2_MAX_MEASURED) ---------------------------------------------
  const int nsel = d.nsel[s];
  int feat = -1;
  if (tid < d.Nmax && tid < nsel) {
    const int i = d.job_feat[fb + tid];
    if (i >= 0 && d.found[fb + i] == 2) feat = i;
  }
  const int k = block_gather(feat, mf, wcount, RESC_THREADS / 32);
  if (k == 0) return;  // block-uniform
  load_stream_cam(d, s, sc);
  for (int e = tid; e < 169; e += RESC_THREADS) Pxx[e] = P[(e % 13) + (size_t)ld * (e / 13)];
  if (tid < SL2_NXV) xv[tid] = x[tid];

  // ---- the first update's terms, for the step record ---------------------------------------------------------------
  update_sums(d, s, d.upd_m[s], SL2_NXV + 3 * d.nfeat[s], s_nis, s_ld);  // its barriers publish the loads above
  if (tid == 0) {
    nis1[s] = s_nis[0];
    logdet1[s] = mul_(2.0, s_ld[0]);
  }

  // ---- the gate, one thread per rejected match ---------------------------------------------------------------------
  for (int j = tid; j < k; j += RESC_THREADS) {
    const int i = mf[j];
    const size_t g = fb + i;
    const int pos = SL2_NXV + 3 * i;
    const rd yi[3] = {rd(x[pos]), rd(x[pos + 1]), rd(x[pos + 2])};
    FeatPred fp;
    predict_feature(sc.cam, xv, yi, Pxx, P + (size_t)ld * pos, ld, pos, fp);
    const rd nu0 = rd(match_z(d, sp, g, 0)) - fp.h[0], nu1 = rd(match_z(d, sp, g, 1)) - fp.h[1];
    rd si[3];
    sinv_from_S(fp.S[0][0], fp.S[1][0], fp.S[1][1], si);
    const rd w0 = si[0] * nu0 + si[1] * nu1, w1 = si[1] * nu0 + si[2] * nu1;
    const rd q = nu0 * w0 + nu1 * w1;
    if (fp.depth.v > 0.0 && q.v <= c2) {
      d.found[g] = SL2_FOUND_RESCUED;
      d.h[g * 2 + 0] = fp.h[0].v;
      d.h[g * 2 + 1] = fp.h[1].v;
      for (int r = 0; r < 2; ++r) {
        for (int c = 0; c < 7; ++c) d.dh_dxp[g * 14 + r * 7 + c] = fp.dxp[r][c].v;
        for (int c = 0; c < 3; ++c) d.dh_dy[g * 6 + r * 3 + c] = fp.dy[r][c].v;
      }
      d.Rvar[g] = fp.var.v;
      d.S[g * 4 + 0] = fp.S[0][0].v;
      d.S[g * 4 + 1] = fp.S[1][0].v;
      d.S[g * 4 + 2] = fp.S[0][1].v;
      d.S[g * 4 + 3] = fp.S[1][1].v;
    }
  }
}

}  // namespace

cudaError_t sl2_launch_rescue(const Sl2Dev &d, int stream_lo, int stream_cnt, const Sl2Rescue &r, const Sl2Subpix &sp,
                              Sl2Queue q) {
  if (stream_cnt <= 0) return cudaSuccess;
  const cudaError_t e = sl2_launch_kernel(rescue_kernel, dim3(stream_cnt), dim3(RESC_THREADS), 0, q,
                                          sl2_use_pdl(stream_cnt), d, stream_lo, r.chi2, r.tau2, r.nis1, r.logdet1, sp);
  if (e != cudaSuccess) return e;
  return sl2_launch_update_rescued(d, stream_lo, stream_cnt, r.m2, sp, q);
}

namespace sl2 {

Sl2Rescue rescue_args(const sl2_ctx *c) {
  Sl2Rescue r = c->resc_dev;
  r.chi2 = c->resc_chi2_dev;
  r.tau2 = c->cons_tau2;
  return r;
}

int rescue_streams(sl2_ctx *c, int lo, int cnt, Sl2Queue q) {
  CU_TRY(c, sl2_launch_rescue(c->d, lo, cnt, rescue_args(c), subpixel_args(c, lo, cnt), q));
  return SL2_OK;
}

}  // namespace sl2

extern "C" {

int sl2_set_stream_rescue(sl2_ctx *c, int32_t s, double chi2) {
  if (bad_stream(c, s)) return fail(c, SL2_ERR_ARG, "sl2_set_stream_rescue: bad stream");
  if (!std::isfinite(chi2) || chi2 < 0.0)
    return fail(c, SL2_ERR_ARG, "sl2_set_stream_rescue: chi2 must be finite and >= 0");
  const double v = chi2 == 0.0 ? 0.0 : chi2;  // -0 is off like +0
  if (v > 0.0 && !c->resc_buf) {
    const size_t B = c->d.B;
    Sl2Rescue &r = c->resc_dev;
    const int rc = alloc_sections(
        c, c->resc_buf, {{&r.nis1, B * sizeof(double)}, {&r.logdet1, B * sizeof(double)}, {&r.m2, B * sizeof(int)}});
    if (rc) return rc;
  }
  // a pageable copy has read v when it returns; ordered on the stream like a launch, and no launch of its own
  CU_TRY(c, cudaMemcpyAsync(c->resc_chi2_dev + s, &v, sizeof(double), cudaMemcpyHostToDevice, c->stream));
  c->opt[s].chi2 = v;
  return SL2_OK;
}

int sl2_get_stream_rescue(sl2_ctx *c, int32_t s, double *chi2) {
  if (bad_stream(c, s) || !chi2) return fail(c, SL2_ERR_ARG, "sl2_get_stream_rescue: bad argument");
  *chi2 = c->opt[s].chi2;
  return SL2_OK;
}

}  // extern "C"
