// records.cu — step records: one sl2_step_record per camera stream per fused step, written into the ring Sl2Dev::rec
// by one CTA per stream after the cull (include/sl2b200.h).  The kernel reads and writes nothing but the ring.
//
// Where the update leaves what the record needs (update.cu), for the step's m = upd_m rows:
//   w = U^-T nu   upd_solve writes Y = U^-T [H P | nu] over the [H P | nu] part of G, so w_i = G(i, m + n) with
//                 n = 13 + 3 nfeat the state size OF THE UPDATE.  The cull ran in between and deleted ncull features,
//                 so n = 13 + 3 (nfeat + ncull).  NIS = nu^T S^-1 nu = w^T w.
//   U_ii          upd_chol leaves U (true diagonal) in G's S block, but the cull uses row 0 of G as scratch when it
//                 deletes features, which overwrites U_00.  upd_chol also keeps W_pp = U_pp^-T of every 16-row panel in
//                 Sl2Dev::Wp for the solve, and nothing else writes Wp: its diagonal holds the reciprocal pivots
//                 W_ii = 1 / U_ii the solve applied.  log det S = 2 sum log U_ii = -2 sum log W_ii.
// When m == 0 the update wrote neither G nor Wp (they hold another update's values) and the kernel reads neither.
// A step that ran the consensus rescue's second update (rescue.cu) overwrote G and Wp with its rows; rescue_kernel kept
// the first update's NIS and log det S, and the record holds the sums of both updates' rows and terms.
// Entry points: sl2_enable_records (the ring) and sl2_get_records* (the most recent records, oldest first).
#include <algorithm>

#include "sl2_context.cuh"

using namespace sl2;

namespace {

constexpr int REC_THREADS = 256;  // one thread per row of S: m <= 2 * SL2_MAX_MEASURED
static_assert(2 * SL2_MAX_MEASURED <= REC_THREADS, "one thread per measurement row");
static_assert(sizeof(sl2_step_record) == 256, "sl2_step_record is 256 bytes without padding");

static_assert(REC_THREADS == 256, "update_sums reduces over 256 slots");

// With the consensus rescue's scratch (resc), a stream whose step ran a second update (m2[s] > 0) records the sums of
// both: G and Wp hold the second update's rows, the scratch the first's NIS and log det S.
__global__ void __launch_bounds__(REC_THREADS) record_kernel(const Sl2Dev d, int stream_lo, long long step,
                                                             const int *resc_m2, const double *resc_nis1,
                                                             const double *resc_logdet1) {
  pdl_prologue();
  const int s = stream_lo + blockIdx.x, tid = threadIdx.x;
  __shared__ double s_nis[REC_THREADS], s_ld[REC_THREADS];
  const int m = d.upd_m[s], nf = d.nfeat[s], nc = d.ncull[s];
  const int m2 = resc_m2 ? resc_m2[s] : 0;
  update_sums(d, s, m2 > 0 ? m2 : m, SL2_NXV + 3 * (nf + nc), s_nis, s_ld);
  sl2_step_record *r = d.rec + (size_t)s * d.rec_depth + (size_t)(step % d.rec_depth);
  if (tid < SL2_NXV) {
    const size_t ld = d.ld;
    r->xv[tid] = d.x[(size_t)s * ld + tid];
    r->pxx_diag[tid] = d.P[(size_t)s * ld * ld + (size_t)tid * (ld + 1)];
  } else if (tid == 32) {
    r->step = step;
    r->nfeat = nf;
    r->nvisible = d.nvisible[s];
    r->nsel = d.nsel[s];
    r->nmeas = d.nmeas[s];
    r->nculled = nc;
    if (m2 > 0) {
      r->m = m + m2;
      r->nis = add_(resc_nis1[s], s_nis[0]);
      r->logdet_s = add_(resc_logdet1[s], mul_(2.0, s_ld[0]));
    } else {
      r->m = m;
      r->nis = s_nis[0];
      r->logdet_s = mul_(2.0, s_ld[0]);
    }
  }
}

}  // namespace

cudaError_t sl2_launch_records(const Sl2Dev &d, int stream_lo, int stream_cnt, int64_t step, const Sl2Rescue *resc,
                               Sl2Queue q) {
  if (stream_cnt <= 0) return cudaSuccess;
  return sl2_launch_kernel(record_kernel, dim3(stream_cnt), dim3(REC_THREADS), 0, q, sl2_use_pdl(stream_cnt), d,
                           stream_lo, (long long)step, resc ? resc->m2 : nullptr, resc ? resc->nis1 : nullptr,
                           resc ? resc->logdet1 : nullptr);
}

extern "C" {

int sl2_enable_records(sl2_ctx *c, int32_t depth) {
  if (!c) return SL2_ERR_ARG;
  enter(c);
  if (depth < 0 || depth > SL2_MAX_RECORDS)
    return fail(c, SL2_ERR_ARG, "sl2_enable_records: depth outside [0, SL2_MAX_RECORDS]");
  // the new ring first, so that a failed allocation leaves the old one in place
  DevPtr<sl2_step_record> ring;
  cudaError_t e = cudaSuccess;
  if (depth) {
    const size_t bytes = (size_t)c->d.B * depth * sizeof(sl2_step_record);
    CU_TRY(c, cuda_malloc(ring, bytes));
    e = cudaMemsetAsync(ring.get(), 0, bytes, c->stream);
  }
  // steps queued before the call (either group: enter() joined them) have written the old ring
  if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
  if (e != cudaSuccess) return fail(c, SL2_ERR_CUDA, std::string("sl2_enable_records: ") + cudaGetErrorString(e));
  c->rec = std::move(ring);
  c->d.rec = c->rec.get();
  c->d.rec_depth = depth;
  c->rec_steps = 0;
  return SL2_OK;
}

// The most recent k records of streams [lo, lo + cnt), oldest first, as one or two 2-D copies (two when the k rows
// wrap around the end of the ring): row pitch `depth` records in the ring, `mx` records in the output.
static int get_records(sl2_ctx *c, int32_t lo, int32_t cnt, int32_t mx, void *out, cudaMemcpyKind kind,
                       const char *who) {
  if (bad_range(c, lo, cnt) || !out || mx < 1 ||
      (kind == cudaMemcpyDeviceToDevice && ((uintptr_t)out & 7)))
    return fail(c, SL2_ERR_ARG, std::string(who) + ": bad argument");
  const int64_t depth = c->d.rec_depth;
  if (!depth) return fail(c, SL2_ERR_STATE, std::string(who) + ": records are off (sl2_enable_records)");
  const int k = (int)std::min<int64_t>(std::min<int64_t>(mx, c->rec_steps), depth);
  if (k == 0 || cnt == 0) return k;
  const size_t R = sizeof(sl2_step_record);
  const int r0 = (int)((c->rec_steps - k) % depth);  // ring row of the oldest record returned
  const int k1 = (int)std::min<int64_t>(k, depth - r0);
  const sl2_step_record *src = c->d.rec + (size_t)lo * depth;
  uint8_t *dst = static_cast<uint8_t *>(out);
  CU_TRY(c, cudaMemcpy2DAsync(dst, (size_t)mx * R, src + r0, (size_t)depth * R, (size_t)k1 * R, cnt, kind, c->stream));
  if (k1 < k)
    CU_TRY(c, cudaMemcpy2DAsync(dst + (size_t)k1 * R, (size_t)mx * R, src, (size_t)depth * R, (size_t)(k - k1) * R,
                                cnt, kind, c->stream));
  if (kind == cudaMemcpyDeviceToHost) CU_TRY(c, cudaStreamSynchronize(c->stream));
  return k;
}

int sl2_get_records(sl2_ctx *c, int32_t lo, int32_t cnt, int32_t max, sl2_step_record *out) {
  return get_records(c, lo, cnt, max, out, cudaMemcpyDeviceToHost, "sl2_get_records");
}

int sl2_get_records_dev(sl2_ctx *c, int32_t lo, int32_t cnt, int32_t max, void *out_dev) {
  return get_records(c, lo, cnt, max, out_dev, cudaMemcpyDeviceToDevice, "sl2_get_records_dev");
}

}  // extern "C"
