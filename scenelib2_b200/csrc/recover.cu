// recover.cu — stream recovery inside the fused step on sm_90a: a per-stream loss detector that stops the selection of
// a lost stream (so the cull keeps its map) and tries the relocalisation of reloc.cu on the step's own frame.
// Semantics and the order of every operation: include/sl2b200.h, sl2_set_stream_recovery (which, with the other
// recovery entry points, ends this file); tests/recovery_ref.py restates the decision rule.
//
// At the end of the step of a group holding a stream with recovery on (after the cull and the records), three launches:
//   recover_kernel: one CTA per stream of the group.  Thread 0 applies rules 1-2 to the stream's state from the step's
//     nmeas and sets `attempted`; then the threads write the stream's row of the job table: for a stream that tries,
//     one full-image job per map feature (the jobs sl2_relocalise packs on the host), else -1 everywhere, so the
//     search's warps of that stream return at once.
//   the full-image search (search.cu) over the job table, into the recovery's own outputs: the step's job slots and
//     per-feature results are not touched.
//   reloc_kernel (reloc.cu) with the states: a stream that does not try returns at once; a try writes its result into
//     the state and, when accepted, the stream's x and P and its return to tracking.
// predict_kernel (ekf.cu) reads the states' lost flags at the next step: a lost stream selects nothing.
#include <algorithm>
#include <cmath>

#include "sl2_context.cuh"

using namespace sl2;

namespace {

constexpr int RECOVER_THREADS = 128;  // job slots per pass

struct RecoverLaunch {
  int stream_lo;
  const sl2_stream_recovery *set;  // [B]
  sl2_recovery_result *state;      // [B]
  int *job_feat;                   // [B][Nmax]
  double *job_centre, *job_puinv;  // [B][Nmax][2], [B][Nmax][3]
};

__global__ void __launch_bounds__(RECOVER_THREADS) recover_kernel(const Sl2Dev d, const RecoverLaunch R) {
  pdl_prologue();
  const int s = R.stream_lo + blockIdx.x;
  const int tid = threadIdx.x;
  __shared__ int s_try;
  if (tid == 0) {
    int tries = 0;
    const int lost_after = R.set[s].lost_after;
    if (lost_after > 0) {
      sl2_recovery_result &st = R.state[s];
      if (st.lost) {  // 2. entered the step lost
        st.lost_steps += 1;
        tries = st.lost_steps % R.set[s].retry_period == 0;
      } else {  // 1. entered the step tracking
        st.failed_steps = d.nmeas[s] < R.set[s].min_matches ? st.failed_steps + 1 : 0;
        if (st.failed_steps >= lost_after) {
          st.lost = 1;
          st.lost_steps = 0;
          tries = 1;
        }
      }
      st.attempted = tries;
    }
    s_try = tries;
  }
  __syncthreads();
  const int tries = s_try, nf = d.nfeat[s];
  const size_t jb = (size_t)s * d.Nmax;
  // 3. the full-image job of sl2_relocalise: centre ((w - 1) / 2, (h - 1) / 2), PuInv = diag(eps, eps) with
  // eps = 9 / (w w + h h), every operation correctly rounded as on the host
  const Sl2StreamCam &cam = d.cams[s];
  const int w = (int)cam.cam[0], h = (int)cam.cam[1];
  const double eps = (rd(9.0) / (rd((double)w) * rd((double)w) + rd((double)h) * rd((double)h))).v;
  const double cx = 0.5 * (double)(w - 1), cy = 0.5 * (double)(h - 1);
  for (int f = tid; f < d.Nmax; f += RECOVER_THREADS) {
    R.job_feat[jb + f] = tries && f < nf ? f : -1;
    if (tries) {
      R.job_centre[(jb + f) * 2 + 0] = cx;
      R.job_centre[(jb + f) * 2 + 1] = cy;
      R.job_puinv[(jb + f) * 3 + 0] = eps;
      R.job_puinv[(jb + f) * 3 + 1] = 0.0;
      R.job_puinv[(jb + f) * 3 + 2] = eps;
    }
  }
}

// the setting's checks of include/sl2b200.h; an empty string when it is accepted
std::string recovery_setting_error(const sl2_stream_recovery *r) {
  if (r->reserved != 0) return "reserved must be 0";
  if (r->lost_after < 0) return "lost_after must be >= 0";
  if (r->lost_after == 0) return "";
  if (r->min_matches < 1 || r->retry_period < 1) return "min_matches and retry_period must be >= 1";
  return reloc_params_error(&r->reloc, r->Pxx);
}

}  // namespace

namespace sl2 {

const sl2_recovery_result *recovery_args(const sl2_ctx *c, int lo, int cnt) {
  return any_stream(c, lo, cnt, [](const StreamOptions &o) { return o.recov.lost_after > 0; }) ? c->recov_state
                                                                                                 : nullptr;
}

int recover_streams(sl2_ctx *c, int slot, int lo, int cnt, Sl2Queue q) {
  const Sl2Dev &d = c->d;
  const size_t jb = (size_t)lo * d.Nmax;
  RecoverLaunch R = {};
  R.stream_lo = lo;
  R.set = c->recov_set;
  R.state = c->recov_state;
  R.job_feat = c->recov_job_feat;
  R.job_centre = c->recov_job_centre;
  R.job_puinv = c->recov_job_puinv;
  CU_TRY(c, sl2_launch_kernel(recover_kernel, dim3(cnt), dim3(RECOVER_THREADS), 0, q, sl2_use_pdl(cnt), d, R));
  SearchLaunch L = {};
  L.job_feat = c->recov_job_feat + jb;
  L.job_centre = c->recov_job_centre + jb * 2;
  L.job_puinv = c->recov_job_puinv + jb * 3;
  L.jobs_per_stream = d.Nmax;
  L.stream_lo = lo;
  L.stream_cnt = cnt;
  L.slot = slot;
  L.out_uv = c->recov_uv + jb * 2;
  L.out_found = c->recov_found + jb;
  L.scatter_to_features = 0;
  CU_TRY(c, sl2_launch_search(d, c->tmap, L, q));
  CU_TRY(c, sl2_launch_reloc(d, cnt, nullptr, lo, L.out_uv, L.out_found, &c->recov_set[0].reloc, c->recov_set[0].Pxx,
                             sizeof(sl2_stream_recovery), nullptr, c->recov_zuv + jb * 2, c->recov_flags + jb,
                             c->recov_state, q));
  return SL2_OK;
}

int recovery_reset(sl2_ctx *c, int lo, int cnt) {
  if (!c->recov_buf || cnt <= 0) return SL2_OK;
  // lost, failed_steps, lost_steps: the leading three fields of each state
  CU_TRY(c, cudaMemset2DAsync(c->recov_state + lo, sizeof(sl2_recovery_result), 0, 3 * sizeof(int32_t), cnt,
                              c->stream));
  return SL2_OK;
}

}  // namespace sl2

extern "C" {

int sl2_set_stream_recovery(sl2_ctx *c, int32_t s, const sl2_stream_recovery *r) {
  if (bad_stream(c, s) || !r) return fail(c, SL2_ERR_ARG, "sl2_set_stream_recovery: bad argument");
  const std::string why = recovery_setting_error(r);
  if (!why.empty()) return fail(c, SL2_ERR_ARG, "sl2_set_stream_recovery: " + why);
  if (r->lost_after > 0 && !c->recov_buf) {
    const size_t B = c->d.B, BN = (size_t)c->d.B * c->d.Nmax;
    const int rc = alloc_sections(
        c, c->recov_buf,
        {{&c->recov_set, B * sizeof(sl2_stream_recovery)}, {&c->recov_state, B * sizeof(sl2_recovery_result)},
         {&c->recov_job_feat, BN * sizeof(int)}, {&c->recov_job_centre, BN * 2 * sizeof(double)},
         {&c->recov_job_puinv, BN * 3 * sizeof(double)}, {&c->recov_uv, BN * 2 * sizeof(int)}, {&c->recov_found, BN},
         {&c->recov_zuv, BN * 2 * sizeof(int)}, {&c->recov_flags, BN}});
    if (rc) return rc;
  }
  if (c->recov_buf) {  // pageable copies have read their sources when they return; ordered on the stream, no launch
    CU_TRY(c, cudaMemcpyAsync(c->recov_set + s, r, sizeof *r, cudaMemcpyHostToDevice, c->stream));
    CU_TRY(c, cudaMemsetAsync(c->recov_state + s, 0, sizeof(sl2_recovery_result), c->stream));  // tracking, no result
  }
  c->opt[s].recov = *r;
  return SL2_OK;
}

int sl2_get_stream_recovery(sl2_ctx *c, int32_t s, sl2_stream_recovery *r) {
  if (bad_stream(c, s) || !r) return fail(c, SL2_ERR_ARG, "sl2_get_stream_recovery: bad argument");
  *r = c->opt[s].recov;
  return SL2_OK;
}

int sl2_get_recovery_results(sl2_ctx *c, int32_t lo, int32_t cnt, sl2_recovery_result *out) {
  if (bad_range(c, lo, cnt) || (cnt > 0 && !out)) return fail(c, SL2_ERR_ARG, "sl2_get_recovery_results: bad argument");
  return read_results(c, c->recov_buf != nullptr, lo, cnt, {{out, c->recov_state, sizeof(sl2_recovery_result)}});
}

}  // extern "C"
