// iterate.cu — the iterated EKF update on sm_90a: Gauss-Newton on the posterior cost (Bell & Cathey, IEEE TAC 1993),
// before the fused step's update.  Semantics: include/sl2b200.h, sl2_set_stream_iterated (which, with
// sl2_get_stream_iterated and sl2_get_iterated_results, ends this file).
//
// An iteration pass i is upd_hp + upd_chol (update.cu, sl2_launch_iterate_factor) at the stream's linearisation L_i,
// then iterate_kernel, one CTA per stream.  After upd_chol, G holds U (U^T U = S_i) in the upper triangle of its S
// block, H_i P0 in its H P block and nu_i in column m + n; Wp holds W_pp = U_pp^-T of every 16-row panel, lower
// triangular and zero past a ragged panel's rows.  That is all the pass needs: t = S^-1 nu by two panel-serial
// triangular solves on one vector, then x_{i+1} = x0 + (H P0)^T t; upd_solve does not run.  Then the step test and, if
// the stream iterates on, the rows of M relinearised at x_{i+1} with predict_kernel's model code (measure_feature,
// sl2_model.cuh) into the iteration's feature-indexed tables, which upd_hp reads from the next pass on.
#include <cmath>

#include "sl2_context.cuh"
#include "sl2_model.cuh"

using namespace sl2;

namespace {

constexpr int IT_THREADS = 256;  // one thread per row (m <= 256) of the solves
static_assert(2 * SL2_MAX_MEASURED <= IT_THREADS, "one thread per measurement row");

__global__ void __launch_bounds__(IT_THREADS) iterate_kernel(const Sl2Dev d, int stream_lo, const Sl2Iter it) {
  pdl_prologue();
  const int s = stream_lo + blockIdx.x;
  const int N = it.max_it[s];
  const int pass = it.pass;
  if (N <= 0 || pass >= N || (pass > 0 && !it.active[s])) return;  // block-uniform
  const int tid = threadIdx.x;
  const int m = d.upd_m[s];
  if (m == 0) {  // pass 0 of a stream that measured nothing
    if (tid == 0) {
      it.active[s] = 0;
      it.iters[s] = 0;
      it.status[s] = 0;
      it.delta[s] = 0.0;
    }
    return;
  }
  const int ld = d.ld, ldg = d.ldg;
  const int n = SL2_NXV + 3 * d.nfeat[s];
  const size_t fb = (size_t)s * d.Nmax;
  const double *__restrict__ G = d.G + (size_t)s * d.mmax * ldg;
  const double *__restrict__ Wp = d.Wp + (size_t)s * SL2_MAX_PANELS * 256;
  const double *__restrict__ P = d.P + (size_t)s * ld * ld;
  const double *__restrict__ x0 = d.x + (size_t)s * ld;
  double *__restrict__ xi = it.x + (size_t)s * ld;

  __shared__ double v[IT_THREADS];
  __shared__ double red[IT_THREADS];
  __shared__ double xn[SL2_NXV];
  __shared__ int mf[SL2_MAX_MEASURED];
  __shared__ int wcount[IT_THREADS / 32];
  __shared__ double th[SL2_MAX_MEASURED][2], tx[SL2_MAX_MEASURED][14], ty[SL2_MAX_MEASURED][6];
  __shared__ Sl2StreamCam sc;

  // ---- t = S^-1 nu: U^T w = nu panel by panel (w_p = W_pp r_p, then every later row r_j -= U(p0 + a, j) w_a), then
  // U t = w from the last panel (t_p = W_pp^T r_p, then every earlier row r_j -= U(j, p0 + a) t_a) -----------------
  if (tid < m) v[tid] = G[(size_t)tid * ldg + m + n];
  __syncthreads();
  const int np = (m + 15) >> 4;
  for (int p = 0; p < np; ++p) {
    const int p0 = 16 * p, nb = min(16, m - p0);
    const double *Wpp = Wp + (size_t)p * 256;
    double w = 0.0;
    if (tid < nb) {
      w = mul_(Wpp[tid * 16], v[p0]);
      for (int b = 1; b < nb; ++b) w = add_(w, mul_(Wpp[tid * 16 + b], v[p0 + b]));
    }
    __syncthreads();
    if (tid < nb) v[p0 + tid] = w;
    __syncthreads();
    if (tid >= p0 + nb && tid < m) {
      double r = v[tid];
      for (int a = 0; a < nb; ++a) r = sub_(r, mul_(G[(size_t)(p0 + a) * ldg + tid], v[p0 + a]));
      v[tid] = r;
    }
    __syncthreads();
  }
  for (int p = np - 1; p >= 0; --p) {
    const int p0 = 16 * p, nb = min(16, m - p0);
    const double *Wpp = Wp + (size_t)p * 256;
    double t = 0.0;
    if (tid < nb) {
      t = mul_(Wpp[tid], v[p0]);
      for (int b = 1; b < nb; ++b) t = add_(t, mul_(Wpp[b * 16 + tid], v[p0 + b]));
    }
    __syncthreads();
    if (tid < nb) v[p0 + tid] = t;
    __syncthreads();
    if (tid < p0) {
      double r = v[tid];
      for (int a = 0; a < nb; ++a) r = sub_(r, mul_(G[(size_t)tid * ldg + p0 + a], v[p0 + a]));
      v[tid] = r;
    }
    __syncthreads();
  }

  // ---- x_{i+1} = x0 + (H P0)^T t, the step delta_i and the finiteness of x_{i+1} ----------------------------------
  double dmax = 0.0;
  bool fin = true;
  for (int j = tid; j < n; j += IT_THREADS) {
    double acc = mul_(G[(size_t)m + j], v[0]);
    for (int r = 1; r < m; ++r) acc = add_(acc, mul_(G[(size_t)r * ldg + m + j], v[r]));
    const double xnew = add_(x0[j], acc);
    const double xold = pass == 0 ? x0[j] : xi[j];
    const double pjj = P[(size_t)j * ld + j];
    if (pjj > 0.0) dmax = fmax(dmax, div_(fabs(sub_(xnew, xold)), sqrt_(pjj)));
    fin = fin && isfinite(xnew);
    xi[j] = xnew;
    if (j < SL2_NXV) xn[j] = xnew;
  }
  red[tid] = dmax;
  const int all_fin = __syncthreads_and(fin);
  for (int h = IT_THREADS / 2; h > 0; h >>= 1) {
    if (tid < h) red[tid] = fmax(red[tid], red[tid + h]);
    __syncthreads();
  }
  const double delta = all_fin ? red[0] : NAN;  // a non-finite x_{i+1}: NaN, never converged, then invalid
  if (delta <= it.tol[s]) {  // converged: the final update uses L_i (block-uniform)
    if (tid == 0) {
      it.active[s] = 0;
      if (pass == 0) it.iters[s] = 0;
      it.status[s] = 1;
      it.delta[s] = delta;
    }
    return;
  }

  // ---- relinearise every row of M at x_{i+1} (M: job slots r < nsel with found == 1, in rank order) ---------------
  const int nsel = d.nsel[s];
  int feat = -1;
  if (tid < d.Nmax && tid < nsel) {
    const int i = d.job_feat[fb + tid];
    if (i >= 0 && d.found[fb + i] == 1) feat = i;
  }
  const int K = block_gather(feat, mf, wcount, IT_THREADS / 32);
  load_stream_cam(d, s, sc);
  __syncthreads();  // mf, sc, xn and this block's writes of x_{i+1} are visible
  bool ok = all_fin != 0;
  for (int k = tid; k < K; k += IT_THREADS) {
    const int pos = SL2_NXV + 3 * mf[k];
    const rd y[3] = {rd(xi[pos]), rd(xi[pos + 1]), rd(xi[pos + 2])};
    rd h[2], dxp[2][7], dy[2][3], depth;
    measure_feature(sc.cam, xn, y, h, dxp, dy, depth);
    rd dx[7], dyv[3];
    for (int c = 0; c < 7; ++c) dx[c] = rd(x0[c]) - rd(xn[c]);
    for (int c = 0; c < 3; ++c) dyv[c] = rd(x0[pos + c]) - y[c];
    bool good = depth.v > 0.0;
    for (int r = 0; r < 2; ++r) {
      rd acc = dxp[r][0] * dx[0];
      for (int c = 1; c < 7; ++c) acc = acc + dxp[r][c] * dx[c];
      for (int c = 0; c < 3; ++c) acc = acc + dy[r][c] * dyv[c];
      th[k][r] = (h[r] + acc).v;
      good = good && isfinite(th[k][r]);
      for (int c = 0; c < 7; ++c) {
        tx[k][r * 7 + c] = dxp[r][c].v;
        good = good && isfinite(dxp[r][c].v);
      }
      for (int c = 0; c < 3; ++c) {
        ty[k][r * 3 + c] = dy[r][c].v;
        good = good && isfinite(dy[r][c].v);
      }
    }
    ok = ok && good;
  }
  if (!__syncthreads_and(ok)) {  // invalid: the final update uses L_i
    if (tid == 0) {
      it.active[s] = 0;
      if (pass == 0) it.iters[s] = 0;
      it.status[s] = 3;
      it.delta[s] = delta;
    }
    return;
  }
  for (int e = tid; e < K * 22; e += IT_THREADS) {
    const int k = e / 22, q = e - k * 22;
    const size_t f = fb + mf[k];
    if (q < 2) it.h[f * 2 + q] = th[k][q];
    else if (q < 16) it.Hxp[f * 14 + q - 2] = tx[k][q - 2];
    else it.Hy[f * 6 + q - 16] = ty[k][q - 16];
  }
  if (tid == 0) {
    const bool last = pass + 1 >= N;
    it.active[s] = last ? 0 : 1;
    it.iters[s] = pass + 1;
    it.status[s] = last ? 2 : 0;
    it.delta[s] = delta;
  }
}

// the most iteration passes any stream of [lo, lo + cnt) runs
int iter_passes(const sl2_ctx *c, int lo, int cnt) {
  int N = 0;
  for (int s = lo; s < lo + cnt; ++s) N = std::max(N, (int)c->opt[s].iter.max_iterations);
  return N;
}

}  // namespace

cudaError_t sl2_launch_iterate_pass(const Sl2Dev &d, int stream_lo, int stream_cnt, const Sl2Subpix &sp,
                                    const Sl2Iter &it, Sl2Queue q) {
  if (stream_cnt <= 0) return cudaSuccess;
  const cudaError_t e = sl2_launch_iterate_factor(d, stream_lo, stream_cnt, sp, it, q);
  if (e != cudaSuccess) return e;
  return sl2_launch_kernel(iterate_kernel, dim3(stream_cnt), dim3(IT_THREADS), 0, q, sl2_use_pdl(stream_cnt), d,
                           stream_lo, it);
}

namespace sl2 {

Sl2Iter iterate_args(const sl2_ctx *c, int lo, int cnt) {
  if (!c->iter_buf || iter_passes(c, lo, cnt) == 0) return {};
  return c->iter_dev;  // pass -1
}

int iterate_streams(sl2_ctx *c, int lo, int cnt, Sl2Queue q) {
  const int N = c->iter_buf ? iter_passes(c, lo, cnt) : 0;
  if (N == 0) return SL2_OK;
  const Sl2Subpix sp = subpixel_args(c, lo, cnt);
  Sl2Iter it = c->iter_dev;
  for (int i = 0; i < N; ++i) {
    it.pass = i;
    CU_TRY(c, sl2_launch_iterate_pass(c->d, lo, cnt, sp, it, q));
  }
  return SL2_OK;
}

}  // namespace sl2

extern "C" {

int sl2_set_stream_iterated(sl2_ctx *c, int32_t s, const sl2_stream_iterated *v) {
  if (bad_stream(c, s) || !v) return fail(c, SL2_ERR_ARG, "sl2_set_stream_iterated: bad argument");
  if (v->reserved != 0 || v->max_iterations < 0 || v->max_iterations > SL2_MAX_ITERATIONS)
    return fail(c, SL2_ERR_ARG, "sl2_set_stream_iterated: max_iterations must be in [0, SL2_MAX_ITERATIONS], reserved 0");
  if (!std::isfinite(v->tol) || !(v->tol >= 0.0))
    return fail(c, SL2_ERR_ARG, "sl2_set_stream_iterated: tol must be finite and >= 0");
  sl2_stream_iterated w = *v;
  if (w.tol == 0.0) w.tol = 0.0;  // -0 like +0
  if (w.max_iterations > 0 && !c->iter_buf) {
    const size_t B = c->d.B, F = (size_t)c->d.B * c->d.Nmax;
    Sl2Iter &t = c->iter_dev;  // pass -1: the final update
    const int rc = alloc_sections(c, c->iter_buf,
                                  {{&t.max_it, B * sizeof(int)}, {&t.tol, B * sizeof(double)},
                                   {&t.h, F * 2 * sizeof(double)}, {&t.Hxp, F * 14 * sizeof(double)},
                                   {&t.Hy, F * 6 * sizeof(double)}, {&t.x, B * (size_t)c->d.ld * sizeof(double)},
                                   {&t.active, B * sizeof(int)}, {&t.iters, B * sizeof(int)},
                                   {&t.status, B * sizeof(int)}, {&t.delta, B * sizeof(double)}});
    if (rc) return rc;
    t.pass = -1;
  }
  if (c->iter_buf) {  // pageable copies have read their sources when they return; ordered on the stream, no launch
    const int nmax = w.max_iterations;
    CU_TRY(c, cudaMemcpyAsync(c->iter_dev.max_it + s, &nmax, sizeof(int), cudaMemcpyHostToDevice, c->stream));
    CU_TRY(c, cudaMemcpyAsync(c->iter_dev.tol + s, &w.tol, sizeof(double), cudaMemcpyHostToDevice, c->stream));
    // the results describe steps the stream ran with this setting
    CU_TRY(c, cudaMemsetAsync(c->iter_dev.iters + s, 0, sizeof(int), c->stream));
    CU_TRY(c, cudaMemsetAsync(c->iter_dev.status + s, 0, sizeof(int), c->stream));
    CU_TRY(c, cudaMemsetAsync(c->iter_dev.delta + s, 0, sizeof(double), c->stream));
  }
  c->opt[s].iter = w;
  return SL2_OK;
}

int sl2_get_stream_iterated(sl2_ctx *c, int32_t s, sl2_stream_iterated *v) {
  if (bad_stream(c, s) || !v) return fail(c, SL2_ERR_ARG, "sl2_get_stream_iterated: bad argument");
  *v = c->opt[s].iter;
  return SL2_OK;
}

int sl2_get_iterated_results(sl2_ctx *c, int32_t lo, int32_t cnt, int32_t *iterations, int32_t *status,
                             double *last_delta) {
  if (bad_range(c, lo, cnt)) return fail(c, SL2_ERR_ARG, "sl2_get_iterated_results: bad range");
  const Sl2Iter &t = c->iter_dev;
  return read_results(c, c->iter_buf != nullptr, lo, cnt,
                      {{iterations, t.iters, sizeof(int)}, {status, t.status, sizeof(int)},
                       {last_delta, t.delta, sizeof(double)}});
}

}  // extern "C"
