// select.cu — greedy mutual-information selection on sm_90a: which of a stream's visible features the step measures,
// picked by what each measurement, conditioned on the ones already picked, tells about the state (Davison, "Active
// Search for Real-Time Vision", ICCV 2005).  Semantics: include/sl2b200.h, sl2_set_stream_selection (which, with
// sl2_get_stream_selection, ends this file).
//
// predict_kernel (ekf.cu) leaves, for a stream with SL2_SELECT_INFORMATION, the reference rank rho of every candidate
// in sel_rank.  select_kernel then runs a block-pivoted Cholesky factorisation of the candidates' joint innovation
// covariance H P H^T + R, one 2x2 block per pick:
//   q_j = (C00 C11 - C10 C10) / (R_j R_j) over the unpicked j; the pick i has the largest q_j with C00 > 0 and q_j > t
//   (ties: smallest rho); L_i = chol(C_i); u = P H_i^T on rows 0..6 and every unpicked candidate's y rows;
//   c_j = A_j u[0:7] + B_j u[y_j] - sum_{p<r} g_{j,p} g_{i,p}^T, g_{j,r} = c_j L_i^-T, C_j -= g_{j,r} g_{j,r}^T.
// Every operation is one correctly rounded, never-fused FP64 op (rd) in the order written here; tests/selection_ref.py
// restates them op for op.
// Shape: one CTA of SEL_THREADS per stream (a stream with the setting off returns at once).  Threads span the
// candidates for q, c_j, g and C, and the needed rows for u.  P[:, 0:7] of the needed rows, the Jacobians, C and R are
// staged once in shared memory; the factors g stay there too when they fit (SEL_SMEM_MAX), else in the context's
// scratch [B][kmax][Nmax][4].
#include <algorithm>
#include <cmath>

#include "sl2_context.cuh"
#include "sl2_model.cuh"

using namespace sl2;

namespace {

#define SEL_THREADS 128
#define SEL_WARPS (SEL_THREADS / 32)
// two CTAs per SM: 2 x (113 KB + 1 KB reserved) = the SM's 228 KB
#define SEL_SMEM_MAX (113 * 1024)

// shared memory of a stream with capacity N, without the factors: P rows [7 + 3N][7], u [7 + 3N][2], A [N][14],
// B [N][6], C [N][3], R [N] (doubles), then feat, rho, picked [N] (ints)
size_t sel_base_bytes(int N) { return ((size_t)(7 + 3 * N) * 9 + (size_t)N * 24) * 8 + (size_t)N * 12; }
// the factors g [npick][N][2][2]
size_t sel_g_bytes(int N, int npick) { return (size_t)N * npick * 32; }

// candidate row rr of the needed rows: 0..6 the camera pose, then the three y rows of each candidate
__device__ __forceinline__ int sel_row(int rr, const int *feat) {
  return rr < 7 ? rr : SL2_NXV + 3 * feat[(rr - 7) / 3] + (rr - 7) % 3;
}

// (q, j) beats (bq, bj): a larger q, ties to the smaller reference rank (then the smaller candidate index)
__device__ __forceinline__ bool sel_better(double q, int j, double bq, int bj, const int *rho) {
  if (bj < 0) return true;
  if (q != bq) return q > bq;
  return rho[j] != rho[bj] ? rho[j] < rho[bj] : j < bj;
}

__global__ void __launch_bounds__(SEL_THREADS) select_kernel(const Sl2Dev d, const SelectLaunch L) {
  pdl_prologue();
  const int s = L.stream_lo + blockIdx.x;
  if (L.mode[s] != SL2_SELECT_INFORMATION) return;
  extern __shared__ __align__(16) double sm[];
  __shared__ int wcount[SEL_WARPS], s_rj[SEL_WARPS], s_pick;
  __shared__ double s_rq[SEL_WARPS];
  const int N = d.Nmax, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int ld = d.ld, nf = d.nfeat[s];
  const size_t fb = (size_t)s * N;
  const double *P = d.P + (size_t)s * ld * ld;
  double *Pc = sm;                  // [7 + 3N][7]  P[row][0:7] of the needed rows
  double *u = Pc + (7 + 3 * N) * 7;  // [7 + 3N][2]  P H_i^T of the current pick
  double *A = u + (7 + 3 * N) * 2;   // [N][2][7]    dh_dxp
  double *Bm = A + N * 14;           // [N][2][3]    dh_dy
  double *Cm = Bm + N * 6;           // [N][3]       C00, C10, C11 of the conditioned innovation covariance
  double *R = Cm + N * 3;            // [N]          Rvar
  // [gstride][N][2][2]: pick-major, so the candidates' threads read one pick's factors from consecutive addresses
  double *g = L.g ? L.g + (size_t)s * N * L.gstride * 4 : R + N;
  int *feat = reinterpret_cast<int *>(L.g ? R + N : R + N + (size_t)N * L.gstride * 4);  // [N] ascending features
  int *rho = feat + N;                                                                   // [N] reference ranks
  int *picked = rho + N;                                                                 // [N]

  // ---- the candidates in feature order, every one unselected until picked -----------------------------------------
  int V = 0;
  for (int i0 = 0; i0 < nf; i0 += SEL_THREADS) {
    const int i = i0 + tid;
    const int rk = i < nf ? d.sel_rank[fb + i] : -1;
    int at;
    const int cnt = block_gather(rk >= 0 ? i : -1, feat + V, wcount, SEL_WARPS, &at);
    if (at >= 0) {
      rho[V + at] = rk;
      d.sel_rank[fb + i] = -1;
    }
    V += cnt;
    __syncthreads();  // wcount is rewritten by the next chunk
  }
  for (int j = tid; j < V; j += SEL_THREADS) {
    const size_t gj = fb + feat[j];
    for (int e = 0; e < 14; ++e) A[j * 14 + e] = d.dh_dxp[gj * 14 + e];
    for (int e = 0; e < 6; ++e) Bm[j * 6 + e] = d.dh_dy[gj * 6 + e];
    Cm[j * 3 + 0] = d.S[gj * 4 + 0];
    Cm[j * 3 + 1] = d.S[gj * 4 + 1];
    Cm[j * 3 + 2] = d.S[gj * 4 + 3];
    R[j] = d.Rvar[gj];
    picked[j] = 0;
  }
  const int rows = 7 + 3 * V;
  for (int e = tid; e < rows * 7; e += SEL_THREADS) {  // row fastest: coalesced down each of the 7 columns
    const int k = e / rows, rr = e - k * rows;
    Pc[rr * 7 + k] = P[sel_row(rr, feat) + (size_t)ld * k];
  }
  __syncthreads();

  const int nmax = min(d.cams[s].n_select, V);
  const double t = L.t[s];
  int r = 0;
  for (; r < nmax; ++r) {
    // ---- pick: the largest qualifying q ----------------------------------------------------------------------------
    double bq = 0.0;
    int bj = -1;
    for (int j = tid; j < V; j += SEL_THREADS) {
      if (picked[j]) continue;
      const rd c00(Cm[j * 3 + 0]), c10(Cm[j * 3 + 1]), c11(Cm[j * 3 + 2]), rv(R[j]);
      const double q = ((c00 * c11 - c10 * c10) / (rv * rv)).v;
      if (c00.v > 0.0 && q > t && sel_better(q, j, bq, bj, rho)) {
        bq = q;
        bj = j;
      }
    }
    for (int o = 16; o > 0; o >>= 1) {
      const double oq = __shfl_down_sync(0xffffffffu, bq, o);
      const int oj = __shfl_down_sync(0xffffffffu, bj, o);
      if (oj >= 0 && sel_better(oq, oj, bq, bj, rho)) {
        bq = oq;
        bj = oj;
      }
    }
    if (lane == 0) {
      s_rq[warp] = bq;
      s_rj[warp] = bj;
    }
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < SEL_WARPS; ++w)
        if (s_rj[w] >= 0 && sel_better(s_rq[w], s_rj[w], bq, bj, rho)) {
          bq = s_rq[w];
          bj = s_rj[w];
        }
      s_pick = bj;
      if (bj >= 0) {
        picked[bj] = 1;
        // the job slot exactly as the trace rule writes a selected feature: the centre and ellipse of the prediction
        const int fi = feat[bj];
        const size_t gi = fb + fi, jr = fb + r;
        d.sel_rank[gi] = r;
        d.job_feat[jr] = fi;
        d.job_centre[jr * 2 + 0] = d.h[gi * 2 + 0];
        d.job_centre[jr * 2 + 1] = d.h[gi * 2 + 1];
        rd pu[3] = {rd(d.ovr[0]), rd(d.ovr[1]), rd(d.ovr[2])};  // the fixed search ellipse, else S^-1
        if (!(d.ovr[0] > 0.0)) sinv_from_S(rd(d.S[gi * 4 + 0]), rd(d.S[gi * 4 + 1]), rd(d.S[gi * 4 + 3]), pu);
        for (int e = 0; e < 3; ++e) d.job_puinv[jr * 3 + e] = pu[e].v;
      }
    }
    __syncthreads();
    const int i = s_pick;
    if (i < 0) break;
    // ---- L_i = chol(C_i) --------------------------------------------------------------------------------------------
    const rd l00 = rsqrt_(rd(Cm[i * 3 + 0]));
    const rd l10 = rd(Cm[i * 3 + 1]) / l00;
    const rd l11 = rsqrt_(rd(Cm[i * 3 + 2]) - l10 * l10);
    // ---- u = P H_i^T on rows 0..6 and the unpicked candidates' y rows ----------------------------------------------
    const int yi = SL2_NXV + 3 * feat[i];
    for (int e = tid; e < 2 * rows; e += SEL_THREADS) {
      const int rr = e >> 1, c = e & 1;
      if (rr >= 7 && picked[(rr - 7) / 3]) continue;
      rd acc(0.0);
      for (int k = 0; k < 7; ++k) acc = acc + rd(Pc[rr * 7 + k]) * rd(A[i * 14 + c * 7 + k]);
      const double *Prow = P + sel_row(rr, feat);
      for (int k = 0; k < 3; ++k) acc = acc + rd(Prow[(size_t)ld * (yi + k)]) * rd(Bm[i * 6 + c * 3 + k]);
      u[rr * 2 + c] = acc.v;
    }
    __syncthreads();
    // ---- condition every unpicked candidate on the pick -------------------------------------------------------------
    for (int j = tid; j < V; j += SEL_THREADS) {
      if (picked[j]) continue;
      const int rj = 7 + 3 * j;
      // the four sums of c_j side by side: each keeps its own order, and each factor is read once per pick
      rd cj[2][2];
      for (int a = 0; a < 2; ++a)
        for (int b = 0; b < 2; ++b) {
          rd acc(0.0);
          for (int k = 0; k < 7; ++k) acc = acc + rd(A[j * 14 + a * 7 + k]) * rd(u[k * 2 + b]);
          for (int k = 0; k < 3; ++k) acc = acc + rd(Bm[j * 6 + a * 3 + k]) * rd(u[(rj + k) * 2 + b]);
          cj[a][b] = acc;
        }
      for (int p = 0; p < r; ++p) {
        const double *gjp = g + ((size_t)p * N + j) * 4, *gip = g + ((size_t)p * N + i) * 4;
        const rd gj[4] = {rd(gjp[0]), rd(gjp[1]), rd(gjp[2]), rd(gjp[3])};
        const rd gi[4] = {rd(gip[0]), rd(gip[1]), rd(gip[2]), rd(gip[3])};
        for (int a = 0; a < 2; ++a)
          for (int b = 0; b < 2; ++b)
            for (int e = 0; e < 2; ++e) cj[a][b] = cj[a][b] - gj[a * 2 + e] * gi[b * 2 + e];
      }
      rd gn[2][2];
      for (int a = 0; a < 2; ++a) {
        gn[a][0] = cj[a][0] / l00;
        gn[a][1] = (cj[a][1] - gn[a][0] * l10) / l11;
      }
      double *gr = g + ((size_t)r * N + j) * 4;
      for (int a = 0; a < 2; ++a)
        for (int e = 0; e < 2; ++e) gr[a * 2 + e] = gn[a][e].v;
      Cm[j * 3 + 0] = (rd(Cm[j * 3 + 0]) - gn[0][0] * gn[0][0] - gn[0][1] * gn[0][1]).v;
      Cm[j * 3 + 1] = (rd(Cm[j * 3 + 1]) - gn[1][0] * gn[0][0] - gn[1][1] * gn[0][1]).v;
      Cm[j * 3 + 2] = (rd(Cm[j * 3 + 2]) - gn[1][0] * gn[1][0] - gn[1][1] * gn[1][1]).v;
    }
    __syncthreads();
  }
  if (tid == 0) d.nsel[s] = r;
}

// the context's largest factor table would not fit beside the staged rows: the factors go to the scratch
bool sel_needs_scratch(const Sl2Dev &d) { return sel_base_bytes(d.Nmax) + sel_g_bytes(d.Nmax, d.kmax) > SEL_SMEM_MAX; }

}  // namespace

cudaError_t sl2_launch_select(const Sl2Dev &d, const SelectLaunch &L, Sl2Queue q) {
  if (L.stream_cnt <= 0) return cudaSuccess;
  const size_t smem = sel_base_bytes(d.Nmax) + (L.g ? 0 : sel_g_bytes(d.Nmax, L.gstride));
  if (smem > SEL_SMEM_MAX) return cudaErrorInvalidValue;
  return sl2_launch_kernel(select_kernel, dim3(L.stream_cnt), dim3(SEL_THREADS), smem, q, sl2_use_pdl(L.stream_cnt), d,
                           L);
}

namespace sl2 {

int select_streams(sl2_ctx *c, int lo, int cnt, Sl2Queue q) {
  const Sl2Dev &d = c->d;
  int npick = 1;  // the most picks a stream of the launch can make
  for (int s = lo; s < lo + cnt; ++s)
    if (c->opt[s].sel.mode == SL2_SELECT_INFORMATION)
      npick = std::max(npick, std::min(d.kmax, (int)c->cams[s].number_of_features_to_select));
  SelectLaunch L = {};
  L.stream_lo = lo;
  L.stream_cnt = cnt;
  L.mode = c->sel_mode_dev;
  L.t = c->sel_t_dev;
  L.gstride = npick;
  if (sel_base_bytes(d.Nmax) + sel_g_bytes(d.Nmax, npick) > SEL_SMEM_MAX) {
    L.g = c->sel_g.get();
    L.gstride = d.kmax;
  }
  CU_TRY(c, sl2_launch_select(d, L, q));
  return SL2_OK;
}

}  // namespace sl2

extern "C" {

int sl2_set_stream_selection(sl2_ctx *c, int32_t s, const sl2_stream_selection *sel) {
  if (bad_stream(c, s) || !sel) return fail(c, SL2_ERR_ARG, "sl2_set_stream_selection: bad argument");
  const int mode = sel->mode;
  const double bits = sel->min_bits;
  if (mode != SL2_SELECT_TRACE && mode != SL2_SELECT_INFORMATION)
    return fail(c, SL2_ERR_ARG, "sl2_set_stream_selection: unknown mode");
  if (sel->reserved != 0) return fail(c, SL2_ERR_ARG, "sl2_set_stream_selection: reserved must be 0");
  if (!std::isfinite(bits) || bits < 0.0 || (mode == SL2_SELECT_TRACE && bits != 0.0))
    return fail(c, SL2_ERR_ARG, "sl2_set_stream_selection: min_bits must be finite and >= 0, and 0 for the trace rule");
  const Sl2Dev &d = c->d;
  if (mode == SL2_SELECT_INFORMATION) {
    if (sel_needs_scratch(d)) {  // the factors of every stream, once
      const int rc = grow_scratch(c, (size_t)d.B * sel_g_bytes(d.Nmax, d.kmax), c->sel_g_bytes, c->sel_g);
      if (rc) return rc;
    }
    CU_TRY(c, cudaFuncSetAttribute(select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SEL_SMEM_MAX));
  }
  // ordered on the stream; a pageable source is staged before the copies return, so no launch is needed
  c->sel_mode[s] = mode;
  c->sel_t[s] = std::exp2(2.0 * bits);  // a pick must have q > t: (1/2) log2 q > min_bits
  CU_TRY(c, cudaMemcpyAsync(c->sel_mode_dev + s, &c->sel_mode[s], sizeof(int), cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, cudaMemcpyAsync(c->sel_t_dev + s, &c->sel_t[s], sizeof(double), cudaMemcpyHostToDevice, c->stream));
  sl2_stream_selection v = {};
  v.mode = mode;
  v.min_bits = bits == 0.0 ? 0.0 : bits;  // -0 like +0
  c->opt[s].sel = v;
  return SL2_OK;
}

int sl2_get_stream_selection(sl2_ctx *c, int32_t s, sl2_stream_selection *sel) {
  if (bad_stream(c, s) || !sel) return fail(c, SL2_ERR_ARG, "sl2_get_stream_selection: bad argument");
  *sel = c->opt[s].sel;
  return SL2_OK;
}

}  // extern "C"
