// gyro.cu — the gyroscope update on sm_90a, between the motion prediction and the feature prediction of the fused
// step: a linear measurement of the state's omega, x[10:13] (Pinies, Lupton, Sukkarieh, Tardos, "Inertial Aiding of
// Inverse Depth SLAM using a Monocular Camera", ICRA 2007).  Semantics and the order of every operation:
// include/sl2b200.h, sl2_set_stream_gyro (which, with the other gyro entry points, ends this file); tests/gyro_ref.py
// restates both kernels op for op.
//
// gyro_prep_kernel: one CTA per stream of the launch; streams that are off return at once, streams without a valid
// sample write status 0 and return.  Thread 0 forms zc, S, L, nu, w and the NIS, and consumes the sample; then the
// threads take the rows r < n: W[r] = P(r, 10:13) L^-T by forward substitution into the scratch (column c of P is
// contiguous in r, so the reads are coalesced), and x[r] += W[r] . w.
// gyro_downdate_kernel: P(i, j) -= W[i] . W[j] over each applied stream's n x n block, one read and one write per
// element, coalesced along columns.  It is a second launch because any tile that writes rows or columns 10..12 would
// race with the CTAs still reading them to form W: W is taken out of P before anything of P changes.
#include <algorithm>
#include <cmath>

#include "sl2_context.cuh"

using namespace sl2;

namespace {

constexpr int GYRO_THREADS = 128;  // prep: rows of W per pass
constexpr int DD_THREADS = 128;    // downdate: rows per pass
constexpr int DD_COLS = 16;        // downdate: columns per CTA

__device__ __forceinline__ bool finite_(rd v) { return isfinite(v.v); }

__global__ void __launch_bounds__(GYRO_THREADS) gyro_prep_kernel(const Sl2Dev d, const GyroLaunch G) {
  pdl_prologue();
  const int s = G.stream_lo + blockIdx.x;
  if (!G.on[s]) return;
  const int tid = threadIdx.x;
  const int ld = d.ld;
  const int n = SL2_NXV + 3 * d.nfeat[s];
  const double *P = d.P + (size_t)s * ld * ld;
  double *x = d.x + (size_t)s * ld;
  __shared__ double Ls[6], ws[3];  // l00 l10 l20 l11 l21 l22; w
  __shared__ int st;

  if (tid == 0) {
    const int k = s - G.sample_lo;
    int status = 0;
    double nis = 0.0;
    if (G.valid[k]) {
      G.valid[k] = 0;  // a sample is used by one step
      const Sl2GyroParam &p = G.prm[s];
      // 1. zc = R^T (z - b)
      rd dz[3], zc[3];
      for (int i = 0; i < 3; ++i) dz[i] = rd(G.rate[3 * k + i]) - rd(p.b[i]);
      for (int i = 0; i < 3; ++i) zc[i] = (rd(p.R[i]) * dz[0] + rd(p.R[3 + i]) * dz[1]) + rd(p.R[6 + i]) * dz[2];
      // 2. S = P(10:13, 10:13) + Rc (lower triangle) and its Cholesky factor
      const auto Pw = [&](int i, int j) { return rd(P[(10 + i) + (size_t)ld * (10 + j)]); };
      const rd S00 = Pw(0, 0) + rd(p.Rc[0]), S10 = Pw(1, 0) + rd(p.Rc[3]), S20 = Pw(2, 0) + rd(p.Rc[6]);
      const rd S11 = Pw(1, 1) + rd(p.Rc[4]), S21 = Pw(2, 1) + rd(p.Rc[7]), S22 = Pw(2, 2) + rd(p.Rc[8]);
      const rd l00 = rsqrt_(S00), l10 = S10 / l00, l20 = S20 / l00;
      const rd a11 = S11 - l10 * l10, l11 = rsqrt_(a11);
      const rd l21 = (S21 - l20 * l10) / l11;
      const rd a22 = (S22 - l20 * l20) - l21 * l21, l22 = rsqrt_(a22);
      // 3. nu, w = L^-1 nu, NIS = w . w
      const rd nu0 = zc[0] - rd(x[10]), nu1 = zc[1] - rd(x[11]), nu2 = zc[2] - rd(x[12]);
      const rd w0 = nu0 / l00, w1 = (nu1 - l10 * w0) / l11, w2 = ((nu2 - l20 * w0) - l21 * w1) / l22;
      const rd q = (w0 * w0 + w1 * w1) + w2 * w2;
      const rd all[] = {S00, S10, S20, S11, S21, S22, l00, l10, l20, l11, l21, l22, nu0, nu1, nu2, w0, w1, w2, q};
      bool ok = S00.v > 0.0 && a11.v > 0.0 && a22.v > 0.0;  // NaN: not > 0
      for (const rd &v : all) ok = ok && finite_(v);
      status = ok ? 1 : 2;
      if (ok) {
        nis = q.v;
        Ls[0] = l00.v, Ls[1] = l10.v, Ls[2] = l20.v, Ls[3] = l11.v, Ls[4] = l21.v, Ls[5] = l22.v;
        ws[0] = w0.v, ws[1] = w1.v, ws[2] = w2.v;
      }
    }
    st = status;
    G.nis[s] = nis;
    G.status[s] = status;
  }
  __syncthreads();
  if (st != 1) return;  // block-uniform: a skipped stream keeps x and P exactly

  // 4. W = P(0:n, 10:13) L^-T, row by row; 5. x += W w
  const rd l00(Ls[0]), l10(Ls[1]), l20(Ls[2]), l11(Ls[3]), l21(Ls[4]), l22(Ls[5]);
  const rd w0(ws[0]), w1(ws[1]), w2(ws[2]);
  double *W = G.W + (size_t)s * 3 * ld;
  for (int r = tid; r < n; r += GYRO_THREADS) {
    const rd p0(P[r + (size_t)ld * 10]), p1(P[r + (size_t)ld * 11]), p2(P[r + (size_t)ld * 12]);
    const rd W0 = p0 / l00;
    const rd W1 = (p1 - W0 * l10) / l11;
    const rd W2 = ((p2 - W0 * l20) - W1 * l21) / l22;
    W[r] = W0.v;
    W[ld + r] = W1.v;
    W[2 * ld + r] = W2.v;
    x[r] = (rd(x[r]) + ((W0 * w0 + W1 * w1) + W2 * w2)).v;
  }
}

// P(i, j) -= (W[i][0] W[j][0] + W[i][1] W[j][1]) + W[i][2] W[j][2], the products in the order (i, j).  IEEE
// multiplication is commutative, so P(j, i) gets the bits of P(i, j): each entry is formed on its own and the kernel
// treats the two triangles independently, with no mirror pass.  Grid: (stream, DD_COLS columns); threads over rows.
__global__ void __launch_bounds__(DD_THREADS) gyro_downdate_kernel(const Sl2Dev d, const GyroLaunch G) {
  pdl_prologue();
  const int s = G.stream_lo + blockIdx.x;
  if (!G.on[s] || G.status[s] != 1) return;
  const int tid = threadIdx.x;
  const int ld = d.ld;
  const int n = SL2_NXV + 3 * d.nfeat[s];
  const int j0 = blockIdx.y * DD_COLS;
  if (j0 >= n) return;
  const int jn = n - j0 < DD_COLS ? n - j0 : DD_COLS;
  const double *W = G.W + (size_t)s * 3 * ld;
  __shared__ double wj[3][DD_COLS];
  if (tid < 3 * DD_COLS) {
    const int c = tid / DD_COLS, jj = tid % DD_COLS;
    wj[c][jj] = jj < jn ? W[(size_t)c * ld + j0 + jj] : 0.0;
  }
  __syncthreads();
  double *P = d.P + (size_t)s * ld * ld + (size_t)ld * j0;
  for (int i = tid; i < n; i += DD_THREADS) {
    const double a0 = W[i], a1 = W[ld + i], a2 = W[2 * ld + i];
    double v[DD_COLS];
#pragma unroll
    for (int jj = 0; jj < DD_COLS; ++jj)  // every load of the row first: DD_COLS reads in flight
      if (jj < jn) v[jj] = P[i + (size_t)ld * jj];
#pragma unroll
    for (int jj = 0; jj < DD_COLS; ++jj)
      if (jj < jn)
        P[i + (size_t)ld * jj] = sub_(v[jj], add_(add_(mul_(a0, wj[0][jj]), mul_(a1, wj[1][jj])), mul_(a2, wj[2][jj])));
  }
}

}  // namespace

cudaError_t sl2_launch_gyro(const Sl2Dev &d, const GyroLaunch &G, Sl2Queue q) {
  if (G.stream_cnt <= 0) return cudaSuccess;
  const bool pdl = sl2_use_pdl(G.stream_cnt);
  const cudaError_t e = sl2_launch_kernel(gyro_prep_kernel, dim3(G.stream_cnt), dim3(GYRO_THREADS), 0, q, pdl, d, G);
  if (e != cudaSuccess) return e;
  return sl2_launch_kernel(gyro_downdate_kernel, dim3(G.stream_cnt, (d.ld + DD_COLS - 1) / DD_COLS), dim3(DD_THREADS),
                           0, q, pdl, d, G);
}

namespace {

GyroLaunch gyro_args(const sl2_ctx *c, int lo, int cnt) {
  GyroLaunch G = {};
  G.stream_lo = lo;
  G.stream_cnt = cnt;
  G.on = c->gyro_on_dev;
  G.prm = c->gyro_prm;
  G.W = c->gyro_W;
  G.nis = c->gyro_nis;
  G.status = c->gyro_status;
  return G;
}

// the setting's checks of include/sl2b200.h; an empty string when it is accepted
std::string gyro_setting_error(const sl2_stream_gyro *g) {
  if (g->reserved != 0 || (g->on != 0 && g->on != 1)) return "reserved must be 0 and on 0 or 1";
  if (!finite_all(g->R_gc, 9) || !finite_all(g->bias, 3) || !finite_all(g->cov, 9)) return "non-finite value";
  return sensor_frame_error(g->R_gc, g->cov, "R_gc");
}

Sl2GyroParam gyro_param(const sl2_stream_gyro &g) {
  Sl2GyroParam p;
  sensor_cov_in_camera(g.R_gc, g.cov, p.Rc);
  for (int i = 0; i < 9; ++i) p.R[i] = g.R_gc[i];
  for (int i = 0; i < 3; ++i) p.b[i] = g.bias[i];
  return p;
}

}  // namespace

namespace sl2 {

bool finite_all(const double *v, int n) {
  for (int i = 0; i < n; ++i)
    if (!std::isfinite(v[i])) return false;
  return true;
}

std::string sensor_frame_error(const double *R, const double *C, const std::string &rname) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      const double rr = R[3 * i] * R[3 * j] + R[3 * i + 1] * R[3 * j + 1] + R[3 * i + 2] * R[3 * j + 2];
      if (!(std::fabs(rr - (i == j ? 1.0 : 0.0)) <= 1e-9)) return rname + " is not a rotation";
    }
  const double det = R[0] * (R[4] * R[8] - R[5] * R[7]) - R[1] * (R[3] * R[8] - R[5] * R[6]) +
                     R[2] * (R[3] * R[7] - R[4] * R[6]);
  if (!(det > 0.0)) return rname + " is not a rotation";
  if (C[1] != C[3] || C[2] != C[6] || C[5] != C[7]) return "cov is not symmetric";
  const double l00 = std::sqrt(C[0]), l10 = C[3] / l00, l20 = C[6] / l00;
  const double a11 = C[4] - l10 * l10, l11 = std::sqrt(a11);
  const double l21 = (C[7] - l20 * l10) / l11;
  const double a22 = (C[8] - l20 * l20) - l21 * l21;
  if (!(C[0] > 0.0) || !(a11 > 0.0) || !(a22 > 0.0)) return "cov is not positive definite";
  return "";
}

// Rc = R^T C R: M = C R, then the upper triangle of R^T M, mirrored (include/sl2b200.h states the order)
void sensor_cov_in_camera(const double *R, const double *C, double Rc[9]) {
  double M[9];
  for (int k = 0; k < 3; ++k)
    for (int j = 0; j < 3; ++j) {
      double a = C[3 * k] * R[j];
      a = a + C[3 * k + 1] * R[3 + j];
      M[3 * k + j] = a + C[3 * k + 2] * R[6 + j];
    }
  for (int i = 0; i < 3; ++i)
    for (int j = i; j < 3; ++j) {
      double a = R[i] * M[j];
      a = a + R[3 + i] * M[3 + j];
      Rc[3 * i + j] = Rc[3 * j + i] = a + R[6 + i] * M[6 + j];
    }
}

int gyro_streams(sl2_ctx *c, int slot, int lo, int cnt, Sl2Queue q) {
  GyroLaunch G = gyro_args(c, lo, cnt);
  G.rate = c->gyro_rate + (size_t)slot * c->d.B * 3;
  G.valid = c->gyro_valid + (size_t)slot * c->d.B;
  G.sample_lo = 0;
  CU_TRY(c, sl2_launch_gyro(c->d, G, q));
  return SL2_OK;
}

}  // namespace sl2

extern "C" {

int sl2_set_stream_gyro(sl2_ctx *c, int32_t s, const sl2_stream_gyro *g) {
  if (bad_stream(c, s) || !g) return fail(c, SL2_ERR_ARG, "sl2_set_stream_gyro: bad argument");
  const std::string why = gyro_setting_error(g);
  if (!why.empty()) return fail(c, SL2_ERR_ARG, "sl2_set_stream_gyro: " + why);
  const Sl2Dev &d = c->d;
  if (g->on && !c->gyro_buf) {
    const size_t B = d.B, slots = d.slots;
    const int rc = alloc_sections(c, c->gyro_buf,
                                  {{&c->gyro_on_dev, B}, {&c->gyro_prm, B * sizeof(Sl2GyroParam)},
                                   {&c->gyro_rate, slots * B * 3 * sizeof(double)}, {&c->gyro_valid, slots * B},
                                   {&c->gyro_W, B * 3 * (size_t)d.ld * sizeof(double)},
                                   {&c->gyro_nis, B * sizeof(double)}, {&c->gyro_status, B * sizeof(int)}});
    if (rc) return rc;
  }
  const sl2_stream_gyro &old = c->opt[s].gyro;
  if (c->gyro_buf) {  // pageable copies have read their sources when they return; ordered on the stream, no launch
    const Sl2GyroParam p = gyro_param(*g);
    const uint8_t on = (uint8_t)g->on;
    CU_TRY(c, cudaMemcpyAsync(c->gyro_prm + s, &p, sizeof p, cudaMemcpyHostToDevice, c->stream));
    if (g->on && !old.on)  // turned on: no stale sample
      CU_TRY(c, cudaMemset2DAsync(c->gyro_valid + s, d.B, 0, 1, d.slots, c->stream));
    if (g->on != old.on) {  // turned on or off: no stale result
      CU_TRY(c, cudaMemsetAsync(c->gyro_nis + s, 0, sizeof(double), c->stream));
      CU_TRY(c, cudaMemsetAsync(c->gyro_status + s, 0, sizeof(int), c->stream));
    }
    CU_TRY(c, cudaMemcpyAsync(c->gyro_on_dev + s, &on, 1, cudaMemcpyHostToDevice, c->stream));
  }
  c->opt[s].gyro = *g;
  return SL2_OK;
}

int sl2_get_stream_gyro(sl2_ctx *c, int32_t s, sl2_stream_gyro *g) {
  if (bad_stream(c, s) || !g) return fail(c, SL2_ERR_ARG, "sl2_get_stream_gyro: bad argument");
  *g = c->opt[s].gyro;
  return SL2_OK;
}

int sl2_set_gyro_samples(sl2_ctx *c, int32_t slot, int32_t lo, int32_t cnt, const double *rates,
                         const uint8_t *valid) {
  if (bad_range(c, lo, cnt) || bad_slot(c, slot) || (cnt > 0 && !rates))
    return fail(c, SL2_ERR_ARG, "sl2_set_gyro_samples: bad argument");
  std::vector<uint8_t> v(cnt);
  for (int i = 0; i < cnt; ++i) {
    v[i] = (uint8_t)(!valid || valid[i] ? 1 : 0);
    if (v[i] && !finite_all(rates + 3 * (size_t)i, 3))
      return fail(c, SL2_ERR_ARG, "sl2_set_gyro_samples: a valid sample with a non-finite rate");
  }
  if (!c->gyro_buf) return fail(c, SL2_ERR_STATE, "sl2_set_gyro_samples: no stream has the gyroscope on");
  if (cnt == 0) return SL2_OK;
  const size_t at = (size_t)slot * c->d.B + lo;
  CU_TRY(c, cudaMemcpyAsync(c->gyro_rate + 3 * at, rates, sizeof(double) * 3 * cnt, cudaMemcpyHostToDevice,
                            c->stream));
  CU_TRY(c, cudaMemcpyAsync(c->gyro_valid + at, v.data(), cnt, cudaMemcpyHostToDevice, c->stream));
  return SL2_OK;
}

int sl2_gyro_update(sl2_ctx *c, int32_t s, const double *rate3) {
  if (bad_stream(c, s) || !rate3 || !finite_all(rate3, 3))
    return fail(c, SL2_ERR_ARG, "sl2_gyro_update: bad argument");
  if (!c->opt[s].gyro.on) return fail(c, SL2_ERR_STATE, "sl2_gyro_update: the stream's gyroscope is off");
  Stage r{STAGE_IN, 24, rate3}, v{STAGE_IN, 1};
  return staged_call(c, {&r, &v}, [&] { v.h[0] = 1; }, [&] {
    GyroLaunch G = gyro_args(c, s, 1);
    G.rate = r.dev<double>();
    G.valid = v.d;
    G.sample_lo = s;
    CU_TRY(c, sl2_launch_gyro(c->d, G, queue(c)));
    return SL2_OK;
  });
}

int sl2_get_gyro_results(sl2_ctx *c, int32_t lo, int32_t cnt, double *nis, int32_t *status) {
  if (bad_range(c, lo, cnt)) return fail(c, SL2_ERR_ARG, "sl2_get_gyro_results: bad range");
  return read_results(c, c->gyro_buf != nullptr, lo, cnt,
                      {{nis, c->gyro_nis, sizeof(double)}, {status, c->gyro_status, sizeof(int)}});
}

}  // extern "C"
