// consensus.cu — the match consensus on sm_90a, between the patch search and the EKF update of the fused step.
// One-point RANSAC with exhaustive hypotheses (Civera, Grasa, Davison, Montiel, J. Field Robotics 2010), one CTA per
// camera stream of the launch; streams whose tau2[s] (= fl(tau * tau), 0 = off) is not > 0 return at once.
// Semantics: include/sl2b200.h, sl2_set_stream_consensus.
//
// M = the job slots r < nsel whose feature has found == 1, in rank order (match j, k = |M| <= SL2_MAX_MEASURED);
// x, P are the predicted state and covariance.  Every operation is one correctly rounded, never-fused op (rd), in
// this order (tests/consensus_oracle.cpp restates it op for op):
//   per match j:  nu = (double)z - h;  (Sinv00, Sinv01, Sinv11) = sinv_from_S(S00, S10, S11);
//                 w0 = Sinv00 nu0 + Sinv01 nu1;  w1 = Sinv01 nu0 + Sinv11 nu1;
//                 a[c] = dh_dxp[0][c] w0 + dh_dxp[1][c] w1 (c < 7);  b[c] = dh_dy[0][c] w0 + dh_dy[1][c] w1 (c < 3)
//   hypothesis i: xp'[r] = x[r] + s,  s = ((0 + P[r,0] a_i[0]) + ... + P[r,6] a_i[6]) + P[r,yi] b_i[0] + ...
//                                        + P[r,yi+2] b_i[2]                                      (r < 7)
//                 RRW = pose_RRW(xp')
//   match j of i: y'[r] = y_j[r] + s,  s = the same sum over P[yj+r, 0..6] a_i then P[yj+r, yi..yi+2] b_i   (r < 3)
//                 reproj_inlier(RRW, y', xp', z_j): zeroed_point, project_point -> g;  du = (double)z_u - g_u, dv
//                 likewise; inlier iff the camera-frame depth is > 0 and du du + dv dv <= tau2 (NaN: never)
//   support(i) = inliers of i (i itself included); winner = largest support, ties to the lowest rank; when the
//   winner's support is >= 2 every match outside its inlier set gets found = 2 (matched, rejected by the consensus).
// Shape: warp w takes hypotheses w, w + CONS_WARPS, ...; its lanes take the matches j = lane + 32 c and count the
// support (warp_support).  The per-match terms and P[yj, 0:7] sit in shared memory, P[0:7, yi] and the 3x3 blocks
// P[yj, yi] are read from L2.
#include "sl2_model.cuh"

namespace {

#define CONS_WARPS 8
#define CONS_WORDS (SL2_MAX_MEASURED / 32)
__global__ void __launch_bounds__(32 * CONS_WARPS) consensus_kernel(const Sl2Dev d, int stream_lo,
                                                                  const double *__restrict__ tau2) {
  pdl_prologue();
  const int s = stream_lo + blockIdx.x;
  const double t2 = tau2[s];
  if (!(t2 > 0.0)) return;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int ld = d.ld;
  const size_t fb = (size_t)s * d.Nmax;
  const double *P = d.P + (size_t)s * ld * ld;
  const double *x = d.x + (size_t)s * ld;

  __shared__ int mf[SL2_MAX_MEASURED];                  // feature of match j
  __shared__ double mz[SL2_MAX_MEASURED][2];            // z_j
  __shared__ double my[SL2_MAX_MEASURED][3];            // y_j
  __shared__ double ma[SL2_MAX_MEASURED][7];            // a_j = dh_dxp^T w_j
  __shared__ double mb[SL2_MAX_MEASURED][3];            // b_j = dh_dy^T w_j
  __shared__ double pyx[SL2_MAX_MEASURED][21];          // P[yj + r, c], r < 3, c < 7: [r * 7 + c]
  __shared__ double pxx[49], xp0[7];                    // P[0:7, 0:7] column-major, x[0:7]
  __shared__ double hxp[CONS_WARPS][7];                 // xp' of each warp's hypothesis
  __shared__ unsigned mask[SL2_MAX_MEASURED][CONS_WORDS];  // inlier set of hypothesis i
  __shared__ int support[SL2_MAX_MEASURED];
  __shared__ int wcount[CONS_WARPS], s_win;
  __shared__ Sl2StreamCam sc;

  // ---- M in rank order (job slots < nsel <= kmax <= SL2_MAX_MEASURED) ---------------------------------------------
  const int nsel = d.nsel[s];
  int feat = -1;
  if (tid < d.Nmax && tid < nsel) {
    const int i = d.job_feat[fb + tid];
    if (i >= 0 && d.found[fb + i] == 1) feat = i;
  }
  load_stream_cam(d, s, sc);
  if (tid < 49) pxx[tid] = P[(tid % 7) + (size_t)ld * (tid / 7)];
  if (tid < 7) xp0[tid] = x[tid];
  const int k = block_gather(feat, mf, wcount, CONS_WARPS);
  __syncthreads();
  if (k < 2) return;  // no two matches can agree: nothing is rejected

  // ---- per-match terms ---------------------------------------------------------------------------------------------
  for (int j = tid; j < k; j += blockDim.x) {
    const size_t g = fb + mf[j];
    const int pos = SL2_NXV + 3 * mf[j];
    const rd zu((double)d.z_uv[g * 2]), zv((double)d.z_uv[g * 2 + 1]);
    const rd nu0 = zu - rd(d.h[g * 2]), nu1 = zv - rd(d.h[g * 2 + 1]);
    rd si[3];
    sinv_from_S(rd(d.S[g * 4 + 0]), rd(d.S[g * 4 + 1]), rd(d.S[g * 4 + 3]), si);
    const rd w0 = si[0] * nu0 + si[1] * nu1, w1 = si[1] * nu0 + si[2] * nu1;
    for (int c = 0; c < 7; ++c)
      ma[j][c] = (rd(d.dh_dxp[g * 14 + c]) * w0 + rd(d.dh_dxp[g * 14 + 7 + c]) * w1).v;
    for (int c = 0; c < 3; ++c) mb[j][c] = (rd(d.dh_dy[g * 6 + c]) * w0 + rd(d.dh_dy[g * 6 + 3 + c]) * w1).v;
    mz[j][0] = zu.v;
    mz[j][1] = zv.v;
    for (int r = 0; r < 3; ++r) {
      my[j][r] = x[pos + r];
      for (int c = 0; c < 7; ++c) pyx[j][r * 7 + c] = P[(pos + r) + (size_t)ld * c];
    }
  }
  __syncthreads();

  // ---- hypotheses: one warp each --------------------------------------------------------------------------------
  for (int i = warp; i < k; i += CONS_WARPS) {
    const int pi = SL2_NXV + 3 * mf[i];
    if (lane < 7) {
      rd acc(0.0);
      for (int c = 0; c < 7; ++c) acc = acc + rd(pxx[lane + 7 * c]) * rd(ma[i][c]);
      for (int c = 0; c < 3; ++c) acc = acc + rd(P[lane + (size_t)ld * (pi + c)]) * rd(mb[i][c]);
      hxp[warp][lane] = (rd(xp0[lane]) + acc).v;
    }
    __syncwarp();
    rd RRW[3][3];
    pose_RRW(hxp[warp], RRW);
    const int sup = warp_support(k, lane, mask[i], [&](int j) {
      const int pj = SL2_NXV + 3 * mf[j];
      rd yj[3];
      for (int r = 0; r < 3; ++r) {
        rd acc(0.0);
        for (int c = 0; c < 7; ++c) acc = acc + rd(pyx[j][r * 7 + c]) * rd(ma[i][c]);
        for (int c = 0; c < 3; ++c) acc = acc + rd(P[(pj + r) + (size_t)ld * (pi + c)]) * rd(mb[i][c]);
        yj[r] = rd(my[j][r]) + acc;
      }
      double d2;
      return reproj_inlier(sc.cam, RRW, hxp[warp], yj, mz[j], t2, &d2);
    });
    if (lane == 0) support[i] = sup;
    __syncwarp();  // hxp[warp] is rewritten by the next hypothesis
  }
  __syncthreads();
  if (tid == 0) {
    int best = -1, win = -1;
    for (int i = 0; i < k; ++i)
      if (support[i] > best) {
        best = support[i];
        win = i;
      }
    s_win = best >= 2 ? win : -1;
  }
  __syncthreads();
  const int win = s_win;
  if (win < 0) return;
  for (int j = tid; j < k; j += blockDim.x)
    if (!((mask[win][j >> 5] >> (j & 31)) & 1u)) d.found[fb + mf[j]] = 2;
}

}  // namespace

cudaError_t sl2_launch_consensus(const Sl2Dev &d, int stream_lo, int stream_cnt, const double *tau2_dev, Sl2Queue q) {
  if (stream_cnt <= 0) return cudaSuccess;
  return sl2_launch_kernel(consensus_kernel, dim3(stream_cnt), dim3(32 * CONS_WARPS), 0, q, sl2_use_pdl(stream_cnt), d,
                           stream_lo, tau2_dev);
}
