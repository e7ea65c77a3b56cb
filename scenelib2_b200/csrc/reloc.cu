// reloc.cu — relocalisation on sm_90a (Williams, Klein, Reid, ICCV 2007): after the full-image search, the camera pose
// of a lost stream from its matches with a three-point consensus.  Semantics: include/sl2b200.h, sl2_relocalise.
#include <math_constants.h>

#include "sl2_model.cuh"

namespace {

// splitmix64 (Steele, Lea, Flood, OOPSLA 2014) of state x: the hypothesis sequence of sl2_relocalise
__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  uint64_t z = x + 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// the three distinct match indices of hypothesis h among k >= 3 matches
__device__ __forceinline__ void reloc_triple(int h, int k, int t[3]) {
  const uint64_t x = 3ull * (uint64_t)h;
  int i0 = (int)(splitmix64(x) % (uint64_t)k);
  int i1 = (int)(splitmix64(x + 1) % (uint64_t)(k - 1));
  int i2 = (int)(splitmix64(x + 2) % (uint64_t)(k - 2));
  if (i1 >= i0) ++i1;
  if (i2 >= min(i0, i1)) ++i2;
  if (i2 >= max(i0, i1)) ++i2;
  t[0] = i0, t[1] = i1, t[2] = i2;
}

__device__ __forceinline__ void cross3(const double a[3], const double b[3], double o[3]) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}
__device__ __forceinline__ double dot3(const double a[3], const double b[3]) {
  return a[0] * b[0] + a[1] * b[1] + a[2] * b[2];
}
__device__ __forceinline__ double norm3(const double a[3]) { return sqrt(dot3(a, a)); }

// the largest real root of m^3 + a m^2 + b m + c (Cardano / trigonometric form), polished by two Newton steps
__device__ double cubic_max_root(double a, double b, double c) {
  const double a3 = a / 3.0;
  const double P = b - a * a3, Q = 2.0 * a3 * a3 * a3 - a3 * b + c;
  const double D = 0.25 * Q * Q + P * P * P / 27.0;
  double t;
  if (D > 0.0) {
    const double sD = sqrt(D);
    t = cbrt(-0.5 * Q + sD) + cbrt(-0.5 * Q - sD);
  } else {
    const double rr = sqrt(fmax(-P / 3.0, 0.0));
    const double cs = rr > 0.0 ? fmin(fmax(-0.5 * Q / (rr * rr * rr), -1.0), 1.0) : 0.0;
    t = 2.0 * rr * cos(acos(cs) / 3.0);
  }
  double m = t - a3;
  for (int it = 0; it < 2; ++it) {
    const double f = ((m + a) * m + b) * m + c, fp = (3.0 * m + 2.0 * a) * m + b;
    if (fp != 0.0) m -= f / fp;
  }
  return m;
}

// the real roots of a4 x^4 + a3 x^3 + a2 x^2 + a1 x + a0 (Ferrari, resolvent cubic), each polished by Newton steps
// that are kept only while they reduce |f|; returns how many (<= 4) in a fixed order
__device__ int quartic_roots(const double a[5], double x[4]) {
  if (!(fabs(a[0]) > 0.0)) return 0;
  const double B = a[1] / a[0], C = a[2] / a[0], D = a[3] / a[0], E = a[4] / a[0];
  const double BB = B * B;
  const double p = C - 0.375 * BB, q = D - 0.5 * B * C + 0.125 * BB * B,
               r = E - 0.25 * B * D + 0.0625 * BB * C - 3.0 / 256.0 * BB * BB;
  const double m = cubic_max_root(p, 0.25 * p * p - r, -0.125 * q * q);
  int n = 0;
  double y[4];
  if (!(m > 0.0)) {  // biquadratic: y^4 + p y^2 + r
    const double disc = p * p - 4.0 * r;
    if (disc >= 0.0) {
      const double sd = sqrt(disc);
      const double t2[2] = {0.5 * (-p + sd), 0.5 * (-p - sd)};
      for (int i = 0; i < 2; ++i)
        if (t2[i] >= 0.0) {
          y[n++] = sqrt(t2[i]);
          y[n++] = -sqrt(t2[i]);
        }
    }
  } else {  // (y^2 + p/2 + m)^2 = (s y - q / (2 s))^2, s = sqrt(2 m)
    const double s = sqrt(2.0 * m), qs = q / (2.0 * s);
    for (int sg = 0; sg < 2; ++sg) {
      const double bq = sg == 0 ? -s : s, cq = 0.5 * p + m + (sg == 0 ? qs : -qs);
      const double disc = bq * bq - 4.0 * cq;
      if (disc >= 0.0) {
        const double sd = sqrt(disc);
        y[n++] = 0.5 * (-bq + sd);
        y[n++] = 0.5 * (-bq - sd);
      }
    }
  }
  for (int i = 0; i < n; ++i) {
    double xi = y[i] - 0.25 * B;
    double f = (((a[0] * xi + a[1]) * xi + a[2]) * xi + a[3]) * xi + a[4];
    for (int it = 0; it < 3; ++it) {
      const double fp = ((4.0 * a[0] * xi + 3.0 * a[1]) * xi + 2.0 * a[2]) * xi + a[3];
      if (!(fp != 0.0)) break;
      const double xn = xi - f / fp;
      const double fn = (((a[0] * xn + a[1]) * xn + a[2]) * xn + a[3]) * xn + a[4];
      if (!(fabs(fn) < fabs(f))) break;
      xi = xn;
      f = fn;
    }
    x[i] = xi;
  }
  return n;
}

// rotation matrix (row-major) -> unit quaternion (w, x, y, z), w >= 0 (Shepperd's branch on the largest pivot)
__device__ void rot_to_quat(const double R[3][3], double q[4]) {
  const double tr = R[0][0] + R[1][1] + R[2][2];
  double w, x, y, z;
  if (tr > 0.0) {
    const double s = 2.0 * sqrt(tr + 1.0);
    w = 0.25 * s, x = (R[2][1] - R[1][2]) / s, y = (R[0][2] - R[2][0]) / s, z = (R[1][0] - R[0][1]) / s;
  } else if (R[0][0] > R[1][1] && R[0][0] > R[2][2]) {
    const double s = 2.0 * sqrt(1.0 + R[0][0] - R[1][1] - R[2][2]);
    w = (R[2][1] - R[1][2]) / s, x = 0.25 * s, y = (R[0][1] + R[1][0]) / s, z = (R[0][2] + R[2][0]) / s;
  } else if (R[1][1] > R[2][2]) {
    const double s = 2.0 * sqrt(1.0 + R[1][1] - R[0][0] - R[2][2]);
    w = (R[0][2] - R[2][0]) / s, x = (R[0][1] + R[1][0]) / s, y = 0.25 * s, z = (R[1][2] + R[2][1]) / s;
  } else {
    const double s = 2.0 * sqrt(1.0 + R[2][2] - R[0][0] - R[1][1]);
    w = (R[1][0] - R[0][1]) / s, x = (R[0][2] + R[2][0]) / s, y = (R[1][2] + R[2][1]) / s, z = 0.25 * s;
  }
  double n = sqrt(w * w + x * x + y * y + z * z);
  if (w < 0.0) n = -n;
  q[0] = w / n, q[1] = x / n, q[2] = y / n, q[3] = z / n;
}

// Kneip, Scaramuzza, Siegwart, "A Novel Parametrization of the Perspective-Three-Point Problem for a Direct
// Computation of Absolute Camera Position and Orientation", CVPR 2011: the camera poses xp = (r, qWR) under which the
// world points P[i] lie along the unit bearings f[i] (camera frame).  Returns the number of poses written (<= 4); a
// degenerate triple gives 0, and every pose written is finite.
__device__ int p3p_kneip(const double Pw[3][3], const double fb[3][3], double xp[4][7]) {
  double P1[3], P2[3], P3[3], f1[3], f2[3], f3[3];
  for (int i = 0; i < 3; ++i) P1[i] = Pw[0][i], P2[i] = Pw[1][i], P3[i] = Pw[2][i];
  for (int i = 0; i < 3; ++i) f1[i] = fb[0][i], f2[i] = fb[1][i], f3[i] = fb[2][i];
  double v1[3], v2[3], nw[3];
  for (int i = 0; i < 3; ++i) v1[i] = P2[i] - P1[i], v2[i] = P3[i] - P1[i];
  cross3(v1, v2, nw);
  if (!(norm3(nw) > 1e-10 * norm3(v1) * norm3(v2))) return 0;  // coincident or collinear points
  double nf[3];
  for (int a = 0; a < 3; ++a) {  // parallel bearings
    cross3(fb[a], fb[(a + 1) % 3], nf);
    if (!(norm3(nf) > 1e-10)) return 0;
  }
  // camera-side frame T: e1 = f1, e3 = f1 x f2 / |.|, e2 = e3 x e1; f3 in it must have a non-positive z
  double T[3][3], f3t[3];
  const auto frame = [&]() {
    double e3[3], e2[3];
    cross3(f1, f2, e3);
    const double ne = norm3(e3);
    for (int i = 0; i < 3; ++i) e3[i] /= ne;
    cross3(e3, f1, e2);
    for (int i = 0; i < 3; ++i) T[0][i] = f1[i], T[1][i] = e2[i], T[2][i] = e3[i];
    for (int i = 0; i < 3; ++i) f3t[i] = dot3(T[i], f3);
  };
  frame();
  if (f3t[2] > 0.0) {
    for (int i = 0; i < 3; ++i) {
      double t = f1[i];
      f1[i] = f2[i], f2[i] = t;
      t = P1[i];
      P1[i] = P2[i], P2[i] = t;
    }
    frame();
  }
  // world-side frame N: n1 = (P2 - P1) / |.|, n3 = n1 x (P3 - P1) / |.|, n2 = n3 x n1
  double N[3][3], n1[3], n2[3], n3[3], d31[3];
  const double d_12 = sqrt((P2[0] - P1[0]) * (P2[0] - P1[0]) + (P2[1] - P1[1]) * (P2[1] - P1[1]) +
                           (P2[2] - P1[2]) * (P2[2] - P1[2]));
  for (int i = 0; i < 3; ++i) n1[i] = (P2[i] - P1[i]) / d_12, d31[i] = P3[i] - P1[i];
  cross3(n1, d31, n3);
  const double nn3 = norm3(n3);
  for (int i = 0; i < 3; ++i) n3[i] /= nn3;
  cross3(n3, n1, n2);
  for (int i = 0; i < 3; ++i) N[0][i] = n1[i], N[1][i] = n2[i], N[2][i] = n3[i];
  const double p_1 = dot3(N[0], d31), p_2 = dot3(N[1], d31);
  const double f_1 = f3t[0] / f3t[2], f_2 = f3t[1] / f3t[2];
  const double cos_beta = dot3(f1, f2);
  double b = 1.0 / (1.0 - cos_beta * cos_beta) - 1.0;
  b = cos_beta < 0.0 ? -sqrt(b) : sqrt(b);
  const double f_1_pw2 = f_1 * f_1, f_2_pw2 = f_2 * f_2, p_1_pw2 = p_1 * p_1, p_1_pw3 = p_1_pw2 * p_1,
               p_1_pw4 = p_1_pw3 * p_1, p_2_pw2 = p_2 * p_2, p_2_pw3 = p_2_pw2 * p_2, p_2_pw4 = p_2_pw3 * p_2,
               d_12_pw2 = d_12 * d_12, b_pw2 = b * b;
  double fac[5];
  fac[0] = -f_2_pw2 * p_2_pw4 - p_2_pw4 * f_1_pw2 - p_2_pw4;
  fac[1] = 2 * p_2_pw3 * d_12 * b + 2 * f_2_pw2 * p_2_pw3 * d_12 * b - 2 * f_2 * p_2_pw3 * f_1 * d_12;
  fac[2] = -f_2_pw2 * p_2_pw2 * p_1_pw2 - f_2_pw2 * p_2_pw2 * d_12_pw2 * b_pw2 - f_2_pw2 * p_2_pw2 * d_12_pw2 +
           f_2_pw2 * p_2_pw4 + p_2_pw4 * f_1_pw2 + 2 * p_1 * p_2_pw2 * d_12 + 2 * f_1 * f_2 * p_1 * p_2_pw2 * d_12 * b -
           p_2_pw2 * p_1_pw2 * f_1_pw2 + 2 * p_1 * p_2_pw2 * f_2_pw2 * d_12 - p_2_pw2 * d_12_pw2 * b_pw2 -
           2 * p_1_pw2 * p_2_pw2;
  fac[3] = 2 * p_1_pw2 * p_2 * d_12 * b + 2 * f_2 * p_2_pw3 * f_1 * d_12 - 2 * f_2_pw2 * p_2_pw3 * d_12 * b -
           2 * p_1 * p_2 * d_12_pw2 * b;
  fac[4] = -2 * f_2 * p_2_pw2 * f_1 * p_1 * d_12 * b + f_2_pw2 * p_2_pw2 * d_12_pw2 + 2 * p_1_pw3 * d_12 -
           p_1_pw2 * d_12_pw2 + f_2_pw2 * p_2_pw2 * p_1_pw2 - p_1_pw4 - 2 * f_2_pw2 * p_2_pw2 * p_1 * d_12 +
           p_2_pw2 * f_1_pw2 * p_1_pw2 + f_2_pw2 * p_2_pw2 * d_12_pw2 * b_pw2;
  double roots[4];
  const int nr = quartic_roots(fac, roots);
  int ns = 0;
  for (int i = 0; i < nr; ++i) {
    const double cos_theta = roots[i];
    const double cot_alpha = (-f_1 * p_1 / f_2 - cos_theta * p_2 + d_12 * b) /
                             (-f_1 * cos_theta * p_2 / f_2 + p_1 - d_12);
    const double sin_theta = sqrt(1.0 - cos_theta * cos_theta);
    const double sin_alpha = sqrt(1.0 / (cot_alpha * cot_alpha + 1.0));
    double cos_alpha = sqrt(1.0 - sin_alpha * sin_alpha);
    if (cot_alpha < 0.0) cos_alpha = -cos_alpha;
    const double k1 = d_12 * sin_alpha * (sin_alpha * b + cos_alpha);
    const double Cn[3] = {d_12 * cos_alpha * (sin_alpha * b + cos_alpha), cos_theta * k1, sin_theta * k1};
    const double Rn[3][3] = {{-cos_alpha, -sin_alpha * cos_theta, -sin_alpha * sin_theta},
                             {sin_alpha, -cos_alpha * cos_theta, -cos_alpha * sin_theta},
                             {0.0, -sin_theta, cos_theta}};
    // r = P1 + N^T Cn;  R(qWR) = N^T Rn^T T
    double r[3], M[3][3], R[3][3];
    for (int a = 0; a < 3; ++a) r[a] = P1[a] + N[0][a] * Cn[0] + N[1][a] * Cn[1] + N[2][a] * Cn[2];
    for (int a = 0; a < 3; ++a)
      for (int c = 0; c < 3; ++c) M[a][c] = N[0][a] * Rn[c][0] + N[1][a] * Rn[c][1] + N[2][a] * Rn[c][2];
    for (int a = 0; a < 3; ++a)
      for (int c = 0; c < 3; ++c) R[a][c] = M[a][0] * T[0][c] + M[a][1] * T[1][c] + M[a][2] * T[2][c];
    double q[4];
    rot_to_quat(R, q);
    bool ok = true;
    for (int a = 0; a < 3; ++a) ok = ok && isfinite(r[a]);
    for (int a = 0; a < 4; ++a) ok = ok && isfinite(q[a]);
    if (!ok) continue;
    for (int a = 0; a < 3; ++a) xp[ns][a] = r[a];
    for (int a = 0; a < 4; ++a) xp[ns][3 + a] = q[a];
    ++ns;
  }
  return ns;
}

#define RELOC_WARPS 8
#define RELOC_THREADS (32 * RELOC_WARPS)  // one hypothesis per thread per round; >= SL2_MAX_FEATURES
#define RELOC_WORDS (SL2_MAX_FEATURES / 32)
static_assert(RELOC_THREADS >= SL2_MAX_FEATURES && RELOC_WORDS <= RELOC_WARPS, "one thread per feature");
static_assert(SL2_RELOC_HYPOTHESES % RELOC_THREADS == 0, "whole rounds of hypotheses");

struct RelocSmem {
  int mf[SL2_MAX_FEATURES];                     // feature of match j, j < k
  double mz[SL2_MAX_FEATURES][2];               // z_j
  rd my[SL2_MAX_FEATURES][3];                   // y_j
  double mbr[SL2_MAX_FEATURES][3];              // unit bearing of z_j
  double md2[SL2_MAX_FEATURES];                 // squared reprojection error under the refined pose
  double sol[RELOC_THREADS][4][7];              // the P3P poses of this round's hypotheses
  int nsol[RELOC_THREADS];
  double wpose[RELOC_WARPS][7];                 // each warp's best pose so far
  int wsup[RELOC_WARPS], widx[RELOC_WARPS], wcount[RELOC_WARPS];
  unsigned inl[RELOC_WORDS];                    // inlier set (winner, then refined pose)
  double pose[7];
  int k, win_sup, win_idx, n_inl, gn_ok;
  Sl2StreamCam sc;
};

// inliers of the pose xp over the k matches, one warp; lane 0 writes the inlier words to mask unless it is nullptr
template <typename Mask>
__device__ int reloc_support(const RelocSmem &S, const double *xp, double t2, int k, int lane, Mask mask) {
  rd RRW[3][3];
  pose_RRW(xp, RRW);
  return warp_support(k, lane, mask, [&](int j) {
    double d2;
    return reproj_inlier(S.sc.cam, RRW, xp, S.my[j], S.mz[j], t2, &d2);
  });
}

// One CTA per listed stream.  search_uv / search_found: the full-image search's results by job, job = (stream -
// stream_lo) * Nmax + feature.  Rounds of RELOC_THREADS hypotheses: every thread solves one P3P into shared memory,
// then warp w scores the poses of hypotheses w, w + RELOC_WARPS, ... of the round (lanes over the matches, ballot /
// popc), keeping its best (largest support, then lowest index: it visits indices in increasing order); thread 0
// reduces the warps' bests in the same order.  Warp 0 refines, the CTA recounts and, on acceptance, writes x and P.
__global__ void __launch_bounds__(RELOC_THREADS) reloc_kernel(const Sl2Dev d, const int *__restrict__ ids,
                                                              int stream_lo, const int *__restrict__ search_uv,
                                                              const uint8_t *__restrict__ search_found,
                                                              const sl2_reloc_params *__restrict__ prm,
                                                              const double *__restrict__ Pxx,
                                                              sl2_reloc_result *__restrict__ res, int *__restrict__ zuv_out,
                                                              uint8_t *__restrict__ flags_out) {
  extern __shared__ __align__(16) uint8_t reloc_smem[];
  RelocSmem &S = *reinterpret_cast<RelocSmem *>(reloc_smem);
  const int i = blockIdx.x, s = ids[i];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int ld = d.ld, nf = d.nfeat[s], n = SL2_NXV + 3 * nf;
  double *P = d.P + (size_t)s * ld * ld;
  double *x = d.x + (size_t)s * ld;
  const size_t jb = (size_t)(s - stream_lo) * d.Nmax;
  const double t2 = (rd(prm->inlier_px) * rd(prm->inlier_px)).v;

  // ---- M in feature-index order ------------------------------------------------------------------------------------
  const bool matched = tid < nf && search_found[jb + tid] == 1;
  load_stream_cam(d, s, S.sc);
  int myj;
  const int k = block_gather(matched ? tid : -1, S.mf, S.wcount, RELOC_WARPS, &myj);
  if (matched) {
    const rd zz[2] = {rd((double)search_uv[(jb + tid) * 2]), rd((double)search_uv[(jb + tid) * 2 + 1])};
    rd bv[3];
    unproject_point(S.sc.cam, zz, bv);
    const rd nb = rsqrt_(bv[0] * bv[0] + bv[1] * bv[1] + bv[2] * bv[2]);
    for (int r = 0; r < 3; ++r) {
      S.mbr[myj][r] = (bv[r] / nb).v;
      S.my[myj][r] = x[SL2_NXV + 3 * tid + r];
    }
    S.mz[myj][0] = zz[0].v;
    S.mz[myj][1] = zz[1].v;
  }
  __syncthreads();

  // ---- hypotheses, support, winner ---------------------------------------------------------------------------------
  int best_sup = -1, best_idx = -1;
  for (int h0 = 0; h0 < SL2_RELOC_HYPOTHESES; h0 += RELOC_THREADS) {
    int ns = 0;
    if (k >= 3) {
      int t[3];
      reloc_triple(h0 + tid, k, t);
      double Pw[3][3], fb[3][3];
      for (int a = 0; a < 3; ++a)
        for (int c = 0; c < 3; ++c) Pw[a][c] = S.my[t[a]][c].v, fb[a][c] = S.mbr[t[a]][c];
      ns = p3p_kneip(Pw, fb, S.sol[tid]);
    }
    S.nsol[tid] = ns;
    __syncthreads();
    for (int hl = warp; hl < RELOC_THREADS; hl += RELOC_WARPS)
      for (int q = 0; q < S.nsol[hl]; ++q) {
        const int sup = reloc_support(S, S.sol[hl][q], t2, k, lane, nullptr);
        if (sup > best_sup) {
          best_sup = sup;
          best_idx = (h0 + hl) * 4 + q;
          if (lane < 7) S.wpose[warp][lane] = S.sol[hl][q][lane];
        }
      }
    __syncthreads();  // S.sol is rewritten by the next round
  }
  if (lane == 0) {
    S.wsup[warp] = best_sup;
    S.widx[warp] = best_idx;
  }
  __syncthreads();
  if (tid == 0) {
    int bs = -1, bi = -1, bw = -1;
    for (int w = 0; w < RELOC_WARPS; ++w)
      if (S.wsup[w] > bs || (S.wsup[w] == bs && bs >= 0 && S.widx[w] < bi)) {
        bs = S.wsup[w];
        bi = S.widx[w];
        bw = w;
      }
    S.win_sup = bs;
    S.win_idx = bi;
    for (int e = 0; e < 7; ++e) S.pose[e] = bw >= 0 && bs >= 0 ? S.wpose[bw][e] : CUDART_NAN;
    S.k = k;
  }
  __syncthreads();
  const bool have = S.win_sup >= 0;

  // ---- refinement on the winner's inliers (warp 0) -------------------------------------------------------------------
  if (have && warp == 0) {
    reloc_support(S, S.pose, t2, k, lane, S.inl);
    __syncwarp();
    for (int it = 0; it < SL2_RELOC_GN_ITERS; ++it) {
      double acc[27];
      for (int e = 0; e < 27; ++e) acc[e] = 0.0;
      rd RRW[3][3];
      pose_RRW(S.pose, RRW);
      for (int j = lane; j < k; j += 32) {
        if (!((S.inl[j >> 5] >> (j & 31)) & 1u)) continue;
        rd dd[3], z[3], hh[2], J[2][3];
        zeroed_point(RRW, S.my[j], S.pose, dd, z);
        project(S.sc.cam, z, hh, J);
        // dz/d(dr) = -RRW, dz/d(dtheta) = [z]x (RWR' = RWR Exp(dtheta))
        const double Zx[3][3] = {{0.0, -z[2].v, z[1].v}, {z[2].v, 0.0, -z[0].v}, {-z[1].v, z[0].v, 0.0}};
        double A[2][6];
        for (int r = 0; r < 2; ++r)
          for (int c = 0; c < 3; ++c) {
            double a = 0.0, b = 0.0;
            for (int m = 0; m < 3; ++m) {
              a -= J[r][m].v * RRW[m][c].v;
              b += J[r][m].v * Zx[m][c];
            }
            A[r][c] = a;
            A[r][3 + c] = b;
          }
        const double e0 = S.mz[j][0] - hh[0].v, e1 = S.mz[j][1] - hh[1].v;
        int o = 0;
        for (int r = 0; r < 6; ++r)
          for (int c = r; c < 6; ++c) acc[o++] += A[0][r] * A[0][c] + A[1][r] * A[1][c];
        for (int r = 0; r < 6; ++r) acc[21 + r] += A[0][r] * e0 + A[1][r] * e1;
      }
      for (int e = 0; e < 27; ++e)
        for (int off = 16; off > 0; off >>= 1) acc[e] += __shfl_xor_sync(0xffffffffu, acc[e], off);
      if (lane == 0) {
        // Cholesky solve of the 6 x 6 normal equations (upper triangle packed row by row in acc[0..20])
        double L[6][6], y[6], dlt[6];
        int o = 0;
        for (int r = 0; r < 6; ++r)
          for (int c = r; c < 6; ++c) L[c][r] = acc[o++];
        bool ok = true;
        for (int j = 0; j < 6 && ok; ++j) {
          double sj = L[j][j];
          for (int m = 0; m < j; ++m) sj -= L[j][m] * L[j][m];
          if (!(sj > 0.0)) {
            ok = false;
            break;
          }
          L[j][j] = sqrt(sj);
          for (int r = j + 1; r < 6; ++r) {
            double v = L[r][j];
            for (int m = 0; m < j; ++m) v -= L[r][m] * L[j][m];
            L[r][j] = v / L[j][j];
          }
        }
        if (ok) {
          for (int r = 0; r < 6; ++r) {
            double v = acc[21 + r];
            for (int m = 0; m < r; ++m) v -= L[r][m] * y[m];
            y[r] = v / L[r][r];
          }
          for (int r = 5; r >= 0; --r) {
            double v = y[r];
            for (int m = r + 1; m < 6; ++m) v -= L[m][r] * dlt[m];
            dlt[r] = v / L[r][r];
          }
          double np[7];
          for (int a = 0; a < 3; ++a) np[a] = S.pose[a] + dlt[a];
          const double ang = sqrt(dlt[3] * dlt[3] + dlt[4] * dlt[4] + dlt[5] * dlt[5]);
          Quat dq;
          dq.w = rd(cos(0.5 * ang));
          const double sc = ang > 0.0 ? sin(0.5 * ang) / ang : 0.5;
          dq.x = rd(sc * dlt[3]), dq.y = rd(sc * dlt[4]), dq.z = rd(sc * dlt[5]);
          const Quat qn = quat_mul(Quat{rd(S.pose[3]), rd(S.pose[4]), rd(S.pose[5]), rd(S.pose[6])}, dq);
          double nq = sqrt(qn.w.v * qn.w.v + qn.x.v * qn.x.v + qn.y.v * qn.y.v + qn.z.v * qn.z.v);
          if (qn.w.v < 0.0) nq = -nq;
          np[3] = qn.w.v / nq, np[4] = qn.x.v / nq, np[5] = qn.y.v / nq, np[6] = qn.z.v / nq;
          for (int a = 0; a < 7; ++a) ok = ok && isfinite(np[a]);
          if (ok)
            for (int a = 0; a < 7; ++a) S.pose[a] = np[a];
        }
        S.gn_ok = ok;
      }
      __syncwarp();
      if (!S.gn_ok) break;
    }
  }
  __syncthreads();

  // ---- recount with the refined pose: warp w takes the matches 32 w .. 32 w + 31 ----------------------------------
  if (have) {
    rd RRW[3][3];
    pose_RRW(S.pose, RRW);
    const int j = warp * 32 + lane;
    double d2 = 0.0;
    const bool in = j < k && reproj_inlier(S.sc.cam, RRW, S.pose, S.my[j], S.mz[j], t2, &d2);
    if (j < SL2_MAX_FEATURES) S.md2[j] = d2;
    const unsigned b = __ballot_sync(0xffffffffu, in);
    if (lane == 0 && warp < RELOC_WORDS) S.inl[warp] = b;
  } else if (tid < RELOC_WORDS) {
    S.inl[tid] = 0u;
  }
  __syncthreads();
  if (tid == 0) {
    int cntin = 0;
    double sum = 0.0;
    for (int j = 0; j < k; ++j)
      if ((S.inl[j >> 5] >> (j & 31)) & 1u) {
        ++cntin;
        sum += S.md2[j];
      }
    S.n_inl = cntin;
    const bool accept = have && cntin >= prm->min_inliers;
    sl2_reloc_result &o = res[i];
    o.status = accept ? 1 : 0;
    o.matches = k;
    o.support = have ? S.win_sup : 0;
    o.inliers = cntin;
    o.rms_px = cntin > 0 ? sqrt(sum / (double)cntin) : CUDART_NAN;
    for (int e = 0; e < 7; ++e) o.pose[e] = S.pose[e];
  }
  // ---- per-feature results -------------------------------------------------------------------------------------------
  if (tid < d.Nmax) {
    const size_t o = (size_t)i * d.Nmax + tid;
    const bool has = tid < nf;
    zuv_out[o * 2 + 0] = has ? search_uv[(jb + tid) * 2 + 0] : -1;
    zuv_out[o * 2 + 1] = has ? search_uv[(jb + tid) * 2 + 1] : -1;
    uint8_t fl = matched ? 1 : 0;
    if (matched && ((S.inl[myj >> 5] >> (myj & 31)) & 1u)) fl |= 2;
    flags_out[o] = fl;
  }
  __syncthreads();
  if (!(have && S.n_inl >= prm->min_inliers)) return;

  // ---- acceptance: x[0:13], P[0:13, 0:13] = Pxx, the camera-map blocks zero ---------------------------------------
  if (tid < 7) x[tid] = S.pose[tid];
  if (tid < 3) {
    x[7 + tid] = prm->v[tid];
    x[10 + tid] = prm->omega[tid];
  }
  for (int e = tid; e < 169; e += blockDim.x) P[(e % 13) + (size_t)ld * (e / 13)] = Pxx[e];
  for (int e = tid; e < SL2_NXV * (n - SL2_NXV); e += blockDim.x) {
    const int r = e % SL2_NXV, c = SL2_NXV + e / SL2_NXV;
    P[r + (size_t)ld * c] = 0.0;
    P[c + (size_t)ld * r] = 0.0;
  }
}

}  // namespace

cudaError_t sl2_launch_reloc(const Sl2Dev &d, int cnt, const int *ids_dev, int stream_lo, const int *search_uv,
                             const uint8_t *search_found, const sl2_reloc_params *prm_dev, const double *Pxx_dev,
                             sl2_reloc_result *res_dev, int *zuv_dev, uint8_t *flags_dev, Sl2Queue q) {
  if (cnt <= 0) return cudaSuccess;
  const cudaError_t e =
      cudaFuncSetAttribute(reloc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(RelocSmem));
  if (e != cudaSuccess) return e;
  return sl2_launch_kernel(reloc_kernel, dim3(cnt), dim3(RELOC_THREADS), sizeof(RelocSmem), q, false, d, ids_dev,
                           stream_lo, search_uv, search_found, prm_dev, Pxx_dev, res_dev, zuv_dev, flags_dev);
}
