// ekf.cu — EKF predict / measurement prediction + selection / cull on sm_90a (the update is update.cu).
//
// Replaces, per camera stream (one CTA per stream, all streams of a context in one launch):
//   Kalman::KalmanFilterPredict            kalman.cpp:50-69   (+ motion_model.cpp:84-217)
//   MonoSLAM::auto_select_n_features       monoslam.cpp:187-254 (+ :289-308,
//                                          full_feature_model.cpp:67-195, camera.cpp:90-300)
//   MonoSLAM::delete_bad_features          monoslam.cpp:644-703, 770-812
// and, per partially-initialised feature of one stream (one CTA per feature, one thread per depth particle):
//   MonoSLAM::predict_partially_initialised_feature_measurements   monoslam.cpp:1347-1400
//                                          (+ part_feature_model.cpp:80-143, 231-265, feature_init_info.cpp:57-65)
// Map features and depth particles share the camera and feature models of sl2_model.cuh.
//
// State layout in HBM: ONE dense column-major P (ld x ld) per stream in the order of
// construct_total_covariance (monoslam.cpp:518-546): [xv(13) | y_0 | y_1 | ...], with both
// triangles kept bit-consistent (the reference rebuilds the lower triangle from the upper blocks
// on every gather, so P is exactly block-symmetric whenever it is read).
#include "sl2_model.cuh"

namespace {

// ---------------------------------------------------------------------------------------------
// motion model on one thread: fv, F (13x13 col-major), G (13x6 col-major) -- motion_model.cpp
// ---------------------------------------------------------------------------------------------
__device__ void dqomegadt_by_domega(const rd om[3], rd dt, rd m[4][3]) {
  const rd omega = rsqrt_(om[0] * om[0] + om[1] * om[1] + om[2] * om[2]);
  const rd two(2.0), one(1.0);
  const double sn = sin((omega * dt / two).v), cs = cos((omega * dt / two).v);
  const rd s(sn), c(cs);
  // motion_model.cpp:318-349
  auto dq0 = [&](rd a) { return ((-dt) / two) * (a / omega) * s; };
  auto dqA_A = [&](rd a) {
    return (dt / two) * a * a / (omega * omega) * c +
           (one / omega) * (one - a * a / (omega * omega)) * s;
  };
  auto dqA_B = [&](rd a, rd b) {
    return (a * b / (omega * omega)) * ((dt / two) * c - (one / omega) * s);
  };
  m[0][0] = dq0(om[0]);
  m[0][1] = dq0(om[1]);
  m[0][2] = dq0(om[2]);
  m[1][0] = dqA_A(om[0]);
  m[1][1] = dqA_B(om[0], om[1]);
  m[1][2] = dqA_B(om[0], om[2]);
  m[2][0] = dqA_B(om[1], om[0]);
  m[2][1] = dqA_A(om[1]);
  m[2][2] = dqA_B(om[1], om[2]);
  m[3][0] = dqA_B(om[2], om[0]);
  m[3][1] = dqA_B(om[2], om[1]);
  m[3][2] = dqA_A(om[2]);
}

__device__ void dq3_by_dq1(const Quat &q, rd m[4][4]) {  // math_util.cpp:82-97
  const rd x = q.x, y = q.y, z = q.z, w = q.w;
  const rd v[16] = {w, -x, -y, -z, x, w, -z, y, y, z, w, -x, z, -y, x, w};
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) m[i][j] = v[i * 4 + j];
}
__device__ void dq3_by_dq2(const Quat &q, rd m[4][4]) {  // math_util.cpp:99-114
  const rd x = q.x, y = q.y, z = q.z, w = q.w;
  const rd v[16] = {w, -x, -y, -z, x, w, z, -y, y, -z, w, x, z, y, -x, w};
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) m[i][j] = v[i * 4 + j];
}

// F and Gn are shared-memory col-major arrays (13x13, 13x6); fv 13.
__device__ void motion_model(const double *xv, const double *u3, double dt_, double *fv, double *F,
                             double *Gn) {
  const rd dt(dt_);
  const Quat qold = {rd(xv[3]), rd(xv[4]), rd(xv[5]), rd(xv[6])};
  const rd om[3] = {rd(xv[10]), rd(xv[11]), rd(xv[12])};
  // QuaternionFromAngularVelocity(omega * dt), math_util.cpp:61-80
  const rd av[3] = {om[0] * dt, om[1] * dt, om[2] * dt};
  const rd angle = rsqrt_(av[0] * av[0] + av[1] * av[1] + av[2] * av[2]);
  Quat qwt;
  if (angle.v > 0.0) {
    const rd sn(sin((angle / rd(2.0)).v)), cs(cos((angle / rd(2.0)).v));
    const rd s = sn / angle;
    qwt.x = s * av[0];
    qwt.y = s * av[1];
    qwt.z = s * av[2];
    qwt.w = cs;
  } else {
    qwt.w = rd(1.0);
  }
  const Quat qnew = quat_mul(qold, qwt);
  for (int i = 0; i < 3; ++i) fv[i] = (rd(xv[i]) + rd(xv[7 + i]) * dt).v;
  fv[3] = qnew.w.v;
  fv[4] = qnew.x.v;
  fv[5] = qnew.y.v;
  fv[6] = qnew.z.v;
  for (int i = 0; i < 3; ++i) fv[7 + i] = (rd(xv[7 + i]) + rd(u3 ? u3[i] : 0.0) * dt).v;
  for (int i = 0; i < 3; ++i) fv[10 + i] = om[i].v;

  for (int i = 0; i < 169; ++i) F[i] = 0.0;
  for (int i = 0; i < 13; ++i) F[i + 13 * i] = 1.0;
  for (int i = 0; i < 3; ++i) F[i + 13 * (7 + i)] = (rd(1.0) * dt).v;
  rd m44[4][4], m43[4][3], t44[4][4];
  dq3_by_dq2(qwt, m44);
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) F[(3 + i) + 13 * (3 + j)] = m44[i][j].v;
  dq3_by_dq1(qold, t44);
  dqomegadt_by_domega(om, dt, m43);
  for (int i = 0; i < 78; ++i) Gn[i] = 0.0;
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 3; ++j) {
      rd sacc(0.0);
      for (int k = 0; k < 4; ++k) sacc = sacc + t44[i][k] * m43[k][j];
      F[(3 + i) + 13 * (10 + j)] = sacc.v;
      Gn[(3 + i) + 13 * (3 + j)] = sacc.v;  // same product in func_Q (motion_model.cpp:202-213)
    }
  for (int i = 0; i < 3; ++i) {
    Gn[(7 + i) + 13 * i] = 1.0;
    Gn[(10 + i) + 13 * (3 + i)] = 1.0;
    Gn[i + 13 * i] = (rd(1.0) * dt).v;
  }
}

struct FeatPred {
  rd h[2];
  rd dxp[2][7];
  rd dy[2][3];
  rd var;
  rd S[2][2];
};

// Pxx: shared 13x13 col-major; Pcol: global pointer to P(0, pos) (column-major, ld)
__device__ void predict_feature(const double *cam, const double *xv, const rd yi[3],
                                const double *Pxx, const double *Pcol, int ld, int pos,
                                FeatPred &o) {
  rd z[3], dz_dxp[3][7], RRW[3][3], J[2][3];
  zeroedyi(yi, xv, z, dz_dxp, RRW);
  project(cam, z, o.h, J);
  for (int i = 0; i < 2; ++i) {
    for (int j = 0; j < 7; ++j) {
      rd s(0.0);
      for (int k = 0; k < 3; ++k) s = s + J[i][k] * dz_dxp[k][j];
      o.dxp[i][j] = s;
    }
    for (int j = 0; j < 3; ++j) {
      rd s(0.0);
      for (int k = 0; k < 3; ++k) s = s + J[i][k] * RRW[k][j];
      o.dy[i][j] = s;
    }
  }
  o.var = measurement_noise(cam, o.h);
  func_Si<3>(o.dxp, o.dy, o.var, Pxx, 13, Pcol, ld, Pcol + pos, ld, o.S);
}

__device__ int visibility_test(const double *cam, const double *xp, const rd yi[3],
                               const double *xp_orig, const rd h[2]) {
  int cant = 0;
  const double bound = 20.0;  // kImageSearchBoundary_, full_feature_model.cpp:51
  if (h[0].v < 0.0 + bound || h[0].v > (double)((int)cam[0] - 1 - bound)) cant |= 1;
  if (h[1].v < 0.0 + bound || h[1].v > (double)((int)cam[1] - 1 - bound)) cant |= 2;
  rd z[3], t[3][7], R1[3][3], RWR[3][3];
  zeroedyi(yi, xp, z, t, R1);
  if (z[2].v <= 0) cant |= 16;
  rd a[3], b[3];
  quat_to_R(Quat{rd(xp[3]), rd(xp[4]), rd(xp[5]), rd(xp[6])}, RWR);
  mat3_vec(RWR, z, a);
  zeroedyi(yi, xp_orig, z, t, R1);
  quat_to_R(Quat{rd(xp_orig[3]), rd(xp_orig[4]), rd(xp_orig[5]), rd(xp_orig[6])}, RWR);
  mat3_vec(RWR, z, b);
  const rd ma = rsqrt_(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
  const rd mb = rsqrt_(b[0] * b[0] + b[1] * b[1] + b[2] * b[2]);
  const rd ratio = ma / mb;
  if (ratio.v > 2.0 || ratio.v < (1.0 / 2.0)) cant |= 4;
  const rd dot = a[0] * b[0] + a[1] * b[1] + a[2] * b[2];
  double angle = acos((dot / (ma * mb)).v);
  angle = (angle >= 0.0 ? angle : -angle);
  if (angle > 3.14159265358979323846 * 45.0 / 180.0) cant |= 8;
  return cant;
}

// ---------------------------------------------------------------------------------------------
// kernel 1: predict (kalman.cpp:50-69) + measurement prediction / selection (monoslam.cpp:187-254)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) predict_kernel(const Sl2Dev d, int stream_lo,
                                                      const double *u3, int do_predict,
                                                      int do_measure) {
  pdl_prologue();
  const int s = stream_lo + blockIdx.x;
  const int tid = threadIdx.x;
  const int nf = d.nfeat[s];
  const int n = SL2_NXV + 3 * nf;
  const int ld = d.ld;
  double *P = d.P + (size_t)s * ld * ld;
  double *x = d.x + (size_t)s * ld;

  __shared__ double F[169], Gn[78], Pxx[169], TT[169], Qm[169], xv[13], fv[13];
  __shared__ double score[SL2_MAX_FEAT_SMEM];
  __shared__ int vis[SL2_MAX_FEAT_SMEM];
  __shared__ int s_nvis, s_r0;
  __shared__ Sl2StreamCam sc;  // this stream's camera row, loaded once per CTA

  load_stream_cam(d, s, sc);
  if (tid < 13) xv[tid] = x[tid];
  for (int e = tid; e < 169; e += blockDim.x) Pxx[e] = P[(e % 13) + (size_t)ld * (e / 13)];
  __syncthreads();

  if (do_predict) {
    if (tid == 0) motion_model(xv, u3, sc.dt, fv, F, Gn);
    __syncthreads();
    // Q = (G * Pnn) * G^T, Pnn = diag(lin x3, ang x3)   (motion_model.cpp:157-216)
    // TT = F * Pxx
    for (int e = tid; e < 169; e += blockDim.x) {
      const int i = e % 13, j = e / 13;
      const rd dt(sc.dt);
      const rd lin = rd(4.0) * rd(4.0) * dt * dt, ang = rd(6.0) * rd(6.0) * dt * dt;
      rd q(0.0), t(0.0);
      for (int k = 0; k < 6; ++k) {
        const rd gp = rd(0.0) + rd(Gn[i + 13 * k]) * (k < 3 ? lin : ang);  // (G*Pnn)(i,k)
        q = q + gp * rd(Gn[j + 13 * k]);
      }
      for (int k = 0; k < 13; ++k) t = t + rd(F[i + 13 * k]) * rd(Pxx[k + 13 * j]);
      Qm[e] = q.v;
      TT[e] = t.v;
    }
    __syncthreads();
    // Pxx = TT * F^T + Q
    for (int e = tid; e < 169; e += blockDim.x) {
      const int i = e % 13, j = e / 13;
      rd a(0.0);
      for (int k = 0; k < 13; ++k) a = a + rd(TT[i + 13 * k]) * rd(F[j + 13 * k]);
      const double v = (a + rd(Qm[e])).v;
      Pxx[e] = v;  // own element only: no hazard with TT/F readers
      P[i + (size_t)ld * j] = v;
    }
    // Pxy_i = F * Pxy_i  (one thread per column of the 13 x 3N panel), mirrored below the diagonal
    for (int c = SL2_NXV + tid; c < n; c += blockDim.x) {
      double col[13], out[13];
      for (int k = 0; k < 13; ++k) col[k] = P[k + (size_t)ld * c];
      for (int i = 0; i < 13; ++i) {
        rd a(0.0);
        for (int k = 0; k < 13; ++k) a = a + rd(F[i + 13 * k]) * rd(col[k]);
        out[i] = a.v;
      }
      for (int i = 0; i < 13; ++i) {
        P[i + (size_t)ld * c] = out[i];
        P[c + (size_t)ld * i] = out[i];
      }
    }
    if (tid < 13) {
      x[tid] = fv[tid];
      xv[tid] = fv[tid];
    }
    __syncthreads();
  }
  if (!do_measure) return;

  // ---- per-feature prediction, visibility, score ---------------------------------------------
  const size_t fb = (size_t)s * d.Nmax;
  for (int i0 = 0; i0 < d.Nmax; i0 += blockDim.x) {
    const int i = i0 + tid;
    if (i < d.Nmax) {
      vis[i] = 0;
      score[i] = 0.0;
      d.sel_rank[fb + i] = -1;
      // d.found keeps its previous value for features that are not measured this frame, like
      // Feature::successful_measurement_flag_ (only written by make_measurements, monoslam.cpp:479-496)
      d.job_feat[fb + i] = -1;
    }
    if (i < nf) {
      const int pos = SL2_NXV + 3 * i;
      const rd yi[3] = {rd(x[pos]), rd(x[pos + 1]), rd(x[pos + 2])};
      FeatPred fp;
      predict_feature(sc.cam, xv, yi, Pxx, P + (size_t)ld * pos, ld, pos, fp);
      d.h[(fb + i) * 2 + 0] = fp.h[0].v;
      d.h[(fb + i) * 2 + 1] = fp.h[1].v;
      for (int r = 0; r < 2; ++r) {
        for (int j = 0; j < 7; ++j) d.dh_dxp[(fb + i) * 14 + r * 7 + j] = fp.dxp[r][j].v;
        for (int j = 0; j < 3; ++j) d.dh_dy[(fb + i) * 6 + r * 3 + j] = fp.dy[r][j].v;
      }
      d.Rvar[fb + i] = fp.var.v;
      d.S[(fb + i) * 4 + 0] = fp.S[0][0].v;
      d.S[(fb + i) * 4 + 1] = fp.S[1][0].v;
      d.S[(fb + i) * 4 + 2] = fp.S[0][1].v;
      d.S[(fb + i) * 4 + 3] = fp.S[1][1].v;
      const int cant = visibility_test(sc.cam, xv, yi, d.xp_org + (fb + i) * 7, fp.h);
      vis[i] = (cant == 0);
      score[i] = (fp.S[0][0] + fp.S[1][1]).v;  // trace, full_feature_model.cpp:172-176
    }
  }
  __syncthreads();
  // ---- insertion sort of monoslam.cpp:211-230 as a rank: strictly larger scores first, ties in
  //      feature order; selection stops at the first zero score or after n_select (:241-249)
  if (tid == 0) {
    s_nvis = 0;
    s_r0 = 1 << 30;
  }
  __syncthreads();
  for (int i = tid; i < nf; i += blockDim.x) {
    if (vis[i]) {
      int rank = 0;
      const double si = score[i];
      for (int j = 0; j < nf; ++j)
        if (vis[j] && (score[j] > si || (j < i && !(si > score[j])))) ++rank;
      d.sel_rank[fb + i] = rank;  // provisional: rank among visible
      atomicAdd(&s_nvis, 1);
      if (si == 0.0) atomicMin(&s_r0, rank);
    }
  }
  __syncthreads();
  const int nsel = min(min(sc.n_select, s_r0), s_nvis);
  for (int i = tid; i < nf; i += blockDim.x) {
    int rank = d.sel_rank[fb + i];
    if (rank >= nsel) rank = -1;
    d.sel_rank[fb + i] = rank;
    if (rank >= 0) {
      d.job_feat[fb + rank] = i;
      d.job_centre[(fb + rank) * 2 + 0] = d.h[(fb + i) * 2 + 0];
      d.job_centre[(fb + rank) * 2 + 1] = d.h[(fb + i) * 2 + 1];
      rd pu[3] = {rd(d.ovr[0]), rd(d.ovr[1]), rd(d.ovr[2])};  // the fixed search ellipse, else S^-1
      if (!(d.ovr[0] > 0.0))
        sinv_from_S(rd(d.S[(fb + i) * 4 + 0]), rd(d.S[(fb + i) * 4 + 1]), rd(d.S[(fb + i) * 4 + 3]), pu);
      for (int e = 0; e < 3; ++e) d.job_puinv[(fb + rank) * 3 + e] = pu[e].v;
    }
  }
  if (tid == 0) {
    d.nsel[s] = nsel;
    d.nvisible[s] = s_nvis;
    d.nmeas[s] = 0;
  }
}

// ---------------------------------------------------------------------------------------------
// particle prediction: predict_partially_initialised_feature_measurements (monoslam.cpp:1347-1400) for the depth
// particles of F partially-initialised features of stream s: h_pi (part_feature_model.cpp:80-143, 231-265), R_i, S_i
// and Particle::set_S (S_i^-1, det S_i; feature_init_info.cpp:57-65).  One CTA per feature, thread k = particle k.
// Ray yi = (r_i, hhat_i): ypi [F][6]; its covariance blocks Pxy [F][13x6], Pyy [F][6x6] column-major.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) particle_predict_kernel(const Sl2Dev d, int s, int Kmax,
                                                               const int *__restrict__ Kf,
                                                               const double *__restrict__ ypi_all,
                                                               const double *__restrict__ Pxy_all,
                                                               const double *__restrict__ Pyy_all,
                                                               const double *__restrict__ lambda_all,
                                                               double *__restrict__ h_out, double *__restrict__ sinv3_out,
                                                               double *__restrict__ detS_out) {
  const int f = blockIdx.x, K = Kf[f];
  const double *ypi = ypi_all + 6 * f, *Pxy = Pxy_all + 78 * f, *Pyy = Pyy_all + 36 * f;
  const double *xv = d.x + (size_t)s * d.ld;
  const double *P = d.P + (size_t)s * d.ld * d.ld;  // Pxx = P(0:13, 0:13), column-major with stride ld
  __shared__ Sl2StreamCam sc;  // this stream's camera row, loaded once per CTA
  load_stream_cam(d, s, sc);
  __syncthreads();
  // qRW and RRW: one camera pose for every particle
  rd R[3][3];
  const Quat qi = pose_RRW(xv, R);
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const size_t o = (size_t)f * Kmax + k;
    const rd lam(lambda_all[o]);
    // zeroedri = RRW (r_i - r), zeroedhhati = RRW hhat_i and their dq columns (part_feature_model.cpp:80-143)
    const rd dv[3] = {rd(ypi[0]) - rd(xv[0]), rd(ypi[1]) - rd(xv[1]), rd(ypi[2]) - rd(xv[2])};
    const rd hh[3] = {rd(ypi[3]), rd(ypi[4]), rd(ypi[5])};
    rd zr[3], zh[3], Dr[3][4], Dh[3][4];
    mat3_vec(R, dv, zr);
    mat3_vec(R, hh, zh);
    dRq_times_a_by_dq(qi, dv, Dr);
    dRq_times_a_by_dq(qi, hh, Dh);
    const rd hLR[3] = {zr[0] + lam * zh[0], zr[1] + lam * zh[1], zr[2] + lam * zh[2]};
    rd h[2], J[2][3];
    project(sc.cam, hLR, h, J);
    // dhpi_by_dxp (2x7) and dhpi_by_dyi (2x6) = J [I | lambda I] dzeroedyi (part_feature_model.cpp:262-264): the
    // lambda columns of dh/dy, and one accumulator for the r and hhat terms of each quaternion column of dh/dxp
    rd dxp[2][7], dy[2][6];
    for (int i = 0; i < 2; ++i) {
      rd Jl[3];
      for (int q = 0; q < 3; ++q) Jl[q] = J[i][q] * lam;
      for (int j = 0; j < 3; ++j) {
        rd a(0.0), b(0.0), c(0.0);
        for (int q = 0; q < 3; ++q) {
          a = a + J[i][q] * (R[q][j] * rd(-1.0));
          b = b + J[i][q] * R[q][j];
          c = c + Jl[q] * R[q][j];
        }
        dxp[i][j] = a;
        dy[i][j] = b;
        dy[i][3 + j] = c;
      }
      for (int j = 0; j < 4; ++j) {
        rd a(0.0);
        for (int q = 0; q < 3; ++q) a = a + J[i][q] * Dr[q][j];
        for (int q = 0; q < 3; ++q) a = a + Jl[q] * Dh[q][j];
        dxp[i][3 + j] = a;
      }
    }
    rd S[2][2], Sinv[3];
    func_Si<6>(dxp, dy, measurement_noise(sc.cam, h), P, d.ld, Pxy, 13, Pyy, 6, S);
    sinv_from_S(S[0][0], S[1][0], S[1][1], Sinv);
    h_out[2 * o] = h[0].v;
    h_out[2 * o + 1] = h[1].v;
    for (int e = 0; e < 3; ++e) sinv3_out[3 * o + e] = Sinv[e].v;
    detS_out[o] = (S[0][0] * S[1][1] - S[0][1] * S[1][0]).v;
  }
}

// ---------------------------------------------------------------------------------------------
// kernel 3: delete_bad_features (monoslam.cpp:644-703) / delete_feature (:770-812)
// removes the rows/columns of the culled features from x and P in place.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) cull_kernel(const Sl2Dev d, int stream_lo, int force_index) {
  pdl_prologue();
  const int s = stream_lo + blockIdx.x;
  const int tid = threadIdx.x;
  const int nf = d.nfeat[s];
  const int ld = d.ld;
  const size_t fb = (size_t)s * d.Nmax;
  if (force_index < 0 && d.ncull[s] == 0) return;  // nothing to cull (decided by the update's finish kernel)
  __shared__ int keep[SL2_MAX_FEAT_SMEM];  // new index of feature i or -1
  __shared__ int s_new;
  if (tid == 0) {
    int k = 0;
    for (int i = 0; i < nf; ++i) {
      bool kill;
      if (force_index >= 0) {
        kill = (i == force_index);
      } else {
        const int att = d.attempted[fb + i], suc = d.successful[fb + i];
        kill = att >= d.min_attempts && (double)suc / (double)att < d.match_fraction;
      }
      keep[i] = kill ? -1 : k++;
    }
    s_new = k;
  }
  __syncthreads();
  const int nk = s_new;
  if (nk == nf) return;
  double *P = d.P + (size_t)s * ld * ld;
  double *x = d.x + (size_t)s * ld;
  double *scr = d.G + (size_t)s * d.mmax * d.ldg;  // scratch >= ld*ld? no: compact column by column
  const int n = SL2_NXV + 3 * nf;
  // destination indices are never larger than source indices, so walking columns in increasing
  // order with a per-column staging buffer in scratch is race-free inside one CTA.
  for (int c = 0; c < n; ++c) {
    int cn;
    if (c < SL2_NXV) {
      cn = c;
    } else {
      const int f = (c - SL2_NXV) / 3;
      cn = keep[f] < 0 ? -1 : SL2_NXV + 3 * keep[f] + (c - SL2_NXV) % 3;
    }
    if (cn < 0) continue;  // uniform across the CTA
    for (int r = tid; r < n; r += blockDim.x) scr[r] = P[r + (size_t)ld * c];
    __syncthreads();
    for (int r = tid; r < n; r += blockDim.x) {
      int rn;
      if (r < SL2_NXV) {
        rn = r;
      } else {
        const int f = (r - SL2_NXV) / 3;
        rn = keep[f] < 0 ? -1 : SL2_NXV + 3 * keep[f] + (r - SL2_NXV) % 3;
      }
      if (rn >= 0) P[rn + (size_t)ld * cn] = scr[r];
    }
    __syncthreads();
  }
  // state vector and per-feature records
  for (int r = tid; r < n; r += blockDim.x) scr[r] = x[r];
  __syncthreads();
  for (int r = SL2_NXV + tid; r < n; r += blockDim.x) {
    const int f = (r - SL2_NXV) / 3;
    if (keep[f] >= 0) x[SL2_NXV + 3 * keep[f] + (r - SL2_NXV) % 3] = scr[r];
  }
  __syncthreads();
  if (tid == 0) {
    // serial compaction of the small per-feature records (rare path)
    // selected_feature_list_.erase (monoslam.cpp:258-281 via :797-798): later entries move up
    for (int i = 0; i < nf; ++i) {
      const int r = d.sel_rank[fb + i];
      if (keep[i] < 0 && r >= 0) {
        for (int j = 0; j < nf; ++j)
          if (d.sel_rank[fb + j] > r) d.sel_rank[fb + j] -= 1;
        d.sel_rank[fb + i] = -1;
      }
    }
    const int box16 = d.box * 16;
    for (int i = 0; i < nf; ++i) {
      const int k = keep[i];
      if (k < 0 || k == i) continue;
      for (int e = 0; e < box16; ++e)
        d.patches[(fb + k) * box16 + e] = d.patches[(fb + i) * box16 + e];
      // every per-feature record moves with the Feature object, as in the reference
#define SL2_MOVE(T, name, per, by, reset) \
  if (by == SL2_BY_FEATURE)               \
    for (int e = 0; e < per; ++e) d.name[(fb + k) * per + e] = d.name[(fb + i) * per + e];
      SL2_STREAM_ARRAYS(SL2_MOVE)
#undef SL2_MOVE
    }
    // the job list of this step indexes the old feature numbering: rebuild it from the compacted ranks
    for (int r = 0; r < d.Nmax; ++r) d.job_feat[fb + r] = -1;
    int nsel_new = 0;
    for (int k = 0; k < nk; ++k) {
      const int r = d.sel_rank[fb + k];
      if (r >= 0) {
        d.job_feat[fb + r] = k;
        ++nsel_new;
      }
    }
    d.nsel[s] = nsel_new;
    d.nfeat[s] = nk;
  }
}

// ---------------------------------------------------------------------------------------------
// kernel 4: append one fully-initialised feature (monoslam.cpp:1278-1289, feature.cpp:108-149): the mirror of
// cull_kernel -- x grows by y, P by three rows / columns (zero like the reference's Pxy_ / Pyy_ /
// matrix_block_list_, or the caller's (n + 3) x 3 block), the per-feature records start like Feature::Initialise.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) append_kernel(const Sl2Dev d, int s, const double *y3, const double *xp7,
                                                     const uint8_t *patch_rows16, const double *Pcol) {
  const int tid = threadIdx.x;
  const int nf = d.nfeat[s];
  const int n = SL2_NXV + 3 * nf, ld = d.ld;
  double *P = d.P + (size_t)s * ld * ld;
  double *x = d.x + (size_t)s * ld;
  const size_t f = (size_t)s * d.Nmax + nf;
  for (int e = tid; e < 3 * (n + 3); e += blockDim.x) {
    const int c = e / (n + 3), r = e - c * (n + 3);
    const double v = Pcol ? Pcol[e] : 0.0;  // column-major (n + 3) x 3
    P[r + (size_t)ld * (n + c)] = v;
    if (r < n) P[(n + c) + (size_t)ld * r] = v;  // mirrored: both triangles stay consistent
  }
  if (Pcol) {
    // the 3x3 diagonal block must be exactly symmetric: take the upper triangle of the caller's block
    __syncthreads();
    if (tid < 9) {
      const int r = tid % 3, c = tid / 3;
      if (r > c) P[(n + r) + (size_t)ld * (n + c)] = P[(n + c) + (size_t)ld * (n + r)];
    }
  }
  if (tid < 3) x[n + tid] = y3[tid];
  if (tid < 7) d.xp_org[f * 7 + tid] = xp7[tid];
  const int box16 = d.box * 16;
  for (int e = tid; e < box16; e += blockDim.x) d.patches[f * box16 + e] = patch_rows16[e];
  if (tid == 0) {
    // every per-feature record but xp_org (written above) starts at its reset value
#define SL2_RESET(T, name, per, by, reset)                          \
  if (by == SL2_BY_FEATURE && SL2_FIELD_##name != SL2_FIELD_xp_org) \
    for (int e = 0; e < per; ++e) d.name[f * per + e] = (T)(reset);
    SL2_STREAM_ARRAYS(SL2_RESET)
#undef SL2_RESET
  }
  __syncthreads();
  if (tid == 0) d.nfeat[s] = nf + 1;
}

}  // namespace

cudaError_t sl2_launch_append(const Sl2Dev &d, int s, const double *y3_dev, const double *xp7_dev,
                              const uint8_t *patch_rows16_dev, const double *Pcol_dev, Sl2Queue q) {
  return sl2_launch_kernel(append_kernel, dim3(1), dim3(256), 0, q, false, d, s, y3_dev, xp7_dev, patch_rows16_dev,
                           Pcol_dev);
}

cudaError_t sl2_launch_predict(const Sl2Dev &d, int stream_lo, int stream_cnt, const double *u3_dev,
                               int do_predict, int do_measure, Sl2Queue q) {
  if (stream_cnt <= 0) return cudaSuccess;
  // 128 threads, one feature each per pass over the map (two passes at SL2_MAX_FEATURES); the kernel needs ~255
  // registers per thread, so 128-thread CTAs are what lets two streams share an SM
  return sl2_launch_kernel(predict_kernel, dim3(stream_cnt), dim3(128), 0, q, sl2_use_pdl(stream_cnt), d,
                           stream_lo, u3_dev, do_predict, do_measure);
}

// F features, Kmax = stride between features in every per-particle array, K_dev[f] particles used
cudaError_t sl2_launch_particle_predict(const Sl2Dev &d, int s, int F, int Kmax, const int *K_dev,
                                        const double *ypi, const double *Pxy, const double *Pyy,
                                        const double *lambda, double *h, double *sinv3, double *detS,
                                        Sl2Queue q) {
  if (F <= 0) return cudaSuccess;
  return sl2_launch_kernel(particle_predict_kernel, dim3(F), dim3(128), 0, q, false, d, s, Kmax, K_dev, ypi, Pxy, Pyy,
                           lambda, h, sinv3, detS);
}

cudaError_t sl2_launch_cull(const Sl2Dev &d, int stream_lo, int stream_cnt, int force_index, Sl2Queue q) {
  if (stream_cnt <= 0) return cudaSuccess;
  return sl2_launch_kernel(cull_kernel, dim3(stream_cnt), dim3(256), 0, q, sl2_use_pdl(stream_cnt), d,
                           stream_lo, force_index);
}
