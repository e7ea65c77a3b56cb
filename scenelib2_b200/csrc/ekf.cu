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
// Entry points of one stream: sl2_ekf_predict, sl2_predict_measurements, sl2_append_feature, sl2_delete_feature.
//
// State layout in HBM: ONE dense column-major P (ld x ld) per stream in the order of
// construct_total_covariance (monoslam.cpp:518-546): [xv(13) | y_0 | y_1 | ...], with both
// triangles kept bit-consistent (the reference rebuilds the lower triangle from the upper blocks
// on every gather, so P is exactly block-symmetric whenever it is read).
#include "sl2_context.cuh"
#include "sl2_model.cuh"

using namespace sl2;

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

// The accelerometer's part of stream s's step (include/sl2b200.h, sl2_set_stream_accel), on thread 0 before
// motion_model: consumes an on stream's sample and writes its result; returns 0 (off or no sample), 1 (applied: the
// world-frame a, D = d(R(q) f_c)/dq (3 x 4 row-major) and the linear block L of Pnn (3 x 3) are in a, D, L) or 2
// (skipped: a, D or L not finite).  Not inlined: the predict kernel's registers stay its own.
__device__ __noinline__ int accel_model(const Sl2Accel &A, int s, const double *xv, double dt_, double *a_out,
                                        double *D_out, double *L_out) {
  if (!A.on[s]) return 0;
  const int k = s - A.sample_lo;
  int status = 0;
  rd a[3];
  if (A.valid[k]) {
    A.valid[k] = 0;  // a sample is used by one step
    const Sl2AccelParam &p = A.prm[s];
    const rd dt(dt_);
    // f_c = R_ac^T (f - b); a = R(q) f_c + g
    rd df[3], fc[3], Rf[3], R[3][3], D[3][4];
    for (int i = 0; i < 3; ++i) df[i] = rd(A.force[3 * k + i]) - rd(p.b[i]);
    for (int i = 0; i < 3; ++i) fc[i] = (rd(p.R[i]) * df[0] + rd(p.R[3 + i]) * df[1]) + rd(p.R[6 + i]) * df[2];
    const Quat q = {rd(xv[3]), rd(xv[4]), rd(xv[5]), rd(xv[6])};
    quat_to_R(q, R);
    mat3_vec(R, fc, Rf);
    for (int i = 0; i < 3; ++i) a[i] = Rf[i] + rd(p.g[i]);
    dRq_times_a_by_dq(q, fc, D);
    // L = ((R(q) Rc R(q)^T + sd_a^2 I) dt) dt: M = R(q) Rc, then the upper triangle of M R(q)^T, mirrored
    rd M[3][3], L[3][3];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        rd t(0.0);
        for (int m = 0; m < 3; ++m) t = t + R[i][m] * rd(p.Rc[3 * m + j]);
        M[i][j] = t;
      }
    for (int i = 0; i < 3; ++i)
      for (int j = i; j < 3; ++j) {
        rd t(0.0);
        for (int m = 0; m < 3; ++m) t = t + M[i][m] * R[j][m];
        if (i == j) t = t + rd(p.sd2);
        L[i][j] = L[j][i] = (t * dt) * dt;
      }
    bool ok = true;
    for (int i = 0; i < 3; ++i) {
      ok = ok && isfinite(a[i].v);
      for (int j = 0; j < 4; ++j) ok = ok && isfinite(D[i][j].v);
      for (int j = 0; j < 3; ++j) ok = ok && isfinite(L[i][j].v);
    }
    status = ok ? 1 : 2;
    if (ok)
      for (int i = 0; i < 3; ++i) {
        a_out[i] = a[i].v;
        for (int j = 0; j < 4; ++j) D_out[4 * i + j] = D[i][j].v;
        for (int j = 0; j < 3; ++j) L_out[3 * i + j] = L[i][j].v;
      }
  }
  for (int i = 0; i < 3; ++i) A.a[3 * s + i] = status == 1 ? a[i].v : 0.0;
  A.status[s] = status;
  return status;
}

// F and Gn are shared-memory col-major arrays (13x13, 13x6); fv 13.  acc_a, acc_D: an applied accelerometer sample's
// a and D (accel_model), or nullptr: the reference's model with the control u3 (nullptr: zero)
__device__ void motion_model(const double *xv, const double *u3, double dt_, double *fv, double *F,
                             double *Gn, const double *acc_a = nullptr, const double *acc_D = nullptr) {
  const rd dt(dt_);
  const Quat qold = {rd(xv[3]), rd(xv[4]), rd(xv[5]), rd(xv[6])};
  const rd om[3] = {rd(xv[10]), rd(xv[11]), rd(xv[12])};
  const rd av[3] = {om[0] * dt, om[1] * dt, om[2] * dt};
  const Quat qwt = quat_from_angular_velocity(av);
  const Quat qnew = quat_mul(qold, qwt);
  const rd hdt2 = (rd(0.5) * dt) * dt;
  for (int i = 0; i < 3; ++i) {
    const rd r = rd(xv[i]) + rd(xv[7 + i]) * dt;
    fv[i] = acc_a ? (r + rd(acc_a[i]) * hdt2).v : r.v;
  }
  fv[3] = qnew.w.v;
  fv[4] = qnew.x.v;
  fv[5] = qnew.y.v;
  fv[6] = qnew.z.v;
  for (int i = 0; i < 3; ++i) fv[7 + i] = (rd(xv[7 + i]) + rd(acc_a ? acc_a[i] : u3 ? u3[i] : 0.0) * dt).v;
  for (int i = 0; i < 3; ++i) fv[10 + i] = om[i].v;

  for (int i = 0; i < 169; ++i) F[i] = 0.0;
  for (int i = 0; i < 13; ++i) F[i + 13 * i] = 1.0;
  for (int i = 0; i < 3; ++i) F[i + 13 * (7 + i)] = (rd(1.0) * dt).v;
  if (acc_D)  // dr'/dq = hdt2 D, dv'/dq = dt D
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 4; ++j) {
        F[i + 13 * (3 + j)] = (hdt2 * rd(acc_D[4 * i + j])).v;
        F[(7 + i) + 13 * (3 + j)] = (dt * rd(acc_D[4 * i + j])).v;
      }
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
// sel_mode: [B] every stream's SL2_SELECT_* (sl2_set_stream_selection), or nullptr: every stream selects by trace.  An
// SL2_SELECT_INFORMATION stream keeps the provisional rank of every candidate (visible, ranked before the first zero
// trace) in sel_rank and leaves the truncation, the job slots and nsel to select_kernel (select.cu).  rv: [B] the
// streams' recovery states (recover.cu), or nullptr: no stream of the launch has recovery on.  A stream that enters
// the step lost selects nothing, under either rule, as with n_select = 0.  acc: the streams' accelerometers (acc.on ==
// nullptr: none); a stream whose step applies a sample predicts with its a, D and linear noise block L.
__global__ void __launch_bounds__(128) predict_kernel(const Sl2Dev d, int stream_lo,
                                                      const double *u3, int do_predict,
                                                      int do_measure, const int *sel_mode,
                                                      const sl2_recovery_result *rv, const Sl2Accel acc) {
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
    __shared__ double acc_a[3], acc_D[12], acc_L[9];
    __shared__ int s_acc;
    if (tid == 0) {
      s_acc = acc.on ? accel_model(acc, s, xv, sc.dt, acc_a, acc_D, acc_L) : 0;
      motion_model(xv, u3, sc.dt, fv, F, Gn, s_acc == 1 ? acc_a : nullptr, s_acc == 1 ? acc_D : nullptr);
    }
    __syncthreads();
    // Q = (G * Pnn) * G^T, Pnn = diag(lin x3, ang x3)   (motion_model.cpp:157-216); with an applied accelerometer
    // sample Pnn's linear block is the full L
    // TT = F * Pxx
    const bool full = s_acc == 1;
    for (int e = tid; e < 169; e += blockDim.x) {
      const int i = e % 13, j = e / 13;
      const rd dt(sc.dt);
      const rd lin = rd(4.0) * rd(4.0) * dt * dt, ang = rd(6.0) * rd(6.0) * dt * dt;
      rd q(0.0), t(0.0);
      for (int k = 0; k < 6; ++k) {
        rd gp;  // (G*Pnn)(i,k)
        if (full && k < 3)
          gp = ((rd(0.0) + rd(Gn[i]) * rd(acc_L[k])) + rd(Gn[i + 13]) * rd(acc_L[3 + k])) +
               rd(Gn[i + 26]) * rd(acc_L[6 + k]);
        else
          gp = rd(0.0) + rd(Gn[i + 13 * k]) * (k < 3 ? lin : ang);
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
  const bool info = sel_mode && sel_mode[s] == SL2_SELECT_INFORMATION;
  // information: the candidates are every rank before the first zero score
  const int nsel = (rv && rv[s].lost) ? 0 : info ? min(s_r0, s_nvis) : min(min(sc.n_select, s_r0), s_nvis);
  for (int i = tid; i < nf; i += blockDim.x) {
    int rank = d.sel_rank[fb + i];
    if (rank >= nsel) rank = -1;
    d.sel_rank[fb + i] = rank;
    if (rank >= 0 && !info) {
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
    d.nsel[s] = info ? 0 : nsel;  // select_kernel writes the information count
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
    times_dqbar_by_dq(Dr);
    times_dqbar_by_dq(Dh);
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
__global__ void __launch_bounds__(256) cull_kernel(const Sl2Dev d, int stream_lo, int force_index,
                                                    const Sl2Subpix sp, const Sl2Normals nrm) {
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
      if (sp.z) {  // and so does its sub-pixel match
        sp.z[(fb + k) * 2 + 0] = sp.z[(fb + i) * 2 + 0];
        sp.z[(fb + k) * 2 + 1] = sp.z[(fb + i) * 2 + 1];
        sp.refined[fb + k] = sp.refined[fb + i];
      }
      if (nrm.prm) {  // and so does its normal estimate
        for (int e = 0; e < 2; ++e) nrm.theta[(fb + k) * 2 + e] = nrm.theta[(fb + i) * 2 + e];
        for (int e = 0; e < 3; ++e) nrm.cov[(fb + k) * 3 + e] = nrm.cov[(fb + i) * 3 + e];
        nrm.count[fb + k] = nrm.count[fb + i];
        nrm.status[fb + k] = nrm.status[fb + i];
      }
    }
    if (sp.z)  // the vacated slots hold no match: a feature appended there starts unrefined
      for (int i = nk; i < nf; ++i) sp.refined[fb + i] = 0;
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

cudaError_t sl2_launch_append(const Sl2Dev &d, int s, const double *y3_dev, const double *xp7_dev,
                              const uint8_t *patch_rows16_dev, const double *Pcol_dev, Sl2Queue q) {
  return sl2_launch_kernel(append_kernel, dim3(1), dim3(256), 0, q, false, d, s, y3_dev, xp7_dev, patch_rows16_dev,
                           Pcol_dev);
}

}  // namespace

cudaError_t sl2_launch_predict(const Sl2Dev &d, int stream_lo, int stream_cnt, const double *u3_dev,
                               int do_predict, int do_measure, const int *sel_mode_dev, Sl2Queue q,
                               const sl2_recovery_result *rv_dev, const Sl2Accel &acc) {
  if (stream_cnt <= 0) return cudaSuccess;
  // 128 threads, one feature each per pass over the map (two passes at SL2_MAX_FEATURES); the kernel needs ~255
  // registers per thread, so 128-thread CTAs are what lets two streams share an SM
  return sl2_launch_kernel(predict_kernel, dim3(stream_cnt), dim3(128), 0, q, sl2_use_pdl(stream_cnt), d,
                           stream_lo, u3_dev, do_predict, do_measure, sel_mode_dev, rv_dev, acc);
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

cudaError_t sl2_launch_cull(const Sl2Dev &d, int stream_lo, int stream_cnt, int force_index, const Sl2Subpix &sp,
                            Sl2Queue q, const Sl2Normals &nrm) {
  if (stream_cnt <= 0) return cudaSuccess;
  return sl2_launch_kernel(cull_kernel, dim3(stream_cnt), dim3(256), 0, q, sl2_use_pdl(stream_cnt), d,
                           stream_lo, force_index, sp, nrm);
}

extern "C" {

int sl2_ekf_predict(sl2_ctx *c, int32_t s, const double *u3) {
  if (bad_stream(c, s)) return fail(c, SL2_ERR_ARG, "bad stream");
  Stage u{STAGE_IN, u3 ? (size_t)24 : 0, u3};
  return staged_call(c, {&u}, [] {}, [&] {
    CU_TRY(c, sl2_launch_predict(c->d, s, 1, u3 ? u.dev<double>() : nullptr, 1, 0, nullptr, queue(c)));
    return SL2_OK;
  });
}

int sl2_predict_measurements(sl2_ctx *c, int32_t s) {
  if (bad_stream(c, s)) return fail(c, SL2_ERR_ARG, "bad stream");
  const bool info = c->opt[s].sel.mode == SL2_SELECT_INFORMATION;
  CU_TRY(c, sl2_launch_predict(c->d, s, 1, nullptr, 0, 1, info ? c->sel_mode_dev : nullptr, queue(c)));
  if (info) {
    const int rc = select_streams(c, s, 1, queue(c));
    if (rc) return rc;
  }
  int nv = 0;
  CU_TRY(c, cudaMemcpyAsync(&nv, c->d.nvisible + s, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return nv;
}

int sl2_delete_feature(sl2_ctx *c, int32_t s, int32_t index) {
  if (bad_stream(c, s)) return fail(c, SL2_ERR_ARG, "bad stream");
  const int n = sl2_num_features(c, s);
  if (n < 0) return n;
  if (index < 0 || index >= n) return fail(c, SL2_ERR_ARG, "sl2_delete_feature: bad index");
  CU_TRY(c, sl2_launch_cull(c->d, s, 1, index, subpixel_args(c, s, 1), queue(c), normals_args(c, s, 1)));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return SL2_OK;
}

int sl2_append_feature(sl2_ctx *c, int32_t s, const double *y, const double *xp_org, const uint8_t *patch,
                       const double *Pcol) {
  if (bad_stream(c, s) || !y || !xp_org || !patch) return fail(c, SL2_ERR_ARG, "sl2_append_feature: bad argument");
  const int nf = sl2_num_features(c, s);
  if (nf < 0) return nf;
  if (nf >= c->cfg.max_features) return fail(c, SL2_ERR_STATE, "sl2_append_feature: the map is full (max_features)");
  const int box = c->d.box, n3 = SL2_NXV + 3 * nf + 3;
  Stage ys{STAGE_IN, 24, y}, xs{STAGE_IN, 56, xp_org}, pc{STAGE_IN, Pcol ? 8 * 3 * (size_t)n3 : 0, Pcol},
      rows{STAGE_IN, (size_t)box * 16};
  int rc = normals_reset(c, s, nf, 1);  // the new feature's normal is unestimated
  if (rc) return rc;
  rc = staged_call(
      c, {&ys, &xs, &pc, &rows}, [&] { pack_patch_rows(rows.h, patch, 1, box); },
      [&] {
        CU_TRY(c, sl2_launch_append(c->d, s, ys.dev<double>(), xs.dev<double>(), rows.d,
                                    Pcol ? pc.dev<double>() : nullptr, queue(c)));
        return SL2_OK;
      });
  return rc ? rc : nf;  // index of the new feature
}

}  // extern "C"
