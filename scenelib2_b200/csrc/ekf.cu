// ekf.cu — EKF predict / measurement prediction + selection / cull on sm_90a (the update is update.cu).
//
// Replaces, per camera stream (one CTA per stream, all streams of a context in one launch):
//   Kalman::KalmanFilterPredict            kalman.cpp:50-69   (+ motion_model.cpp:84-217)
//   MonoSLAM::auto_select_n_features       monoslam.cpp:187-254 (+ :289-308,
//                                          full_feature_model.cpp:67-195, camera.cpp:90-300)
//   MonoSLAM::delete_bad_features          monoslam.cpp:644-703, 770-812
//
// State layout in HBM: ONE dense column-major P (ld x ld) per stream in the order of
// construct_total_covariance (monoslam.cpp:518-546): [xv(13) | y_0 | y_1 | ...], with both
// triangles kept bit-consistent (the reference rebuilds the lower triangle from the upper blocks
// on every gather, so P is exactly block-symmetric whenever it is read).
//
// Small bit-critical prologue math (everything that decides WHICH pixels are searched: S_i,
// Sinv, h_i) uses never-fused __d*_rn ops in the oracle's evaluation order.
#include "sl2_common.cuh"

namespace {

struct Quat {
  rd w, x, y, z;
};

__device__ Quat quat_mul(const Quat &a, const Quat &b) {
  Quat q;
  q.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
  q.x = a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y;
  q.y = a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z;
  q.z = a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x;
  return q;
}

__device__ Quat quat_inverse(const Quat &q) {
  const rd n2 = q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z;
  Quat r;
  if (n2.v > 0.0) {
    r.w = q.w / n2;
    r.x = (-q.x) / n2;
    r.y = (-q.y) / n2;
    r.z = (-q.z) / n2;
  }
  return r;
}

__device__ void quat_to_R(const Quat &q, rd R[3][3]) {
  const rd two(2.0), one(1.0);
  const rd tx = two * q.x, ty = two * q.y, tz = two * q.z;
  const rd twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
  const rd txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
  const rd tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
  R[0][0] = one - (tyy + tzz);
  R[0][1] = txy - twz;
  R[0][2] = txz + twy;
  R[1][0] = txy + twz;
  R[1][1] = one - (txx + tzz);
  R[1][2] = tyz - twx;
  R[2][0] = txz - twy;
  R[2][1] = tyz + twx;
  R[2][2] = one - (txx + tyy);
}

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

// ---------------------------------------------------------------------------------------------
// per-feature measurement prediction (one thread per feature)
// ---------------------------------------------------------------------------------------------
struct FeatPred {
  rd h[2];
  rd dxp[2][7];
  rd dy[2][3];
  rd var;
  rd S[2][2];
};

__device__ void zeroedyi(const rd yi[3], const double *xp, rd z[3], rd dz_dxp[3][7], rd RRW[3][3]) {
  const rd d[3] = {yi[0] - rd(xp[0]), yi[1] - rd(xp[1]), yi[2] - rd(xp[2])};
  const Quat q = {rd(xp[3]), rd(xp[4]), rd(xp[5]), rd(xp[6])};
  const Quat qi = quat_inverse(q);
  quat_to_R(qi, RRW);
  for (int i = 0; i < 3; ++i) {
    rd s(0.0);
    for (int k = 0; k < 3; ++k) s = s + RRW[i][k] * d[k];
    z[i] = s;
  }
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) dz_dxp[i][j] = RRW[i][j] * rd(-1.0);
  // feature_model.cpp:187-238 applied to (qRW, d); then * dqbar_by_dq = diag(1,-1,-1,-1)
  const rd two(2.0);
  const rd w2 = two * qi.w, x2 = two * qi.x, y2 = two * qi.y, z2 = two * qi.z;
  const rd m0[9] = {w2, -z2, y2, z2, w2, -x2, -y2, x2, w2};
  const rd mx[9] = {x2, y2, z2, y2, -x2, -w2, z2, w2, -x2};
  const rd my[9] = {-y2, x2, w2, x2, y2, z2, -w2, z2, -y2};
  const rd mz[9] = {-z2, -w2, x2, w2, -z2, y2, x2, y2, z2};
  for (int i = 0; i < 3; ++i) {
    rd s0(0.0), s1(0.0), s2(0.0), s3(0.0);
    for (int k = 0; k < 3; ++k) {
      s0 = s0 + m0[i * 3 + k] * d[k];
      s1 = s1 + mx[i * 3 + k] * d[k];
      s2 = s2 + my[i * 3 + k] * d[k];
      s3 = s3 + mz[i * 3 + k] * d[k];
    }
    dz_dxp[i][3] = s0;
    dz_dxp[i][4] = -s1;
    dz_dxp[i][5] = -s2;
    dz_dxp[i][6] = -s3;
  }
}

// Pxx: shared 13x13 col-major; Pcol: global pointer to P(0, pos) (column-major, ld)
__device__ void predict_feature(const double *cam, const double *xv, const rd yi[3],
                                const double *Pxx, const double *Pcol, int ld, int pos,
                                FeatPred &o) {
  rd z[3], dz_dxp[3][7], RRW[3][3];
  zeroedyi(yi, xv, z, dz_dxp, RRW);
  const rd fku(cam[2]), fkv(cam[3]), u0(cam[4]), v0(cam[5]), kd1(cam[6]), sd(cam[7]);
  const rd one(1.0), two(2.0);
  // Camera::Project, camera.cpp:90-114
  const rd uc = (-fku) * z[0] / z[2];
  const rd vc = (-fkv) * z[1] / z[2];
  const rd radius2 = uc * uc + vc * vc;
  const rd factor = rsqrt_(one + two * kd1 * radius2);
  o.h[0] = uc / factor + u0;
  o.h[1] = vc / factor + v0;
  // Camera::ProjectionJacobian, camera.cpp:183-215
  const rd fku_yz = fku / z[2], fkv_yz = fkv / z[2];
  rd du[2][3];
  du[0][0] = -fku_yz;
  du[0][1] = rd(0.0);
  du[0][2] = fku_yz * z[0] / z[2];
  du[1][0] = rd(0.0);
  du[1][1] = -fkv_yz;
  du[1][2] = fkv_yz * z[1] / z[2];
  rd dh[2][2];
  dh[0][0] = uc * uc;
  dh[0][1] = uc * vc;
  dh[1][0] = vc * uc;
  dh[1][1] = vc * vc;
  const rd r2 = dh[0][0] + dh[1][1];
  const rd distor = one + two * kd1 * r2;
  const rd distor1_2 = rsqrt_(distor);
  const rd distor3_2 = distor1_2 * distor;
  const rd scale = rd(-2.0) * kd1 / distor3_2;
  for (int i = 0; i < 2; ++i)
    for (int j = 0; j < 2; ++j) dh[i][j] = dh[i][j] * scale;
  dh[0][0] = dh[0][0] + (one / distor1_2);
  dh[1][1] = dh[1][1] + (one / distor1_2);
  rd dhid[2][3];
  for (int i = 0; i < 2; ++i)
    for (int j = 0; j < 3; ++j) {
      rd s(0.0);
      for (int k = 0; k < 2; ++k) s = s + dh[i][k] * du[k][j];
      dhid[i][j] = s;
    }
  for (int i = 0; i < 2; ++i) {
    for (int j = 0; j < 7; ++j) {
      rd s(0.0);
      for (int k = 0; k < 3; ++k) s = s + dhid[i][k] * dz_dxp[k][j];
      o.dxp[i][j] = s;
    }
    for (int j = 0; j < 3; ++j) {
      rd s(0.0);
      for (int k = 0; k < 3; ++k) s = s + dhid[i][k] * RRW[k][j];
      o.dy[i][j] = s;
    }
  }
  // Camera::MeasurementNoise, camera.cpp:282-300
  const rd dx = o.h[0] - u0, dyv = o.h[1] - v0;
  const rd distance = rsqrt_(dx * dx + dyv * dyv);
  const rd max_distance = rsqrt_(u0 * u0 + v0 * v0);
  const rd ratio = distance / max_distance;
  const rd sd_use = sd * (one + ratio);
  o.var = one * (sd_use * sd_use);
  // FeatureModel::func_Si, feature_model.cpp:99-116.  dh_by_dxv = [dh_by_dxp | 0(2x6)]
  // (motion_model.cpp:224-235), so terms with k >= 7 are exact zeros and are skipped.
  rd A[2][7], Bm[2][3], Cm[2][3];
  for (int r = 0; r < 2; ++r) {
    for (int j = 0; j < 7; ++j) {
      rd s(0.0);
      for (int k = 0; k < 7; ++k) s = s + o.dxp[r][k] * rd(Pxx[k + 13 * j]);
      A[r][j] = s;
    }
    for (int j = 0; j < 3; ++j) {
      rd s(0.0);
      for (int k = 0; k < 7; ++k) s = s + o.dxp[r][k] * rd(Pcol[k + (size_t)ld * j]);
      Bm[r][j] = s;
      rd t(0.0);
      for (int k = 0; k < 3; ++k) t = t + o.dy[r][k] * rd(Pcol[(pos + k) + (size_t)ld * j]);
      Cm[r][j] = t;
    }
  }
  for (int r = 0; r < 2; ++r)
    for (int c = 0; c < 2; ++c) {
      rd s1(0.0), t1(0.0), t1t(0.0), s4(0.0);
      for (int k = 0; k < 7; ++k) s1 = s1 + A[r][k] * o.dxp[c][k];
      for (int k = 0; k < 3; ++k) t1 = t1 + Bm[r][k] * o.dy[c][k];
      for (int k = 0; k < 3; ++k) t1t = t1t + Bm[c][k] * o.dy[r][k];
      for (int k = 0; k < 3; ++k) s4 = s4 + Cm[r][k] * o.dy[c][k];
      rd S = rd(0.0) + s1;
      S = S + t1;
      S = S + t1t;
      S = S + s4;
      S = S + (r == c ? o.var : rd(0.0));
      o.S[r][c] = S;
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
  for (int i = 0; i < 3; ++i) {
    rd s(0.0);
    for (int k = 0; k < 3; ++k) s = s + RWR[i][k] * z[k];
    a[i] = s;
  }
  zeroedyi(yi, xp_orig, z, t, R1);
  quat_to_R(Quat{rd(xp_orig[3]), rd(xp_orig[4]), rd(xp_orig[5]), rd(xp_orig[6])}, RWR);
  for (int i = 0; i < 3; ++i) {
    rd s(0.0);
    for (int k = 0; k < 3; ++k) s = s + RWR[i][k] * z[k];
    b[i] = s;
  }
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

  if (tid < 13) xv[tid] = x[tid];
  for (int e = tid; e < 169; e += blockDim.x) Pxx[e] = P[(e % 13) + (size_t)ld * (e / 13)];
  __syncthreads();

  if (do_predict) {
    if (tid == 0) motion_model(xv, u3, d.dt, fv, F, Gn);
    __syncthreads();
    // Q = (G * Pnn) * G^T, Pnn = diag(lin x3, ang x3)   (motion_model.cpp:157-216)
    // TT = F * Pxx
    for (int e = tid; e < 169; e += blockDim.x) {
      const int i = e % 13, j = e / 13;
      const rd dt(d.dt);
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
      predict_feature(d.cam, xv, yi, Pxx, P + (size_t)ld * pos, ld, pos, fp);
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
      const int cant = visibility_test(d.cam, xv, yi, d.xp_org + (fb + i) * 7, fp.h);
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
  const int nsel = min(min(d.n_select, s_r0), s_nvis);
  for (int i = tid; i < nf; i += blockDim.x) {
    int rank = d.sel_rank[fb + i];
    if (rank >= nsel) rank = -1;
    d.sel_rank[fb + i] = rank;
    if (rank >= 0) {
      d.job_feat[fb + rank] = i;
      d.job_centre[(fb + rank) * 2 + 0] = d.h[(fb + i) * 2 + 0];
      d.job_centre[(fb + rank) * 2 + 1] = d.h[(fb + i) * 2 + 1];
      double p00, p01, p11;
      if (d.ovr[0] > 0.0) {
        p00 = d.ovr[0];
        p01 = d.ovr[1];
        p11 = d.ovr[2];
      } else {
        // monoslam.cpp:371-374: LLT, inverse of L, Sinv = Linv^T Linv (closed form, see oracle)
        const rd s00(d.S[(fb + i) * 4 + 0]), s10(d.S[(fb + i) * 4 + 1]), s11(d.S[(fb + i) * 4 + 3]);
        const rd l00 = rsqrt_(s00);
        const rd l10 = s10 / l00;
        const rd l11 = rsqrt_(s11 - l10 * l10);
        const rd x00 = rd(1.0) / l00;
        const rd x10 = (rd(0.0) - l10 * x00) / l11;
        const rd x11 = rd(1.0) / l11;
        p00 = (x00 * x00 + x10 * x10).v;
        p01 = (x10 * x11).v;
        p11 = (x11 * x11).v;
      }
      d.job_puinv[(fb + rank) * 3 + 0] = p00;
      d.job_puinv[(fb + rank) * 3 + 1] = p01;
      d.job_puinv[(fb + rank) * 3 + 2] = p11;
    }
  }
  if (tid == 0) {
    d.nsel[s] = nsel;
    d.nvisible[s] = s_nvis;
    d.nmeas[s] = 0;
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
      for (int e = 0; e < 7; ++e) d.xp_org[(fb + k) * 7 + e] = d.xp_org[(fb + i) * 7 + e];
      d.attempted[fb + k] = d.attempted[fb + i];
      d.successful[fb + k] = d.successful[fb + i];
      for (int e = 0; e < box16; ++e)
        d.patches[(fb + k) * box16 + e] = d.patches[(fb + i) * box16 + e];
      for (int e = 0; e < 2; ++e) {
        d.h[(fb + k) * 2 + e] = d.h[(fb + i) * 2 + e];
        d.z_uv[(fb + k) * 2 + e] = d.z_uv[(fb + i) * 2 + e];
      }
      for (int e = 0; e < 4; ++e) d.S[(fb + k) * 4 + e] = d.S[(fb + i) * 4 + e];
      // Feature::dh_by_dxv_ / dh_by_dy_ / R_ move with the Feature object in the reference
      for (int e = 0; e < 14; ++e) d.dh_dxp[(fb + k) * 14 + e] = d.dh_dxp[(fb + i) * 14 + e];
      for (int e = 0; e < 6; ++e) d.dh_dy[(fb + k) * 6 + e] = d.dh_dy[(fb + i) * 6 + e];
      d.Rvar[fb + k] = d.Rvar[fb + i];
      d.best[fb + k] = d.best[fb + i];
      d.sel_rank[fb + k] = d.sel_rank[fb + i];
      d.found[fb + k] = d.found[fb + i];
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
    d.attempted[f] = 0;
    d.successful[f] = 0;
    d.sel_rank[f] = -1;
    d.found[f] = 0;
    d.best[f] = 0.0;
    d.h[f * 2] = d.h[f * 2 + 1] = 0.0;
    d.z_uv[f * 2] = d.z_uv[f * 2 + 1] = 0;
    for (int e = 0; e < 4; ++e) d.S[f * 4 + e] = 0.0;
    for (int e = 0; e < 14; ++e) d.dh_dxp[f * 14 + e] = 0.0;
    for (int e = 0; e < 6; ++e) d.dh_dy[f * 6 + e] = 0.0;
    d.Rvar[f] = 0.0;
  }
  __syncthreads();
  if (tid == 0) d.nfeat[s] = nf + 1;
}

}  // namespace

cudaError_t sl2_launch_append(const Sl2Dev &d, int s, const double *y3_dev, const double *xp7_dev,
                              const uint8_t *patch_rows16_dev, const double *Pcol_dev, cudaStream_t st) {
  append_kernel<<<1, 256, 0, st>>>(d, s, y3_dev, xp7_dev, patch_rows16_dev, Pcol_dev);
  return cudaGetLastError();
}

cudaError_t sl2_launch_predict(const Sl2Dev &d, int stream_lo, int stream_cnt, const double *u3_dev,
                               int do_predict, int do_measure, cudaStream_t st) {
  if (stream_cnt <= 0) return cudaSuccess;
  // 128 threads = one per feature (SL2_MAX_FEATURES); the kernel needs ~255 registers per thread,
  // so 128-thread CTAs are what lets two streams share an SM
  return sl2_launch_kernel(predict_kernel, dim3(stream_cnt), dim3(128), 0, st, sl2_use_pdl(d, stream_cnt), d,
                           stream_lo, u3_dev, do_predict, do_measure);
}

cudaError_t sl2_launch_cull(const Sl2Dev &d, int stream_lo, int stream_cnt, int force_index,
                            cudaStream_t st) {
  if (stream_cnt <= 0) return cudaSuccess;
  return sl2_launch_kernel(cull_kernel, dim3(stream_cnt), dim3(256), 0, st, sl2_use_pdl(d, stream_cnt), d,
                           stream_lo, force_index);
}
