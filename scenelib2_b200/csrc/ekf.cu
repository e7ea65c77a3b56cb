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
// Map features and depth particles share one statement of the camera and feature models
// (quat_inverse .. sinv_from_S below).
//
// State layout in HBM: ONE dense column-major P (ld x ld) per stream in the order of
// construct_total_covariance (monoslam.cpp:518-546): [xv(13) | y_0 | y_1 | ...], with both
// triangles kept bit-consistent (the reference rebuilds the lower triangle from the upper blocks
// on every gather, so P is exactly block-symmetric whenever it is read).
//
// Small bit-critical prologue math (everything that decides WHICH pixels are searched: S_i,
// Sinv, h_i) uses never-fused __d*_rn ops in the oracle's evaluation order.
#include <math_constants.h>

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

// Eigen::Quaterniond::inverse(): conjugate / squaredNorm, the zero quaternion when the norm is 0
__device__ __forceinline__ Quat quat_inverse(const Quat &q) {
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

// Eigen::Quaterniond::toRotationMatrix()
__device__ __forceinline__ void quat_to_R(const Quat &q, rd R[3][3]) {
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

// M a, every row summed from 0.0 in ascending order like the oracle
__device__ __forceinline__ void mat3_vec(const rd M[3][3], const rd a[3], rd out[3]) {
  for (int i = 0; i < 3; ++i) {
    rd s(0.0);
    for (int k = 0; k < 3; ++k) s = s + M[i][k] * a[k];
    out[i] = s;
  }
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
// measurement models, one thread per map feature (predict_kernel) or per depth particle
// (particle_predict_kernel)
// ---------------------------------------------------------------------------------------------
// dRq_times_a_by_dq(qRW, a) * dqbar_by_dq (feature_model.cpp:187-238, 152-162), dqbar_by_dq = diag(1,-1,-1,-1)
__device__ __forceinline__ void dRq_times_a_by_dq(const Quat &qi, const rd a[3], rd D[3][4]) {
  const rd two(2.0);
  const rd w2 = two * qi.w, x2 = two * qi.x, y2 = two * qi.y, z2 = two * qi.z;
  const rd m0[9] = {w2, -z2, y2, z2, w2, -x2, -y2, x2, w2};
  const rd mx[9] = {x2, y2, z2, y2, -x2, -w2, z2, w2, -x2};
  const rd my[9] = {-y2, x2, w2, x2, y2, z2, -w2, z2, -y2};
  const rd mz[9] = {-z2, -w2, x2, w2, -z2, y2, x2, y2, z2};
  for (int i = 0; i < 3; ++i) {
    rd s0(0.0), s1(0.0), s2(0.0), s3(0.0);
    for (int k = 0; k < 3; ++k) {
      s0 = s0 + m0[i * 3 + k] * a[k];
      s1 = s1 + mx[i * 3 + k] * a[k];
      s2 = s2 + my[i * 3 + k] * a[k];
      s3 = s3 + mz[i * 3 + k] * a[k];
    }
    D[i][0] = s0;
    D[i][1] = -s1;
    D[i][2] = -s2;
    D[i][3] = -s3;
  }
}

// RRW of the camera pose xp (position r, quaternion qWR): the rotation of qRW = qWR^-1; returns qRW
__device__ __forceinline__ Quat pose_RRW(const double *xp, rd RRW[3][3]) {
  const Quat qi = quat_inverse(Quat{rd(xp[3]), rd(xp[4]), rd(xp[5]), rd(xp[6])});
  quat_to_R(qi, RRW);
  return qi;
}

// z = RRW (yi - r) with d = yi - r: the camera-frame point of yi seen from xp, RRW = pose_RRW(xp)
__device__ __forceinline__ void zeroed_point(const rd RRW[3][3], const rd yi[3], const double *xp, rd d[3], rd z[3]) {
  for (int i = 0; i < 3; ++i) d[i] = yi[i] - rd(xp[i]);
  mat3_vec(RRW, d, z);
}

// feature_model.cpp:187-238: z = RRW (yi - r), dz/dxp = [-RRW | dRq_times_a_by_dq(qRW, yi - r) dqbar_by_dq]
__device__ __forceinline__ void zeroedyi(const rd yi[3], const double *xp, rd z[3], rd dz_dxp[3][7],
                                         rd RRW[3][3]) {
  rd d[3];
  const Quat qi = pose_RRW(xp, RRW);
  zeroed_point(RRW, yi, xp, d, z);
  rd D[3][4];
  dRq_times_a_by_dq(qi, d, D);
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) dz_dxp[i][j] = RRW[i][j] * rd(-1.0);
    for (int j = 0; j < 4; ++j) dz_dxp[i][3 + j] = D[i][j];
  }
}

// Camera::Project (camera.cpp:90-114) of the camera-frame point z; uc, vc = the undistorted image-centred point
__device__ __forceinline__ void project_point(const double *cam, const rd z[3], rd h[2], rd &uc, rd &vc) {
  const rd fku(cam[2]), fkv(cam[3]), u0(cam[4]), v0(cam[5]), kd1(cam[6]);
  const rd one(1.0), two(2.0);
  uc = (-fku) * z[0] / z[2];
  vc = (-fkv) * z[1] / z[2];
  const rd radius2 = uc * uc + vc * vc;
  const rd factor = rsqrt_(one + two * kd1 * radius2);
  h[0] = uc / factor + u0;
  h[1] = vc / factor + v0;
}

// Camera::Unproject (camera.cpp:133-157) of the image point h: the camera-frame direction (x, y, 1) that
// project_point maps to h (NaN where 1 - 2 kd1 r^2 < 0, outside the model's reach)
__device__ __forceinline__ void unproject_point(const double *cam, const rd h[2], rd out[3]) {
  const rd fku(cam[2]), fkv(cam[3]), u0(cam[4]), v0(cam[5]), kd1(cam[6]);
  const rd one(1.0), two(2.0);
  const rd c0 = h[0] - u0, c1 = h[1] - v0;
  const rd radius2 = c0 * c0 + c1 * c1;
  const rd factor = rsqrt_(one - two * kd1 * radius2);
  out[0] = (c0 / factor) / (-fku);
  out[1] = (c1 / factor) / (-fkv);
  out[2] = one;
}

// Camera::Project (camera.cpp:90-114) of the camera-frame point z, and J = dh/dz
// (Camera::ProjectionJacobian, camera.cpp:183-215)
__device__ __forceinline__ void project(const double *cam, const rd z[3], rd h[2], rd J[2][3]) {
  const rd fku(cam[2]), fkv(cam[3]), kd1(cam[6]);
  const rd one(1.0), two(2.0);
  rd uc, vc;
  project_point(cam, z, h, uc, vc);
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
  for (int i = 0; i < 2; ++i)
    for (int j = 0; j < 3; ++j) {
      rd s(0.0);
      for (int k = 0; k < 2; ++k) s = s + dh[i][k] * du[k][j];
      J[i][j] = s;
    }
}

// Camera::MeasurementNoise, camera.cpp:282-300: R = var I
__device__ __forceinline__ rd measurement_noise(const double *cam, const rd h[2]) {
  const rd u0(cam[4]), v0(cam[5]), sd(cam[7]), one(1.0);
  const rd dx = h[0] - u0, dy = h[1] - v0;
  const rd distance = rsqrt_(dx * dx + dy * dy);
  const rd max_distance = rsqrt_(u0 * u0 + v0 * v0);
  const rd ratio = distance / max_distance;
  const rd sd_use = sd * (one + ratio);
  return one * (sd_use * sd_use);
}

// FeatureModel::func_Si, feature_model.cpp:99-116, for a feature state of NY entries (3: map feature, 6: ray).
// dh_by_dxv = [dh_by_dxp | 0(2x6)] (motion_model.cpp:224-235), so terms with k >= 7 are exact zeros and are
// skipped.  Column-major blocks: Pxx (7 x 7 used) with leading dimension ldxx, Pxy (7 x NY used) ldxy, Pyy ldyy.
template <int NY>
__device__ __forceinline__ void func_Si(const rd dxp[2][7], const rd dy[2][NY], rd var, const double *Pxx,
                                        int ldxx, const double *Pxy, int ldxy, const double *Pyy, int ldyy,
                                        rd S[2][2]) {
  rd A[2][7], Bm[2][NY], Cm[2][NY];
  for (int r = 0; r < 2; ++r) {
    for (int j = 0; j < 7; ++j) {
      rd s(0.0);
      for (int k = 0; k < 7; ++k) s = s + dxp[r][k] * rd(Pxx[k + (size_t)ldxx * j]);
      A[r][j] = s;
    }
    for (int j = 0; j < NY; ++j) {
      rd s(0.0);
      for (int k = 0; k < 7; ++k) s = s + dxp[r][k] * rd(Pxy[k + (size_t)ldxy * j]);
      Bm[r][j] = s;
      rd t(0.0);
      for (int k = 0; k < NY; ++k) t = t + dy[r][k] * rd(Pyy[k + (size_t)ldyy * j]);
      Cm[r][j] = t;
    }
  }
  for (int r = 0; r < 2; ++r)
    for (int c = 0; c < 2; ++c) {
      rd s1(0.0), t1(0.0), t1t(0.0), s4(0.0);
      for (int k = 0; k < 7; ++k) s1 = s1 + A[r][k] * dxp[c][k];
      for (int k = 0; k < NY; ++k) t1 = t1 + Bm[r][k] * dy[c][k];
      for (int k = 0; k < NY; ++k) t1t = t1t + Bm[c][k] * dy[r][k];
      for (int k = 0; k < NY; ++k) s4 = s4 + Cm[r][k] * dy[c][k];
      rd v = rd(0.0) + s1;
      v = v + t1;
      v = v + t1t;
      v = v + s4;
      v = v + (r == c ? var : rd(0.0));
      S[r][c] = v;
    }
}

// (S^-1)00, 01, 11 of a 2x2 S: LLT, L^-1 in closed form, L^-T L^-1 (monoslam.cpp:371-374; Particle::set_S,
// feature_init_info.cpp:57-65; the oracle's puinv_from_S)
__device__ __forceinline__ void sinv_from_S(rd s00, rd s10, rd s11, rd Sinv[3]) {
  const rd l00 = rsqrt_(s00);
  const rd l10 = s10 / l00;
  const rd l11 = rsqrt_(s11 - l10 * l10);
  const rd x00 = rd(1.0) / l00;
  const rd x10 = (rd(0.0) - l10 * x00) / l11;
  const rd x11 = rd(1.0) / l11;
  Sinv[0] = x00 * x00 + x10 * x10;
  Sinv[1] = x10 * x11;
  Sinv[2] = x11 * x11;
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

  if (tid < (int)(sizeof(Sl2StreamCam) / sizeof(double)))
    reinterpret_cast<double *>(&sc)[tid] = reinterpret_cast<const double *>(d.cams + s)[tid];
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
// kernel 2b: match consensus (one-point RANSAC with exhaustive hypotheses; Civera, Grasa, Davison, Montiel, J. Field
// Robotics 2010) between the patch search and the EKF update, one CTA per camera stream of the launch; streams whose
// tau2[s] (= fl(tau * tau), 0 = off) is not > 0 return at once.  Semantics: include/sl2b200.h, sl2_set_stream_consensus.
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
//                 zeroed_point(RRW, y', xp'), project_point -> g;  du = (double)z_u - g_u, dv likewise;
//                 inlier iff the camera-frame depth is > 0 and du du + dv dv <= tau2 (NaN: never)
//   support(i) = inliers of i (i itself included); winner = largest support, ties to the lowest rank; when the
//   winner's support is >= 2 every match outside its inlier set gets found = 2 (matched, rejected by the consensus).
// Shape: warp w takes hypotheses w, w + CONS_WARPS, ...; its lanes take the matches j = lane + 32 c and count the
// support with ballot / popc.  The per-match terms and P[yj, 0:7] sit in shared memory, P[0:7, yi] and the 3x3 blocks
// P[yj, yi] are read from L2.
// ---------------------------------------------------------------------------------------------
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
  const unsigned bal = __ballot_sync(0xffffffffu, feat >= 0);
  if (lane == 0) wcount[warp] = __popc(bal);
  if (tid < (int)(sizeof(Sl2StreamCam) / sizeof(double)))
    reinterpret_cast<double *>(&sc)[tid] = reinterpret_cast<const double *>(d.cams + s)[tid];
  if (tid < 49) pxx[tid] = P[(tid % 7) + (size_t)ld * (tid / 7)];
  if (tid < 7) xp0[tid] = x[tid];
  __syncthreads();
  int base = 0, k = 0;
  for (int w = 0; w < CONS_WARPS; ++w) {
    if (w < warp) base += wcount[w];
    k += wcount[w];
  }
  if (feat >= 0) mf[base + __popc(bal & ((1u << lane) - 1u))] = feat;
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
    int sup = 0;
    for (int c32 = 0; c32 * 32 < k; ++c32) {
      const int j = c32 * 32 + lane;
      bool in = false;
      if (j < k) {
        const int pj = SL2_NXV + 3 * mf[j];
        rd yj[3];
        for (int r = 0; r < 3; ++r) {
          rd acc(0.0);
          for (int c = 0; c < 7; ++c) acc = acc + rd(pyx[j][r * 7 + c]) * rd(ma[i][c]);
          for (int c = 0; c < 3; ++c) acc = acc + rd(P[(pj + r) + (size_t)ld * (pi + c)]) * rd(mb[i][c]);
          yj[r] = rd(my[j][r]) + acc;
        }
        rd dd[3], zc[3], g[2], uc, vc;
        zeroed_point(RRW, yj, hxp[warp], dd, zc);
        if (zc[2].v > 0.0) {
          project_point(sc.cam, zc, g, uc, vc);
          const rd du = rd(mz[j][0]) - g[0], dv = rd(mz[j][1]) - g[1];
          in = (du * du + dv * dv).v <= t2;
        }
      }
      const unsigned b = __ballot_sync(0xffffffffu, in);
      if (lane == 0) mask[i][c32] = b;
      sup += __popc(b);
    }
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

// ---------------------------------------------------------------------------------------------
// relocalisation (sl2_relocalise; Williams, Klein, Reid, ICCV 2007): after the full-image search, the camera pose of
// a lost stream from its matches with a three-point consensus.  Semantics: include/sl2b200.h, sl2_relocalise.
// ---------------------------------------------------------------------------------------------
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

// match j against the pose xp (RRW = pose_RRW(xp)): in front of the camera and d2 = |z_j - h(y_j)|^2 <= t2 (NaN: no)
__device__ __forceinline__ bool reloc_inlier(const double *cam, const rd RRW[3][3], const double *xp,
                                             const double *y, const double *z, double t2, double *d2) {
  const rd yi[3] = {rd(y[0]), rd(y[1]), rd(y[2])};
  rd dd[3], zc[3];
  zeroed_point(RRW, yi, xp, dd, zc);
  if (!(zc[2].v > 0.0)) return false;
  rd g[2], uc, vc;
  project_point(cam, zc, g, uc, vc);
  const rd du = rd(z[0]) - g[0], dv = rd(z[1]) - g[1];
  *d2 = (du * du + dv * dv).v;
  return *d2 <= t2;
}

#define RELOC_WARPS 8
#define RELOC_THREADS (32 * RELOC_WARPS)  // one hypothesis per thread per round; >= SL2_MAX_FEATURES
#define RELOC_WORDS (SL2_MAX_FEATURES / 32)
static_assert(RELOC_THREADS >= SL2_MAX_FEATURES && RELOC_WORDS <= RELOC_WARPS, "one thread per feature");
static_assert(SL2_RELOC_HYPOTHESES % RELOC_THREADS == 0, "whole rounds of hypotheses");

struct RelocSmem {
  int mf[SL2_MAX_FEATURES];                     // feature of match j, j < k
  double mz[SL2_MAX_FEATURES][2];               // z_j
  double my[SL2_MAX_FEATURES][3];               // y_j
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

// inliers of the pose xp over the k matches, one warp; lane 0 writes the inlier words when `mask` is given
__device__ int reloc_support(const RelocSmem &S, const double *xp, double t2, int k, int lane, unsigned *mask) {
  rd RRW[3][3];
  pose_RRW(xp, RRW);
  int sup = 0;
  for (int c32 = 0; c32 * 32 < k; ++c32) {
    const int j = c32 * 32 + lane;
    double d2;
    const bool in = j < k && reloc_inlier(S.sc.cam, RRW, xp, S.my[j], S.mz[j], t2, &d2);
    const unsigned b = __ballot_sync(0xffffffffu, in);
    if (mask && lane == 0) mask[c32] = b;
    sup += __popc(b);
  }
  return sup;
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
  const unsigned bal = __ballot_sync(0xffffffffu, matched);
  if (lane == 0) S.wcount[warp] = __popc(bal);
  if (tid < (int)(sizeof(Sl2StreamCam) / sizeof(double)))
    reinterpret_cast<double *>(&S.sc)[tid] = reinterpret_cast<const double *>(d.cams + s)[tid];
  __syncthreads();
  int base = 0, k = 0;
  for (int w = 0; w < RELOC_WARPS; ++w) {
    if (w < warp) base += S.wcount[w];
    k += S.wcount[w];
  }
  const int myj = matched ? base + __popc(bal & ((1u << lane) - 1u)) : -1;
  if (matched) {
    S.mf[myj] = tid;
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
        for (int c = 0; c < 3; ++c) Pw[a][c] = S.my[t[a]][c], fb[a][c] = S.mbr[t[a]][c];
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
        const rd yi[3] = {rd(S.my[j][0]), rd(S.my[j][1]), rd(S.my[j][2])};
        rd dd[3], z[3], hh[2], J[2][3];
        zeroed_point(RRW, yi, S.pose, dd, z);
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
    const bool in = j < k && reloc_inlier(S.sc.cam, RRW, S.pose, S.my[j], S.mz[j], t2, &d2);
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
  if (threadIdx.x < sizeof(Sl2StreamCam) / sizeof(double))
    reinterpret_cast<double *>(&sc)[threadIdx.x] = reinterpret_cast<const double *>(d.cams + s)[threadIdx.x];
  __syncthreads();
  // qRW and RRW: one camera pose for every particle
  const Quat qi = quat_inverse(Quat{rd(xv[3]), rd(xv[4]), rd(xv[5]), rd(xv[6])});
  rd R[3][3];
  quat_to_R(qi, R);
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

cudaError_t sl2_launch_consensus(const Sl2Dev &d, int stream_lo, int stream_cnt, const double *tau2_dev, Sl2Queue q) {
  if (stream_cnt <= 0) return cudaSuccess;
  return sl2_launch_kernel(consensus_kernel, dim3(stream_cnt), dim3(32 * CONS_WARPS), 0, q, sl2_use_pdl(stream_cnt), d,
                           stream_lo, tau2_dev);
}

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
