// ORACLE — TEST INFRASTRUCTURE ONLY (see dense.hpp header).
//
// CPU restatement of the closed-form models that feed the SceneLib2 hot path:
//   camera            scenelib2/camera.cpp:49-300
//   motion model      scenelib2/motion_model.cpp:84-380
//   quaternion utils  scenelib2/support/math_util.cpp:61-114
//   measurement model scenelib2/full_feature_model.cpp:67-200,
//                     scenelib2/feature_model.cpp:99-238
// Every function cites the lines it follows.  Scalar expressions keep the reference's
// left-to-right evaluation order; Eigen quaternion helpers follow Eigen3's generic
// (non-vectorised) formulas.
// Pinning: every function here is checked against the reference's OWN source files compiled
// unmodified against oracle/stubs_arith (tests/test_oracle_ref.py, _ref/libsl2refmodels.so): the
// formulas are pinned (agreement < 1e-13, scalar Jacobians bit-exact); PARITY UNPINNED only for
// Eigen's summation order inside matrix products (Eigen absent, no reference goldens).
#pragma once
#include "dense.hpp"

namespace sl2o {

struct Quat {
  double w, x, y, z;
};

// Eigen::Quaterniond operator* (generic path).
inline Quat quat_mul(const Quat &a, const Quat &b) {
  Quat q;
  q.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
  q.x = a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y;
  q.y = a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z;
  q.z = a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x;
  return q;
}

// Eigen::Quaterniond::inverse(): conjugate / squaredNorm.
inline Quat quat_inverse(const Quat &q) {
  const double n2 = q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z;
  Quat r;
  if (n2 > 0.0) {
    r.w = q.w / n2;
    r.x = -q.x / n2;
    r.y = -q.y / n2;
    r.z = -q.z / n2;
  } else {
    r.w = r.x = r.y = r.z = 0.0;
  }
  return r;
}

// Eigen::Quaterniond::toRotationMatrix().
inline void quat_to_R(const Quat &q, double R[3][3]) {
  const double tx = 2.0 * q.x, ty = 2.0 * q.y, tz = 2.0 * q.z;
  const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
  const double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
  const double tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
  R[0][0] = 1.0 - (tyy + tzz);
  R[0][1] = txy - twz;
  R[0][2] = txz + twy;
  R[1][0] = txy + twz;
  R[1][1] = 1.0 - (txx + tzz);
  R[1][2] = tyz - twx;
  R[2][0] = txz - twy;
  R[2][1] = tyz + twx;
  R[2][2] = 1.0 - (txx + tyy);
}

// support/math_util.cpp:61-80
inline Quat quaternion_from_angular_velocity(const double av[3]) {
  Quat q;
  const double angle = std::sqrt(av[0] * av[0] + av[1] * av[1] + av[2] * av[2]);
  if (angle > 0.0) {
    const double s = std::sin(angle / 2.0) / angle;
    const double c = std::cos(angle / 2.0);
    q.x = s * av[0];
    q.y = s * av[1];
    q.z = s * av[2];
    q.w = c;
  } else {
    q.x = q.y = q.z = 0.0;
    q.w = 1.0;
  }
  return q;
}

// support/math_util.cpp:82-97 : d(q2 x q1)/dq1
inline Mat dq3_by_dq1(const Quat &q) {
  Mat m(4, 4);
  const double x = q.x, y = q.y, z = q.z, w = q.w;
  const double v[16] = {w, -x, -y, -z, x, w, -z, y, y, z, w, -x, z, -y, x, w};
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) m(i, j) = v[i * 4 + j];
  return m;
}

// support/math_util.cpp:99-114 : d(q2 x q1)/dq2
inline Mat dq3_by_dq2(const Quat &q) {
  Mat m(4, 4);
  const double x = q.x, y = q.y, z = q.z, w = q.w;
  const double v[16] = {w, -x, -y, -z, x, w, z, -y, y, -z, w, x, z, y, -x, w};
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) m(i, j) = v[i * 4 + j];
  return m;
}

// ---------------------------------------------------------------------------------------
// Camera  (camera.cpp)
// ---------------------------------------------------------------------------------------
struct Camera {
  int width = 320, height = 240;
  double fku = 195, fkv = 195, u0 = 162, v0 = 125, kd1 = 9e-6, sd = 1.0;
  // remembered by Project() for ProjectionJacobian() (camera.cpp:94,108)
  double last_camera[3] = {0, 0, 1};
  double last_image_centred[2] = {0, 0};

  // camera.cpp:90-114
  void project(const double cam[3], double h[2]) {
    last_camera[0] = cam[0];
    last_camera[1] = cam[1];
    last_camera[2] = cam[2];
    const double uc = -fku * cam[0] / cam[2];
    const double vc = -fkv * cam[1] / cam[2];
    last_image_centred[0] = uc;
    last_image_centred[1] = vc;
    const double radius2 = (uc * uc + vc * vc);
    const double factor = std::sqrt(1 + 2 * kd1 * radius2);
    h[0] = uc / factor + u0;
    h[1] = vc / factor + v0;
  }

  // camera.cpp:183-215 ; returns 2x3
  Mat projection_jacobian() const {
    const double fku_yz = fku / last_camera[2];
    const double fkv_yz = fkv / last_camera[2];
    Mat du_by_dy(2, 3);
    du_by_dy(0, 0) = -fku_yz;
    du_by_dy(0, 1) = 0.0;
    du_by_dy(0, 2) = fku_yz * last_camera[0] / last_camera[2];
    du_by_dy(1, 0) = 0.0;
    du_by_dy(1, 1) = -fkv_yz;
    du_by_dy(1, 2) = fkv_yz * last_camera[1] / last_camera[2];

    Mat dh_by_du(2, 2);
    const double uc = last_image_centred[0], vc = last_image_centred[1];
    dh_by_du(0, 0) = uc * uc;
    dh_by_du(0, 1) = uc * vc;
    dh_by_du(1, 0) = vc * uc;
    dh_by_du(1, 1) = vc * vc;
    const double radius2 = dh_by_du(0, 0) + dh_by_du(1, 1);
    const double distor = 1 + 2 * kd1 * radius2;
    const double distor1_2 = std::sqrt(distor);
    const double distor3_2 = distor1_2 * distor;
    const double scale = -2 * kd1 / distor3_2;
    for (double &e : dh_by_du.a) e *= scale;
    dh_by_du(0, 0) += (1 / distor1_2);
    dh_by_du(1, 1) += (1 / distor1_2);
    return mul(dh_by_du, du_by_dy);
  }

  // camera.cpp:282-300 ; R_i = var * I2
  double measurement_noise_variance(const double h[2]) const {
    const double dx = h[0] - u0, dy = h[1] - v0;
    const double distance = std::sqrt(dx * dx + dy * dy);
    const double max_distance = std::sqrt(u0 * u0 + v0 * v0);
    const double ratio = distance / max_distance;
    const double sd_use = sd * (1.0 + ratio);
    return sd_use * sd_use;
  }
};

// ---------------------------------------------------------------------------------------
// Motion model (motion_model.cpp).  State xv = [r(3) q(w,x,y,z) v(3) omega(3)].
// ---------------------------------------------------------------------------------------
struct MotionModel {
  static constexpr double kSdA = 4.0;      // motion_model.cpp:45
  static constexpr double kSdAlpha = 6.0;  // motion_model.cpp:45

  // motion_model.cpp:318-349
  static double dq0_by_domegaA(double omegaA, double omega, double dt) {
    return (-dt / 2.0) * (omegaA / omega) * std::sin(omega * dt / 2.0);
  }
  static double dqA_by_domegaA(double omegaA, double omega, double dt) {
    return (dt / 2.0) * omegaA * omegaA / (omega * omega) * std::cos(omega * dt / 2.0) +
           (1.0 / omega) * (1.0 - omegaA * omegaA / (omega * omega)) * std::sin(omega * dt / 2.0);
  }
  static double dqA_by_domegaB(double omegaA, double omegaB, double omega, double dt) {
    return (omegaA * omegaB / (omega * omega)) *
           ((dt / 2.0) * std::cos(omega * dt / 2.0) - (1.0 / omega) * std::sin(omega * dt / 2.0));
  }

  // motion_model.cpp:290-311 ; 4x3.  Divides by |omega| (quirk Q5: NaN at omega = 0).
  static Mat dqomegadt_by_domega(const double om[3], double dt) {
    const double omegamod = std::sqrt(om[0] * om[0] + om[1] * om[1] + om[2] * om[2]);
    Mat m(4, 3);
    m(0, 0) = dq0_by_domegaA(om[0], omegamod, dt);
    m(0, 1) = dq0_by_domegaA(om[1], omegamod, dt);
    m(0, 2) = dq0_by_domegaA(om[2], omegamod, dt);
    m(1, 0) = dqA_by_domegaA(om[0], omegamod, dt);
    m(1, 1) = dqA_by_domegaB(om[0], om[1], omegamod, dt);
    m(1, 2) = dqA_by_domegaB(om[0], om[2], omegamod, dt);
    m(2, 0) = dqA_by_domegaB(om[1], om[0], omegamod, dt);
    m(2, 1) = dqA_by_domegaA(om[1], omegamod, dt);
    m(2, 2) = dqA_by_domegaB(om[1], om[2], omegamod, dt);
    m(3, 0) = dqA_by_domegaB(om[2], om[0], omegamod, dt);
    m(3, 1) = dqA_by_domegaB(om[2], om[1], omegamod, dt);
    m(3, 2) = dqA_by_domegaA(om[2], omegamod, dt);
    return m;
  }

  // motion_model.cpp:84-146 : fv (13) and F = dfv/dxv (13x13)
  static void fv_and_dfv_by_dxv(const double xv[13], const double u[3], double dt, double fv[13],
                                Mat &F) {
    const Quat qold = {xv[3], xv[4], xv[5], xv[6]};
    const double omegaold[3] = {xv[10], xv[11], xv[12]};
    const double omdt[3] = {omegaold[0] * dt, omegaold[1] * dt, omegaold[2] * dt};
    const Quat qwt = quaternion_from_angular_velocity(omdt);
    const Quat qnew = quat_mul(qold, qwt);
    for (int i = 0; i < 3; ++i) fv[i] = xv[i] + xv[7 + i] * dt;
    fv[3] = qnew.w;
    fv[4] = qnew.x;
    fv[5] = qnew.y;
    fv[6] = qnew.z;
    for (int i = 0; i < 3; ++i) fv[7 + i] = xv[7 + i] + u[i] * dt;
    for (int i = 0; i < 3; ++i) fv[10 + i] = omegaold[i];

    F = Mat(13, 13);
    F.identity();
    for (int i = 0; i < 3; ++i) F(i, 7 + i) = 1.0 * dt;  // Temp33A = I * delta_t (:122-126)
    set_block(F, 3, 3, dq3_by_dq2(qwt));                 // :130-131
    const Mat T44 = dq3_by_dq1(qold);                    // :134
    const Mat T43 = dqomegadt_by_domega(omegaold, dt);   // :137-138
    set_block(F, 3, 10, mul(T44, T43));                  // :141-145
  }

  // motion_model.cpp:148-217 : Q = G * Pnn * G^T (13x13)
  static Mat Q(const double xv[13], double dt) {
    const double lin = kSdA * kSdA * dt * dt;
    const double ang = kSdAlpha * kSdAlpha * dt * dt;
    Mat Pnn(6, 6);
    for (int i = 0; i < 3; ++i) {
      Pnn(i, i) = lin;
      Pnn(3 + i, 3 + i) = ang;
    }
    Mat G(13, 6);
    for (int i = 0; i < 3; ++i) {
      G(7 + i, i) = 1.0;
      G(10 + i, 3 + i) = 1.0;
      G(i, i) = 1.0 * dt;
    }
    const Quat qold = {xv[3], xv[4], xv[5], xv[6]};
    const double omegaold[3] = {xv[10], xv[11], xv[12]};
    set_block(G, 3, 3, mul(dq3_by_dq1(qold), dqomegadt_by_domega(omegaold, dt)));
    return mul_nt(mul(G, Pnn), G);
  }

  // motion_model.cpp:351-380 (quirk Q2: qq = |q|^2 used where |q| would be exact)
  static Mat dqnorm_by_dq(const Quat &q) {
    const double qq = q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z;
    const double e[4] = {q.w, q.x, q.y, q.z};
    Mat M(4, 4);
    for (int i = 0; i < 4; ++i)
      for (int j = 0; j < 4; ++j)
        M(i, j) = (i == j) ? (1 - e[i] * e[i] / (qq * qq)) / qq : -e[i] * e[j] / (qq * qq * qq);
    return M;
  }

  // motion_model.cpp:237-263 : J = dxvnorm/dxv (13x13); xv itself is returned unchanged
  // (quirk Q1: Tempqb is a plain copy that is never normalised).
  static Mat dxvnorm_by_dxv(const double xv[13]) {
    Mat J(13, 13);
    J.identity();
    const Quat q = {xv[3], xv[4], xv[5], xv[6]};
    set_block(J, 3, 3, dqnorm_by_dq(q));
    return J;
  }
};

// ---------------------------------------------------------------------------------------
// Fully-initialised point feature measurement model (full_feature_model.cpp, feature_model.cpp)
// ---------------------------------------------------------------------------------------
struct FeaturePrediction {
  double h[2];
  Mat dh_by_dxp;  // 2x7
  Mat dh_by_dy;   // 2x3
  Mat dh_by_dxv;  // 2x13
  Mat R;          // 2x2
  Mat S;          // 2x2
};

struct FullFeatureModel {
  static constexpr double kMaximumLengthRatio = 2.0;                          // full_feature_model.cpp:49
  static constexpr double kImageSearchBoundary = 20.0;                        // :51
  static double maximum_angle_difference() { return M_PI * 45.0 / 180.0; }    // :50

  // feature_model.cpp:187-238 : the four dR/dq_i matrices applied to a.
  static Mat dRq_times_a_by_dq(const Quat &q, const double a[3]) {
    const double m0[9] = {2 * q.w, -2 * q.z, 2 * q.y, 2 * q.z, 2 * q.w, -2 * q.x, -2 * q.y, 2 * q.x, 2 * q.w};
    const double mx[9] = {2 * q.x, 2 * q.y, 2 * q.z, 2 * q.y, -2 * q.x, -2 * q.w, 2 * q.z, 2 * q.w, -2 * q.x};
    const double my[9] = {-2 * q.y, 2 * q.x, 2 * q.w, 2 * q.x, 2 * q.y, 2 * q.z, -2 * q.w, 2 * q.z, -2 * q.y};
    const double mz[9] = {-2 * q.z, -2 * q.w, 2 * q.x, 2 * q.w, -2 * q.z, 2 * q.y, 2 * q.x, 2 * q.y, 2 * q.z};
    const double *ms[4] = {m0, mx, my, mz};
    Mat out(3, 4);
    for (int c = 0; c < 4; ++c)
      for (int i = 0; i < 3; ++i) {
        double s = 0.0;
        for (int k = 0; k < 3; ++k) s += ms[c][i * 3 + k] * a[k];
        out(i, c) = s;
      }
    return out;
  }

  // full_feature_model.cpp:67-101
  static void zeroedyi(const double yi[3], const double xp[7], double zeroed[3], Mat &dz_by_dxp,
                       Mat &dz_by_dyi) {
    const double d[3] = {yi[0] - xp[0], yi[1] - xp[1], yi[2] - xp[2]};
    const Quat q = {xp[3], xp[4], xp[5], xp[6]};
    const Quat qRW = quat_inverse(q);
    double RRW[3][3];
    quat_to_R(qRW, RRW);
    for (int i = 0; i < 3; ++i) {
      double s = 0.0;
      for (int k = 0; k < 3; ++k) s += RRW[i][k] * d[k];
      zeroed[i] = s;
    }
    dz_by_dyi = Mat(3, 3);
    dz_by_dxp = Mat(3, 7);
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        dz_by_dyi(i, j) = RRW[i][j];
        dz_by_dxp(i, j) = RRW[i][j] * -1.0;
      }
    const Mat dz_by_dqRW = dRq_times_a_by_dq(qRW, d);
    Mat dqbar(4, 4);  // feature_model.cpp:152-162
    dqbar(0, 0) = 1.0;
    dqbar(1, 1) = -1.0;
    dqbar(2, 2) = -1.0;
    dqbar(3, 3) = -1.0;
    set_block(dz_by_dxp, 0, 3, mul(dz_by_dqRW, dqbar));
  }

  // full_feature_model.cpp:178-195 + monoslam.cpp:289-308 + feature_model.cpp:99-116,147-150
  static void predict(Camera &cam, const double xv[13], const double yi[3], const Mat &Pxx,
                      const Mat &Pxy, const Mat &Pyy, FeaturePrediction &out) {
    double zeroed[3];
    Mat dz_by_dxp, dz_by_dyi;
    zeroedyi(yi, xv, zeroed, dz_by_dxp, dz_by_dyi);  // xp = xv[0..6] (motion_model.cpp:219-222)
    cam.project(zeroed, out.h);
    const Mat dhid = cam.projection_jacobian();
    out.dh_by_dxp = mul(dhid, dz_by_dxp);
    out.dh_by_dy = mul(dhid, dz_by_dyi);
    Mat dxp_by_dxv(7, 13);  // motion_model.cpp:224-235
    for (int i = 0; i < 7; ++i) dxp_by_dxv(i, i) = 1.0;
    out.dh_by_dxv = mul(out.dh_by_dxp, dxp_by_dxv);
    const double var = cam.measurement_noise_variance(out.h);
    out.R = Mat(2, 2);
    out.R(0, 0) = 1.0 * var;
    out.R(1, 1) = 1.0 * var;
    // func_Si, feature_model.cpp:99-116
    Mat S(2, 2);
    add_inplace(S, mul_nt(mul(out.dh_by_dxv, Pxx), out.dh_by_dxv));
    const Mat T1 = mul_nt(mul(out.dh_by_dxv, Pxy), out.dh_by_dy);
    add_inplace(S, T1);
    add_inplace(S, transpose(T1));
    add_inplace(S, mul_nt(mul(out.dh_by_dy, Pyy), out.dh_by_dy));
    add_inplace(S, out.R);
    out.S = S;
  }

  // full_feature_model.cpp:103-170 ; 0 = visible
  static int visibility_test(const Camera &cam, const double xp[7], const double yi[3],
                             const double xp_orig[7], const double hi[2]) {
    int cant_see = 0;
    if (hi[0] < 0.0 + kImageSearchBoundary ||
        hi[0] > (double)(cam.width - 1 - kImageSearchBoundary))
      cant_see |= 1;  // kLeftRightFail_
    if (hi[1] < 0.0 + kImageSearchBoundary ||
        hi[1] > (double)(cam.height - 1 - kImageSearchBoundary))
      cant_see |= 2;  // kUpDownFail_
    double z[3];
    Mat t1, t2;
    zeroedyi(yi, xp, z, t1, t2);
    if (z[2] <= 0) cant_see |= 16;  // kBehindCameraFail_ (full_feature_model.h:74-78)
    double RWR[3][3];
    quat_to_R(Quat{xp[3], xp[4], xp[5], xp[6]}, RWR);
    double hLWi[3], hLWi_orig[3];
    for (int i = 0; i < 3; ++i) {
      double s = 0.0;
      for (int k = 0; k < 3; ++k) s += RWR[i][k] * z[k];
      hLWi[i] = s;
    }
    zeroedyi(yi, xp_orig, z, t1, t2);
    quat_to_R(Quat{xp_orig[3], xp_orig[4], xp_orig[5], xp_orig[6]}, RWR);
    for (int i = 0; i < 3; ++i) {
      double s = 0.0;
      for (int k = 0; k < 3; ++k) s += RWR[i][k] * z[k];
      hLWi_orig[i] = s;
    }
    const double mod = std::sqrt(hLWi[0] * hLWi[0] + hLWi[1] * hLWi[1] + hLWi[2] * hLWi[2]);
    const double mod_orig = std::sqrt(hLWi_orig[0] * hLWi_orig[0] + hLWi_orig[1] * hLWi_orig[1] +
                                      hLWi_orig[2] * hLWi_orig[2]);
    const double length_ratio = mod / mod_orig;
    if (length_ratio > kMaximumLengthRatio || length_ratio < (1.0 / kMaximumLengthRatio))
      cant_see |= 4;  // kDistanceFail_
    const double dot = hLWi[0] * hLWi_orig[0] + hLWi[1] * hLWi_orig[1] + hLWi[2] * hLWi_orig[2];
    double angle = std::acos(dot / (mod * mod_orig));
    angle = (angle >= 0.0 ? angle : -angle);
    if (angle > maximum_angle_difference()) cant_see |= 8;  // kAngleFail_
    return cant_see;
  }
};

// ---------------------------------------------------------------------------------------
// Partially-initialised feature (a ray r + lambda * hhat) measured through one depth particle
// (part_feature_model.cpp:80-143, 231-265; monoslam.cpp:1375-1392; feature_init_info.cpp:57-65)
// ---------------------------------------------------------------------------------------
struct ParticlePrediction {
  double h[2];
  Mat dh_by_dxp;  // 2x7
  Mat dh_by_dy;   // 2x6
  Mat S;          // 2x2
  double var;     // R = var * I
  double Sinv[4]; // Particle::m_SInv_ (column-major 2x2)
  double detS;
};

struct PartFeatureModel {
  // part_feature_model.cpp:80-143: yi = (ri, hhati) -> zeroedyi = (RRW (ri - r), RRW hhati) and its Jacobians
  static void zeroedyi(const double yi[6], const double xp[7], double zeroed[6], Mat &dz_by_dxp,
                       Mat &dz_by_dyi) {
    const double d[3] = {yi[0] - xp[0], yi[1] - xp[1], yi[2] - xp[2]};
    const double hh[3] = {yi[3], yi[4], yi[5]};
    const Quat q = {xp[3], xp[4], xp[5], xp[6]};
    const Quat qRW = quat_inverse(q);
    double RRW[3][3];
    quat_to_R(qRW, RRW);
    for (int i = 0; i < 3; ++i) {
      double s = 0.0, t = 0.0;
      for (int k = 0; k < 3; ++k) {
        s += RRW[i][k] * d[k];
        t += RRW[i][k] * hh[k];
      }
      zeroed[i] = s;
      zeroed[3 + i] = t;
    }
    Mat R(3, 3), Rneg(3, 3);
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        R(i, j) = RRW[i][j];
        Rneg(i, j) = RRW[i][j] * -1.0;
      }
    Mat dqbar(4, 4);  // feature_model.cpp:152-162
    dqbar(0, 0) = 1.0;
    dqbar(1, 1) = -1.0;
    dqbar(2, 2) = -1.0;
    dqbar(3, 3) = -1.0;
    dz_by_dxp = Mat(6, 7);
    set_block(dz_by_dxp, 0, 0, Rneg);
    set_block(dz_by_dxp, 0, 3, mul(FullFeatureModel::dRq_times_a_by_dq(qRW, d), dqbar));
    set_block(dz_by_dxp, 3, 3, mul(FullFeatureModel::dRq_times_a_by_dq(qRW, hh), dqbar));
    dz_by_dyi = Mat(6, 6);
    set_block(dz_by_dyi, 0, 0, R);
    set_block(dz_by_dyi, 3, 3, R);
  }

  // One particle of MonoSLAM::predict_partially_initialised_feature_measurements (monoslam.cpp:1375-1392):
  // func_hpi_and_dhpi_by_dxp_and_dhpi_by_dyi (part_feature_model.cpp:231-265), func_Ri, func_Si
  // (feature_model.cpp:99-116) with the 13x6 / 6x6 covariance blocks of the 6-dimensional feature state,
  // Particle::set_S (feature_init_info.cpp:57-65; the L^-1 of the 2x2 factor in closed form like puinv_from_S).
  static void predict_particle(Camera &cam, const double xv[13], const double ypi[6], double lambda,
                               const Mat &Pxx, const Mat &Pxy, const Mat &Pyy, ParticlePrediction &out) {
    double z[6];
    Mat dz_by_dxp, dz_by_dyi;
    zeroedyi(ypi, xv, z, dz_by_dxp, dz_by_dyi);  // xp = xv[0..6]
    const double hLR[3] = {z[0] + lambda * z[3], z[1] + lambda * z[4], z[2] + lambda * z[5]};
    cam.project(hLR, out.h);
    const Mat J = cam.projection_jacobian();
    Mat D(3, 6);  // dhLRi_by_dzeroedyi
    for (int i = 0; i < 3; ++i) {
      D(i, i) = 1.0;
      D(i, 3 + i) = lambda;
    }
    const Mat M1 = mul(J, D);
    out.dh_by_dxp = mul(M1, dz_by_dxp);
    out.dh_by_dy = mul(M1, dz_by_dyi);
    Mat dxp_by_dxv(7, 13);  // motion_model.cpp:224-235
    for (int i = 0; i < 7; ++i) dxp_by_dxv(i, i) = 1.0;
    const Mat dh_by_dxv = mul(out.dh_by_dxp, dxp_by_dxv);
    out.var = cam.measurement_noise_variance(out.h);
    Mat R(2, 2);
    R(0, 0) = 1.0 * out.var;
    R(1, 1) = 1.0 * out.var;
    Mat S(2, 2);
    add_inplace(S, mul_nt(mul(dh_by_dxv, Pxx), dh_by_dxv));
    const Mat T1 = mul_nt(mul(dh_by_dxv, Pxy), out.dh_by_dy);
    add_inplace(S, T1);
    add_inplace(S, transpose(T1));
    add_inplace(S, mul_nt(mul(out.dh_by_dy, Pyy), out.dh_by_dy));
    add_inplace(S, R);
    out.S = S;
    const double s00 = S(0, 0), s10 = S(1, 0), s11 = S(1, 1);
    const double l00 = std::sqrt(s00);
    const double l10 = s10 / l00;
    const double l11 = std::sqrt(s11 - l10 * l10);
    const double x00 = 1.0 / l00;
    const double x10 = (0.0 - l10 * x00) / l11;
    const double x11 = 1.0 / l11;
    out.Sinv[0] = x00 * x00 + x10 * x10;
    out.Sinv[1] = x10 * x11;
    out.Sinv[2] = x10 * x11;
    out.Sinv[3] = x11 * x11;
    out.detS = S(0, 0) * S(1, 1) - S(0, 1) * S(1, 0);
  }
};

}  // namespace sl2o
