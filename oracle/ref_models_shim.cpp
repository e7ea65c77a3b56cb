// ORACLE — TEST INFRASTRUCTURE ONLY.  C entry points into the REFERENCE'S OWN model classes
// (MotionModel, Camera, FullFeatureModel), compiled unmodified from the original scenelib2/ against the
// arithmetic stand-in of oracle/stubs_arith (see its header for what is and is not pinned).  Signatures
// mirror the oracle's orc_* functions so tests can compare the two directly.
#include <cstring>

#include "camera.h"
#include "feature_init_info.h"
#include "full_feature_model.h"
#include "motion_model.h"
#include "part_feature_model.h"

using namespace SceneLib2;

namespace {
Eigen::VectorXd vec(const double *p, int n) {
  Eigen::VectorXd v(n);
  for (int i = 0; i < n; ++i) v(i) = p[i];
  return v;
}
Eigen::MatrixXd mat(const double *p, int r, int c) {  // column-major in, column-major stored
  Eigen::MatrixXd m(r, c);
  std::memcpy(m.data(), p, sizeof(double) * r * c);
  return m;
}
void out(const Eigen::MatrixXd &m, double *p) { std::memcpy(p, m.data(), sizeof(double) * m.size()); }
void set_camera(Camera &cam, const double *c8) {
  cam.SetCameraParameters((int)c8[0], (int)c8[1], c8[2], c8[3], c8[4], c8[5], c8[6], (int)c8[7]);
}
}  // namespace

extern "C" {

// motion_model.cpp:84-217
void ref_motion(const double *xv, const double *u, double delta_t, double *fv, double *F, double *Q) {
  MotionModel mm;
  const Eigen::VectorXd x = vec(xv, 13), uu = vec(u, 3);
  mm.func_fv_and_dfv_by_dxv(x, uu, delta_t);
  mm.func_Q(x, uu, delta_t);
  out(mm.fvRES_, fv);
  out(mm.dfv_by_dxvRES_, F);
  out(mm.QxRES_, Q);
}

// motion_model.cpp:237-263
void ref_dxvnorm_by_dxv(const double *xv, double *J, double *xvnorm) {
  MotionModel mm;
  mm.func_xvnorm_and_dxvnorm_by_dxv(vec(xv, 13));
  out(mm.dxvnorm_by_dxvRES_, J);
  out(mm.xvnormRES_, xvnorm);
}

// the body of MonoSLAM::predict_single_feature_measurements (monoslam.cpp:289-308) on the reference's
// own model objects: h_i, dh_i/dx_v, dh_i/dy_i, R_i, S_i
void ref_predict_feature(const double *cam8, const double *xv, const double *y, const double *Pxx,
                         const double *Pxy, const double *Pyy, double *h, double *dh_by_dxv,
                         double *dh_by_dy, double *R, double *S) {
  Camera cam;
  set_camera(cam, cam8);
  MotionModel mm;
  FullFeatureModel fm(2, 3, 3, &cam, &mm);
  const Eigen::VectorXd x = vec(xv, 13);
  mm.func_xp(x);
  const Eigen::VectorXd xp = mm.xpRES_;
  fm.func_hi_and_dhi_by_dxp_and_dhi_by_dyi(vec(y, 3), xp);
  mm.func_dxp_by_dxv(x);
  const Eigen::MatrixXd dh_dxv = fm.dhi_by_dxpRES_ * mm.dxp_by_dxvRES_;
  fm.func_Ri(fm.hiRES_);
  fm.func_Si(mat(Pxx, 13, 13), mat(Pxy, 13, 3), mat(Pyy, 3, 3), dh_dxv, fm.dhi_by_dyiRES_, fm.RiRES_);
  out(fm.hiRES_, h);
  out(dh_dxv, dh_by_dxv);
  out(fm.dhi_by_dyiRES_, dh_by_dy);
  out(fm.RiRES_, R);
  out(fm.SiRES_, S);
}

// full_feature_model.cpp:103-170
int ref_visibility_test(const double *cam8, const double *xp, const double *y, const double *xp_org,
                        const double *h) {
  Camera cam;
  set_camera(cam, cam8);
  MotionModel mm;
  FullFeatureModel fm(2, 3, 3, &cam, &mm);
  return fm.visibility_test(vec(xp, 7), vec(y, 3), vec(xp_org, 7), vec(h, 2));
}

// camera.cpp:90-170
void ref_project(const double *cam8, const double *c3, double *h2, double *J23) {
  Camera cam;
  set_camera(cam, cam8);
  const Eigen::Vector2d hh = cam.Project(Eigen::Vector3d(c3[0], c3[1], c3[2]));
  out(hh, h2);
  out(cam.ProjectionJacobian(), J23);
}
void ref_unproject(const double *cam8, const double *h2, double *c3, double *J32) {
  Camera cam;
  set_camera(cam, cam8);
  const Eigen::Vector3d cc = cam.Unproject(Eigen::Vector2d(h2[0], h2[1]));
  out(cc, c3);
  out(cam.UnprojectionJacobian(), J32);
}

// Particle::set_S (feature_init_info.cpp:55-63): S (2x2, column-major) -> SInv (2x2), det S.  The same
// LLT -> matrixL -> inverse -> L^-T L^-1 sequence as MonoSLAM::measure_feature (monoslam.cpp:371-374).
void ref_particle_set_S(const double *S4, double *Sinv4, double *detS) {
  Eigen::VectorXd l(1);
  Particle p(l, 1.0, 2);
  p.set_S(mat(S4, 2, 2));
  out(p.m_SInv_, Sinv4);
  *detS = p.m_detS_;
}

// one particle of MonoSLAM::predict_partially_initialised_feature_measurements (monoslam.cpp:1375-1392) on the
// reference's own PartFeatureModel / Particle objects: h_pi, S_i, S_i^-1, det S_i
void ref_predict_particle(const double *cam8, const double *xv, const double *ypi, double lambda,
                          const double *Pxx, const double *Pxy, const double *Pyy, double *h, double *S4,
                          double *Sinv4, double *detS) {
  Camera cam;
  set_camera(cam, cam8);
  MotionModel mm;
  PartFeatureModel pm(2, 6, 6, &cam, &mm, 3);
  const Eigen::VectorXd x = vec(xv, 13);
  mm.func_xp(x);
  const Eigen::VectorXd local_xp = mm.xpRES_;
  mm.func_dxp_by_dxv(x);
  const Eigen::MatrixXd local_dxp_by_dxv = mm.dxp_by_dxvRES_;
  Eigen::VectorXd lam(1);
  lam(0) = lambda;
  pm.func_hpi_and_dhpi_by_dxp_and_dhpi_by_dyi(vec(ypi, 6), local_xp, lam);
  const Eigen::VectorXd m_h = pm.hpiRES_;
  pm.func_Ri(m_h);
  pm.func_Si(mat(Pxx, 13, 13), mat(Pxy, 13, 6), mat(Pyy, 6, 6), pm.dhpi_by_dxpRES_ * local_dxp_by_dxv,
             pm.dhpi_by_dyiRES_, pm.RiRES_);
  Particle p(lam, 1.0, 2);
  p.set_S(pm.SiRES_);
  out(m_h, h);
  out(pm.SiRES_, S4);
  out(p.m_SInv_, Sinv4);
  *detS = p.m_detS_;
}

}  // extern "C"
