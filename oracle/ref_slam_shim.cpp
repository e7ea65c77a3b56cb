// ORACLE — TEST INFRASTRUCTURE ONLY.  C entry points into the REFERENCE'S OWN MonoSLAM tracking step:
// monoslam.cpp, kalman.cpp, feature.cpp, part_feature_model.cpp, the model files, support/*.cpp and improc/*.cpp
// are compiled UNMODIFIED where they lie in a SceneLib2 checkout against the stand-ins of oracle/stubs_arith
// (matrix class with plain-loop arithmetic instead of Eigen, pixel container instead of OpenCV, "key = value;"
// parser instead of Pangolin; GUI and frame grabber reduced to the empty definitions below).
// So GoOneStep, KalmanFilterPredict/Update, auto_select_n_features, make_measurements, measure_feature,
// elliptical_search, construct_total_*, fill_*, normalise_state, delete_bad_features ... executed by the
// functions below ARE the reference's code; only Eigen's internal summation order is not reproduced.
// Signatures mirror the oracle's orc_slam_* API (oracle/sl2_oracle.h).
#include <cstdint>
#include <cstring>
#include <string>

#include "kalman.h"
#include "monoslam.h"

namespace SceneLib2 {
// the two collaborators MonoSLAM::Init creates that are out of scope here (monoslam.cpp:1961-1963)
GraphicTool::GraphicTool(MonoSLAM *)
    : kQR0_(0.0, 0.0, 1.0, 0.0), kMoveClippingPlaneFactor_(0.0), kSemiInfiniteLineLength_(0.0),
      kCovariancesNumberOfSigma_(0.0), kDrawNOverlappingEllipses_(0) {}
GraphicTool::~GraphicTool() {}
FrameGrabber::FrameGrabber() : file_grabber_(nullptr), usb_cam_grabber_(nullptr) {}
FrameGrabber::~FrameGrabber() {}
void FrameGrabber::Init(const std::string &, const bool) {}
}  // namespace SceneLib2

using namespace SceneLib2;

extern "C" {

// MonoSLAM::Init (monoslam.cpp:1576-1969): camera, models, initial state and the four known features of the cfg
void *ref_slam_create(const char *cfg_path) {
  MonoSLAM *m = new MonoSLAM();
  m->Init(cfg_path);
  return m;
}
void ref_slam_destroy(void *p) { delete static_cast<MonoSLAM *>(p); }

// MonoSLAM::AddNewKnownFeature (monoslam.cpp:1278-1289); the template is read by cv::imread (feature.cpp:119)
void ref_slam_add_feature(void *p, const double *y, const double *xp_org, const char *patch_path) {
  MonoSLAM *m = static_cast<MonoSLAM *>(p);
  Eigen::VectorXd yy(3), xp(7);
  for (int i = 0; i < 3; ++i) yy(i) = y[i];
  for (int i = 0; i < 7; ++i) xp(i) = xp_org[i];
  m->AddNewKnownFeature(yy, xp, patch_path);
}
void ref_slam_set_params(void *p, int n_select, int min_attempts, double match_fraction) {
  MonoSLAM *m = static_cast<MonoSLAM *>(p);
  if (n_select >= 0) m->kNumberOfFeaturesToSelect_ = n_select;
  if (min_attempts >= 0) m->minimum_attempted_measurements_of_feature_ = min_attempts;
  if (match_fraction >= 0.0) m->successful_match_fraction_ = match_fraction;
}
int32_t ref_slam_num_features(void *p) { return (int32_t) static_cast<MonoSLAM *>(p)->feature_list_.size(); }
int32_t ref_slam_state_size(void *p) { return static_cast<MonoSLAM *>(p)->total_state_size_; }

// fill_states / fill_covariances (monoslam.cpp:574-614); P column-major n x n
void ref_slam_set_state(void *p, const double *x, const double *P) {
  MonoSLAM *m = static_cast<MonoSLAM *>(p);
  const int n = m->total_state_size_;
  Eigen::VectorXd V(n);
  Eigen::MatrixXd M(n, n);
  std::memcpy(V.data(), x, sizeof(double) * n);
  std::memcpy(M.data(), P, sizeof(double) * n * n);
  m->fill_states(V);
  m->fill_covariances(M);
}
// construct_total_state / construct_total_covariance (monoslam.cpp:501-546)
void ref_slam_get_state(void *p, double *x, double *P) {
  MonoSLAM *m = static_cast<MonoSLAM *>(p);
  const int n = m->total_state_size_;
  Eigen::VectorXd V(n);
  Eigen::MatrixXd M(n, n);
  V.setZero();
  M.setZero();
  m->construct_total_state(V);
  m->construct_total_covariance(M);
  std::memcpy(x, V.data(), sizeof(double) * n);
  std::memcpy(P, M.data(), sizeof(double) * n * n);
}
// MonoSLAM::GoOneStep (monoslam.cpp:108-180), tracking only
void ref_slam_step(void *p, const uint8_t *frame, int32_t width, int32_t height) {
  MonoSLAM *m = static_cast<MonoSLAM *>(p);
  cv::Mat f(height, width, CV_8UC1, const_cast<uint8_t *>(frame));
  m->GoOneStep(f, false, false);
}
void ref_slam_get_features(void *p, int32_t *label, double *h, double *z, double *S, uint8_t *flags,
                           int32_t *attempted, int32_t *successful, int32_t *select_rank) {
  MonoSLAM *m = static_cast<MonoSLAM *>(p);
  int i = 0;
  for (Feature *f : m->feature_list_) {
    label[i] = f->label_;
    for (int k = 0; k < 2; ++k) {
      h[2 * i + k] = f->h_.size() == 2 ? f->h_(k) : 0.0;
      z[2 * i + k] = f->z_.size() == 2 ? f->z_(k) : 0.0;
    }
    for (int k = 0; k < 4; ++k) S[4 * i + k] = f->S_.size() == 4 ? f->S_.data()[k] : 0.0;
    // Feature::Initialise (feature.cpp:150-160) leaves successful_measurement_flag_ uninitialised; it only has
    // a defined value once the feature has been measured at least once
    const bool succ = f->attempted_measurements_of_feature_ > 0 && f->successful_measurement_flag_;
    flags[i] = (f->selected_flag_ ? 1 : 0) | (succ ? 2 : 0);
    attempted[i] = f->attempted_measurements_of_feature_;
    successful[i] = f->successful_measurements_of_feature_;
    select_rank[i] = -1;
    int r = 0;
    for (Feature *s : m->selected_feature_list_) {
      if (s == f) select_rank[i] = r;
      ++r;
    }
    ++i;
  }
}

// MonoSLAM::InitialiseFeature (monoslam.cpp:1211-1236): a partially-initialised feature with
// kNumberOfParticles_ depth particles at pixel (u, v) of `frame`
void ref_slam_init_partial(void *p, const uint8_t *frame, int32_t width, int32_t height, int32_t u, int32_t v) {
  MonoSLAM *m = static_cast<MonoSLAM *>(p);
  cv::Mat f(height, width, CV_8UC1, const_cast<uint8_t *>(frame));
  m->uu_ = u;
  m->vv_ = v;
  m->location_selected_flag_ = true;
  m->InitialiseFeature(f);
}

// One particle cycle of the FIRST partially-initialised feature, split exactly like
// MonoSLAM::MatchPartiallyInitialisedFeatures (monoslam.cpp:1299-1340) so that the inputs and outputs of the
// measurement / re-weighting step can be read: predict_partially_initialised_feature_measurements ->
// [h, SInv, detS, lambda, probability] -> measure_feature_with_multiple_priors -> [z, flags] ->
// update_partially_initialised_feature_probabilities -> [probability, cumulative, survivors, mean, covariance].
// Returns the number of particles before the cycle, -1 when the feature makes no measurement on this step
// (the first step after initialisation, monoslam.cpp:1367-1369), -2 when there is no such feature.
int32_t ref_slam_particle_cycle(void *p, const uint8_t *frame, int32_t width, int32_t height, int32_t cap,
                                double *h, double *sinv3, double *detS, double *lambda, double *prob_before,
                                int32_t *z_uv, uint8_t *found, double *prob_after, uint8_t *keep,
                                double *cumulative, double *mean_var, int32_t *k_after) {
  MonoSLAM *m = static_cast<MonoSLAM *>(p);
  if (m->feature_init_info_vector_.empty()) return -2;
  cv::Mat f(height, width, CV_8UC1, const_cast<uint8_t *>(frame));
  m->predict_partially_initialised_feature_measurements();
  FeatureInitInfo *feat = &m->feature_init_info_vector_.front();
  if (!feat->making_measurement_on_this_step_flag_) return -1;
  const int K = (int)feat->particle_vector_.size();
  if (K > cap) return -3;
  for (int k = 0; k < K; ++k) {
    const Particle &q = feat->particle_vector_[k];
    h[2 * k] = q.m_h_(0);
    h[2 * k + 1] = q.m_h_(1);
    sinv3[3 * k] = q.m_SInv_(0, 0);
    sinv3[3 * k + 1] = q.m_SInv_(0, 1);
    sinv3[3 * k + 2] = q.m_SInv_(1, 1);
    detS[k] = q.m_detS_;
    lambda[k] = q.lambda_(0);
    prob_before[k] = q.probability_;
  }
  m->measure_feature_with_multiple_priors(f, feat->fp_->patch_, feat->particle_vector_);
  for (int k = 0; k < K; ++k) {
    const Particle &q = feat->particle_vector_[k];
    found[k] = q.m_successful_measurement_flag_ ? 1 : 0;
    z_uv[2 * k] = found[k] ? (int)q.m_z_(0) : 0;
    z_uv[2 * k + 1] = found[k] ? (int)q.m_z_(1) : 0;
    keep[k] = 0;
    prob_after[k] = 0.0;
    cumulative[k] = 0.0;
  }
  m->update_partially_initialised_feature_probabilities(m->kPruneProbabilityThreshold_);
  mean_var[0] = mean_var[1] = 0.0;
  *k_after = 0;
  if (m->feature_init_info_vector_.empty()) return K;  // every match failed: the feature was deleted
  feat = &m->feature_init_info_vector_.front();
  size_t j = 0;
  for (int k = 0; k < K && j < feat->particle_vector_.size(); ++k)
    if (feat->particle_vector_[j].lambda_(0) == lambda[k]) {
      keep[k] = 1;
      prob_after[k] = feat->particle_vector_[j].probability_;
      cumulative[k] = feat->particle_vector_[j].cumulative_probability_;
      ++j;
    }
  mean_var[0] = feat->mean_(0);
  mean_var[1] = feat->covariance_(0, 0);
  *k_after = (int)feat->particle_vector_.size();
  return K;
}

// MonoSLAM::elliptical_search (monoslam.cpp:401-477) on its own: PuInv3 = (P00, P01, P11); returns the bool
int32_t ref_elliptical_search(const uint8_t *image, int32_t width, int32_t height, const uint8_t *patch,
                              int32_t boxsize, const double *centre, const double *PuInv3, int32_t *u,
                              int32_t *v) {
  MonoSLAM m;  // no Init needed: the search only uses the constructor's constants
  cv::Mat img(height, width, CV_8UC1, const_cast<uint8_t *>(image));
  cv::Mat pat(boxsize, boxsize, CV_8UC1, const_cast<uint8_t *>(patch));
  Eigen::Vector2d c(centre[0], centre[1]);
  Eigen::Matrix2d P;
  P(0, 0) = PuInv3[0];
  P(0, 1) = P(1, 0) = PuInv3[1];
  P(1, 1) = PuInv3[2];
  int uu = *u, vv = *v;
  const bool ok = m.elliptical_search(img, pat, c, P, &uu, &vv, boxsize);
  *u = uu;
  *v = vv;
  return ok ? 1 : 0;
}

// MonoSLAM::measure_feature (monoslam.cpp:368-386): S (2x2 column-major) -> LLT -> PuInv -> elliptical_search
int32_t ref_measure_feature(const uint8_t *image, int32_t width, int32_t height, const uint8_t *patch,
                            const double *h, const double *S4, double *z) {
  MonoSLAM m;
  cv::Mat img(height, width, CV_8UC1, const_cast<uint8_t *>(image));
  cv::Mat pat(11, 11, CV_8UC1, const_cast<uint8_t *>(patch));  // kBoxSize_ (monoslam.cpp:48)
  Eigen::VectorXd zz(2), hh(2);
  hh(0) = h[0];
  hh(1) = h[1];
  zz(0) = z[0];
  zz(1) = z[1];
  Eigen::MatrixXd S(2, 2);
  std::memcpy(S.data(), S4, sizeof(double) * 4);
  const bool ok = m.measure_feature(img, pat, zz, hh, S);
  z[0] = zz(0);
  z[1] = zz(1);
  return ok ? 1 : 0;
}

// MonoSLAM::find_best_patch_inside_region (monoslam.cpp:1070-1205), region4 = (ustart, vstart, ufinish, vfinish)
void ref_find_best_patch(const uint8_t *image, int32_t width, int32_t height, int32_t boxsize,
                         const int32_t *region4, int32_t *ubest, int32_t *vbest, double *evbest) {
  MonoSLAM m;
  cv::Mat img(height, width, CV_8UC1, const_cast<uint8_t *>(image));
  int u = *ubest, v = *vbest;
  m.find_best_patch_inside_region(img, &u, &v, evbest, boxsize, region4[0], region4[1], region4[2], region4[3]);
  *ubest = u;
  *vbest = v;
}

}  // extern "C"
