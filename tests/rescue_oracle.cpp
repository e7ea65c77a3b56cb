// TEST INFRASTRUCTURE ONLY.  The consensus rescue (include/sl2b200.h, sl2_set_stream_rescue) on top of the CPU oracle
// (oracle/slam.hpp, used as it is) and of the consensus oracle (tests/consensus_oracle.cpp, included as it is): the
// rescue gate as a pure function in the operation order of csrc/rescue.cu rescue_kernel, and a whole step that runs
//   predict, select, measure, consensus, update 1 (inliers), re-predict, gate, update 2 (rescued), cull.
// Compiled by tests/rescue_oracle.py with the oracle's flags (-O3 -ffp-contract=off).
#include "consensus_oracle.cpp"

namespace {

// One rejected match seen from the updated state: depth zc[2], the prediction p and q = nu'^T S'^-1 nu'.
// Returns whether the match is rescued (in front of the camera and q <= chi2; a NaN q never is).
bool rescue_gate(Camera &cam, const double *xv, const double *y, const Mat &Pxx, const Mat &Pxy, const Mat &Pyy,
                 const double z[2], double chi2, FeaturePrediction &p, double *q_out) {
  FullFeatureModel::predict(cam, xv, y, Pxx, Pxy, Pyy, p);
  double zc[3];
  Mat a, b;
  FullFeatureModel::zeroedyi(y, xv, zc, a, b);
  const double nu0 = z[0] - p.h[0], nu1 = z[1] - p.h[1];
  double si[4];
  puinv_from_S(p.S.a.data(), si);  // (00, 10, 01, 11): the sinv_from_S sequence
  const double w0 = si[0] * nu0 + si[2] * nu1, w1 = si[2] * nu0 + si[3] * nu1;
  const double q = nu0 * w0 + nu1 * w1;
  *q_out = q;
  return zc[2] > 0.0 && q <= chi2;
}

}  // namespace

// The consensus oracle's Slam with the rescue stage after update 1.  `rescued` holds the labels rescued in the last
// step, returned only by resc_slam_rescued; the flags read-back shows a rescued match as a plain success, like the
// device.
struct resc_slam : cons_slam {
  double chi2 = 0.0;
  std::set<int> rescued;
  explicit resc_slam(const SlamConfig &c) : cons_slam(c) {}

  void rescue() {
    rescued.clear();
    if (!(chi2 > 0.0)) return;
    std::vector<Feature *> in1, res;
    std::vector<FeaturePrediction> preds;
    for (Feature *f : s.selected_feature_list) {
      if (f->successful_measurement_flag) {
        in1.push_back(f);
      } else if (rejected.count(f->label)) {
        FeaturePrediction p;
        double q;
        if (rescue_gate(s.cam, s.xv, f->y, s.Pxx, f->Pxy, f->Pyy, f->z, chi2, p, &q)) {
          res.push_back(f);
          preds.push_back(p);
        }
      }
    }
    if (res.empty()) return;
    for (Feature *f : in1) f->successful_measurement_flag = false;
    for (size_t r = 0; r < res.size(); ++r) {
      Feature *f = res[r];
      const FeaturePrediction &p = preds[r];
      f->h[0] = p.h[0];
      f->h[1] = p.h[1];
      f->dh_by_dy = p.dh_by_dy;
      f->dh_by_dxv = p.dh_by_dxv;
      f->R = p.R;
      f->S = p.S;
      f->nu[0] = f->z[0] - f->h[0];
      f->nu[1] = f->z[1] - f->h[1];
      f->successful_measurement_flag = true;
    }
    s.successful_measurement_vector_size = 2 * (int)res.size();
    s.kalman_update();
    s.normalise_state();
    for (Feature *f : in1) f->successful_measurement_flag = true;
    for (Feature *f : res) {
      ++f->successful_measurements_of_feature;
      rejected.erase(f->label);
      rescued.insert(f->label);
    }
    s.successful_measurement_vector_size += 2 * (int)in1.size();
  }

  void step(const uint8_t *frame) {
    const double u[3] = {0.0, 0.0, 0.0};
    s.kalman_predict(u);
    s.number_of_visible_features = s.auto_select_n_features(s.cfg.number_of_features_to_select);
    rescued.clear();
    if (!s.selected_feature_list.empty()) {
      s.make_measurements(frame);
      for (const Feature *f : s.selected_feature_list) rejected.erase(f->label);
      apply_consensus();
      if (s.successful_measurement_vector_size != 0) {
        s.kalman_update();
        s.normalise_state();
        rescue();
      }
    }
    s.delete_bad_features();
    Mat P = s.dense_P();
    const Mat PT = transpose(P);
    for (size_t i = 0; i < P.a.size(); ++i) P.a[i] = P.a[i] * 0.5 + PT.a[i] * 0.5;
    s.fill_covariances(P);
  }
};

extern "C" {

// k rejected matches of one state: x (n), P (n x n column-major); pos[j] = index of y_j in x; z (k x 2).
// rescued[j] = the gate's decision, q[j] = nu'^T S'^-1 nu'; h (k x 2) and S (k x 4 column-major) = the re-prediction.
void resc_gate(const double *cam8, const double *x, const double *P, int32_t n, int32_t k, const int32_t *pos,
               const double *z, double chi2, uint8_t *rescued, double *q, double *h, double *S) {
  Camera cam;
  cam.width = (int)cam8[0];
  cam.height = (int)cam8[1];
  cam.fku = cam8[2];
  cam.fkv = cam8[3];
  cam.u0 = cam8[4];
  cam.v0 = cam8[5];
  cam.kd1 = cam8[6];
  cam.sd = cam8[7];
  auto Pat = [&](int r, int c) { return P[r + (size_t)n * c]; };
  Mat Pxx(13, 13);
  for (int r = 0; r < 13; ++r)
    for (int c = 0; c < 13; ++c) Pxx(r, c) = Pat(r, c);
  for (int j = 0; j < k; ++j) {
    Mat Pxy(13, 3), Pyy(3, 3);
    for (int r = 0; r < 13; ++r)
      for (int c = 0; c < 3; ++c) Pxy(r, c) = Pat(r, pos[j] + c);
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) Pyy(r, c) = Pat(pos[j] + r, pos[j] + c);
    FeaturePrediction p;
    rescued[j] = rescue_gate(cam, x, x + pos[j], Pxx, Pxy, Pyy, z + 2 * j, chi2, p, q + j) ? 1 : 0;
    h[2 * j] = p.h[0];
    h[2 * j + 1] = p.h[1];
    for (int e = 0; e < 4; ++e) S[4 * j + e] = p.S.a[e];
  }
}

resc_slam *resc_slam_create(const orc_config *c) {
  cons_slam *b = cons_slam_create(c);
  resc_slam *r = new resc_slam(b->s.cfg);
  delete b;
  return r;
}
void resc_slam_destroy(resc_slam *s) { delete s; }
void resc_slam_set(resc_slam *s, double tau, double chi2) {
  s->tau = tau;
  s->chi2 = chi2;
}
cons_slam *resc_slam_base(resc_slam *s) { return s; }
void resc_slam_step(resc_slam *s, const uint8_t *frame) { s->step(frame); }
// labels of the features rescued in the last step; returns their count
int32_t resc_slam_rescued(const resc_slam *s, int32_t *labels) {
  int32_t n = 0;
  for (int l : s->rescued) labels[n++] = l;
  return n;
}

}  // extern "C"
