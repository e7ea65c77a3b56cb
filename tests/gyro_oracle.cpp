// TEST INFRASTRUCTURE ONLY.  The gyroscope update (include/sl2b200.h, sl2_set_stream_gyro) on top of the CPU oracle
// (oracle/slam.hpp, used as it is) and of the consensus oracle (tests/consensus_oracle.cpp, included as it is, with
// its consensus off): a whole step that runs
//   predict, gyro update (when a sample is pending), select, measure, update, cull,
// the gyro update in the header's operation order on the oracle's dense P.  Compiled by tests/gyro_oracle.py with the
// oracle's flags (-O3 -ffp-contract=off).
#include <cmath>

#include "consensus_oracle.cpp"

struct gyro_slam : cons_slam {
  double R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, b[3] = {0, 0, 0}, Rc[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  double z[3] = {0, 0, 0};
  bool pending = false;
  int status = 0;
  double nis = 0.0;
  explicit gyro_slam(const SlamConfig &c) : cons_slam(c) {}

  void set(const double *R9, const double *b3, const double *C) {
    for (int i = 0; i < 9; ++i) R[i] = R9[i];
    for (int i = 0; i < 3; ++i) b[i] = b3[i];
    double M[9];  // Rc = R^T C R: M = C R, the upper triangle of R^T M, mirrored
    for (int k = 0; k < 3; ++k)
      for (int j = 0; j < 3; ++j) M[3 * k + j] = (C[3 * k] * R[j] + C[3 * k + 1] * R[3 + j]) + C[3 * k + 2] * R[6 + j];
    for (int i = 0; i < 3; ++i)
      for (int j = i; j < 3; ++j) Rc[3 * i + j] = Rc[3 * j + i] = (R[i] * M[j] + R[3 + i] * M[3 + j]) + R[6 + i] * M[6 + j];
  }

  void gyro_update() {
    status = 0;
    nis = 0.0;
    if (!pending) return;
    pending = false;
    const int n = s.total_state_size;
    Vec x((size_t)n, 0.0);
    s.construct_total_state(x);
    Mat P = s.dense_P();
    double d[3], zc[3];
    for (int i = 0; i < 3; ++i) d[i] = z[i] - b[i];
    for (int i = 0; i < 3; ++i) zc[i] = (R[i] * d[0] + R[3 + i] * d[1]) + R[6 + i] * d[2];
    auto Pw = [&](int i, int j) { return P(10 + i, 10 + j); };
    const double S00 = Pw(0, 0) + Rc[0], S10 = Pw(1, 0) + Rc[3], S20 = Pw(2, 0) + Rc[6];
    const double S11 = Pw(1, 1) + Rc[4], S21 = Pw(2, 1) + Rc[7], S22 = Pw(2, 2) + Rc[8];
    const double l00 = std::sqrt(S00), l10 = S10 / l00, l20 = S20 / l00;
    const double a11 = S11 - l10 * l10, l11 = std::sqrt(a11);
    const double l21 = (S21 - l20 * l10) / l11;
    const double a22 = (S22 - l20 * l20) - l21 * l21, l22 = std::sqrt(a22);
    const double nu0 = zc[0] - x[10], nu1 = zc[1] - x[11], nu2 = zc[2] - x[12];
    const double w0 = nu0 / l00, w1 = (nu1 - l10 * w0) / l11, w2 = ((nu2 - l20 * w0) - l21 * w1) / l22;
    const double q = (w0 * w0 + w1 * w1) + w2 * w2;
    const double all[] = {S00, S10, S20, S11, S21, S22, l00, l10, l20, l11, l21, l22, nu0, nu1, nu2, w0, w1, w2, q};
    bool ok = S00 > 0.0 && a11 > 0.0 && a22 > 0.0;
    for (double v : all) ok = ok && std::isfinite(v);
    if (!ok) {
      status = 2;
      return;
    }
    std::vector<double> W(3 * (size_t)n);
    for (int r = 0; r < n; ++r) {
      const double W0 = P(r, 10) / l00;
      const double W1 = (P(r, 11) - W0 * l10) / l11;
      const double W2 = ((P(r, 12) - W0 * l20) - W1 * l21) / l22;
      W[3 * r] = W0, W[3 * r + 1] = W1, W[3 * r + 2] = W2;
      x[r] = x[r] + ((W0 * w0 + W1 * w1) + W2 * w2);
    }
    for (int j = 0; j < n; ++j)
      for (int i = 0; i < n; ++i)
        P(i, j) = P(i, j) - ((W[3 * i] * W[3 * j] + W[3 * i + 1] * W[3 * j + 1]) + W[3 * i + 2] * W[3 * j + 2]);
    s.fill_states(x);
    s.fill_covariances(P);
    status = 1;
    nis = q;
  }

  // cons_slam::step with the gyro update between the predict and the selection
  void step(const uint8_t *frame) {
    const double u[3] = {0.0, 0.0, 0.0};
    s.kalman_predict(u);
    gyro_update();
    s.number_of_visible_features = s.auto_select_n_features(s.cfg.number_of_features_to_select);
    if (!s.selected_feature_list.empty()) {
      s.make_measurements(frame);
      for (const Feature *f : s.selected_feature_list) rejected.erase(f->label);
      apply_consensus();
      if (s.successful_measurement_vector_size != 0) {
        s.kalman_update();
        s.normalise_state();
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

gyro_slam *gyro_slam_create(const orc_config *c) {
  cons_slam *b = cons_slam_create(c);
  gyro_slam *g = new gyro_slam(b->s.cfg);
  delete b;
  return g;
}
void gyro_slam_destroy(gyro_slam *s) { delete s; }
cons_slam *gyro_slam_base(gyro_slam *s) { return s; }
void gyro_slam_set(gyro_slam *s, const double *R9, const double *b3, const double *cov9) { s->set(R9, b3, cov9); }
void gyro_slam_sample(gyro_slam *s, const double *z3) {
  for (int i = 0; i < 3; ++i) s->z[i] = z3[i];
  s->pending = true;
}
void gyro_slam_step(gyro_slam *s, const uint8_t *frame) { s->step(frame); }
int32_t gyro_slam_result(const gyro_slam *s, double *nis) {
  *nis = s->nis;
  return s->status;
}

}  // extern "C"
