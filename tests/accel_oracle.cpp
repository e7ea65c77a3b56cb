// TEST INFRASTRUCTURE ONLY.  The accelerometer (include/sl2b200.h, sl2_set_stream_accel) on top of the CPU oracle
// (oracle/slam.hpp, used as it is) and of the consensus oracle (tests/consensus_oracle.cpp, included as it is, with its
// consensus off): a whole step whose predict, when a sample is pending, is the header's prediction built from the
// oracle's own motion model (MotionModel::fv_and_dfv_by_dxv with u = a, FullFeatureModel::dRq_times_a_by_dq, the
// reference's Gn) and its dense products, then select, measure, update, cull.  Compiled by tests/accel_oracle.py with
// the oracle's flags (-O3 -ffp-contract=off).
#include <cmath>

#include "consensus_oracle.cpp"

struct accel_slam : cons_slam {
  double R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, b[3] = {0, 0, 0}, Rc[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  double g[3] = {0, 0, 0}, sd2 = 16.0;
  double f[3] = {0, 0, 0};
  bool pending = false;
  int status = 0;
  double a_last[3] = {0, 0, 0};
  explicit accel_slam(const SlamConfig &c) : cons_slam(c) {}

  void set(const double *R9, const double *b3, const double *C, const double *g3, double sd_a) {
    for (int i = 0; i < 9; ++i) R[i] = R9[i];
    for (int i = 0; i < 3; ++i) b[i] = b3[i], g[i] = g3[i];
    sd2 = sd_a * sd_a;
    double M[9];  // Rc = R^T C R: M = C R, the upper triangle of R^T M, mirrored
    for (int k = 0; k < 3; ++k)
      for (int j = 0; j < 3; ++j) M[3 * k + j] = (C[3 * k] * R[j] + C[3 * k + 1] * R[3 + j]) + C[3 * k + 2] * R[6 + j];
    for (int i = 0; i < 3; ++i)
      for (int j = i; j < 3; ++j) Rc[3 * i + j] = Rc[3 * j + i] = (R[i] * M[j] + R[3 + i] * M[3 + j]) + R[6 + i] * M[6 + j];
  }

  // kalman_predict with the accelerometer's a, F blocks and linear noise block; the plain predict without a sample or
  // when a, D or the block is not finite
  void predict() {
    status = 0;
    for (double &v : a_last) v = 0.0;
    const double zero[3] = {0.0, 0.0, 0.0};
    if (!pending) {
      s.kalman_predict(zero);
      return;
    }
    pending = false;
    const double dt = s.cfg.delta_t;
    const Quat q = {s.xv[3], s.xv[4], s.xv[5], s.xv[6]};
    double d[3], fc[3], Rq[3][3], a[3];
    for (int i = 0; i < 3; ++i) d[i] = f[i] - b[i];
    for (int i = 0; i < 3; ++i) fc[i] = (R[i] * d[0] + R[3 + i] * d[1]) + R[6 + i] * d[2];
    quat_to_R(q, Rq);
    for (int i = 0; i < 3; ++i) a[i] = (Rq[i][0] * fc[0] + Rq[i][1] * fc[1]) + Rq[i][2] * fc[2] + g[i];
    const Mat D = FullFeatureModel::dRq_times_a_by_dq(q, fc);
    double L[3][3];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        double t = 0.0;
        for (int m = 0; m < 3; ++m)
          for (int k = 0; k < 3; ++k) t += Rq[i][m] * Rc[3 * m + k] * Rq[j][k];
        L[i][j] = (t + (i == j ? sd2 : 0.0)) * dt * dt;
      }
    bool ok = true;
    for (int i = 0; i < 3; ++i) {
      ok = ok && std::isfinite(a[i]);
      for (int j = 0; j < 4; ++j) ok = ok && std::isfinite(D(i, j));
      for (int j = 0; j < 3; ++j) ok = ok && std::isfinite(L[i][j]);
    }
    if (!ok) {
      status = 2;
      s.kalman_predict(zero);
      return;
    }
    double fv[13];
    Mat F;
    MotionModel::fv_and_dfv_by_dxv(s.xv, a, dt, fv, F);  // v' = v + a dt
    const double h = 0.5 * dt * dt;
    for (int i = 0; i < 3; ++i) {
      fv[i] = fv[i] + a[i] * h;
      for (int j = 0; j < 4; ++j) {
        F(i, 3 + j) = h * D(i, j);
        F(7 + i, 3 + j) = dt * D(i, j);
      }
    }
    Mat G(13, 6), Pnn(6, 6);
    for (int i = 0; i < 3; ++i) {
      G(7 + i, i) = 1.0;
      G(10 + i, 3 + i) = 1.0;
      G(i, i) = 1.0 * dt;
      for (int j = 0; j < 3; ++j) Pnn(i, j) = L[i][j];
      Pnn(3 + i, 3 + i) = MotionModel::kSdAlpha * MotionModel::kSdAlpha * dt * dt;
    }
    const double om[3] = {s.xv[10], s.xv[11], s.xv[12]};
    set_block(G, 3, 3, mul(dq3_by_dq1(q), MotionModel::dqomegadt_by_domega(om, dt)));
    const Mat Q = mul_nt(mul(G, Pnn), G);
    for (int i = 0; i < 13; ++i) s.xv[i] = fv[i];
    s.Pxx = add(mul_nt(mul(F, s.Pxx), F), Q);
    for (auto &ft : s.feature_list) ft->Pxy = mul(F, ft->Pxy);
    status = 1;
    for (int i = 0; i < 3; ++i) a_last[i] = a[i];
  }

  // cons_slam::step with the accelerometer's predict
  void step(const uint8_t *frame) {
    predict();
    s.number_of_visible_features = s.auto_select_n_features(s.cfg.number_of_features_to_select);
    if (!s.selected_feature_list.empty()) {
      s.make_measurements(frame);
      for (const Feature *ft : s.selected_feature_list) rejected.erase(ft->label);
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

accel_slam *accel_slam_create(const orc_config *c) {
  cons_slam *b = cons_slam_create(c);
  accel_slam *a = new accel_slam(b->s.cfg);
  delete b;
  return a;
}
void accel_slam_destroy(accel_slam *s) { delete s; }
cons_slam *accel_slam_base(accel_slam *s) { return s; }
void accel_slam_set(accel_slam *s, const double *R9, const double *b3, const double *cov9, const double *g3,
                    double sd_a) {
  s->set(R9, b3, cov9, g3, sd_a);
}
void accel_slam_sample(accel_slam *s, const double *f3) {
  for (int i = 0; i < 3; ++i) s->f[i] = f3[i];
  s->pending = true;
}
void accel_slam_step(accel_slam *s, const uint8_t *frame) { s->step(frame); }
int32_t accel_slam_result(const accel_slam *s, double *a3) {
  for (int i = 0; i < 3; ++i) a3[i] = s->a_last[i];
  return s->status;
}

}  // extern "C"
