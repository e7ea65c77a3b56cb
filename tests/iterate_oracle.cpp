// TEST INFRASTRUCTURE ONLY.  The iterated EKF update (include/sl2b200.h, sl2_set_stream_iterated) on top of the CPU
// oracle (oracle/slam.hpp, used as it is) and of the sub-pixel oracle (tests/subpixel_oracle.cpp, which includes the
// rescue and consensus oracles; all included as they are): the first update of the step replaced by the iterated one,
// written from the header's definition with the oracle's own dense algebra and feature model, and a whole step that
// runs
//   predict, select, measure, refine, consensus, iterated update 1, rescue and update 2, cull.
// Compiled by tests/iterate_oracle.py with the oracle's flags (-O3 -ffp-contract=off).
#include <cmath>

#include "subpixel_oracle.cpp"

// The sub-pixel oracle's Slam with the iterated first update.  iterations / status / delta: the last step's results,
// as sl2_get_iterated_results returns them.
struct iter_slam : sub_slam {
  int max_iterations = 0;
  double tol = 0.0;
  int iterations = 0, status = 0;
  double delta = 0.0;
  explicit iter_slam(const SlamConfig &c) : sub_slam(c) {}

  // update 1: N relinearisations at most, then the oracle's kalman_update at the last accepted linearisation from the
  // prediction's state; the features' h, H and nu are the prediction's again afterwards (sl2_get_features shows them)
  void iterated_update() {
    iterations = status = 0;
    delta = 0.0;
    std::vector<Feature *> rows;
    for (Feature *f : s.selected_feature_list)
      if (f->successful_measurement_flag) rows.push_back(f);
    if (max_iterations == 0 || rows.empty()) {
      s.kalman_update();
      return;
    }
    struct Saved {
      double h[2], nu[2];
      Mat dxv, dy;
    };
    std::vector<Saved> saved;
    for (Feature *f : rows) saved.push_back({{f->h[0], f->h[1]}, {f->nu[0], f->nu[1]}, f->dh_by_dxv, f->dh_by_dy});
    const int n = s.total_state_size, m = s.successful_measurement_vector_size;
    Vec x0((size_t)n, 0.0);
    Mat P0(n, n);
    s.construct_total_state(x0);
    s.construct_total_covariance(P0);
    Vec xi = x0;
    status = 2;
    for (int i = 0; i < max_iterations; ++i) {
      Vec nu((size_t)m, 0.0);
      Mat H(m, n), R(m, m);
      s.construct_total_measurement_stuff(nu, H, R);
      const Mat HP = mul(H, P0);
      Mat S = mul_nt(HP, H);
      add_inplace(S, R);
      const Mat Li = lower_inverse(cholesky_lower(S));
      const Vec t = mul(mul_tn(Li, Li), nu);
      Vec xn = x0;
      for (int j = 0; j < n; ++j) {
        double a = 0.0;
        for (int r = 0; r < m; ++r) a += HP(r, j) * t[r];
        xn[j] = x0[j] + a;
      }
      bool fin = true;
      double d = 0.0;
      for (int j = 0; j < n; ++j) {
        fin = fin && std::isfinite(xn[j]);
        if (P0(j, j) > 0.0) d = std::fmax(d, std::fabs(xn[j] - xi[j]) / std::sqrt(P0(j, j)));
      }
      delta = fin ? d : NAN;
      if (delta <= tol) {
        status = 1;
        break;
      }
      // relinearise every row at x_{i+1} with the oracle's feature model
      std::vector<FeaturePrediction> ps(rows.size());
      std::vector<double> heff(2 * rows.size());
      bool ok = fin;
      for (size_t k = 0; k < rows.size() && ok; ++k) {
        const int pos = rows[k]->position_in_total_state_vector;
        const double *y = xn.data() + pos;
        FullFeatureModel::predict(s.cam, xn.data(), y, s.Pxx, rows[k]->Pxy, rows[k]->Pyy, ps[k]);
        double zc[3];
        Mat a, b;
        FullFeatureModel::zeroedyi(y, xn.data(), zc, a, b);
        ok = zc[2] > 0.0;
        for (int r = 0; r < 2; ++r) {
          double c = 0.0;
          for (int q = 0; q < 7; ++q) c += ps[k].dh_by_dxv(r, q) * (x0[q] - xn[q]);
          for (int q = 0; q < 3; ++q) c += ps[k].dh_by_dy(r, q) * (x0[pos + q] - xn[pos + q]);
          heff[2 * k + r] = ps[k].h[r] + c;
          ok = ok && std::isfinite(heff[2 * k + r]);
        }
        for (double v : ps[k].dh_by_dxv.a) ok = ok && std::isfinite(v);
        for (double v : ps[k].dh_by_dy.a) ok = ok && std::isfinite(v);
      }
      if (!ok) {
        status = 3;
        break;
      }
      for (size_t k = 0; k < rows.size(); ++k) {
        Feature *f = rows[k];
        f->h[0] = heff[2 * k];
        f->h[1] = heff[2 * k + 1];
        f->dh_by_dxv = ps[k].dh_by_dxv;
        f->dh_by_dy = ps[k].dh_by_dy;
        f->nu[0] = f->z[0] - f->h[0];
        f->nu[1] = f->z[1] - f->h[1];
      }
      iterations = i + 1;
      xi = xn;
    }
    s.kalman_update();
    for (size_t k = 0; k < rows.size(); ++k) {
      Feature *f = rows[k];
      f->h[0] = saved[k].h[0];
      f->h[1] = saved[k].h[1];
      f->nu[0] = saved[k].nu[0];
      f->nu[1] = saved[k].nu[1];
      f->dh_by_dxv = saved[k].dxv;
      f->dh_by_dy = saved[k].dy;
    }
  }

  // sub_slam::step with the iterated update 1
  void step(const uint8_t *frame) {
    const double u[3] = {0.0, 0.0, 0.0};
    s.kalman_predict(u);
    s.number_of_visible_features = s.auto_select_n_features(s.cfg.number_of_features_to_select);
    rescued.clear();
    iterations = status = 0;
    delta = 0.0;
    if (!s.selected_feature_list.empty()) {
      s.make_measurements(frame);
      refine(frame);
      for (const Feature *f : s.selected_feature_list) rejected.erase(f->label);
      apply_consensus();
      if (s.successful_measurement_vector_size != 0) {
        iterated_update();
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

iter_slam *iter_slam_create(const orc_config *c) {
  cons_slam *b = cons_slam_create(c);
  iter_slam *r = new iter_slam(b->s.cfg);
  delete b;
  return r;
}
void iter_slam_destroy(iter_slam *s) { delete s; }
void iter_slam_set(iter_slam *s, double tau, double chi2, int32_t max_iterations, double tol) {
  s->tau = tau;
  s->chi2 = chi2;
  s->max_iterations = max_iterations;
  s->tol = tol;
}
cons_slam *iter_slam_base(iter_slam *s) { return s; }
sub_slam *iter_slam_sub(iter_slam *s) { return s; }
void iter_slam_step(iter_slam *s, const uint8_t *frame) { s->step(frame); }
void iter_slam_results(const iter_slam *s, int32_t *iterations, int32_t *status, double *delta) {
  *iterations = s->iterations;
  *status = s->status;
  *delta = s->delta;
}

}  // extern "C"
