// TEST INFRASTRUCTURE ONLY.  The mutual-information selection (include/sl2b200.h, sl2_set_stream_selection) on top
// of the CPU oracle (oracle/slam.hpp, used as it is): the oracle's trace ranking with no limit gives the candidates in
// rank order, then the picks are made in the operation order of csrc/select.cu select_kernel, and the oracle's step
// goes on with them as its selected list.  Compiled by tests/selection_oracle.py with the oracle's flags
// (-O3 -ffp-contract=off).
#include <climits>
#include <cmath>
#include <cstring>
#include <vector>

#include "sl2_oracle.h"
#include "slam.hpp"

using namespace sl2o;

// The oracle's Slam whose selection follows `mode` (SL2_SELECT_*; t = exp2(2 min_bits))
struct sel_slam {
  Slam s;
  int mode = 0;
  double t = 1.0;
  explicit sel_slam(const SlamConfig &c) : s(c) {}

  // the picks among cand (the trace rule's candidates in rank order, so a strict > keeps the smallest rank on ties)
  std::vector<Feature *> information(const std::vector<Feature *> &cand, int n_select) {
    const int V = (int)cand.size();
    const Mat P = s.dense_P();
    std::vector<double> A((size_t)14 * V), B((size_t)6 * V), C00(V), C10(V), C11(V), R(V);
    std::vector<int> y(V), picked(V, 0);
    for (int j = 0; j < V; ++j) {
      const Feature *f = cand[j];
      for (int a = 0; a < 2; ++a) {
        for (int k = 0; k < 7; ++k) A[14 * j + 7 * a + k] = f->dh_by_dxv(a, k);
        for (int k = 0; k < 3; ++k) B[6 * j + 3 * a + k] = f->dh_by_dy(a, k);
      }
      C00[j] = f->S(0, 0);
      C10[j] = f->S(1, 0);
      C11[j] = f->S(1, 1);
      R[j] = f->R(0, 0);
      y[j] = f->position_in_total_state_vector;
    }
    const int nmax = std::min(n_select, V);
    std::vector<double> g((size_t)4 * V * (nmax > 0 ? nmax : 1)), u7(14), uy((size_t)6 * V);
    auto G = [&](int p, int j) { return &g[((size_t)p * V + j) * 4]; };
    std::vector<Feature *> out;
    for (int r = 0; r < nmax; ++r) {
      int i = -1;
      double bq = 0.0;
      for (int j = 0; j < V; ++j) {
        if (picked[j]) continue;
        const double q = (C00[j] * C11[j] - C10[j] * C10[j]) / (R[j] * R[j]);
        if (C00[j] > 0.0 && q > t && (i < 0 || q > bq)) {
          i = j;
          bq = q;
        }
      }
      if (i < 0) break;
      picked[i] = 1;
      out.push_back(cand[i]);
      const double l00 = std::sqrt(C00[i]);
      const double l10 = C10[i] / l00;
      const double l11 = std::sqrt(C11[i] - l10 * l10);
      auto urow = [&](int row, int c) {
        double acc = 0.0;
        for (int k = 0; k < 7; ++k) acc = acc + P(row, k) * A[14 * i + 7 * c + k];
        for (int k = 0; k < 3; ++k) acc = acc + P(row, y[i] + k) * B[6 * i + 3 * c + k];
        return acc;
      };
      for (int row = 0; row < 7; ++row)
        for (int c = 0; c < 2; ++c) u7[2 * row + c] = urow(row, c);
      for (int j = 0; j < V; ++j)
        if (!picked[j])
          for (int k = 0; k < 3; ++k)
            for (int c = 0; c < 2; ++c) uy[6 * j + 2 * k + c] = urow(y[j] + k, c);
      for (int j = 0; j < V; ++j) {
        if (picked[j]) continue;
        double cj[2][2], gn[2][2];
        for (int a = 0; a < 2; ++a)
          for (int b = 0; b < 2; ++b) {
            double acc = 0.0;
            for (int k = 0; k < 7; ++k) acc = acc + A[14 * j + 7 * a + k] * u7[2 * k + b];
            for (int k = 0; k < 3; ++k) acc = acc + B[6 * j + 3 * a + k] * uy[6 * j + 2 * k + b];
            for (int p = 0; p < r; ++p)
              for (int e = 0; e < 2; ++e) acc = acc - G(p, j)[2 * a + e] * G(p, i)[2 * b + e];
            cj[a][b] = acc;
          }
        for (int a = 0; a < 2; ++a) {
          gn[a][0] = cj[a][0] / l00;
          gn[a][1] = (cj[a][1] - gn[a][0] * l10) / l11;
        }
        for (int a = 0; a < 2; ++a)
          for (int e = 0; e < 2; ++e) G(r, j)[2 * a + e] = gn[a][e];
        C00[j] = C00[j] - gn[0][0] * gn[0][0] - gn[0][1] * gn[0][1];
        C10[j] = C10[j] - gn[1][0] * gn[0][0] - gn[1][1] * gn[0][1];
        C11[j] = C11[j] - gn[1][0] * gn[1][0] - gn[1][1] * gn[1][1];
      }
    }
    return out;
  }

  // Slam::go_one_step (monoslam.cpp:108-180) with the selection of `mode`
  void step(const uint8_t *frame) {
    const double u[3] = {0.0, 0.0, 0.0};
    s.kalman_predict(u);
    if (mode == 1) {
      s.number_of_visible_features = s.auto_select_n_features(INT_MAX);
      const std::vector<Feature *> cand = s.selected_feature_list;
      for (Feature *f : cand) f->selected_flag = false;
      s.selected_feature_list = information(cand, s.cfg.number_of_features_to_select);
      for (Feature *f : s.selected_feature_list) f->selected_flag = true;
    } else {
      s.number_of_visible_features = s.auto_select_n_features(s.cfg.number_of_features_to_select);
    }
    if (!s.selected_feature_list.empty()) {
      s.make_measurements(frame);
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

sel_slam *sel_slam_create(const orc_config *c) {
  SlamConfig k;
  k.width = c->width;
  k.height = c->height;
  k.fku = c->fku;
  k.fkv = c->fkv;
  k.u0 = c->u0;
  k.v0 = c->v0;
  k.kd1 = c->kd1;
  k.sd = c->sd;
  k.delta_t = c->delta_t;
  k.number_of_features_to_select = c->number_of_features_to_select;
  k.boxsize = c->boxsize;
  for (int i = 0; i < 3; ++i) k.search_override[i] = c->search_override[i];
  k.minimum_attempted_measurements_of_feature = c->minimum_attempted_measurements_of_feature;
  k.successful_match_fraction = c->successful_match_fraction;
  return new sel_slam(k);
}
void sel_slam_destroy(sel_slam *s) { delete s; }
void sel_slam_set_mode(sel_slam *s, int32_t mode, double t) {
  s->mode = mode;
  s->t = t;
}
void sel_slam_add_feature(sel_slam *s, const double *y, const double *xp_org, const uint8_t *patch) {
  s->s.add_known_feature(y, xp_org, patch);
}
int32_t sel_slam_num_features(const sel_slam *s) { return (int32_t)s->s.feature_list.size(); }
int32_t sel_slam_state_size(const sel_slam *s) { return s->s.total_state_size; }
void sel_slam_set_state(sel_slam *s, const double *x, const double *P) {
  const int n = s->s.total_state_size;
  s->s.fill_states(Vec(x, x + n));
  Mat m(n, n);
  std::memcpy(m.a.data(), P, sizeof(double) * (size_t)n * n);
  s->s.fill_covariances(m);
}
void sel_slam_get_state(const sel_slam *s, double *x, double *P) {
  const int n = s->s.total_state_size;
  Vec xv((size_t)n, 0.0);
  s->s.construct_total_state(xv);
  std::memcpy(x, xv.data(), sizeof(double) * n);
  const Mat Pm = s->s.dense_P();
  std::memcpy(P, Pm.a.data(), sizeof(double) * (size_t)n * n);
}
void sel_slam_step(sel_slam *s, const uint8_t *frame) { s->step(frame); }
// what orc_slam_get_features reads back
void sel_slam_get_features(const sel_slam *s, int32_t *label, double *h, double *z, double *S, uint8_t *flags,
                            int32_t *attempted, int32_t *successful, int32_t *select_rank) {
  const auto &fl = s->s.feature_list;
  for (size_t i = 0; i < fl.size(); ++i) {
    const Feature &f = *fl[i];
    label[i] = f.label;
    h[2 * i] = f.h[0];
    h[2 * i + 1] = f.h[1];
    z[2 * i] = f.z[0];
    z[2 * i + 1] = f.z[1];
    for (int k = 0; k < 4; ++k) S[4 * i + k] = f.S.a.size() == 4 ? f.S.a[k] : 0.0;
    flags[i] = (uint8_t)((f.selected_flag ? 1 : 0) | (f.successful_measurement_flag ? 2 : 0));
    attempted[i] = f.attempted_measurements_of_feature;
    successful[i] = f.successful_measurements_of_feature;
    select_rank[i] = -1;
  }
  for (size_t r = 0; r < s->s.selected_feature_list.size(); ++r)
    select_rank[s->s.selected_feature_list[r]->position_in_list] = (int32_t)r;
}

}  // extern "C"
