// TEST INFRASTRUCTURE ONLY.  The match consensus (include/sl2b200.h, sl2_set_stream_consensus) on top of the CPU
// oracle (oracle/slam.hpp, used as it is): the consensus as a pure function in the operation order of csrc/ekf.cu
// consensus_kernel, and a whole step that runs it between the oracle's measure and update.  Compiled by
// tests/consensus_oracle.py with the oracle's flags (-O3 -ffp-contract=off).
#include <cstring>
#include <set>
#include <vector>

#include "sl2_oracle.h"
#include "slam.hpp"

using namespace sl2o;

namespace {

// k matches in selection-rank order; x (n) and P (column-major, leading dimension ld) the predicted state and
// covariance; pos[j] = index of y_j in x; z, h (k x 2); S (k x 4 column-major); dh_dxp (k x 2 x 7 row-major), dh_dy
// (k x 2 x 3 row-major).  keep[j] = 0 for a rejected match, support[i] = inliers of hypothesis i; returns the winner or
// -1 when nothing is rejected.
int consensus(const Camera &cam0, const double *x, const double *P, int ld, int k, const int *pos, const double *z,
              const double *h, const double *S, const double *dh_dxp, const double *dh_dy, double tau, uint8_t *keep,
              int *support) {
  Camera cam = cam0;
  const double tau2 = tau * tau;
  auto Pat = [&](int r, int c) { return P[r + (size_t)ld * c]; };
  std::vector<double> a((size_t)7 * k), b((size_t)3 * k);
  for (int j = 0; j < k; ++j) {
    const double nu0 = z[2 * j] - h[2 * j], nu1 = z[2 * j + 1] - h[2 * j + 1];
    double si[4];
    puinv_from_S(S + 4 * j, si);  // (00, 10, 01, 11): the sinv_from_S sequence of the search
    const double w0 = si[0] * nu0 + si[2] * nu1, w1 = si[2] * nu0 + si[3] * nu1;
    for (int c = 0; c < 7; ++c) a[7 * j + c] = dh_dxp[14 * j + c] * w0 + dh_dxp[14 * j + 7 + c] * w1;
    for (int c = 0; c < 3; ++c) b[3 * j + c] = dh_dy[6 * j + c] * w0 + dh_dy[6 * j + 3 + c] * w1;
  }
  std::vector<std::vector<uint8_t>> in((size_t)k, std::vector<uint8_t>((size_t)k, 0));
  int best = -1, win = -1;
  for (int i = 0; i < k; ++i) {
    const double *ai = &a[7 * i], *bi = &b[3 * i];
    double xp[7];
    for (int r = 0; r < 7; ++r) {
      double s = 0.0;
      for (int c = 0; c < 7; ++c) s = s + Pat(r, c) * ai[c];
      for (int c = 0; c < 3; ++c) s = s + Pat(r, pos[i] + c) * bi[c];
      xp[r] = x[r] + s;
    }
    int sup = 0;
    for (int j = 0; j < k; ++j) {
      double y[3];
      for (int r = 0; r < 3; ++r) {
        double s = 0.0;
        for (int c = 0; c < 7; ++c) s = s + Pat(pos[j] + r, c) * ai[c];
        for (int c = 0; c < 3; ++c) s = s + Pat(pos[j] + r, pos[i] + c) * bi[c];
        y[r] = x[pos[j] + r] + s;
      }
      double zc[3], g[2];
      Mat dz_dxp, dz_dy;
      FullFeatureModel::zeroedyi(y, xp, zc, dz_dxp, dz_dy);
      if (zc[2] > 0.0) {
        cam.project(zc, g);
        const double du = z[2 * j] - g[0], dv = z[2 * j + 1] - g[1];
        in[i][j] = (du * du + dv * dv <= tau2) ? 1 : 0;
      }
      sup += in[i][j];
    }
    support[i] = sup;
    if (sup > best) {
      best = sup;
      win = i;
    }
  }
  if (best < 2) win = -1;
  for (int j = 0; j < k; ++j) keep[j] = win < 0 ? 1 : in[win][j];
  return win;
}

Camera cam_of(const SlamConfig &c) {
  Camera cam;
  cam.width = c.width;
  cam.height = c.height;
  cam.fku = c.fku;
  cam.fkv = c.fkv;
  cam.u0 = c.u0;
  cam.v0 = c.v0;
  cam.kd1 = c.kd1;
  cam.sd = c.sd;
  return cam;
}

}  // namespace

// The oracle's Slam with a consensus: `rejected` holds the labels of the features whose last match the consensus
// rejected (found = 2 on the device), kept like Feature::successful_measurement_flag_ until the next measurement.
struct cons_slam {
  Slam s;
  double tau = 0.0;
  std::set<int> rejected;
  explicit cons_slam(const SlamConfig &c) : s(c) {}

  void apply_consensus() {
    std::vector<Feature *> M;
    for (Feature *f : s.selected_feature_list)
      if (f->successful_measurement_flag) M.push_back(f);
    const int k = (int)M.size(), n = s.total_state_size;
    if (!(tau > 0.0) || k < 2) return;
    Vec x((size_t)n, 0.0);
    Mat P(n, n);
    s.construct_total_state(x);
    s.construct_total_covariance(P);
    std::vector<int> pos(k), support(k);
    std::vector<double> z(2 * k), h(2 * k), S(4 * k), dxp(14 * k), dy(6 * k);
    for (int j = 0; j < k; ++j) {
      const Feature *f = M[j];
      pos[j] = f->position_in_total_state_vector;
      for (int e = 0; e < 2; ++e) {
        z[2 * j + e] = f->z[e];
        h[2 * j + e] = f->h[e];
      }
      for (int e = 0; e < 4; ++e) S[4 * j + e] = f->S.a[e];
      for (int r = 0; r < 2; ++r) {
        for (int c = 0; c < 7; ++c) dxp[14 * j + 7 * r + c] = f->dh_by_dxv(r, c);
        for (int c = 0; c < 3; ++c) dy[6 * j + 3 * r + c] = f->dh_by_dy(r, c);
      }
    }
    std::vector<uint8_t> keep(k);
    consensus(cam_of(s.cfg), x.data(), P.a.data(), n, k, pos.data(), z.data(), h.data(), S.data(), dxp.data(),
              dy.data(), tau, keep.data(), support.data());
    for (int j = 0; j < k; ++j)
      if (!keep[j]) {  // an attempted, unsuccessful measurement: out of the update, counted by the cull
        Feature *f = M[j];
        f->successful_measurement_flag = false;
        --f->successful_measurements_of_feature;
        s.successful_measurement_vector_size -= 2;
        rejected.insert(f->label);
      }
  }

  // Slam::go_one_step (monoslam.cpp:108-180) with the consensus between make_measurements and the update
  void step(const uint8_t *frame) {
    const double u[3] = {0.0, 0.0, 0.0};
    s.kalman_predict(u);
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

int32_t cons_consensus(const double *cam8, const double *x, const double *P, int32_t ld, int32_t k,
                       const int32_t *positions, const double *z, const double *h, const double *S,
                       const double *dh_dxp, const double *dh_dy, double tau, uint8_t *keep, int32_t *support) {
  Camera cam;
  cam.width = (int)cam8[0];
  cam.height = (int)cam8[1];
  cam.fku = cam8[2];
  cam.fkv = cam8[3];
  cam.u0 = cam8[4];
  cam.v0 = cam8[5];
  cam.kd1 = cam8[6];
  cam.sd = cam8[7];
  return consensus(cam, x, P, ld, k, positions, z, h, S, dh_dxp, dh_dy, tau, keep, support);
}

cons_slam *cons_slam_create(const orc_config *c) {
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
  return new cons_slam(k);
}
void cons_slam_destroy(cons_slam *s) { delete s; }
void cons_slam_set_tau(cons_slam *s, double tau) { s->tau = tau; }
void cons_slam_add_feature(cons_slam *s, const double *y, const double *xp_org, const uint8_t *patch) {
  s->s.add_known_feature(y, xp_org, patch);
}
int32_t cons_slam_num_features(const cons_slam *s) { return (int32_t)s->s.feature_list.size(); }
int32_t cons_slam_state_size(const cons_slam *s) { return s->s.total_state_size; }
void cons_slam_set_state(cons_slam *s, const double *x, const double *P) {
  const int n = s->s.total_state_size;
  s->s.fill_states(Vec(x, x + n));
  Mat m(n, n);
  std::memcpy(m.a.data(), P, sizeof(double) * (size_t)n * n);
  s->s.fill_covariances(m);
}
void cons_slam_get_state(const cons_slam *s, double *x, double *P) {
  const int n = s->s.total_state_size;
  Vec xv((size_t)n, 0.0);
  s->s.construct_total_state(xv);
  std::memcpy(x, xv.data(), sizeof(double) * n);
  const Mat Pm = s->s.dense_P();
  std::memcpy(P, Pm.a.data(), sizeof(double) * (size_t)n * n);
}
void cons_slam_step(cons_slam *s, const uint8_t *frame) { s->step(frame); }
// what orc_slam_get_features reads back, with flags bit 2 = the last match was rejected by the consensus
void cons_slam_get_features(const cons_slam *s, int32_t *label, double *h, double *z, double *S, uint8_t *flags,
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
    flags[i] = (uint8_t)((f.selected_flag ? 1 : 0) | (f.successful_measurement_flag ? 2 : 0) |
                         (s->rejected.count(f.label) ? 4 : 0));
    attempted[i] = f.attempted_measurements_of_feature;
    successful[i] = f.successful_measurements_of_feature;
    select_rank[i] = -1;
  }
  for (size_t r = 0; r < s->s.selected_feature_list.size(); ++r)
    select_rank[s->s.selected_feature_list[r]->position_in_list] = (int32_t)r;
}

}  // extern "C"
