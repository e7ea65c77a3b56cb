// ORACLE — TEST INFRASTRUCTURE ONLY (see dense.hpp header).
//
// CPU restatement of the per-frame EKF-MonoSLAM step of SceneLib2, tracking only
// (enable_mapping = false, no partially-initialised features):
//   step order            scenelib2/monoslam.cpp:108-180
//   selection             scenelib2/monoslam.cpp:187-323
//   measurement           scenelib2/monoslam.cpp:336-496
//   gather / scatter      scenelib2/monoslam.cpp:501-614
//   normalise, symmetrise scenelib2/monoslam.cpp:616-637, 143-150
//   feature culling       scenelib2/monoslam.cpp:644-703, 770-812
//   EKF predict / update  scenelib2/kalman.cpp:50-119
//   feature state layout  scenelib2/feature.h:56-143, feature.cpp:108-149
// "Faithful" storage: per-feature Pxy_ / Pyy_ / matrix_block_list_ blocks exactly like the
// reference, dense P assembled and scattered around the update (4 gather/scatter passes per
// frame).
// Pinning: tests/test_oracle_ref.py runs this step against the reference's OWN monoslam.cpp / kalman.cpp /
// feature.cpp (+ models, improc) compiled unmodified against oracle/stubs_arith (_ref/libsl2refmodels.so,
// ref_slam_shim.cpp): selection, match positions, counters, deletion identical frame by frame and over a
// 1 000-step trajectory; state / covariance agree to ~1e-13.  PARITY UNPINNED only at the last ulp
// (Eigen's own product order cannot be reproduced without Eigen), see dense.hpp.
#pragma once
#include <chrono>
#include <memory>

#include "improc.hpp"
#include "models.hpp"

namespace sl2o {

struct Feature {
  double y[3];
  double xp_org[7];
  Mat Pyy;                            // 3x3
  Mat Pxy;                            // 13x3
  std::vector<uint8_t> patch;         // B*B
  std::vector<Mat> matrix_block_list;  // P_{y_j y_i}, j < i, each 3x3
  double h[2] = {0, 0}, z[2] = {0, 0}, nu[2] = {0, 0};
  Mat dh_by_dxv, dh_by_dy, R, S;
  int label = 0;
  int position_in_list = 0;
  int position_in_total_state_vector = 0;
  int attempted_measurements_of_feature = 0;
  int successful_measurements_of_feature = 0;
  bool selected_flag = false;
  bool scheduled_for_termination_flag = false;
  bool successful_measurement_flag = false;
};

struct SlamConfig {
  int width = 320, height = 240;
  double fku = 195, fkv = 195, u0 = 162, v0 = 125, kd1 = 9e-6, sd = 1.0;
  double delta_t = 0.033333333;
  int number_of_features_to_select = 10;
  int boxsize = 11;
  // Benchmark-only: when search_override[0] > 0 the search ellipse of every feature is
  // PuInv = (search_override[0], search_override[1], search_override[2]) instead of S_i^-1.
  double search_override[3] = {0, 0, 0};
  int minimum_attempted_measurements_of_feature = 10;  // monoslam.cpp:1875
  double successful_match_fraction = 0.5;              // monoslam.cpp:1876
};

struct Slam {
  SlamConfig cfg;
  Camera cam;
  double xv[13];
  Mat Pxx;  // 13x13
  std::vector<std::unique_ptr<Feature>> feature_list;
  std::vector<Feature *> selected_feature_list;
  int total_state_size = 13;
  int next_free_label = 0;
  int successful_measurement_vector_size = 0;
  int number_of_visible_features = 0;
  // benchmark bookkeeping only: seconds spent in the 4 gather / scatter passes per frame (monoslam.cpp:518-614
  // around the update and the symmetrisation); "dense-resident" CPU figure = run time minus this
  double gather_scatter_seconds = 0.0;
  struct GsTimer {
    double &acc;
    std::chrono::steady_clock::time_point t0;
    explicit GsTimer(double &a) : acc(a), t0(std::chrono::steady_clock::now()) {}
    ~GsTimer() { acc += std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count(); }
  };

  explicit Slam(const SlamConfig &c) : cfg(c), Pxx(13, 13) {
    cam.width = c.width;
    cam.height = c.height;
    cam.fku = c.fku;
    cam.fkv = c.fkv;
    cam.u0 = c.u0;
    cam.v0 = c.v0;
    cam.kd1 = c.kd1;
    cam.sd = c.sd;
    for (double &e : xv) e = 0.0;
    xv[3] = 1.0;
  }

  // monoslam.cpp:1278-1289 + feature.cpp:108-149 (known, fully-initialised feature)
  void add_known_feature(const double y[3], const double xp_org[7], const uint8_t *patch) {
    std::unique_ptr<Feature> f(new Feature);
    for (int i = 0; i < 3; ++i) f->y[i] = y[i];
    for (int i = 0; i < 7; ++i) f->xp_org[i] = xp_org[i];
    f->patch.assign(patch, patch + cfg.boxsize * cfg.boxsize);
    f->label = next_free_label;
    f->position_in_list = (int)feature_list.size();
    f->position_in_total_state_vector = total_state_size;
    f->Pxy = Mat(13, 3);
    f->Pyy = Mat(3, 3);
    for (int i = 0; i < f->position_in_list; ++i) f->matrix_block_list.push_back(Mat(3, 3));
    feature_list.push_back(std::move(f));
    total_state_size += 3;
    ++next_free_label;
  }

  // ---- gather / scatter (monoslam.cpp:501-614) -------------------------------------------
  void construct_total_state(Vec &V) const {
    int pos = 0;
    for (int i = 0; i < 13; ++i) V[pos + i] = xv[i];
    pos += 13;
    for (const auto &f : feature_list) {
      for (int i = 0; i < 3; ++i) V[pos + i] = f->y[i];
      pos += 3;
    }
  }
  void construct_total_covariance(Mat &M) const {
    set_block(M, 0, 0, Pxx);
    int x_position = 13;
    for (const auto &f : feature_list) {
      int y_position = 0;
      set_block(M, y_position, x_position, f->Pxy);
      set_block_transposed(M, x_position, y_position, f->Pxy);
      y_position += 13;
      for (const Mat &blk : f->matrix_block_list) {
        set_block(M, y_position, x_position, blk);
        set_block_transposed(M, x_position, y_position, blk);
        y_position += blk.r;
      }
      set_block(M, y_position, x_position, f->Pyy);
      x_position += 3;
    }
  }
  void fill_states(const Vec &V) {
    int pos = 0;
    for (int i = 0; i < 13; ++i) xv[i] = V[pos + i];
    pos += 13;
    for (auto &f : feature_list) {
      if (pos >= (int)V.size()) break;
      for (int i = 0; i < 3; ++i) f->y[i] = V[pos + i];
      pos += 3;
    }
  }
  void fill_covariances(const Mat &M) {
    Pxx = block(M, 0, 0, 13, 13);
    int x_position = 13;
    for (auto &f : feature_list) {
      if (x_position >= M.c) break;
      int y_position = 0;
      f->Pxy = block(M, y_position, x_position, 13, 3);
      y_position += 13;
      for (Mat &blk : f->matrix_block_list) {
        blk = block(M, y_position, x_position, blk.r, blk.c);
        y_position += blk.r;
      }
      f->Pyy = block(M, y_position, x_position, 3, 3);
      x_position += 3;
    }
  }
  Mat dense_P() const {
    Mat P(total_state_size, total_state_size);
    construct_total_covariance(P);
    return P;
  }

  // ---- kalman.cpp:50-69 ------------------------------------------------------------------
  void kalman_predict(const double u[3]) {
    double fv[13];
    Mat F;
    MotionModel::fv_and_dfv_by_dxv(xv, u, cfg.delta_t, fv, F);
    const Mat Q = MotionModel::Q(xv, cfg.delta_t);  // func_Q uses the OLD xv (:55 before :57)
    for (int i = 0; i < 13; ++i) xv[i] = fv[i];
    Pxx = add(mul_nt(mul(F, Pxx), F), Q);
    for (auto &f : feature_list) f->Pxy = mul(F, f->Pxy);
  }

  // ---- monoslam.cpp:289-308 --------------------------------------------------------------
  void predict_single_feature_measurements(Feature *f) {
    FeaturePrediction p;
    FullFeatureModel::predict(cam, xv, f->y, Pxx, f->Pxy, f->Pyy, p);
    f->h[0] = p.h[0];
    f->h[1] = p.h[1];
    f->dh_by_dy = p.dh_by_dy;
    f->dh_by_dxv = p.dh_by_dxv;
    f->R = p.R;
    f->S = p.S;
  }

  // ---- monoslam.cpp:187-254 --------------------------------------------------------------
  int auto_select_n_features(int n) {
    for (Feature *f : selected_feature_list) f->selected_flag = false;
    selected_feature_list.clear();
    std::vector<std::pair<double, Feature *>> fas;
    for (auto &fp : feature_list) {
      Feature *f = fp.get();
      predict_single_feature_measurements(f);
      const int cant_see = FullFeatureModel::visibility_test(cam, xv, f->y, f->xp_org, f->h);
      if (cant_see == 0) {
        const double score = f->S(0, 0) + f->S(1, 1);  // trace, full_feature_model.cpp:172-176
        bool added = false;
        for (auto it = fas.begin(); it != fas.end(); ++it) {
          if (score > it->first) {
            fas.insert(it, std::make_pair(score, f));
            added = true;
            break;
          }
        }
        if (!added) fas.push_back(std::make_pair(score, f));
      }
    }
    int n_actual = 0;
    if (fas.empty()) return 0;
    for (auto &e : fas) {
      if (e.first == 0.0 || n_actual == n) return (int)fas.size();
      if (!e.second->selected_flag) {
        e.second->selected_flag = true;
        selected_feature_list.push_back(e.second);
      }
      ++n_actual;
    }
    return (int)fas.size();
  }

  // ---- monoslam.cpp:336-386, 479-496 -----------------------------------------------------
  int make_measurements(const uint8_t *image) {
    int count = 0;
    if (selected_feature_list.empty()) return 0;
    successful_measurement_vector_size = 0;
    for (Feature *f : selected_feature_list) {
      double PuInv[4];
      if (cfg.search_override[0] > 0.0) {
        PuInv[0] = cfg.search_override[0];
        PuInv[1] = PuInv[2] = cfg.search_override[1];
        PuInv[3] = cfg.search_override[2];
      } else {
        puinv_from_S(f->S.a.data(), PuInv);
      }
      int u_found = 0, v_found = 0;
      const bool ok = elliptical_search(image, cfg.width, cfg.height, f->patch.data(), f->h,
                                        PuInv[0], PuInv[2], PuInv[3], &u_found, &v_found,
                                        cfg.boxsize);
      if (!ok) {
        f->successful_measurement_flag = false;
        ++f->attempted_measurements_of_feature;
      } else {
        f->z[0] = (double)u_found;
        f->z[1] = (double)v_found;
        f->successful_measurement_flag = true;
        successful_measurement_vector_size += 2;
        f->nu[0] = f->z[0] - f->h[0];  // full_feature_model.cpp:197-200
        f->nu[1] = f->z[1] - f->h[1];
        ++f->successful_measurements_of_feature;
        ++f->attempted_measurements_of_feature;
        ++count;
      }
    }
    return count;
  }

  // ---- monoslam.cpp:548-572 --------------------------------------------------------------
  void construct_total_measurement_stuff(Vec &nu_tot, Mat &H, Mat &R_tot) const {
    int pos = 0;
    for (const Feature *f : selected_feature_list) {
      if (!f->successful_measurement_flag) continue;
      nu_tot[pos] = f->nu[0];
      nu_tot[pos + 1] = f->nu[1];
      set_block(H, pos, 0, f->dh_by_dxv);
      set_block(H, pos, f->position_in_total_state_vector, f->dh_by_dy);
      set_block(R_tot, pos, pos, f->R);
      pos += 2;
    }
  }

  // ---- kalman.cpp:72-119 (dense, as written) ---------------------------------------------
  static void kalman_update_dense(Vec &x, Mat &P, const Mat &H, const Mat &R, const Vec &nu) {
    Mat S = mul_nt(mul(H, P), H);  // (H*P)*H^T
    add_inplace(S, R);
    const Mat S_L = cholesky_lower(S);
    const Mat S_Linv = lower_inverse(S_L);
    const Mat Sinv = mul_tn(S_Linv, S_Linv);
    const Mat W = mul(mul_nt(P, H), Sinv);  // (P*H^T)*Sinv
    const Vec dx = mul(W, nu);
    for (size_t i = 0; i < x.size(); ++i) x[i] += dx[i];
    sub_inplace(P, mul_nt(mul(W, S), W));  // P -= (W*S)*W^T
  }

  void kalman_update() {
    const int size = successful_measurement_vector_size;
    const int size2 = total_state_size;
    Vec x((size_t)size2, 0.0);
    Mat P(size2, size2);
    {
      GsTimer tm(gather_scatter_seconds);
      construct_total_state(x);
      construct_total_covariance(P);
    }
    Vec nu_tot((size_t)size, 0.0);
    Mat H(size, size2), R_tot(size, size);
    construct_total_measurement_stuff(nu_tot, H, R_tot);
    kalman_update_dense(x, P, H, R_tot, nu_tot);
    {
      GsTimer tm(gather_scatter_seconds);
      fill_states(x);
      fill_covariances(P);
    }
  }

  // ---- monoslam.cpp:616-637 --------------------------------------------------------------
  void normalise_state() {
    const Mat J = MotionModel::dxvnorm_by_dxv(xv);
    Pxx = mul_nt(mul(J, Pxx), J);
    for (auto &f : feature_list) f->Pxy = mul(J, f->Pxy);
  }

  // ---- monoslam.cpp:644-703, 770-812 -----------------------------------------------------
  void delete_feature_at(size_t idx) {
    Feature *del = feature_list[idx].get();
    for (size_t j = idx + 1; j < feature_list.size(); ++j) {
      Feature *f = feature_list[j].get();
      --f->position_in_list;
      f->matrix_block_list.erase(f->matrix_block_list.begin() + del->position_in_list);
      f->position_in_total_state_vector -= 3;
    }
    if (del->selected_flag) {
      for (auto it = selected_feature_list.begin(); it != selected_feature_list.end(); ++it)
        if (*it == del) {
          selected_feature_list.erase(it);
          break;
        }
    }
    total_state_size -= 3;
    feature_list.erase(feature_list.begin() + idx);
  }
  void delete_bad_features() {
    for (auto &f : feature_list) {
      if (f->attempted_measurements_of_feature >= cfg.minimum_attempted_measurements_of_feature &&
          double(f->successful_measurements_of_feature) /
                  double(f->attempted_measurements_of_feature) <
              cfg.successful_match_fraction)
        f->scheduled_for_termination_flag = true;
    }
    for (size_t i = 0; i < feature_list.size();) {
      if (feature_list[i]->scheduled_for_termination_flag)
        delete_feature_at(i);
      else
        ++i;
    }
  }

  // ---- monoslam.cpp:108-180 (tracking only) ----------------------------------------------
  void go_one_step(const uint8_t *frame) {
    const double u[3] = {0.0, 0.0, 0.0};
    kalman_predict(u);
    number_of_visible_features = auto_select_n_features(cfg.number_of_features_to_select);
    if (!selected_feature_list.empty()) {
      make_measurements(frame);
      if (successful_measurement_vector_size != 0) {
        kalman_update();
        normalise_state();
      }
    }
    delete_bad_features();
    Mat P(total_state_size, total_state_size);
    {
      GsTimer tm(gather_scatter_seconds);
      construct_total_covariance(P);
    }
    const Mat PT = transpose(P);
    for (size_t i = 0; i < P.a.size(); ++i) P.a[i] = P.a[i] * 0.5 + PT.a[i] * 0.5;
    {
      GsTimer tm(gather_scatter_seconds);
      fill_covariances(P);
    }
  }
};

}  // namespace sl2o
