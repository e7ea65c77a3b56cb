// TEST INFRASTRUCTURE ONLY.  The sub-pixel refinement (include/sl2b200.h, sl2_set_stream_subpixel) on top of the CPU
// oracle (oracle/slam.hpp, used as it is) and of the rescue oracle (tests/rescue_oracle.cpp, which includes the
// consensus oracle; both included as they are): the refinement of every successful match right after the oracle's
// elliptical_search, scored with its correlate2_warning, in the operation order of csrc/subpixel.cu subpixel_kernel,
// and a whole step that runs
//   predict, select, measure, refine, consensus, update 1, rescue and update 2, cull.
// Compiled by tests/subpixel_oracle.py with the oracle's flags (-O3 -ffp-contract=off).
#include <map>

#include "rescue_oracle.cpp"

namespace {

// The refinement of the successful match (u, v) of `patch` (B x B) in the width x height `image`: returns whether it
// is refined, with z = (u + du, v + dv) when it is.
bool subpixel_refine(const uint8_t *image, int width, int height, const uint8_t *patch, int B, int u, int v,
                     double z[2]) {
  const int half = (B - 1) / 2;
  if (u - 1 - half < 0 || u + 1 + half > width - 1 || v - 1 - half < 0 || v + 1 + half > height - 1) return false;
  double c[3][3];
  for (int a = -1; a <= 1; ++a)
    for (int b = -1; b <= 1; ++b) {
      double sd0, sd1;
      c[a + 1][b + 1] = correlate2_warning(0, 0, B, B, u + a - half, v + b - half, patch, B, image, width, &sd0, &sd1);
      if (sd1 < kCorrelationSigmaThreshold) return false;
    }
  const double gu = (c[2][1] - c[0][1]) * 0.5, gv = (c[1][2] - c[1][0]) * 0.5;
  const double huu = (c[2][1] + c[0][1]) - 2.0 * c[1][1], hvv = (c[1][2] + c[1][0]) - 2.0 * c[1][1];
  const double huv = ((c[2][2] - c[2][0]) - (c[0][2] - c[0][0])) * 0.25;
  const double det = huu * hvv - huv * huv;
  if (!(huu > 0.0 && det > 0.0)) return false;
  const double du = (huv * gv - hvv * gu) / det, dv = (huv * gu - huu * gv) / det;
  if (!(du >= -0.5 && du <= 0.5 && dv >= -0.5 && dv <= 0.5)) return false;
  z[0] = (double)u + du;
  z[1] = (double)v + dv;
  return true;
}

}  // namespace

// The rescue oracle's Slam with the refinement between the measurement and the consensus.  `refined` holds, per label,
// whether the feature's last match was refined (flags bit 3 on the device): every selected feature's entry is
// rewritten each step, the others keep theirs.
struct sub_slam : resc_slam {
  std::map<int, bool> refined;
  explicit sub_slam(const SlamConfig &c) : resc_slam(c) {}

  void refine(const uint8_t *frame) {
    for (Feature *f : s.selected_feature_list) {
      bool ok = false;
      if (f->successful_measurement_flag) {
        double z[2];
        ok = subpixel_refine(frame, s.cfg.width, s.cfg.height, f->patch.data(), s.cfg.boxsize, (int)f->z[0],
                             (int)f->z[1], z);
        if (ok) {
          f->z[0] = z[0];
          f->z[1] = z[1];
          f->nu[0] = f->z[0] - f->h[0];
          f->nu[1] = f->z[1] - f->h[1];
        }
      }
      refined[f->label] = ok;
    }
  }

  // resc_slam::step with refine() after make_measurements
  void step(const uint8_t *frame) {
    const double u[3] = {0.0, 0.0, 0.0};
    s.kalman_predict(u);
    s.number_of_visible_features = s.auto_select_n_features(s.cfg.number_of_features_to_select);
    rescued.clear();
    if (!s.selected_feature_list.empty()) {
      s.make_measurements(frame);
      refine(frame);
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

// the refinement of one match: returns 1 and writes z when it is refined
int32_t sub_refine(const uint8_t *image, int32_t width, int32_t height, const uint8_t *patch, int32_t B, int32_t u,
                   int32_t v, double *z) {
  return subpixel_refine(image, width, height, patch, B, u, v, z) ? 1 : 0;
}

sub_slam *sub_slam_create(const orc_config *c) {
  cons_slam *b = cons_slam_create(c);
  sub_slam *r = new sub_slam(b->s.cfg);
  delete b;
  return r;
}
void sub_slam_destroy(sub_slam *s) { delete s; }
void sub_slam_set(sub_slam *s, double tau, double chi2) {
  s->tau = tau;
  s->chi2 = chi2;
}
cons_slam *sub_slam_base(sub_slam *s) { return s; }
void sub_slam_step(sub_slam *s, const uint8_t *frame) { s->step(frame); }
// flags bit 3 of every feature in map order
void sub_slam_refined(const sub_slam *s, uint8_t *out) {
  const auto &fl = s->s.feature_list;
  for (size_t i = 0; i < fl.size(); ++i) {
    const auto it = s->refined.find(fl[i]->label);
    out[i] = (it != s->refined.end() && it->second) ? 1 : 0;
  }
}

}  // extern "C"
