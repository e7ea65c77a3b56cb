// ORACLE — TEST INFRASTRUCTURE ONLY.
// extern "C" doorway into the REFERENCE's own improc sources, which oracle/Makefile compiles
// unmodified from the original scenelib2/improc/{improc,search_multiple_overlapping_ellipses}.cpp
// into oracle/_ref/libsl2ref.so against the storage-only stubs in oracle/stubs/.
// Used to pin the oracle's A1 / A11 restatements bit-for-bit (tests/test_oracle_ref.py).
#include <cstdint>

#include "improc/improc.h"
#include "improc/search_multiple_overlapping_ellipses.h"

extern "C" {

double ref_correlate2_warning(const uint8_t *patch, int32_t patch_width, int32_t patch_height,
                              int32_t x0lim, int32_t y0lim, const uint8_t *image,
                              int32_t image_width, int32_t image_height, int32_t x1, int32_t y1,
                              double *sd0, double *sd1) {
  cv::Mat p0(patch_height, patch_width, CV_8UC1, (void *)patch);
  cv::Mat p1(image_height, image_width, CV_8UC1, (void *)image);
  return SceneLib2::correlate2_warning(0, 0, x0lim, y0lim, x1, y1, p0, p1, sd0, sd1);
}

void ref_smoe_search(const uint8_t *image, int32_t width, int32_t height, const uint8_t *patch,
                     int32_t boxsize, int32_t K, const double *PuInv3, const double *centres,
                     int32_t *res_u, int32_t *res_v, uint8_t *res_flag) {
  cv::Mat img(height, width, CV_8UC1, (void *)image);
  cv::Mat pat(boxsize, boxsize, CV_8UC1, (void *)patch);
  SceneLib2::SearchMultipleOverlappingEllipses smoe(img, pat, boxsize);
  for (int k = 0; k < K; ++k) {
    Eigen::Matrix2d P;
    P(0, 0) = PuInv3[3 * k + 0];
    P(0, 1) = PuInv3[3 * k + 1];
    P(1, 0) = PuInv3[3 * k + 1];
    P(1, 1) = PuInv3[3 * k + 2];
    Eigen::Vector2d c;
    c(0) = centres[2 * k + 0];
    c(1) = centres[2 * k + 1];
    smoe.add_ellipse(P, c);
  }
  smoe.search();
  int k = 0;
  for (auto it = smoe.begin(); it != smoe.end(); ++it, ++k) {
    res_u[k] = it->result_u_;
    res_v[k] = it->result_v_;
    res_flag[k] = it->result_flag_ ? 1 : 0;
  }
}

}  // extern "C"
