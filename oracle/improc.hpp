// ORACLE — TEST INFRASTRUCTURE ONLY (see dense.hpp header).
//
// CPU restatement of the SceneLib2 patch-correlation search:
//   A1  correlate2_warning                  scenelib2/improc/improc.cpp:55-134
//   A2  MonoSLAM::elliptical_search         scenelib2/monoslam.cpp:401-477
//   A3  MonoSLAM::measure_feature (S->PuInv) scenelib2/monoslam.cpp:368-386
//   A11 SearchMultipleOverlappingEllipses   scenelib2/improc/
//                                            search_multiple_overlapping_ellipses.cpp:41-196
// Images are raw row-major u8 with an explicit width (the reference reads cv::Mat::data
// with stride = size().width, improc.cpp:66-67,81-82).
//
// Pinning: A1 and A11 are checked bit-for-bit against the reference's OWN source files
// compiled unmodified into oracle/_ref/libsl2ref.so (storage-only cv::Mat / Eigen stubs, see
// oracle/Makefile and tests/test_oracle_ref.py).  A2/A3 live in monoslam.cpp; they are pinned
// through the reference's own monoslam.cpp compiled against oracle/stubs_arith
// (_ref/libsl2refmodels.so): identical match positions on every frame of the whole-step tests and
// of the 1 000-step trajectory, and S -> PuInv against Particle::set_S (same operation sequence) to
// 4e-15 (closed form per SURVEY.md 8(c): l11 = sqrt(s11), l21 = s21/l11, l22 = sqrt(s22 - l21^2),
// inverse by forward substitution, Sinv = Linv^T * Linv; last-ulp differences to the stand-in's
// Gauss-Jordan inverse / to real Eigen remain unpinned).
#pragma once
#include <cstdint>

#include "dense.hpp"

namespace sl2o {

static const double kNoSigma = 3.0;                     // monoslam.cpp:48, smoe.h:55
static const double kCorrThresh2 = 0.40;                // monoslam.cpp:48, smoe.h:50
static const double kCorrelationSigmaThreshold = 10.0;  // monoslam.cpp:49, smoe.h:53
static const double kLowSigmaPenalty = 5.0;             // smoe.h:57

// A1. improc.cpp:55-134.  Note the loop bounds run x0lim / y0lim iterations (not lim-start),
// exactly like the reference (:84-85); all callers pass x0 = y0 = 0.
inline double correlate2_warning(int x0, int y0, int x0lim, int y0lim, int x1, int y1,
                                 const uint8_t *p0, int p0width, const uint8_t *p1, int p1width,
                                 double *sd0ptr, double *sd1ptr) {
  const int patchwidth = x0lim - x0;
  const int p0skip = p0width - patchwidth;
  const int p1skip = p1width - patchwidth;
  int Sg0 = 0, Sg1 = 0, Sg0g1 = 0, Sg0sq = 0, Sg1sq = 0;
  const double n = (x0lim - x0) * (y0lim - y0);

  const uint8_t *a = p0 + p0width * y0 + x0;
  const uint8_t *b = p1 + p1width * y1 + x1;
  for (int yy = y0lim - 1; yy >= 0; --yy) {
    for (int xx = x0lim - 1; xx >= 0; --xx) {
      const int g0 = *a, g1 = *b;
      Sg0 += g0;
      Sg1 += g1;
      Sg0g1 += g0 * g1;
      Sg0sq += g0 * g0;
      Sg1sq += g1 * g1;
      ++a;
      ++b;
    }
    a += p0skip;
    b += p1skip;
  }
  const double Sg0d = Sg0, Sg1d = Sg1, Sg0g1d = Sg0g1, Sg0sqd = Sg0sq, Sg1sqd = Sg1sq;
  const double g0bar = Sg0d / n;
  const double g1bar = Sg1d / n;
  const double varg0 = Sg0sqd / n - (g0bar * g0bar);
  const double varg1 = Sg1sqd / n - (g1bar * g1bar);
  const double sigmag0 = std::sqrt(varg0);
  const double sigmag1 = std::sqrt(varg1);
  *sd0ptr = sigmag0;
  *sd1ptr = sigmag1;
  if (sigmag0 == 0.0) {
    if (sigmag1 == 0.0) return 0.0;
    return 1.0;
  }
  if (sigmag1 == 0.0) return 1.0;
  const double k = g0bar / sigmag0 - g1bar / sigmag1;
  const double C = Sg0sqd / varg0 + Sg1sqd / varg1 + n * (k * k) -
                   Sg0g1d * 2.0 / (sigmag0 * sigmag1) - Sg0d * 2.0 * k / sigmag0 +
                   Sg1d * 2.0 * k / sigmag1;
  return C / n;
}

// A3. monoslam.cpp:371-374 : S (2x2, col-major s[4]) -> Sinv = Linv^T Linv, as (P00,P01,P10,P11).
inline void puinv_from_S(const double S[4], double PuInv[4]) {
  const double s00 = S[0], s10 = S[1], s11 = S[3];
  const double l00 = std::sqrt(s00);
  const double l10 = s10 / l00;
  const double l11 = std::sqrt(s11 - l10 * l10);
  const double x00 = 1.0 / l00;
  const double x10 = (0.0 - l10 * x00) / l11;
  const double x11 = 1.0 / l11;
  PuInv[0] = x00 * x00 + x10 * x10;  // (0,0)
  PuInv[1] = x10 * x11;              // (1,0)
  PuInv[2] = x10 * x11;              // (0,1)
  PuInv[3] = x11 * x11;              // (1,1)
}

// A2. monoslam.cpp:401-477.  PuInv is given as (P00, P01, P11).  Returns true on success;
// *u,*v are only written when a candidate is accepted (quirk Q6); *best is the final corrmax.
inline bool elliptical_search(const uint8_t *image, int width, int height, const uint8_t *patch,
                              const double centre[2], double P00, double P01, double P11, int *u,
                              int *v, int BOXSIZE, double *best = nullptr) {
  const int halfwidth = (int)(kNoSigma / std::sqrt(P00 - P01 * P01 / P11));
  const int halfheight = (int)(kNoSigma / std::sqrt(P11 - P01 * P01 / P00));
  const int ucentre = int(centre[0] + 0.5);
  const int vcentre = int(centre[1] + 0.5);
  int urelstart = -halfwidth, urelfinish = halfwidth;
  int vrelstart = -halfheight, vrelfinish = halfheight;
  if (ucentre + urelstart - (BOXSIZE - 1) / 2 < 0) urelstart = (BOXSIZE - 1) / 2 - ucentre;
  if (ucentre + urelfinish - (BOXSIZE - 1) / 2 > width - BOXSIZE)
    urelfinish = width - BOXSIZE - ucentre + (BOXSIZE - 1) / 2;
  if (vcentre + vrelstart - (BOXSIZE - 1) / 2 < 0) vrelstart = (BOXSIZE - 1) / 2 - vcentre;
  if (vcentre + vrelfinish - (BOXSIZE - 1) / 2 > height - BOXSIZE)
    vrelfinish = height - BOXSIZE - vcentre + (BOXSIZE - 1) / 2;

  double corrmax = 1000000.0;
  double sdpatch, sdimage;
  for (int urel = urelstart; urel <= urelfinish; ++urel) {
    for (int vrel = vrelstart; vrel <= vrelfinish; ++vrel) {
      if (P00 * urel * urel + 2 * P01 * urel * vrel + P11 * vrel * vrel < kNoSigma * kNoSigma) {
        const double corr = correlate2_warning(
            0, 0, BOXSIZE, BOXSIZE, ucentre + urel - (BOXSIZE - 1) / 2,
            vcentre + vrel - (BOXSIZE - 1) / 2, patch, BOXSIZE, image, width, &sdpatch, &sdimage);
        if (corr <= corrmax) {
          if (sdpatch < kCorrelationSigmaThreshold) {
          } else if (sdimage < kCorrelationSigmaThreshold) {
          } else {
            corrmax = corr;
            *u = urel + ucentre;
            *v = vrel + vcentre;
          }
        }
      }
    }
  }
  if (best) *best = corrmax;
  return !(corrmax > kCorrThresh2);
}

// A11. search_multiple_overlapping_ellipses.cpp:41-48,86-90,106-196.
// K ellipses, one template; PuInv[k] = (P00,P01,P11); results per ellipse.
// Differences from A2 that are reproduced on purpose: centre truncated not rounded (:125-126,
// quirk Q4); low image sigma adds a 5.0 penalty that is cached (:173-177); patch sigma is not
// checked; halfwidth_/halfheight_ are stored as int (smoe.h:110-112).
inline void smoe_search(const uint8_t *image, int width, int height, const uint8_t *patch,
                        int BOXSIZE, int K, const double *PuInv3, const double *centres,
                        int *res_u, int *res_v, uint8_t *res_flag, double *res_best = nullptr) {
  std::vector<double> cache((size_t)width * height, -1.0);
  for (int e = 0; e < K; ++e) {
    const double P00 = PuInv3[3 * e + 0], P01 = PuInv3[3 * e + 1], P11 = PuInv3[3 * e + 2];
    const int halfwidth = (int)(kNoSigma / std::sqrt(P00 - P01 * P01 / P11));
    const int halfheight = (int)(kNoSigma / std::sqrt(P11 - P01 * P01 / P00));
    int urelstart = -halfwidth, urelfinish = halfwidth;
    int vrelstart = -halfheight, vrelfinish = halfheight;
    const int ucentre = int(centres[2 * e + 0]);
    const int vcentre = int(centres[2 * e + 1]);
    if (ucentre + urelstart - (BOXSIZE - 1) / 2 < 0) urelstart = (BOXSIZE - 1) / 2 - ucentre;
    if (ucentre + urelfinish - (BOXSIZE - 1) / 2 > width - BOXSIZE)
      urelfinish = width - BOXSIZE - ucentre + (BOXSIZE - 1) / 2;
    if (vcentre + vrelstart - (BOXSIZE - 1) / 2 < 0) vrelstart = (BOXSIZE - 1) / 2 - vcentre;
    if (vcentre + vrelfinish - (BOXSIZE - 1) / 2 > height - BOXSIZE)
      vrelfinish = height - BOXSIZE - vcentre + (BOXSIZE - 1) / 2;
    double corrmax = 1000000.0;
    double sdpatch, sdimage;
    int ru = 0, rv = 0;  // SearchDatum ctor initialises result_u_/v_ to 0 (:43-44)
    for (int urel = urelstart; urel <= urelfinish; ++urel) {
      for (int vrel = vrelstart; vrel <= vrelfinish; ++vrel) {
        if (P00 * urel * urel + 2 * P01 * urel * vrel + P11 * vrel * vrel < kNoSigma * kNoSigma) {
          double corr;
          double &slot = cache[(size_t)(vcentre + vrel) * width + (ucentre + urel)];
          if (slot != -1.0) {
            corr = slot;
          } else {
            corr = correlate2_warning(0, 0, BOXSIZE, BOXSIZE, ucentre + urel - (BOXSIZE - 1) / 2,
                                      vcentre + vrel - (BOXSIZE - 1) / 2, patch, BOXSIZE, image,
                                      width, &sdpatch, &sdimage);
            if (sdimage < kCorrelationSigmaThreshold) corr += kLowSigmaPenalty;
            slot = corr;
          }
          if (corr <= corrmax) {
            corrmax = corr;
            ru = urel + ucentre;
            rv = vrel + vcentre;
          }
        }
      }
    }
    res_u[e] = ru;
    res_v[e] = rv;
    res_flag[e] = (corrmax > kCorrThresh2) ? 0 : 1;
    if (res_best) res_best[e] = corrmax;
  }
}

// N3. MonoSLAM::find_eigenvalues, monoslam.cpp:1196-1205
inline void find_eigenvalues(double A, double B, double C, double *eval1ptr, double *eval2ptr) {
  const double BB = std::sqrt((A + C) * (A + C) - 4 * (A * C - B * B));
  *eval1ptr = (A + C + BB) / 2.0;
  *eval2ptr = (A + C - BB) / 2.0;
}

// N3. MonoSLAM::find_best_patch_inside_region, monoslam.cpp:1070-1194 (Shi-Tomasi criterion with
// running column sums).  *ubest / *vbest are only written when a position beats evbest = 0, like
// the reference (they keep the caller's values otherwise), except in the empty-region early return.
inline void find_best_patch_inside_region(const uint8_t *image, int width, int height, int *ubest,
                                          int *vbest, double *evbest, const int BOXSIZE, int ustart,
                                          int vstart, int ufinish, int vfinish) {
  if (ustart < (BOXSIZE - 1) / 2 + 1) ustart = (BOXSIZE - 1) / 2 + 1;
  if (ufinish > width - (BOXSIZE - 1) / 2 - 1) ufinish = width - (BOXSIZE - 1) / 2 - 1;
  if (vstart < (BOXSIZE - 1) / 2 + 1) vstart = (BOXSIZE - 1) / 2 + 1;
  if (vfinish > height - (BOXSIZE - 1) / 2 - 1) vfinish = height - (BOXSIZE - 1) / 2 - 1;
  if (vstart >= vfinish || ustart >= ufinish) {
    *ubest = ustart;
    *vbest = vstart;
    *evbest = 0;
    return;
  }
  auto px = [&](int r, int c) { return (int)image[(size_t)r * width + c]; };
  const int calc_width = ufinish - ustart + BOXSIZE - 1;
  std::vector<double> CSgxsq(calc_width), CSgysq(calc_width), CSgxgy(calc_width);
  double TSgxsq = 0.0, TSgysq = 0.0, TSgxgy = 0.0;
  double gx, gy, eval1, eval2;
  const int cstart = ustart - (BOXSIZE - 1) / 2;
  const int cfinish = ufinish + (BOXSIZE - 1) / 2;
  const int rstart = vstart - (BOXSIZE - 1) / 2;
  int i, c, r;
  for (c = cstart, i = 0; c < cfinish; ++c, ++i) {
    CSgxsq[i] = 0;
    CSgysq[i] = 0;
    CSgxgy[i] = 0;
    for (r = rstart; r < rstart + BOXSIZE; ++r) {
      gx = (px(r, c + 1) - px(r, c - 1)) / 2.0;
      gy = (px(r + 1, c) - px(r - 1, c)) / 2.0;
      CSgxsq[i] += gx * gx;
      CSgysq[i] += gy * gy;
      CSgxgy[i] += gx * gy;
    }
  }
  *evbest = 0;
  for (int v = vstart; v < vfinish; ++v) {
    TSgxsq = 0.0, TSgysq = 0.0, TSgxgy = 0.0;
    for (i = 0; i < BOXSIZE; ++i) {
      TSgxsq += CSgxsq[i];
      TSgysq += CSgysq[i];
      TSgxgy += CSgxgy[i];
    }
    for (int u = ustart; u < ufinish; ++u) {
      if (u != ustart) {
        TSgxsq += CSgxsq[u - ustart + BOXSIZE - 1] - CSgxsq[u - ustart - 1];
        TSgysq += CSgysq[u - ustart + BOXSIZE - 1] - CSgysq[u - ustart - 1];
        TSgxgy += CSgxgy[u - ustart + BOXSIZE - 1] - CSgxgy[u - ustart - 1];
      }
      find_eigenvalues(TSgxsq, TSgxgy, TSgysq, &eval1, &eval2);
      if (eval2 > *evbest) {
        *ubest = u;
        *vbest = v;
        *evbest = eval2;
      }
    }
    if (v != vfinish - 1) {
      for (c = cstart, i = 0; c < cfinish; ++c, ++i) {
        gx = (px(v - (BOXSIZE - 1) / 2, c + 1) - px(v - (BOXSIZE - 1) / 2, c - 1)) / 2.0;
        gy = (px(v - (BOXSIZE - 1) / 2 + 1, c) - px(v - (BOXSIZE - 1) / 2 - 1, c)) / 2.0;
        CSgxsq[i] -= gx * gx;
        CSgysq[i] -= gy * gy;
        CSgxgy[i] -= gx * gy;
        gx = (px(v + (BOXSIZE - 1) / 2 + 1, c + 1) - px(v + (BOXSIZE - 1) / 2 + 1, c - 1)) / 2.0;
        gy = (px(v + (BOXSIZE - 1) / 2 + 1 + 1, c) - px(v + (BOXSIZE - 1) / 2 + 1 - 1, c)) / 2.0;
        CSgxsq[i] += gx * gx;
        CSgysq[i] += gy * gy;
        CSgxgy[i] += gx * gy;
      }
    }
  }
}

}  // namespace sl2o
