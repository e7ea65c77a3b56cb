// sl2_score.cuh — the search rules of the reference, stated once for search.cu (MonoSLAM::elliptical_search) and
// smoe.cu (SearchMultipleOverlappingEllipses::search): the template constants and the correlation score of
// improc/improc.cpp:99-133, the search box, the 3-sigma ellipse test, and the scan-order arg-min with its corrmax and
// match threshold.  Each translation unit gets its own copy (anonymous namespace).
#pragma once
#include "sl2_common.cuh"

namespace {

constexpr double CORRMAX = 1000000.0;  // a score above it is never accepted (monoslam.cpp:444, smoe.cpp:150)
constexpr double CORRTHRESH = 0.40;    // the best score matches unless above it (monoslam.cpp:472-476, smoe.cpp:188-193)

// per-template constants of improc.cpp:99-131
struct PatchConst {
  double n, sigmag0, A0, g0s, Sg0x2;
};

// improc.cpp:99-133 op for op (never-fused, IEEE div/sqrt).  Deliberately NOT inlined: the
// filtered kernel reaches it for a handful of candidates per warp, and eight inlined copies of the
// div/sqrt sequences blew the kernel up to ~66 KB of SASS (instruction-cache misses were the top
// stall reason).
__device__ __noinline__ double exact_score_fn(const PatchConst pc, double Sg1d, double Sg1sqd,
                                              double Sg0g1d, double *sigma1_out) {
  const double g1bar = div_(Sg1d, pc.n);
  const double varg1 = sub_(div_(Sg1sqd, pc.n), mul_(g1bar, g1bar));
  const double sigmag1 = sqrt_(varg1);
  *sigma1_out = sigmag1;
  if (pc.sigmag0 == 0.0) return (sigmag1 == 0.0) ? 0.0 : 1.0;
  if (sigmag1 == 0.0) return 1.0;
  const double k = sub_(pc.g0s, div_(g1bar, sigmag1));
  double C = add_(pc.A0, div_(Sg1sqd, varg1));
  C = add_(C, mul_(pc.n, mul_(k, k)));
  C = sub_(C, div_(mul_(Sg0g1d, 2.0), mul_(pc.sigmag0, sigmag1)));
  C = sub_(C, div_(mul_(pc.Sg0x2, k), pc.sigmag0));
  C = add_(C, div_(mul_(mul_(Sg1d, 2.0), k), sigmag1));
  return div_(C, pc.n);
}

// template sums -> constants
__device__ __forceinline__ PatchConst patch_const(int box, int Sg0, int Sg0sq) {
  const double n = (double)(box * box);
  const double Sg0d = (double)Sg0, Sg0sqd = (double)Sg0sq;
  const double g0bar = div_(Sg0d, n);
  const double varg0 = sub_(div_(Sg0sqd, n), mul_(g0bar, g0bar));
  const double sigmag0 = sqrt_(varg0);
  PatchConst pc;
  pc.n = n;
  pc.sigmag0 = sigmag0;
  pc.A0 = div_(Sg0sqd, varg0);
  pc.g0s = div_(g0bar, sigmag0);
  pc.Sg0x2 = mul_(Sg0d, 2.0);
  return pc;
}

// The candidates of a search, relative to its integer centre: the bounding box of the 3-sigma ellipse, clamped so that
// every candidate's window lies inside the stream's W x H image (monoslam.cpp:416-439, smoe.cpp:118-147).
struct SearchBox {
  int us, uf, vs, vf;
  __device__ __forceinline__ int cols() const { return uf - us + 1; }
  __device__ __forceinline__ int rows() const { return vf - vs + 1; }
};
// PuInv = [[P00, P01], [P01, P11]]; the caller rounds (elliptical search) or truncates (SMOE) the centre, as the
// reference does
__device__ __forceinline__ SearchBox search_box(double P00, double P01, double P11, int uc, int vc, int W, int H,
                                                int half) {
  const int halfwidth = __double2int_rz(div_(3.0, sqrt_(sub_(P00, div_(mul_(P01, P01), P11)))));
  const int halfheight = __double2int_rz(div_(3.0, sqrt_(sub_(P11, div_(mul_(P01, P01), P00)))));
  const int box = 2 * half + 1;
  SearchBox b = {-halfwidth, halfwidth, -halfheight, halfheight};
  if (uc + b.us - half < 0) b.us = half - uc;
  if (uc + b.uf - half > W - box) b.uf = W - box - uc + half;
  if (vc + b.vs - half < 0) b.vs = half - vc;
  if (vc + b.vf - half > H - box) b.vf = H - box - vc + half;
  return b;
}

// The 3-sigma test PuInv(0,0) u u + 2 PuInv(0,1) u v + PuInv(1,1) v v < 9 of the candidate (u, v) relative to the
// centre (monoslam.cpp:453-454, SearchDatum::inside_relative), always as ((P00 u) u + (2 P01 u) v) + (P11 v) v.  The
// u terms depend on the column only and the v term on the row only, so a caller may form either once and reuse it.
struct Ellipse {
  double P00, b2, P11;  // PuInv(0,0), 2 PuInv(0,1), PuInv(1,1)
  struct Col {
    double a, b;  // (P00 u) u, (2 P01) u
  };
  __device__ __forceinline__ Col col(double u) const { return {mul_(mul_(P00, u), u), mul_(b2, u)}; }
  __device__ __forceinline__ double vterm(double v) const { return mul_(mul_(P11, v), v); }
  __device__ __forceinline__ bool inside(Col c, double v, double vt) const {  // vt = vterm(v)
    return add_(add_(c.a, mul_(c.b, v)), vt) < 9.0;
  }
  __device__ __forceinline__ bool inside(Col c, double v) const { return inside(c, v, vterm(v)); }
  __device__ __forceinline__ bool inside(int u, int v) const { return inside(col((double)u), (double)v); }
};
__device__ __forceinline__ Ellipse make_ellipse(double P00, double P01, double P11) {
  return {P00, mul_(2.0, P01), P11};
}

// The reference's `corr <= corrmax` scan over a box (monoslam.cpp:457-467, smoe.cpp:178-182) as an order-independent
// arg-min: a smaller score wins, an equal score goes to the later scan index (quirk Q3).
struct ScanBest {
  double corr = CORRMAX;
  int idx = -1;  // scan index of the best candidate, -1: none accepted
  __device__ __forceinline__ void consider(double c, int i) {
    if (c < corr || (c == corr && i > idx)) {
      corr = c;
      idx = i;
    }
  }
  __device__ __forceinline__ void offer(double c, int i) {
    if (c <= CORRMAX) consider(c, i);
  }
  // every lane of the warp ends with the warp's arg-min
  __device__ __forceinline__ void warp_reduce() {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double oc = __shfl_xor_sync(0xffffffffu, corr, o);
      const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
      consider(oc, oi);
    }
  }
  __device__ __forceinline__ uint8_t found() const { return (corr > CORRTHRESH) ? 0 : 1; }
};
// The candidates of a box are visited u major, v minor: scan index idx = (u - us) * rows + (v - vs).  Image position
// of scan index idx, with (u0, v0) = (uc + us, vc + vs) the position of the box's first candidate.
__device__ __forceinline__ int2 scan_position(int idx, int rows, int u0, int v0) {
  return make_int2(u0 + idx / rows, v0 + idx % rows);
}

}  // namespace
