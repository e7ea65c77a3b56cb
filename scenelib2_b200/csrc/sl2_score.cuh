// sl2_score.cuh — the correlation score of improc/improc.cpp:99-133 from the exact integer sums, shared by
// search.cu (elliptical search) and smoe.cu (score map of overlapping ellipses).  Each translation unit gets
// its own copy (anonymous namespace).
#pragma once
#include "sl2_common.cuh"

namespace {

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

// template sums -> constants (the same operations, in the same order, as the prologue of search_kernel)
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

}  // namespace
