// smoe.cu — SearchMultipleOverlappingEllipses::search on sm_90a (SURVEY.md §8 rows A11 / N2).
//
// Replaces improc/search_multiple_overlapping_ellipses.cpp:106-196 for the K ellipses (one per depth particle)
// of each of F partially-initialised features of one frame: the reference evaluates correlate2_warning once per
// image location and caches it in a frame-sized array (:112-114, :160-176), every ellipse then takes the
// arg-min of the cached values inside it.  Here, per feature:
//   smoe_map_kernel     grid = 32x8 tiles of the frame x F.  A tile that no ellipse's box touches exits at once;
//                       otherwise thread = image location: the location is scored if ANY ellipse holds it (the
//                       exact FP64 predicate of SearchDatum::inside_relative, relative to that ellipse's integer
//                       centre), from the tile's pixel window and the template in shared memory, exact int32 sums
//                       and the FP64 chain of improc.cpp:99-133 (+ LOW_SIGMA_PENALTY, :169-171), once.
//   smoe_argmin_kernel  one warp per ellipse: its box in the reference's scan order, the predicate again, the
//                       cached value, `corr <= corrmax` => the LAST minimum in (urel, vrel) order wins.
// The round-1 path ran search_kernel in an "smoe mode" that recomputed the score per ellipse (K = 100 heavily
// overlapping ellipses: up to ~100x redundant work).
#include "sl2_common.cuh"
#include "sl2_score.cuh"

namespace {

constexpr int SM_TW = 32, SM_TH = 8;  // tile of image locations per CTA (thread = location)
constexpr int SM_MAXK = 256;          // ellipses per feature

struct Ell {
  Ellipse ell;
  int uc, vc;     // integer centre: truncated (smoe.cpp:118-147), where the elliptical search rounds
  SearchBox box;  // clamped to the stream's W x H image
};

__device__ __forceinline__ Ell make_ell(int W, int H, int half, const double *centre, const double *puinv) {
  Ell e;
  e.ell = make_ellipse(puinv[0], puinv[1], puinv[2]);
  e.uc = __double2int_rz(centre[0]);
  e.vc = __double2int_rz(centre[1]);
  e.box = search_box(puinv[0], puinv[1], puinv[2], e.uc, e.vc, W, H, half);
  return e;
}

struct SmoeArgs {
  int s, slot, F, Kmax;
  const int *K;          // [F] ellipses of feature f
  const int *feat;       // [F] template index relative to the stream's first template
  const double *centre;  // [F][Kmax][2]
  const double *puinv;   // [F][Kmax][3]
  double *map;           // [F][W][H]  score of location (x, y) at x * H + y
  int *out_uv;           // [F][Kmax][2]
  uint8_t *out_found;    // [F][Kmax]
  double *out_best;      // [F][Kmax] or nullptr
};

template <int BOX>
__global__ void __launch_bounds__(SM_TW *SM_TH) smoe_map_kernel(const Sl2Dev d, const SmoeArgs A) {
  constexpr int HALF = (BOX - 1) / 2;
  constexpr int WW = SM_TW + BOX - 1, WH = SM_TH + BOX - 1;
  __shared__ Ell s_ell[SM_MAXK];
  __shared__ uint8_t s_win[WH][WW + 1];
  __shared__ uint8_t s_tpl[BOX][16];
  __shared__ PatchConst s_pc;
  __shared__ int s_sum[2];
  const int f = blockIdx.y, tid = threadIdx.x;
  const int K = min(A.K[f], SM_MAXK);
  const int tiles_x = (d.W + SM_TW - 1) / SM_TW;
  const int tx0 = (blockIdx.x % tiles_x) * SM_TW, ty0 = (blockIdx.x / tiles_x) * SM_TH;
  const int Ws = stream_width(d.cams[A.s]), Hs = stream_height(d.cams[A.s]);
  // ellipses of this feature; does any box touch the tile?
  int touch = 0;
  for (int k = tid; k < K; k += SM_TW * SM_TH) {
    const size_t j = (size_t)f * A.Kmax + k;
    const Ell e = make_ell(Ws, Hs, HALF, A.centre + j * 2, A.puinv + j * 3);
    s_ell[k] = e;
    if (e.uc + e.box.us < tx0 + SM_TW && e.uc + e.box.uf >= tx0 && e.vc + e.box.vs < ty0 + SM_TH &&
        e.vc + e.box.vf >= ty0)
      touch = 1;
  }
  if (tid < 2) s_sum[tid] = 0;
  if (!__syncthreads_or(touch)) return;
  // this location: inside any ellipse?
  const int X = tx0 + (tid & (SM_TW - 1)), Y = ty0 + tid / SM_TW;
  bool want = false;
  for (int k = 0; k < K && !want; ++k) {
    const int du = X - s_ell[k].uc, dv = Y - s_ell[k].vc;
    const SearchBox &b = s_ell[k].box;
    if (du >= b.us && du <= b.uf && dv >= b.vs && dv <= b.vf) want = s_ell[k].ell.inside(du, dv);
  }
  if (!__syncthreads_or(want)) return;
  // pixel window of the tile's boxes (inside the stream's image: the clamped pixels feed no box) and the template
  const uint8_t *img = d.frames + ((size_t)A.slot * d.B + A.s) * d.H * d.pitch;
  for (int e = tid; e < WH * WW; e += SM_TW * SM_TH) {
    const int r = e / WW, c = e - r * WW;
    const int y = min(max(ty0 - HALF + r, 0), Hs - 1), x = min(max(tx0 - HALF + c, 0), Ws - 1);
    s_win[r][c] = __ldg(img + (size_t)y * d.pitch + x);
  }
  const uint8_t *tp = d.patches + ((size_t)A.s * d.Nmax + A.feat[f]) * (BOX * 16);
  int t1 = 0, t2 = 0;
  for (int e = tid; e < BOX * 16; e += SM_TW * SM_TH) {
    const uint8_t v = __ldg(tp + e);  // rows are zero padded to 16 bytes: the padding adds nothing to the sums
    s_tpl[e >> 4][e & 15] = v;
    t1 += v;
    t2 += (int)v * v;
  }
  if (tid < BOX * 16) {
    atomicAdd(&s_sum[0], t1);
    atomicAdd(&s_sum[1], t2);
  }
  __syncthreads();
  if (tid == 0) s_pc = patch_const(BOX, s_sum[0], s_sum[1]);
  __syncthreads();
  if (!want) return;
  int S1 = 0, S2 = 0, S01 = 0;
  const int lx = tid & (SM_TW - 1), ly = tid / SM_TW;
#pragma unroll 1
  for (int r = 0; r < BOX; ++r) {
#pragma unroll
    for (int c = 0; c < BOX; ++c) {
      const int g1 = s_win[ly + r][lx + c], g0 = s_tpl[r][c];
      S1 += g1;
      S2 += g1 * g1;
      S01 += g0 * g1;
    }
  }
  double sg1;
  double corr = exact_score_fn(s_pc, (double)S1, (double)S2, (double)S01, &sg1);
  if (sg1 < 10.0) corr = add_(corr, 5.0);  // smoe.cpp:169-171
  A.map[((size_t)f * d.W + X) * d.H + Y] = corr;
}

__global__ void __launch_bounds__(128) smoe_argmin_kernel(const Sl2Dev d, const SmoeArgs A, int half) {
  const int f = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k = blockIdx.x * 4 + warp;
  if (k >= A.K[f] || k >= A.Kmax) return;
  const size_t j = (size_t)f * A.Kmax + k;
  const Ell e = make_ell(stream_width(d.cams[A.s]), stream_height(d.cams[A.s]), half, A.centre + j * 2, A.puinv + j * 3);
  const int CW = e.box.cols(), CH = e.box.rows();
  const double *map = A.map + (size_t)f * d.W * d.H;
  ScanBest best;
  if (CW > 0 && CH > 0) {
    for (int idx = lane; idx < CW * CH; idx += 32) {
      const int ui = idx / CH, vi = idx - ui * CH;  // scan index -> box position
      const int du = e.box.us + ui, dv = e.box.vs + vi;
      if (e.ell.inside(du, dv)) best.offer(map[(size_t)(e.uc + du) * d.H + (e.vc + dv)], idx);
    }
  }
  best.warp_reduce();
  if (lane == 0) {
    const int2 uv = best.idx >= 0 ? scan_position(best.idx, CH, e.uc + e.box.us, e.vc + e.box.vs)
                                  : make_int2(0, 0);  // smoe.cpp:43-44 default
    A.out_uv[j * 2 + 0] = uv.x;
    A.out_uv[j * 2 + 1] = uv.y;
    A.out_found[j] = best.found();
    if (A.out_best) A.out_best[j] = best.corr;
  }
}

}  // namespace

size_t sl2_smoe_map_bytes(const Sl2Dev &d, int F) { return (size_t)F * d.W * d.H * sizeof(double); }

// F features x up to Kmax ellipses each (K_dev[f] of them used), templates at feat_dev[f] (relative to the
// stream's first template), all on one frame.  2 launches.
cudaError_t sl2_launch_smoe(const Sl2Dev &d, int s, int slot, int F, int Kmax, const int *K_dev, const int *feat_dev,
                            const double *centre_dev, const double *puinv_dev, double *map_dev, int *out_uv_dev,
                            uint8_t *out_found_dev, double *out_best_dev, Sl2Queue q) {
  if (F <= 0 || Kmax <= 0) return cudaSuccess;
  if (Kmax > SM_MAXK) return cudaErrorInvalidValue;
  SmoeArgs A = {s, slot, F, Kmax, K_dev, feat_dev, centre_dev, puinv_dev, map_dev, out_uv_dev, out_found_dev,
                out_best_dev};
  const int tiles = ((d.W + SM_TW - 1) / SM_TW) * ((d.H + SM_TH - 1) / SM_TH);
  const cudaError_t e = sl2_with_box(d.box, [&](auto box) {
    return sl2_launch_kernel(smoe_map_kernel<decltype(box)::value>, dim3(tiles, F), dim3(SM_TW * SM_TH), 0, q, false,
                             d, A);
  });
  if (e != cudaSuccess) return e;
  return sl2_launch_kernel(smoe_argmin_kernel, dim3((Kmax + 3) / 4, F), dim3(128), 0, q, false, d, A, (d.box - 1) / 2);
}
