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
// Entry points: sl2_smoe_search*, sl2_measure_particles* and sl2_measure_partial_features, each one staged call
// (partial_features) of [particle prediction ->] both SMOE kernels [-> re-weighting, particles.cu].
#include <algorithm>

#include "sl2_context.cuh"
#include "sl2_score.cuh"

using namespace sl2;

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

// ---- partially-initialised features: F features x Kmax particle slots in one pass ------------------------------
// One H2D of everything, [particle_predict] -> smoe map -> smoe argmin -> [reweight], one D2H.
//   feat_index / patches : templates, either map features or raw BOX x BOX templates (scratch slots behind the map)
//   ypi != NULL          : predict h / Sinv3 / detS on the device (they are outputs), else they are inputs
//   prob != NULL         : run the re-weighting (lambda, prob, prune threshold), else search only
struct PartialIO {
  int F, Kmax;
  const int32_t *K;
  const int32_t *feat_index;
  const uint8_t *patches;
  const double *ypi, *Pxy, *Pyy;
  double *h, *Sinv3, *detS;
  const double *lambda;
  double prune;
  double *prob;
  int32_t *z_uv;
  uint8_t *found, *keep;
  double *cumulative, *mean_var;
  int32_t *left;
};

int partial_features(sl2_ctx *c, int32_t s, int32_t slot, const PartialIO &io, const char *who) {
  const Sl2Dev &d = c->d;
  const int F = io.F, Kmax = io.Kmax;
  const bool predict = io.ypi != nullptr, reweight = io.prob != nullptr;
  if (bad_stream(c, s) || bad_slot(c, slot) || F < 0 || F > SL2_MAX_PARTIAL || Kmax < 0 ||
      Kmax > SL2_MAX_PARTICLES || (F && Kmax && (!io.K || (!io.feat_index && !io.patches) || !io.h || !io.Sinv3)) ||
      (predict && (!io.Pxy || !io.Pyy || !io.lambda || !io.detS)) || (reweight && (!io.lambda || !io.detS)))
    return fail(c, SL2_ERR_ARG, std::string(who) + ": bad argument");
  if (F == 0 || Kmax == 0) return SL2_OK;
  for (int f = 0; f < F; ++f)
    if (io.K[f] < 0 || io.K[f] > Kmax) return fail(c, SL2_ERR_ARG, std::string(who) + ": particle count out of range");
  if (io.feat_index) {
    const int rc = check_feature_indices(c, s, io.feat_index, F, std::string(who) + ": feature index out of range");
    if (rc) return rc;
  }
  const int grown = grow_scratch(c, sl2_smoe_map_bytes(d, F), c->smoe_map_bytes, c->smoe_map);
  if (grown) return grown;
  // h / Sinv3 / detS: outputs of the prediction, else inputs; prob: rewritten by the re-weighting
  const size_t n = (size_t)F * Kmax, nF = F;
  Stage K{STAGE_IN, 4 * nF, io.K}, ft{STAGE_IN, 4 * nF}, ypi{STAGE_IN, 48 * nF, io.ypi},
      Pxy{STAGE_IN, 8 * 78 * nF, io.Pxy}, Pyy{STAGE_IN, 8 * 36 * nF, io.Pyy}, lam{STAGE_IN, 8 * n, io.lambda},
      tpl{STAGE_IN, nF * d.box * 16}, prob{STAGE_INOUT, 8 * n, io.prob},
      h{STAGE_INOUT, 16 * n, predict ? nullptr : io.h}, Sinv3{STAGE_INOUT, 24 * n, predict ? nullptr : io.Sinv3},
      detS{STAGE_INOUT, 8 * n, predict ? nullptr : io.detS}, cum{STAGE_OUT, 8 * n}, mv{STAGE_OUT, 16 * nF},
      uv{STAGE_OUT, 8 * n}, left{STAGE_OUT, 4 * nF}, found{STAGE_OUT, n}, keep{STAGE_OUT, n};
  auto pack = [&] {
    for (int f = 0; f < F; ++f) ft.host<int>()[f] = io.feat_index ? io.feat_index[f] : (d.B - s) * d.Nmax + f;
    if (io.patches) pack_patch_rows(tpl.h, io.patches, F, d.box);
  };
  const int rc = staged_call(
      c, {&K, &ft, &ypi, &Pxy, &Pyy, &lam, &tpl, &prob, &h, &Sinv3, &detS, &cum, &mv, &uv, &left, &found, &keep}, pack,
      [&] {
        if (io.patches)  // raw templates -> the scratch slots behind the map templates
          CU_TRY(c, cudaMemcpyAsync(d.patches + (size_t)d.B * d.Nmax * d.box * 16, tpl.d, tpl.bytes,
                                    cudaMemcpyDeviceToDevice, c->stream));
        if (predict)
          CU_TRY(c, sl2_launch_particle_predict(d, s, F, Kmax, K.dev<int>(), ypi.dev<double>(), Pxy.dev<double>(),
                                                Pyy.dev<double>(), lam.dev<double>(), h.dev<double>(),
                                                Sinv3.dev<double>(), detS.dev<double>(), queue(c)));
        // measure_feature_with_multiple_priors (monoslam.cpp:1408-1438): ellipses (SInv_k, h_k), one template per feature
        CU_TRY(c, sl2_launch_smoe(d, s, slot, F, Kmax, K.dev<int>(), ft.dev<int>(), h.dev<double>(), Sinv3.dev<double>(),
                                  c->smoe_map.get(), uv.dev<int>(), found.d, nullptr, queue(c)));
        if (reweight)
          CU_TRY(c, sl2_launch_particles(F, Kmax, K.dev<int>(), h.dev<double>(), Sinv3.dev<double>(),
                                         detS.dev<double>(), lam.dev<double>(), uv.dev<int>(), found.d, io.prune,
                                         prob.dev<double>(), keep.d, cum.dev<double>(), mv.dev<double>(),
                                         left.dev<int>(), queue(c)));
        return SL2_OK;
      });
  if (rc) return rc;
  // Per-particle outputs: feature f's first K[f] slots are this call's results; slots k >= K[f] of the caller's
  // arrays are left as they were (the kernels never write them, so the staging buffer holds whatever an earlier call
  // left there, or zeros).
  auto particles_out = [&](void *dst, const Stage &src, size_t per_particle) {
    if (!dst) return;
    for (int f = 0; f < F; ++f) {
      const size_t o = (size_t)f * Kmax * per_particle;
      memcpy(static_cast<uint8_t *>(dst) + o, src.h + o, (size_t)io.K[f] * per_particle);
    }
  };
  if (predict) {
    particles_out(io.h, h, 16);
    particles_out(io.Sinv3, Sinv3, 24);
    particles_out(io.detS, detS, 8);
  }
  if (reweight) {
    particles_out(io.prob, prob, 8);
    particles_out(io.cumulative, cum, 8);
    particles_out(io.keep, keep, 1);
    if (io.mean_var) memcpy(io.mean_var, mv.h, mv.bytes);
    if (io.left) memcpy(io.left, left.h, left.bytes);
  }
  particles_out(io.z_uv, uv, 8);
  particles_out(io.found, found, 1);
  return SL2_OK;
}

int smoe_one(sl2_ctx *c, int32_t s, int32_t slot, const int32_t *feat_index, const uint8_t *patch, int32_t K,
             const double *PuInv3, const double *centres, int32_t *res_u, int32_t *res_v, uint8_t *res_flag,
             const char *who) {
  if (K < 0 || (K && (!PuInv3 || !centres))) return fail(c, SL2_ERR_ARG, std::string(who) + ": bad argument");
  if (K == 0) return SL2_OK;
  if (K > SL2_MAX_PARTICLES) return fail(c, SL2_ERR_ARG, std::string(who) + ": more than SL2_MAX_PARTICLES ellipses");
  std::vector<int32_t> uv(2 * (size_t)K);
  PartialIO io = {};
  io.F = 1, io.Kmax = K, io.K = &K;
  io.feat_index = feat_index, io.patches = patch;
  io.h = const_cast<double *>(centres), io.Sinv3 = const_cast<double *>(PuInv3);  // inputs (no prediction)
  io.z_uv = uv.data(), io.found = res_flag;
  const int rc = partial_features(c, s, slot, io, who);
  if (rc) return rc;
  for (int i = 0; i < K; ++i) {
    if (res_u) res_u[i] = uv[2 * i];
    if (res_v) res_v[i] = uv[2 * i + 1];
  }
  return SL2_OK;
}

int measure_particles(sl2_ctx *c, int32_t s, int32_t slot, const int32_t *feat_index, const uint8_t *patch,
                      int32_t K, const double *h, const double *Sinv3, const double *detS, const double *lambda,
                      double prune_probability_threshold, double *prob, int32_t *z_uv, uint8_t *found,
                      uint8_t *keep, double *cumulative, double *mean_var) {
  if (K < 0 || (K && (!h || !Sinv3 || !detS || !lambda || !prob)))
    return fail(c, SL2_ERR_ARG, "sl2_measure_particles: bad argument");
  if (K == 0) return 0;
  if (K > SL2_MAX_PARTICLES) return fail(c, SL2_ERR_ARG, "sl2_measure_particles: more than SL2_MAX_PARTICLES particles");
  int32_t left = 0;
  PartialIO io = {};
  io.F = 1, io.Kmax = K, io.K = &K;
  io.feat_index = feat_index, io.patches = patch;
  io.h = const_cast<double *>(h), io.Sinv3 = const_cast<double *>(Sinv3), io.detS = const_cast<double *>(detS);
  io.lambda = lambda, io.prune = prune_probability_threshold, io.prob = prob;
  io.z_uv = z_uv, io.found = found, io.keep = keep, io.cumulative = cumulative, io.mean_var = mean_var;
  io.left = &left;
  const int rc = partial_features(c, s, slot, io, "sl2_measure_particles");
  return rc ? rc : left;
}

}  // namespace

extern "C" {

int sl2_smoe_search(sl2_ctx *c, int32_t s, int32_t slot, int32_t feat_index, int32_t K,
                    const double *PuInv3, const double *centres, int32_t *res_u, int32_t *res_v,
                    uint8_t *res_flag) {
  return smoe_one(c, s, slot, &feat_index, nullptr, K, PuInv3, centres, res_u, res_v, res_flag, "sl2_smoe_search");
}

int sl2_smoe_search_patch(sl2_ctx *c, int32_t s, int32_t slot, const uint8_t *patch, int32_t K,
                          const double *PuInv3, const double *centres, int32_t *res_u, int32_t *res_v,
                          uint8_t *res_flag) {
  if (!patch) return fail(c, SL2_ERR_ARG, "sl2_smoe_search_patch: patch is null");
  return smoe_one(c, s, slot, nullptr, patch, K, PuInv3, centres, res_u, res_v, res_flag, "sl2_smoe_search_patch");
}

int sl2_measure_particles(sl2_ctx *c, int32_t s, int32_t slot, int32_t feat_index, int32_t K,
                          const double *h, const double *Sinv3, const double *detS, const double *lambda,
                          double prune_probability_threshold, double *prob, int32_t *z_uv, uint8_t *found,
                          uint8_t *keep, double *cumulative, double *mean_var) {
  return measure_particles(c, s, slot, &feat_index, nullptr, K, h, Sinv3, detS, lambda,
                           prune_probability_threshold, prob, z_uv, found, keep, cumulative, mean_var);
}

int sl2_measure_particles_patch(sl2_ctx *c, int32_t s, int32_t slot, const uint8_t *patch, int32_t K,
                                const double *h, const double *Sinv3, const double *detS, const double *lambda,
                                double prune_probability_threshold, double *prob, int32_t *z_uv,
                                uint8_t *found, uint8_t *keep, double *cumulative, double *mean_var) {
  if (!patch) return fail(c, SL2_ERR_ARG, "sl2_measure_particles_patch: patch is null");
  return measure_particles(c, s, slot, nullptr, patch, K, h, Sinv3, detS, lambda, prune_probability_threshold,
                           prob, z_uv, found, keep, cumulative, mean_var);
}

int sl2_measure_partial_features(sl2_ctx *c, int32_t s, int32_t slot, int32_t F, int32_t Kmax, const int32_t *K,
                                 const uint8_t *patches, const double *ypi, const double *Pxy, const double *Pyy,
                                 const double *lambda, double prune_probability_threshold, double *prob,
                                 double *h, double *Sinv3, double *detS, int32_t *z_uv, uint8_t *found,
                                 uint8_t *keep, double *cumulative, double *mean_var, int32_t *left) {
  if (F > 0 && Kmax > 0 && (!patches || !ypi || !prob))
    return fail(c, SL2_ERR_ARG, "sl2_measure_partial_features: bad argument");
  // h / Sinv3 / detS are outputs the caller may not want: they still travel through the staging buffer
  std::vector<double> th, ts, td;
  const size_t n = (size_t)std::max(F, 0) * std::max(Kmax, 0);
  if (!h) th.resize(2 * n), h = th.data();
  if (!Sinv3) ts.resize(3 * n), Sinv3 = ts.data();
  if (!detS) td.resize(n), detS = td.data();
  PartialIO io = {};
  io.F = F, io.Kmax = Kmax, io.K = K;
  io.patches = patches;
  io.ypi = ypi, io.Pxy = Pxy, io.Pyy = Pyy;
  io.h = h, io.Sinv3 = Sinv3, io.detS = detS;
  io.lambda = lambda, io.prune = prune_probability_threshold, io.prob = prob;
  io.z_uv = z_uv, io.found = found, io.keep = keep, io.cumulative = cumulative, io.mean_var = mean_var;
  io.left = left;
  return partial_features(c, s, slot, io, "sl2_measure_partial_features");
}

}  // extern "C"
