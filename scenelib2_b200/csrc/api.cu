// api.cu — the context and the fused step: create / destroy, the per-stream camera, the map and the state, the staged
// measurement of one stream, the fused step and its two stream groups, timing and the read-back of the map.  The other
// entry points of include/sl2b200.h live beside the kernels they drive; sl2_context.cuh holds what they share.  Host
// side only orchestrates: every arithmetic step runs in the sm_90a kernels.  There is deliberately no CPU fallback.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "../../include/sl2b200.h"
#include "sl2_context.cuh"

using namespace sl2;

namespace {

thread_local std::string g_create_error;

// A step measures at most min(max_features, SL2_MAX_MEASURED) features; below that capacity the selection is bounded
// by the map itself, so only a larger map needs the bound on the selection.
bool selection_fits(int max_features, int n_select) {
  return !(max_features > SL2_MAX_MEASURED && n_select > SL2_MAX_MEASURED);
}

}  // namespace

namespace sl2 {

cudaError_t cuda_event_create(Event &h, unsigned flags) {
  cudaEvent_t ev = nullptr;
  const cudaError_t e = cudaEventCreateWithFlags(&ev, flags);
  if (e == cudaSuccess) h.reset(ev);
  return e;
}
cudaError_t cuda_stream_create(Stream &h) {
  cudaStream_t st = nullptr;
  const cudaError_t e = cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking);
  if (e == cudaSuccess) h.reset(st);
  return e;
}

int fail(sl2_ctx *c, int code, const std::string &msg) {
  if (code == SL2_ERR_CUDA) cudaGetLastError();  // reported once: sl2_launch_update returns the runtime's last error
  if (c) c->err = msg;
  else g_create_error = msg;
  return code;
}

bool bad_stream(sl2_ctx *c, int s) {
  enter(c);
  return !c || s < 0 || s >= c->cfg.num_streams;
}
bool bad_slot(sl2_ctx *c, int s) { return s < 0 || s >= c->cfg.frame_slots; }
bool bad_range(sl2_ctx *c, int lo, int cnt) {
  enter(c);
  return !c || lo < 0 || cnt < 0 || lo > c->cfg.num_streams - cnt;
}

StreamOptions stream_option_defaults() {
  StreamOptions o = {};  // every feature off, SL2_SELECT_TRACE
  for (int i = 0; i < 3; ++i) {  // a rotation and a covariance the gyro and accel setters accept
    o.gyro.R_gc[4 * i] = o.gyro.cov[4 * i] = 1.0;
    o.accel.R_ac[4 * i] = o.accel.cov[4 * i] = 1.0;
  }
  o.accel.sd_a = 4.0;  // the motion model's
  return o;
}

int alloc_sections(sl2_ctx *c, DevPtr<uint8_t> &buf, std::initializer_list<Section> secs) {
  size_t bytes = 0;
  for (const Section &x : secs) bytes += (x.bytes + 255) & ~(size_t)255;
  DevPtr<uint8_t> h;
  CU_TRY(c, cuda_malloc(h, bytes));
  CU_TRY(c, cudaMemsetAsync(h.get(), 0, bytes, c->stream));
  uint8_t *at = h.get();
  for (const Section &x : secs) {
    x.place(x.ptr, at);
    at += (x.bytes + 255) & ~(size_t)255;
  }
  buf = std::move(h);
  return SL2_OK;
}

int read_results(sl2_ctx *c, bool allocated, int lo, int cnt, std::initializer_list<ResultCopy> outs) {
  for (const ResultCopy &r : outs) {
    if (!r.dst) continue;
    if (!allocated) memset(r.dst, 0, r.per_stream * cnt);
    else if (cnt)
      CU_TRY(c, cudaMemcpyAsync(r.dst, static_cast<const uint8_t *>(r.src) + r.per_stream * lo, r.per_stream * cnt,
                                cudaMemcpyDeviceToHost, c->stream));
  }
  if (allocated) CU_TRY(c, cudaStreamSynchronize(c->stream));
  return SL2_OK;
}

int streams_restarted(sl2_ctx *c, int lo, int cnt) {
  int rc = subpixel_forget(c, lo, cnt);
  if (!rc) rc = recovery_reset(c, lo, cnt);
  for (int s = lo; s < lo + cnt && !rc; ++s) rc = normals_reset(c, s, 0, c->d.Nmax);
  return rc;
}

int stage_reserve(sl2_ctx *c, size_t bytes) {
  return grow_scratch(c, (bytes + 4095) & ~(size_t)4095, c->stg_bytes, c->stg_dev, &c->stg_host);
}

void pack_patch_rows(uint8_t *dst, const uint8_t *src, int n, int box) {
  memset(dst, 0, (size_t)n * box * 16);
  for (size_t r = 0; r < (size_t)n * box; ++r) memcpy(dst + r * 16, src + r * box, box);
}

int device_nfeat(sl2_ctx *c, int s, int *out) {
  CU_TRY(c, cudaMemcpyAsync(out, c->d.nfeat + s, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return SL2_OK;
}

int check_feature_indices(sl2_ctx *c, int s, const int32_t *idx, int n, const std::string &msg) {
  int nf = 0;
  const int rc = device_nfeat(c, s, &nf);
  if (rc) return rc;
  for (int i = 0; i < n; ++i)
    if (idx[i] < 0 || idx[i] >= nf) return fail(c, SL2_ERR_ARG, msg);
  return SL2_OK;
}

// the camera values a stream of this context accepts (sl2_set_stream_config and the snapshot loads)
int check_stream_config(sl2_ctx *c, const sl2_stream_config *sc, const std::string &who) {
  const double v[7] = {sc->fku, sc->fkv, sc->u0, sc->v0, sc->kd1, sc->sd, sc->delta_t};
  for (double x : v)
    if (!std::isfinite(x)) return fail(c, SL2_ERR_ARG, who + ": non-finite value");
  if (!(sc->fku > 0.0) || !(sc->fkv > 0.0) || !(sc->delta_t > 0.0))
    return fail(c, SL2_ERR_ARG, who + ": fku, fkv and delta_t must be > 0");
  const int lo = c->cfg.boxsize > 16 ? c->cfg.boxsize : 16;
  if (sc->width < lo || sc->height < lo || sc->width > c->cfg.width || sc->height > c->cfg.height)
    return fail(c, SL2_ERR_ARG, who + ": image size outside [max(16, boxsize), the context's size]");
  if (sc->number_of_features_to_select < 0 ||
      !selection_fits(c->cfg.max_features, sc->number_of_features_to_select))
    return fail(c, SL2_ERR_ARG,
                who + ": number_of_features_to_select must be >= 0, and <= SL2_MAX_MEASURED (128) "
                      "when max_features > 128");
  return SL2_OK;
}

}  // namespace sl2

namespace {

template <typename T>
cudaError_t dev_alloc(sl2_ctx *c, T **p, size_t count, bool zero = true) {
  DevPtr<void> h;
  cudaError_t e = cuda_malloc(h, count * sizeof(T) + 256);
  if (e != cudaSuccess) return e;
  void *q = h.get();
  c->allocs.push_back(std::move(h));
  if (zero) {
    e = cudaMemsetAsync(q, 0, count * sizeof(T) + 256, c->stream);
    if (e != cudaSuccess) return e;
  }
  *p = static_cast<T *>(q);
  return cudaSuccess;
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *,
                                    const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                                    const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int make_tensor_map(sl2_ctx *c) {
  void *fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  CU_TRY(c, cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
  if (!fn || qres != cudaDriverEntryPointSuccess)
    return fail(c, SL2_ERR_CUDA, "cuTensorMapEncodeTiled not available in this driver");
  const Sl2Dev &d = c->d;
  cuuint64_t dims[3] = {(cuuint64_t)d.W, (cuuint64_t)d.H, (cuuint64_t)d.slots * d.B};
  cuuint64_t strides[2] = {(cuuint64_t)d.pitch, (cuuint64_t)d.pitch * d.H};
  cuuint32_t box[3] = {(cuuint32_t)d.tile_w, (cuuint32_t)d.tile_h, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = ((PFN_encodeTiled)fn)(&c->tmap, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, d.frames, dims,
                                     strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                     CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char b[96];
    snprintf(b, sizeof b, "cuTensorMapEncodeTiled failed (CUresult %d)", (int)r);
    return fail(c, SL2_ERR_CUDA, b);
  }
  return SL2_OK;
}

// the row travels as a kernel parameter, so the write is ordered on the stream like any other launch
__global__ void write_cam_row_kernel(Sl2StreamCam *dst, const Sl2StreamCam row) { *dst = row; }

// The measure stage of the streams [lo, lo + cnt) on q: when some stream of them has the warp or the blur on, every
// job's template at the predicted state (warped, blurred, or the stored one, by each stream's settings) into the
// job-indexed scratch; the patch search over the context's own job arrays (indexed by the stream number local to the
// launch), the sub-pixel refinement when some stream of them has it on, then the match consensus when some stream of
// them has it on
int measure_streams(sl2_ctx *c, int32_t slot, int lo, int cnt, Sl2Queue q) {
  const Sl2Dev &d = c->d;
  const uint8_t *job_patches = nullptr;
  const bool blur = any_stream(c, lo, cnt, [](const StreamOptions &o) { return o.blur.on != 0; });
  if (blur || any_stream(c, lo, cnt, [](const StreamOptions &o) { return o.warp != 0; })) {
    WarpLaunch W = {};
    W.job_feat = d.job_feat + (size_t)lo * d.Nmax;
    W.jobs_per_stream = d.Nmax;
    W.stream_lo = lo;
    W.stream_cnt = cnt;
    W.on = c->warp_on_dev;
    W.out = c->warp_patches.get() + (size_t)lo * d.Nmax * d.box * 16;
    W.nrm = normals_args(c, lo, cnt);
    W.blur = blur ? c->blur_dev : nullptr;
    CU_TRY(c, sl2_launch_warp(d, W, q));
    job_patches = W.out;
  }
  SearchLaunch L = {};
  L.job_patches = job_patches;
  L.job_feat = d.job_feat + (size_t)lo * d.Nmax;
  L.job_centre = d.job_centre + (size_t)lo * d.Nmax * 2;
  L.job_puinv = d.job_puinv + (size_t)lo * d.Nmax * 3;
  L.jobs_per_stream = d.Nmax;
  L.stream_lo = lo;
  L.stream_cnt = cnt;
  L.slot = slot;
  L.scatter_to_features = 1;
  CU_TRY(c, sl2_launch_search(d, c->tmap, L, q));
  const Sl2Subpix sp = subpixel_args(c, lo, cnt);
  if (sp.z) {
    const int rc = subpixel_streams(c, slot, lo, cnt, job_patches, q);
    if (rc) return rc;
  }
  if (any_stream(c, lo, cnt, [](const StreamOptions &o) { return o.inlier_px > 0.0; }))
    CU_TRY(c, sl2_launch_consensus(d, lo, cnt, c->cons_tau2, sp, q));
  return SL2_OK;
}

}  // namespace

extern "C" {

const char *sl2_version(void) { return "sl2b200 0.1.0 sm_90a"; }

void sl2_default_config(sl2_config *cfg) {
  memset(cfg, 0, sizeof *cfg);
  cfg->device = 0;
  cfg->num_streams = 1;
  cfg->frame_slots = 1;
  cfg->width = 320;   // data/SceneLib2.cfg:24-31
  cfg->height = 240;
  cfg->boxsize = 11;  // monoslam.cpp:48
  cfg->max_features = 100;
  cfg->number_of_features_to_select = 10;  // cfg:60
  cfg->search_tile_radius = 20;
  cfg->fku = 195;
  cfg->fkv = 195;
  cfg->u0 = 162;
  cfg->v0 = 125;
  cfg->kd1 = 9e-06;
  cfg->sd = 1;
  cfg->delta_t = 0.033333333;  // cfg:59
  cfg->minimum_attempted_measurements_of_feature = 10;  // monoslam.cpp:1875
  cfg->successful_match_fraction = 0.5;                 // monoslam.cpp:1876
  cfg->cuda_stream = nullptr;
}

const char *sl2_last_error(const sl2_ctx *ctx) {
  return ctx ? ctx->err.c_str() : g_create_error.c_str();
}

int sl2_create(const sl2_config *cfg, sl2_ctx **out) {
  if (!cfg || !out) return fail(nullptr, SL2_ERR_ARG, "null argument");
  *out = nullptr;
  if (cfg->num_streams < 1 || cfg->frame_slots < 1 || cfg->width < 16 || cfg->height < 16 ||
      cfg->max_features < 1 || cfg->max_features > SL2_MAX_FEATURES)
    return fail(nullptr, SL2_ERR_ARG, "bad sizes in sl2_config");
  if (!selection_fits(cfg->max_features, cfg->number_of_features_to_select))
    return fail(nullptr, SL2_ERR_ARG,
                "number_of_features_to_select must be <= SL2_MAX_MEASURED (128) when max_features > 128");
  if (!sl2_box_supported(cfg->boxsize))
    return fail(nullptr, SL2_ERR_ARG, "boxsize must be 11 or 15");
  if (cfg->width < cfg->boxsize || cfg->height < cfg->boxsize)
    return fail(nullptr, SL2_ERR_ARG, "frame smaller than the patch");
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail(nullptr, SL2_ERR_CUDA,
                std::string("no CUDA device: ") + cudaGetErrorString(e) +
                    " (libsl2b200 has no CPU fallback)");
  if (cfg->device < 0 || cfg->device >= ndev) return fail(nullptr, SL2_ERR_ARG, "bad device ordinal");
  cudaDeviceProp prop;
  e = cudaGetDeviceProperties(&prop, cfg->device);
  if (e != cudaSuccess) return fail(nullptr, SL2_ERR_CUDA, cudaGetErrorString(e));
  if (prop.major != 9 || prop.minor != 0)
    return fail(nullptr, SL2_ERR_CUDA, "libsl2b200 is built for sm_90a (H100) only");
  e = cudaSetDevice(cfg->device);
  if (e != cudaSuccess) return fail(nullptr, SL2_ERR_CUDA, cudaGetErrorString(e));

  sl2_ctx *c = new sl2_ctx();
  c->cfg = *cfg;
  // what exists is held by c's handles: a failure releases it through sl2_destroy
  const auto failed = [c](int rc, const std::string &msg) {
    g_create_error = msg;
    sl2_destroy(c);
    return rc;
  };
  if (cfg->cuda_stream) {
    c->stream = static_cast<cudaStream_t>(cfg->cuda_stream);
  } else {
    e = cuda_stream_create(c->owned_stream);
    if (e != cudaSuccess) return failed(SL2_ERR_CUDA, cudaGetErrorString(e));
    c->stream = c->owned_stream.get();
  }
  Sl2Dev &d = c->d;
  memset(&d, 0, sizeof d);
  d.nsm = prop.multiProcessorCount;
  d.B = cfg->num_streams;
  d.Nmax = cfg->max_features;
  d.W = cfg->width;
  d.H = cfg->height;
  d.pitch = (cfg->width + 15) & ~15;
  d.slots = cfg->frame_slots;
  d.box = cfg->boxsize;
  d.ld = ((SL2_NXV + 3 * d.Nmax) + 7) & ~7;
  d.kmax = d.Nmax < SL2_MAX_MEASURED ? d.Nmax : SL2_MAX_MEASURED;  // the measurement capacity of every step
  d.mmax = 2 * d.kmax;
  d.ldg = ((d.mmax + SL2_NXV + 3 * d.Nmax + 1) + 7) & ~7;
  const int radius = cfg->search_tile_radius > 0 ? cfg->search_tile_radius : 20;
  d.tile_h = 2 * radius + d.box;
  if (d.tile_h > 255) d.tile_h = 255;
  d.tile_w = (2 * radius + d.box + 15 + 15) & ~15;  // +15: 16-byte aligned TMA box start
  if (d.tile_w > 256) d.tile_w = 256;
  d.min_attempts = cfg->minimum_attempted_measurements_of_feature;
  d.match_fraction = cfg->successful_match_fraction;
  for (int i = 0; i < 3; ++i) d.ovr[i] = cfg->search_override[i];
  const Sl2StreamCam row0 = sl2_cam_row(*cfg);  // every stream starts with the context's camera
  sl2_stream_config sc0 = {};
  sl2_cam_config(row0, &sc0);
  c->cams.assign(d.B, sc0);
  c->srcs.assign(d.B, sl2_stream_source{});
  c->layout.resize(d.B + 1);
  for (int s = 0; s <= d.B; ++s) c->layout[s] = (size_t)s * d.H * d.W;
  const std::vector<Sl2StreamCam> rows(d.B, row0);  // read by the copy below until the final synchronise

  const auto alloc_failed = [&] {
    return failed(SL2_ERR_CUDA, std::string("cudaMalloc failed: ") + cudaGetErrorString(cudaGetLastError()));
  };
  const size_t B = d.B, N = d.Nmax;
#define ALLOC(ptr, count) \
  if (dev_alloc(c, &(ptr), (count)) != cudaSuccess) return alloc_failed()
  ALLOC(d.cams, B);
  if (cudaMemcpyAsync(d.cams, rows.data(), B * sizeof(Sl2StreamCam), cudaMemcpyHostToDevice, c->stream) != cudaSuccess)
    return alloc_failed();
  ALLOC(d.frames, (size_t)d.slots * B * d.H * d.pitch);
  ALLOC(d.patches, (B * N + SL2_MAX_PARTIAL) * d.box * 16);  // + scratch templates (partially-initialised features)
  ALLOC(d.x, B * d.ld);
  ALLOC(d.P, B * d.ld * d.ld);
  ALLOC(d.G, B * d.mmax * d.ldg);
  ALLOC(d.nfeat, B);
#define SL2_ALLOC(T, name, per, by, reset) ALLOC(d.name, B * N * per);
  SL2_STREAM_ARRAYS(SL2_ALLOC)
#undef SL2_ALLOC
  ALLOC(d.nsel, B);
  ALLOC(d.nvisible, B);
  ALLOC(d.nmeas, B);
  ALLOC(d.ncull, B);
  ALLOC(d.upd_m, B);
  ALLOC(d.Wp, B * SL2_MAX_PANELS * 256);
  ALLOC(c->xv_stage, (size_t)d.slots * B * SL2_NXV);
  c->opt.assign(B, stream_option_defaults());
  ALLOC(c->cons_tau2, B);
  ALLOC(c->resc_chi2_dev, B);
  ALLOC(c->warp_on_dev, B);
  ALLOC(c->blur_dev, B);
  ALLOC(c->sel_mode_dev, B);
  ALLOC(c->sel_t_dev, B);
  c->sel_mode.assign(B, SL2_SELECT_TRACE);
  c->sel_t.assign(B, 1.0);
#undef ALLOC
  int rc = make_tensor_map(c);
  if (rc) return failed(rc, c->err);
  if (sl2_configure_search(d) != cudaSuccess || sl2_configure_update(d) != cudaSuccess)
    return failed(SL2_ERR_CUDA, std::string("kernel configuration failed: ") + cudaGetErrorString(cudaGetLastError()));
  rc = stage_reserve(c, 1 << 20);
  if (rc) return failed(rc, c->err);
  const auto init_failed = [&] { return failed(SL2_ERR_CUDA, "context initialisation failed"); };
  // the step-time events ev / evu keep the default (timing) flags; every other event only orders work
  for (Event &e : c->ev)
    if (cuda_event_create(e, cudaEventDefault) != cudaSuccess) return init_failed();
  for (Event &e : c->evu)
    if (cuda_event_create(e, cudaEventDefault) != cudaSuccess) return init_failed();
  for (Stream *s : {&c->copy_stream, &c->out_stream, &c->stream_b})
    if (cuda_stream_create(*s) != cudaSuccess) return init_failed();
  c->ev_slot.resize(d.slots);
  std::vector<Event *> untimed = {&c->ev_main, &c->ev_a_search, &c->ev_b_search, &c->ev_b_done};
  for (SlotEvents &s : c->ev_slot) untimed.insert(untimed.end(), {&s.h2d, &s.cmp, &s.cmp_b, &s.out});
  for (Event *e : untimed)
    if (cuda_event_create(*e, cudaEventDisableTiming) != cudaSuccess) return init_failed();
  if (cudaStreamSynchronize(c->stream) != cudaSuccess) return init_failed();
  *out = c;
  return SL2_OK;
}

void sl2_destroy(sl2_ctx *c) {
  if (!c) return;
  enter(c);
  for (cudaStream_t s : {c->stream, c->copy_stream.get(), c->out_stream.get(), c->stream_b.get()})
    if (s) cudaStreamSynchronize(s);
  delete c;  // its handles release everything it created
}

int sl2_sync(sl2_ctx *c) {
  if (!c) return SL2_ERR_ARG;
  enter(c);
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  if (c->copy_stream) CU_TRY(c, cudaStreamSynchronize(c->copy_stream.get()));
  if (c->out_stream) CU_TRY(c, cudaStreamSynchronize(c->out_stream.get()));
  return SL2_OK;
}

int64_t sl2_launch_count(const sl2_ctx *c) { return c ? c->launches : 0; }

// ---- per-stream camera --------------------------------------------------------------------------
int sl2_set_stream_config(sl2_ctx *c, int32_t s, const sl2_stream_config *sc) {
  if (bad_stream(c, s) || !sc) return fail(c, SL2_ERR_ARG, "sl2_set_stream_config: bad argument");
  const int rc = check_stream_config(c, sc, "sl2_set_stream_config");
  if (rc) return rc;
  CU_TRY(c, sl2_launch_kernel(write_cam_row_kernel, dim3(1), dim3(1), 0, queue(c), false, c->d.cams + s,
                              sl2_cam_row(*sc)));
  const sl2_stream_config old = c->cams[s];
  c->cams[s] = *sc;
  if (c->srcs[s].format != SL2_SRC_GRAY_RING && (old.width != sc->width || old.height != sc->height))
    return install_sources(c, c->srcs);  // the resize target of the stream's next frame
  return SL2_OK;
}

int sl2_get_stream_config(sl2_ctx *c, int32_t s, sl2_stream_config *sc) {
  if (bad_stream(c, s) || !sc) return fail(c, SL2_ERR_ARG, "sl2_get_stream_config: bad argument");
  *sc = c->cams[s];
  return SL2_OK;
}

// ---- map / state ------------------------------------------------------------------------------
int sl2_set_features(sl2_ctx *c, int32_t s, int32_t n, const double *y, const double *xp_org,
                     const uint8_t *patches) {
  if (bad_stream(c, s) || n < 0 || n > c->cfg.max_features || (n && (!y || !xp_org || !patches)))
    return fail(c, SL2_ERR_ARG, "sl2_set_features: bad argument");
  const Sl2Dev &d = c->d;
  const int box = d.box;
  std::vector<uint8_t> rows((size_t)n * box * 16);  // read by the copies below until the final synchronise
  const size_t fb = (size_t)s * d.Nmax;
  if (n) {
    pack_patch_rows(rows.data(), patches, n, box);
    CU_TRY(c, cudaMemcpyAsync(d.patches + fb * box * 16, rows.data(), rows.size(), cudaMemcpyHostToDevice, c->stream));
    CU_TRY(c, cudaMemcpyAsync(d.x + (size_t)s * d.ld + SL2_NXV, y, (size_t)n * 3 * 8, cudaMemcpyHostToDevice,
                              c->stream));
    CU_TRY(c, cudaMemcpyAsync(d.xp_org + fb * 7, xp_org, (size_t)n * 7 * 8, cudaMemcpyHostToDevice, c->stream));
  }
  CU_TRY(c, cudaMemcpyAsync(d.nfeat + s, &n, sizeof(int), cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, cudaMemsetAsync(d.attempted + fb, 0, sizeof(int) * d.Nmax, c->stream));
  CU_TRY(c, cudaMemsetAsync(d.successful + fb, 0, sizeof(int) * d.Nmax, c->stream));
  CU_TRY(c, cudaMemsetAsync(d.sel_rank + fb, 0xff, sizeof(int) * d.Nmax, c->stream));
  CU_TRY(c, cudaMemsetAsync(d.found + fb, 0, d.Nmax, c->stream));
  CU_TRY(c, cudaMemsetAsync(d.job_feat + fb, 0xff, sizeof(int) * d.Nmax, c->stream));
  const int rc = streams_restarted(c, s, 1);
  if (rc) return rc;
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return SL2_OK;
}

int sl2_num_features(sl2_ctx *c, int32_t s) {
  if (bad_stream(c, s)) return fail(c, SL2_ERR_ARG, "bad stream");
  int n = 0;
  int rc = device_nfeat(c, s, &n);
  return rc ? rc : n;
}

int sl2_state_size(sl2_ctx *c, int32_t s) {
  const int n = sl2_num_features(c, s);
  return n < 0 ? n : SL2_NXV + 3 * n;
}

int sl2_set_state(sl2_ctx *c, int32_t s, const double *x, const double *P) {
  if (bad_stream(c, s) || !x || !P) return fail(c, SL2_ERR_ARG, "sl2_set_state: bad argument");
  const int n = sl2_state_size(c, s);
  if (n < 0) return n;
  const Sl2Dev &d = c->d;
  CU_TRY(c, cudaMemcpyAsync(d.x + (size_t)s * d.ld, x, sizeof(double) * n, cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, cudaMemcpy2DAsync(d.P + (size_t)s * d.ld * d.ld, sizeof(double) * d.ld, P,
                              sizeof(double) * n, sizeof(double) * n, n, cudaMemcpyHostToDevice,
                              c->stream));
  const int rc = recovery_reset(c, s, 1);  // a new state: the stream is tracking
  if (rc) return rc;
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return SL2_OK;
}

int sl2_get_state(sl2_ctx *c, int32_t s, double *x, double *P) {
  if (bad_stream(c, s)) return fail(c, SL2_ERR_ARG, "sl2_get_state: bad argument");
  const int n = sl2_state_size(c, s);
  if (n < 0) return n;
  const Sl2Dev &d = c->d;
  if (x)
    CU_TRY(c, cudaMemcpyAsync(x, d.x + (size_t)s * d.ld, sizeof(double) * n, cudaMemcpyDeviceToHost, c->stream));
  if (P)
    CU_TRY(c, cudaMemcpy2DAsync(P, sizeof(double) * n, d.P + (size_t)s * d.ld * d.ld,
                                sizeof(double) * d.ld, sizeof(double) * n, n,
                                cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return SL2_OK;
}

// ---- staged measurement -------------------------------------------------------------------------
int sl2_make_measurements(sl2_ctx *c, int32_t s, int32_t slot) {
  if (bad_stream(c, s) || bad_slot(c, slot)) return fail(c, SL2_ERR_ARG, "bad stream/slot");
  const int rc = measure_streams(c, slot, s, 1, queue(c));
  if (rc) return rc;
  const Sl2Dev &d = c->d;
  const size_t fb = (size_t)s * d.Nmax;
  // successful measurements of THIS step only: found[] keeps the flag of features that were not
  // selected this frame (Feature::successful_measurement_flag_), so count over the job list
  std::vector<uint8_t> f(d.Nmax);
  std::vector<int> jf(d.Nmax);
  int nsel = 0;
  CU_TRY(c, cudaMemcpyAsync(f.data(), d.found + fb, d.Nmax, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaMemcpyAsync(jf.data(), d.job_feat + fb, sizeof(int) * d.Nmax, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaMemcpyAsync(&nsel, d.nsel + s, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  int cnt = 0;
  for (int r = 0; r < nsel && r < d.Nmax; ++r)
    if (jf[r] >= 0 && jf[r] < d.Nmax && f[jf[r]] == 1) ++cnt;
  return cnt;
}

// ---- fused step ---------------------------------------------------------------------------------
static int step_group(sl2_ctx *c, int32_t slot, int lo, int cnt, Sl2Queue q, cudaEvent_t after_search, bool t) {
  const Sl2Dev &d = c->d;
  const cudaStream_t st = q.stream;
  if (t) CU_TRY(c, cudaEventRecord(c->ev[0].get(), st));
  const bool info = any_stream(c, lo, cnt, [](const StreamOptions &o) { return o.sel.mode == SL2_SELECT_INFORMATION; });
  const sl2_recovery_result *rv = recovery_args(c, lo, cnt);  // a lost stream selects nothing
  const Sl2Accel acc = accel_args(c, slot, lo, cnt);  // inside the motion prediction
  // the motion prediction, the gyro update, then the feature prediction
  if (any_stream(c, lo, cnt, [](const StreamOptions &o) { return o.gyro.on != 0; })) {
    CU_TRY(c, sl2_launch_predict(d, lo, cnt, nullptr, 1, 0, nullptr, q, nullptr, acc));
    const int rc = gyro_streams(c, slot, lo, cnt, q);
    if (rc) return rc;
    CU_TRY(c, sl2_launch_predict(d, lo, cnt, nullptr, 0, 1, info ? c->sel_mode_dev : nullptr, q, rv));
  } else {
    CU_TRY(c, sl2_launch_predict(d, lo, cnt, nullptr, 1, 1, info ? c->sel_mode_dev : nullptr, q, rv, acc));
  }
  if (info) {  // part of the predict's time
    const int rc = select_streams(c, lo, cnt, q);
    if (rc) return rc;
  }
  if (t) CU_TRY(c, cudaEventRecord(c->ev[1].get(), st));
  // the consensus is part of the search's time: the update times still sum to ev[2] .. ev[3]
  const int rc = measure_streams(c, slot, lo, cnt, q);
  if (rc) return rc;
  if (t) CU_TRY(c, cudaEventRecord(c->ev[2].get(), st));
  if (after_search) CU_TRY(c, cudaEventRecord(after_search, st));
  cudaEvent_t evu[6];
  for (int i = 0; i < 6; ++i) evu[i] = c->evu[i].get();
  const Sl2Subpix sp = subpixel_args(c, lo, cnt);
  // the iteration passes are part of the update's time (ev[2] .. ev[3]); the update times are the final pass's
  const int rci = iterate_streams(c, lo, cnt, q);
  if (rci) return rci;
  CU_TRY(c, sl2_launch_update(d, lo, cnt, -1, nullptr, nullptr, nullptr, nullptr, nullptr, 0, sp, q, t ? evu : nullptr,
                              iterate_args(c, lo, cnt)));
  // the rescue and its second update are part of the update's time (ev[2] .. ev[3]); the update times are the first's
  const bool rescue = any_stream(c, lo, cnt, [](const StreamOptions &o) { return o.chi2 > 0.0 && o.inlier_px > 0.0; });
  if (rescue) {
    const int rc2 = rescue_streams(c, lo, cnt, q);
    if (rc2) return rc2;
  }
  // the normal alignment reads the updated state: after the last update, part of the update's time
  const Sl2Normals nrm = normals_args(c, lo, cnt);
  if (nrm.prm) CU_TRY(c, sl2_launch_normals(d, lo, cnt, slot, sp, nrm, q));
  if (t) CU_TRY(c, cudaEventRecord(c->ev[3].get(), st));
  CU_TRY(c, sl2_launch_cull(d, lo, cnt, -1, sp, q, nrm));
  if (t) CU_TRY(c, cudaEventRecord(c->ev[4].get(), st));
  if (d.rec_depth) {  // after ev[4]: the step times keep their meaning
    const Sl2Rescue r = rescue ? rescue_args(c) : Sl2Rescue{};
    CU_TRY(c, sl2_launch_records(d, lo, cnt, c->rec_steps, rescue ? &r : nullptr, q));
  }
  if (rv) return recover_streams(c, slot, lo, cnt, q);  // after the cull and the record: the record keeps its meaning
  return SL2_OK;
}

// number of camera streams in group A when the step runs as two staggered groups, else 0
static int split_point(const sl2_ctx *c) {
  return (c->step_groups >= 2 && !c->timing && c->d.B >= 2) ? (c->d.B + 1) / 2 : 0;
}

static int step_enqueue_groups(sl2_ctx *c, int32_t slot, bool serial) {
  const Sl2Dev &d = c->d;
  const int BA = serial ? 0 : split_point(c);
  if (BA == 0) {
    enter(c);  // serial order on `stream` (timing mode, one stream, or grouping switched off)
    return step_group(c, slot, 0, d.B, queue(c), nullptr, c->timing);
  }
  // group B sees everything `stream` has done so far (uploads, staged calls, the frame copy)
  CU_TRY(c, cudaEventRecord(c->ev_main.get(), c->stream));
  CU_TRY(c, cudaStreamWaitEvent(c->stream_b.get(), c->ev_main.get(), 0));
  if (c->b_search_valid) CU_TRY(c, cudaStreamWaitEvent(c->stream, c->ev_b_search.get(), 0));
  int rc = step_group(c, slot, 0, BA, queue(c), c->ev_a_search.get(), false);
  if (rc) return rc;
  CU_TRY(c, cudaStreamWaitEvent(c->stream_b.get(), c->ev_a_search.get(), 0));
  rc = step_group(c, slot, BA, d.B - BA, {c->stream_b.get(), &c->launches}, c->ev_b_search.get(), false);
  if (rc) return rc;
  c->b_search_valid = true;
  CU_TRY(c, cudaEventRecord(c->ev_b_done.get(), c->stream_b.get()));
  c->b_pending = true;
  return SL2_OK;
}

static int step_enqueue(sl2_ctx *c, int32_t slot, bool serial = false) {
  const int rc = step_enqueue_groups(c, slot, serial);
  if (rc == SL2_OK && c->d.rec_depth) ++c->rec_steps;  // both groups recorded this step under the same index
  return rc;
}

// the slot's frames are busy until everything queued so far on the step stream(s) has run
static int mark_slot_busy(sl2_ctx *c, int32_t slot) {
  CU_TRY(c, cudaEventRecord(c->ev_slot[slot].cmp.get(), c->stream));
  if (c->b_pending) CU_TRY(c, cudaEventRecord(c->ev_slot[slot].cmp_b.get(), c->stream_b.get()));
  return SL2_OK;
}

int sl2_step(sl2_ctx *c, int32_t slot) {
  enter(c, false);
  if (!c || bad_slot(c, slot)) return fail(c, SL2_ERR_ARG, "sl2_step: bad slot");
  const int rc = step_enqueue(c, slot);
  return rc ? rc : mark_slot_busy(c, slot);
}

int sl2_step_host(sl2_ctx *c, int32_t slot, const uint8_t *gray, double *xv_out) {
  enter(c);
  if (!c || bad_slot(c, slot) || !gray) return fail(c, SL2_ERR_ARG, "sl2_step_host: bad argument");
  int rc = sl2_set_frames(c, slot, gray);
  if (rc) return rc;
  rc = step_enqueue(c, slot, true);  // a blocking call has nothing to overlap with: serial kernel order
  if (rc) return rc;
  const Sl2Dev &d = c->d;
  if (xv_out)
    CU_TRY(c, cudaMemcpy2DAsync(xv_out, sizeof(double) * SL2_NXV, d.x, sizeof(double) * d.ld,
                                sizeof(double) * SL2_NXV, d.B, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return SL2_OK;
}

int sl2_step_host_async(sl2_ctx *c, int32_t slot, const uint8_t *gray, double *xv_out) {
  enter(c, false);
  if (!c || bad_slot(c, slot) || !gray) return fail(c, SL2_ERR_ARG, "sl2_step_host_async: bad argument");
  const Sl2Dev &d = c->d;
  cudaStream_t cs = c->copy_stream.get();
  // the frame slot may still be in use by work queued earlier on it: ev_cmp[slot] / ev_cmp_b[slot] are recorded
  // behind EVERY operation that reads or writes the slot (fused steps of either stream group, sl2_set_frame(s));
  // the remaining slot users (staged searches, detector, particles) synchronise the stream before they return.
  // Work on OTHER slots is not waited for: the copy of frame t+1 overlaps the kernels of frame t.
  CU_TRY(c, cudaStreamWaitEvent(cs, c->ev_slot[slot].cmp.get(), 0));
  CU_TRY(c, cudaStreamWaitEvent(cs, c->ev_slot[slot].cmp_b.get(), 0));
  if (!c->src_rows.empty()) CU_TRY(c, cudaStreamWaitEvent(cs, c->ev_src.get(), 0));  // the current source table
  CU_TRY(c, copy_slot_frames(c, slot, gray, cudaMemcpyHostToDevice, {cs, &c->launches}));
  CU_TRY(c, cudaEventRecord(c->ev_slot[slot].h2d.get(), cs));
  CU_TRY(c, cudaStreamWaitEvent(c->stream, c->ev_slot[slot].h2d.get(), 0));
  CU_TRY(c, cudaStreamWaitEvent(c->stream, c->ev_slot[slot].out.get(), 0));  // staging buffer of this slot is free
  int rc = step_enqueue(c, slot);
  if (rc) return rc;
  // camera states of this step -> per-slot staging (each group on its own stream) -> host
  double *stage = c->xv_stage + (size_t)slot * d.B * SL2_NXV;
  const int BA = c->b_pending ? split_point(c) : 0;
  const int nA = BA ? BA : d.B;
  CU_TRY(c, cudaMemcpy2DAsync(stage, sizeof(double) * SL2_NXV, d.x, sizeof(double) * d.ld,
                              sizeof(double) * SL2_NXV, nA, cudaMemcpyDeviceToDevice, c->stream));
  CU_TRY(c, cudaEventRecord(c->ev_slot[slot].cmp.get(), c->stream));
  CU_TRY(c, cudaStreamWaitEvent(c->out_stream.get(), c->ev_slot[slot].cmp.get(), 0));
  if (BA) {
    CU_TRY(c, cudaMemcpy2DAsync(stage + (size_t)BA * SL2_NXV, sizeof(double) * SL2_NXV,
                                d.x + (size_t)BA * d.ld, sizeof(double) * d.ld, sizeof(double) * SL2_NXV,
                                d.B - BA, cudaMemcpyDeviceToDevice, c->stream_b.get()));
    CU_TRY(c, cudaEventRecord(c->ev_slot[slot].cmp_b.get(), c->stream_b.get()));
    CU_TRY(c, cudaEventRecord(c->ev_b_done.get(), c->stream_b.get()));
    CU_TRY(c, cudaStreamWaitEvent(c->out_stream.get(), c->ev_slot[slot].cmp_b.get(), 0));
  }
  if (xv_out)
    CU_TRY(c, cudaMemcpyAsync(xv_out, stage, sizeof(double) * SL2_NXV * d.B, cudaMemcpyDeviceToHost,
                              c->out_stream.get()));
  CU_TRY(c, cudaEventRecord(c->ev_slot[slot].out.get(), c->out_stream.get()));
  return SL2_OK;
}

int sl2_join(sl2_ctx *c) {
  if (!c) return SL2_ERR_ARG;
  enter(c);
  return SL2_OK;
}

int sl2_set_step_groups(sl2_ctx *c, int32_t groups) {
  if (!c || groups < 1 || groups > 2) return fail(c, SL2_ERR_ARG, "sl2_set_step_groups: 1 or 2");
  enter(c);
  c->step_groups = groups;
  return SL2_OK;
}

int sl2_wait_slot(sl2_ctx *c, int32_t slot) {
  enter(c);
  if (!c || bad_slot(c, slot)) return fail(c, SL2_ERR_ARG, "sl2_wait_slot: bad slot");
  CU_TRY(c, cudaEventSynchronize(c->ev_slot[slot].out.get()));
  return SL2_OK;
}

int sl2_enable_timing(sl2_ctx *c, int32_t on) {
  if (!c) return SL2_ERR_ARG;
  enter(c);
  c->timing = on != 0;  // timing mode runs the step in serial order on the context's stream
  return SL2_OK;
}

int sl2_last_step_times(sl2_ctx *c, float *ms4) {
  enter(c);
  if (!c || !ms4) return SL2_ERR_ARG;
  if (!c->timing) return fail(c, SL2_ERR_STATE, "timing not enabled");
  CU_TRY(c, cudaEventSynchronize(c->ev[4].get()));
  for (int i = 0; i < 4; ++i) CU_TRY(c, cudaEventElapsedTime(&ms4[i], c->ev[i].get(), c->ev[i + 1].get()));
  return SL2_OK;
}

}  // extern "C"

// The copies of stream s's sub-pixel matches and refined flags, queued on the context's stream, when it has the
// refinement on; zr and ref stay empty otherwise
static int read_subpixel(sl2_ctx *c, int s, std::vector<double> &zr, std::vector<uint8_t> &ref) {
  const Sl2Subpix sp = subpixel_args(c, s, 1);
  if (!sp.z) return SL2_OK;
  const size_t N = c->d.Nmax, fb = (size_t)s * N;
  zr.resize(2 * N);
  ref.resize(N);
  CU_TRY(c, cudaMemcpyAsync(zr.data(), sp.z + fb * 2, 16 * N, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaMemcpyAsync(ref.data(), sp.refined + fb, N, cudaMemcpyDeviceToHost, c->stream));
  return SL2_OK;
}

extern "C" {

int sl2_get_feature_jacobians(sl2_ctx *c, int32_t s, double *dh_by_dxv, double *dh_by_dy, double *R,
                              double *nu) {
  if (bad_stream(c, s)) return fail(c, SL2_ERR_ARG, "bad stream");
  const Sl2Dev &d = c->d;
  const int N = d.Nmax;
  const size_t fb = (size_t)s * N;
  int nf = 0;
  std::vector<double> xp(14 * (size_t)N), dy(6 * (size_t)N), rv(N), hh(2 * (size_t)N);
  std::vector<int> zz(2 * (size_t)N);
  CU_TRY(c, cudaMemcpyAsync(&nf, d.nfeat + s, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaMemcpyAsync(xp.data(), d.dh_dxp + fb * 14, 8 * xp.size(), cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaMemcpyAsync(dy.data(), d.dh_dy + fb * 6, 8 * dy.size(), cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaMemcpyAsync(rv.data(), d.Rvar + fb, 8 * rv.size(), cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaMemcpyAsync(hh.data(), d.h + fb * 2, 8 * hh.size(), cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaMemcpyAsync(zz.data(), d.z_uv + fb * 2, 4 * zz.size(), cudaMemcpyDeviceToHost, c->stream));
  std::vector<double> zr;
  std::vector<uint8_t> ref;
  int rc = read_subpixel(c, s, zr, ref);
  if (rc) return rc;
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  for (int i = 0; i < nf; ++i) {
    if (dh_by_dxv)
      for (int col = 0; col < 13; ++col)
        for (int r = 0; r < 2; ++r) dh_by_dxv[i * 26 + col * 2 + r] = col < 7 ? xp[i * 14 + r * 7 + col] : 0.0;
    if (dh_by_dy)
      for (int col = 0; col < 3; ++col)
        for (int r = 0; r < 2; ++r) dh_by_dy[i * 6 + col * 2 + r] = dy[i * 6 + r * 3 + col];
    if (R) { R[i * 4 + 0] = rv[i]; R[i * 4 + 1] = 0.0; R[i * 4 + 2] = 0.0; R[i * 4 + 3] = rv[i]; }
    if (nu)
      for (int k = 0; k < 2; ++k) nu[i * 2 + k] = (ref.empty() || !ref[i] ? (double)zz[i * 2 + k] : zr[i * 2 + k]) - hh[i * 2 + k];
  }
  return nf;
}

int sl2_last_update_times(sl2_ctx *c, float *ms5) {
  enter(c);
  if (!c || !ms5) return SL2_ERR_ARG;
  if (!c->timing) return fail(c, SL2_ERR_STATE, "timing not enabled");
  CU_TRY(c, cudaEventSynchronize(c->evu[5].get()));
  for (int i = 0; i < 5; ++i) CU_TRY(c, cudaEventElapsedTime(&ms5[i], c->evu[i].get(), c->evu[i + 1].get()));
  return SL2_OK;
}

// ---- read-back ----------------------------------------------------------------------------------
int sl2_get_features(sl2_ctx *c, int32_t s, double *h, double *z, double *S, uint8_t *flags,
                     int32_t *attempted, int32_t *successful, int32_t *select_rank) {
  if (bad_stream(c, s)) return fail(c, SL2_ERR_ARG, "bad stream");
  const Sl2Dev &d = c->d;
  const int N = d.Nmax;
  const size_t fb = (size_t)s * N;
  int nf = 0;
  std::vector<double> hh(2 * N), SS(4 * N);
  std::vector<int> zz(2 * N), rk(N), at(N), su(N);
  std::vector<uint8_t> fd(N);
  CU_TRY(c, cudaMemcpyAsync(&nf, d.nfeat + s, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaMemcpyAsync(hh.data(), d.h + fb * 2, 16 * (size_t)N, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaMemcpyAsync(SS.data(), d.S + fb * 4, 32 * (size_t)N, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaMemcpyAsync(zz.data(), d.z_uv + fb * 2, 8 * (size_t)N, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaMemcpyAsync(rk.data(), d.sel_rank + fb, 4 * (size_t)N, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaMemcpyAsync(at.data(), d.attempted + fb, 4 * (size_t)N, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaMemcpyAsync(su.data(), d.successful + fb, 4 * (size_t)N, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaMemcpyAsync(fd.data(), d.found + fb, N, cudaMemcpyDeviceToHost, c->stream));
  std::vector<double> zr;
  std::vector<uint8_t> ref;
  const int rc = read_subpixel(c, s, zr, ref);
  if (rc) return rc;
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  for (int i = 0; i < nf; ++i) {
    if (h) { h[2 * i] = hh[2 * i]; h[2 * i + 1] = hh[2 * i + 1]; }
    const bool refined = !ref.empty() && ref[i];
    if (z)
      for (int k = 0; k < 2; ++k) z[2 * i + k] = refined ? zr[2 * i + k] : (double)zz[2 * i + k];
    if (S) for (int k = 0; k < 4; ++k) S[4 * i + k] = SS[4 * i + k];
    if (flags) flags[i] = (uint8_t)((rk[i] >= 0 ? 1 : 0) | (fd[i] == 1 ? 2 : 0) | (fd[i] == 2 ? 4 : 0) |
                                    (refined ? 8 : 0));
    if (attempted) attempted[i] = at[i];
    if (successful) successful[i] = su[i];
    if (select_rank) select_rank[i] = rk[i];
  }
  return nf;
}

}  // extern "C"
