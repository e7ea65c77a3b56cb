// api.cu — context management and the extern "C" surface declared in include/sl2b200.h.
// Host side only orchestrates: every arithmetic step of the hot path runs in the sm_90a
// kernels of search.cu / ekf.cu.  There is deliberately no CPU fallback.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/sl2b200.h"
#include "sl2_common.cuh"

namespace {

thread_local std::string g_create_error;

}  // namespace

struct sl2_ctx {
  sl2_config cfg;
  Sl2Dev d;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  CUtensorMap tmap;
  std::string err;
  std::vector<void *> allocs;
  // staging
  uint8_t *stg_dev = nullptr;   // device scratch for staged API calls
  size_t stg_bytes = 0;
  uint8_t *stg_host = nullptr;  // pinned
  double *smoe_map = nullptr;   // [features of the call][W][H] score cache of the SMOE kernels (lazily sized)
  size_t smoe_map_bytes = 0;
  int64_t launches = 0;
  bool timing = false;
  // timing mode: ev[0..4] bracket predict / search / update / cull, evu[0..5] the five update kernels
  cudaEvent_t ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  cudaEvent_t evu[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  // asynchronous end-to-end path: frames of step t+1 are copied while step t computes
  cudaStream_t copy_stream = nullptr;  // H2D of the frames
  cudaStream_t out_stream = nullptr;   // D2H of the results (own stream: must not block the next H2D)
  std::vector<cudaEvent_t> ev_h2d, ev_cmp, ev_out;  // per frame slot
  double *xv_stage = nullptr;                        // [slots][B][13] device
  // Fused step as two staggered groups of camera streams: group A (first half) on `stream`, group B on
  // `stream_b`; B's predict+search wait for A's search of the same step and A's next step waits for
  // B's search, so the integer-bound search of one group runs under the FP64-bound update of the other
  // and the two update kernels are half a step out of phase.  Results are identical to the serial order
  // (the groups share nothing); every other entry point joins the two streams first (enter()).
  int step_groups = 1;  // off by default: with two streams per SM the update would lose its second CTA per SM
  cudaStream_t stream_b = nullptr;
  cudaEvent_t ev_main = nullptr, ev_a_search = nullptr, ev_b_search = nullptr, ev_b_done = nullptr;
  bool b_pending = false, b_search_valid = false;
  std::vector<cudaEvent_t> ev_cmp_b;  // per frame slot: group B is done with the slot
};

// Defaults of the scheduling knobs; the environment variable SL2_TUNE="key=value,key=value" overrides them at context
// creation (experiments, and the parity tests run once with everything switched on).
static void tune_defaults(Sl2Dev &d) {
  d.tune[SL2_TUNE_PDL] = 2;           // automatic: on for a single camera stream (launch-latency bound), else off
  d.tune[SL2_TUNE_HP_PIPELINED] = 1;
  const char *e = getenv("SL2_TUNE");
  while (e && *e) {
    char *end = nullptr;
    const long k = strtol(e, &end, 10);
    if (end == e || *end != '=') break;
    e = end + 1;
    const long v = strtol(e, &end, 10);
    if (end == e) break;
    if (k >= 0 && k < SL2_TUNE_COUNT && v >= 0) d.tune[k] = (int)v;
    e = (*end == ',') ? end + 1 : end;
  }
}


namespace {

int fail(sl2_ctx *c, int code, const std::string &msg) {
  if (c) c->err = msg;
  else g_create_error = msg;
  return code;
}

#define CU_TRY(c, expr)                                                              \
  do {                                                                               \
    cudaError_t e__ = (expr);                                                        \
    if (e__ != cudaSuccess)                                                          \
      return fail((c), SL2_ERR_CUDA,                                                 \
                  std::string(#expr) + ": " + cudaGetErrorString(e__));             \
  } while (0)

template <typename T>
cudaError_t dev_alloc(sl2_ctx *c, T **p, size_t count, bool zero = true) {
  void *q = nullptr;
  cudaError_t e = cudaMalloc(&q, count * sizeof(T) + 256);
  if (e != cudaSuccess) return e;
  c->allocs.push_back(q);
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

// every entry point runs on the context's device whatever the calling thread's current device is
inline void enter(sl2_ctx *c, bool join = true) {
  if (!c) return;
  cudaSetDevice(c->cfg.device);
  if (join && c->b_pending) {  // the second stream group's step work becomes visible to `stream`
    cudaStreamWaitEvent(c->stream, c->ev_b_done, 0);
    c->b_pending = false;
    c->b_search_valid = false;
  }
}
bool bad_stream(sl2_ctx *c, int s) {
  enter(c);
  return !c || s < 0 || s >= c->cfg.num_streams;
}
bool bad_slot(sl2_ctx *c, int s) { return s < 0 || s >= c->cfg.frame_slots; }

int stage_reserve(sl2_ctx *c, size_t bytes) {
  if (bytes <= c->stg_bytes) return SL2_OK;
  if (c->stg_dev) {
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    cudaFree(c->stg_dev);
    cudaFreeHost(c->stg_host);
    c->stg_dev = nullptr;
    c->stg_host = nullptr;
  }
  bytes = (bytes + 4095) & ~(size_t)4095;
  CU_TRY(c, cudaMalloc((void **)&c->stg_dev, bytes));
  CU_TRY(c, cudaMallocHost((void **)&c->stg_host, bytes));
  c->stg_bytes = bytes;
  return SL2_OK;
}

int device_nfeat(sl2_ctx *c, int s, int *out) {
  CU_TRY(c, cudaMemcpyAsync(out, c->d.nfeat + s, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
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
  if (cfg->boxsize != 11 && cfg->boxsize != 15)
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
  if (cfg->cuda_stream) {
    c->stream = static_cast<cudaStream_t>(cfg->cuda_stream);
  } else {
    e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking);
    if (e != cudaSuccess) {
      delete c;
      return fail(nullptr, SL2_ERR_CUDA, cudaGetErrorString(e));
    }
    c->own_stream = true;
  }
  Sl2Dev &d = c->d;
  memset(&d, 0, sizeof d);
  d.nsm = prop.multiProcessorCount;
  tune_defaults(d);
  d.B = cfg->num_streams;
  d.Nmax = cfg->max_features;
  d.W = cfg->width;
  d.H = cfg->height;
  d.pitch = (cfg->width + 15) & ~15;
  d.slots = cfg->frame_slots;
  d.box = cfg->boxsize;
  d.ld = ((SL2_NXV + 3 * d.Nmax) + 7) & ~7;
  d.mmax = 2 * d.Nmax;
  d.ldg = ((d.mmax + SL2_NXV + 3 * d.Nmax + 1) + 7) & ~7;
  d.n_select = cfg->number_of_features_to_select;
  const int radius = cfg->search_tile_radius > 0 ? cfg->search_tile_radius : 20;
  d.tile_h = 2 * radius + d.box;
  if (d.tile_h > 255) d.tile_h = 255;
  d.tile_w = (2 * radius + d.box + 15 + 15) & ~15;  // +15: 16-byte aligned TMA box start
  if (d.tile_w > 256) d.tile_w = 256;
  d.min_attempts = cfg->minimum_attempted_measurements_of_feature;
  d.match_fraction = cfg->successful_match_fraction;
  d.cam[0] = cfg->width;
  d.cam[1] = cfg->height;
  d.cam[2] = cfg->fku;
  d.cam[3] = cfg->fkv;
  d.cam[4] = cfg->u0;
  d.cam[5] = cfg->v0;
  d.cam[6] = cfg->kd1;
  d.cam[7] = cfg->sd;
  d.dt = cfg->delta_t;
  for (int i = 0; i < 3; ++i) d.ovr[i] = cfg->search_override[i];

  const size_t B = d.B, N = d.Nmax;
  bool ok = true;
#define ALLOC(ptr, count) ok = ok && (dev_alloc(c, &(ptr), (count)) == cudaSuccess)
  ALLOC(d.frames, (size_t)d.slots * B * d.H * d.pitch);
  ALLOC(d.patches, (B * N + SL2_MAX_PARTIAL) * d.box * 16);  // + scratch templates (partially-initialised features)
  ALLOC(d.x, B * d.ld);
  ALLOC(d.P, B * d.ld * d.ld);
  ALLOC(d.G, B * d.mmax * d.ldg);
  ALLOC(d.nfeat, B);
  ALLOC(d.xp_org, B * N * 7);
  ALLOC(d.attempted, B * N);
  ALLOC(d.successful, B * N);
  ALLOC(d.h, B * N * 2);
  ALLOC(d.S, B * N * 4);
  ALLOC(d.Rvar, B * N);
  ALLOC(d.dh_dxp, B * N * 14);
  ALLOC(d.dh_dy, B * N * 6);
  ALLOC(d.sel_rank, B * N);
  ALLOC(d.z_uv, B * N * 2);
  ALLOC(d.found, B * N);
  ALLOC(d.best, B * N);
  ALLOC(d.job_feat, B * N);
  ALLOC(d.job_centre, B * N * 2);
  ALLOC(d.job_puinv, B * N * 3);
  ALLOC(d.nsel, B);
  ALLOC(d.nvisible, B);
  ALLOC(d.nmeas, B);
  ALLOC(d.ncull, B);
  ALLOC(d.upd_m, B);
  ALLOC(d.Wp, B * SL2_MAX_PANELS * 256);
  ALLOC(c->xv_stage, (size_t)d.slots * B * SL2_NXV);
#undef ALLOC
  if (!ok) {
    const std::string m = std::string("cudaMalloc failed: ") + cudaGetErrorString(cudaGetLastError());
    sl2_destroy(c);
    return fail(nullptr, SL2_ERR_CUDA, m);
  }
  int rc = make_tensor_map(c);
  if (rc == SL2_OK && (sl2_configure_search(d) != cudaSuccess || sl2_configure_update(d) != cudaSuccess))
    rc = fail(c, SL2_ERR_CUDA, std::string("kernel configuration failed: ") + cudaGetErrorString(cudaGetLastError()));
  if (rc == SL2_OK) rc = stage_reserve(c, 1 << 20);
  if (rc == SL2_OK) {
    for (int i = 0; i < 5 && rc == SL2_OK; ++i)
      if (cudaEventCreate(&c->ev[i]) != cudaSuccess) rc = SL2_ERR_CUDA;
    for (int i = 0; i < 6 && rc == SL2_OK; ++i)
      if (cudaEventCreate(&c->evu[i]) != cudaSuccess) rc = SL2_ERR_CUDA;
    if (cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking) != cudaSuccess) rc = SL2_ERR_CUDA;
    if (cudaStreamCreateWithFlags(&c->out_stream, cudaStreamNonBlocking) != cudaSuccess) rc = SL2_ERR_CUDA;
    if (cudaStreamCreateWithFlags(&c->stream_b, cudaStreamNonBlocking) != cudaSuccess) rc = SL2_ERR_CUDA;
    for (cudaEvent_t *e : {&c->ev_main, &c->ev_a_search, &c->ev_b_search, &c->ev_b_done})
      if (cudaEventCreateWithFlags(e, cudaEventDisableTiming) != cudaSuccess) rc = SL2_ERR_CUDA;
    for (int i = 0; i < d.slots && rc == SL2_OK; ++i) {
      cudaEvent_t e1, e2, e3, e4;
      if (cudaEventCreateWithFlags(&e1, cudaEventDisableTiming) != cudaSuccess ||
          cudaEventCreateWithFlags(&e2, cudaEventDisableTiming) != cudaSuccess ||
          cudaEventCreateWithFlags(&e3, cudaEventDisableTiming) != cudaSuccess ||
          cudaEventCreateWithFlags(&e4, cudaEventDisableTiming) != cudaSuccess) {
        rc = SL2_ERR_CUDA;
        break;
      }
      c->ev_h2d.push_back(e1);
      c->ev_cmp.push_back(e2);
      c->ev_out.push_back(e3);
      c->ev_cmp_b.push_back(e4);
    }
  }
  if (rc == SL2_OK && cudaStreamSynchronize(c->stream) != cudaSuccess) rc = SL2_ERR_CUDA;
  if (rc != SL2_OK) {
    g_create_error = c->err.empty() ? "context initialisation failed" : c->err;
    sl2_destroy(c);
    return rc;
  }
  *out = c;
  return SL2_OK;
}

void sl2_destroy(sl2_ctx *c) {
  if (!c) return;
  enter(c);
  if (c->stream) cudaStreamSynchronize(c->stream);
  if (c->copy_stream) {
    cudaStreamSynchronize(c->copy_stream);
    cudaStreamDestroy(c->copy_stream);
  }
  if (c->out_stream) {
    cudaStreamSynchronize(c->out_stream);
    cudaStreamDestroy(c->out_stream);
  }
  if (c->stream_b) {
    cudaStreamSynchronize(c->stream_b);
    cudaStreamDestroy(c->stream_b);
  }
  for (auto &v : {c->ev_h2d, c->ev_cmp, c->ev_out, c->ev_cmp_b})
    for (cudaEvent_t e : v) cudaEventDestroy(e);
  for (cudaEvent_t e : {c->ev_main, c->ev_a_search, c->ev_b_search, c->ev_b_done})
    if (e) cudaEventDestroy(e);
  for (void *p : c->allocs) cudaFree(p);
  if (c->stg_dev) cudaFree(c->stg_dev);
  if (c->smoe_map) cudaFree(c->smoe_map);
  if (c->stg_host) cudaFreeHost(c->stg_host);
  for (auto &e : c->ev)
    if (e) cudaEventDestroy(e);
  for (auto &e : c->evu)
    if (e) cudaEventDestroy(e);
  if (c->own_stream && c->stream) cudaStreamDestroy(c->stream);
  delete c;
}

int sl2_sync(sl2_ctx *c) {
  if (!c) return SL2_ERR_ARG;
  enter(c);
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  if (c->copy_stream) CU_TRY(c, cudaStreamSynchronize(c->copy_stream));
  if (c->out_stream) CU_TRY(c, cudaStreamSynchronize(c->out_stream));
  return SL2_OK;
}

int64_t sl2_launch_count(const sl2_ctx *c) { return c ? c->launches : 0; }

// ---- frames -----------------------------------------------------------------------------------
int sl2_set_frame(sl2_ctx *c, int32_t s, int32_t slot, const uint8_t *gray, size_t stride) {
  if (bad_stream(c, s) || bad_slot(c, slot) || !gray) return fail(c, SL2_ERR_ARG, "sl2_set_frame: bad argument");
  const Sl2Dev &d = c->d;
  uint8_t *dst = d.frames + ((size_t)slot * d.B + s) * d.H * d.pitch;
  CU_TRY(c, cudaMemcpy2DAsync(dst, d.pitch, gray, stride, d.W, d.H, cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, cudaEventRecord(c->ev_cmp[slot], c->stream));  // slot busy until the copy has landed
  return SL2_OK;
}

static int set_frames_any(sl2_ctx *c, int32_t slot, const uint8_t *gray, cudaMemcpyKind kind) {
  enter(c);
  if (!c || bad_slot(c, slot) || !gray) return fail(c, SL2_ERR_ARG, "sl2_set_frames: bad argument");
  const Sl2Dev &d = c->d;
  uint8_t *dst = d.frames + (size_t)slot * d.B * d.H * d.pitch;
  if (d.pitch == d.W) {
    CU_TRY(c, cudaMemcpyAsync(dst, gray, (size_t)d.B * d.H * d.W, kind, c->stream));
  } else {
    CU_TRY(c, cudaMemcpy2DAsync(dst, d.pitch, gray, d.W, d.W, (size_t)d.B * d.H, kind, c->stream));
  }
  CU_TRY(c, cudaEventRecord(c->ev_cmp[slot], c->stream));  // slot busy until the copy has landed
  return SL2_OK;
}
int sl2_set_frames(sl2_ctx *c, int32_t slot, const uint8_t *gray) {
  return set_frames_any(c, slot, gray, cudaMemcpyHostToDevice);
}
int sl2_set_frames_dev(sl2_ctx *c, int32_t slot, const uint8_t *gray_dev) {
  return set_frames_any(c, slot, gray_dev, cudaMemcpyDeviceToDevice);
}

// ---- map / state ------------------------------------------------------------------------------
int sl2_set_features(sl2_ctx *c, int32_t s, int32_t n, const double *y, const double *xp_org,
                     const uint8_t *patches) {
  if (bad_stream(c, s) || n < 0 || n > c->cfg.max_features || (n && (!y || !xp_org || !patches)))
    return fail(c, SL2_ERR_ARG, "sl2_set_features: bad argument");
  const Sl2Dev &d = c->d;
  const int box = d.box;
  const size_t pb = (size_t)n * box * 16, yb = (size_t)n * 3 * 8, xb = (size_t)n * 7 * 8;
  int rc = stage_reserve(c, pb + yb + xb + 64);
  if (rc) return rc;
  CU_TRY(c, cudaStreamSynchronize(c->stream));  // staging buffer reuse
  uint8_t *hp = c->stg_host;
  memset(hp, 0, pb);
  for (int i = 0; i < n; ++i)
    for (int r = 0; r < box; ++r)
      memcpy(hp + ((size_t)i * box + r) * 16, patches + ((size_t)i * box + r) * box, box);
  memcpy(hp + pb, y, yb);
  memcpy(hp + pb + yb, xp_org, xb);
  int nn = n;
  memcpy(hp + pb + yb + xb, &nn, sizeof(int));
  const size_t fb = (size_t)s * d.Nmax;
  if (n) {
    CU_TRY(c, cudaMemcpyAsync(d.patches + fb * box * 16, hp, pb, cudaMemcpyHostToDevice, c->stream));
    CU_TRY(c, cudaMemcpyAsync(d.x + (size_t)s * d.ld + SL2_NXV, hp + pb, yb, cudaMemcpyHostToDevice, c->stream));
    CU_TRY(c, cudaMemcpyAsync(d.xp_org + fb * 7, hp + pb + yb, xb, cudaMemcpyHostToDevice, c->stream));
  }
  CU_TRY(c, cudaMemcpyAsync(d.nfeat + s, hp + pb + yb + xb, sizeof(int), cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, cudaMemsetAsync(d.attempted + fb, 0, sizeof(int) * d.Nmax, c->stream));
  CU_TRY(c, cudaMemsetAsync(d.successful + fb, 0, sizeof(int) * d.Nmax, c->stream));
  CU_TRY(c, cudaMemsetAsync(d.sel_rank + fb, 0xff, sizeof(int) * d.Nmax, c->stream));
  CU_TRY(c, cudaMemsetAsync(d.found + fb, 0, d.Nmax, c->stream));
  CU_TRY(c, cudaMemsetAsync(d.job_feat + fb, 0xff, sizeof(int) * d.Nmax, c->stream));
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

int sl2_delete_feature(sl2_ctx *c, int32_t s, int32_t index) {
  if (bad_stream(c, s)) return fail(c, SL2_ERR_ARG, "bad stream");
  const int n = sl2_num_features(c, s);
  if (n < 0) return n;
  if (index < 0 || index >= n) return fail(c, SL2_ERR_ARG, "sl2_delete_feature: bad index");
  CU_TRY(c, sl2_launch_cull(c->d, s, 1, index, c->stream));
  ++c->launches;
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return SL2_OK;
}

int sl2_append_feature(sl2_ctx *c, int32_t s, const double *y, const double *xp_org, const uint8_t *patch,
                       const double *Pcol) {
  if (bad_stream(c, s) || !y || !xp_org || !patch) return fail(c, SL2_ERR_ARG, "sl2_append_feature: bad argument");
  const int nf = sl2_num_features(c, s);
  if (nf < 0) return nf;
  if (nf >= c->cfg.max_features) return fail(c, SL2_ERR_STATE, "sl2_append_feature: the map is full (max_features)");
  const Sl2Dev &d = c->d;
  const int box = d.box, n3 = SL2_NXV + 3 * nf + 3;
  // staging: y(3) xp(7) Pcol(3 * n3) | patch rows (box x 16)
  const size_t o_xp = 24, o_p = 80, o_patch = o_p + 8 * 3 * (size_t)n3, total = o_patch + (size_t)box * 16 + 64;
  int rc = stage_reserve(c, total);
  if (rc) return rc;
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  uint8_t *hp = c->stg_host;
  memset(hp, 0, total);
  memcpy(hp, y, 24);
  memcpy(hp + o_xp, xp_org, 56);
  if (Pcol) memcpy(hp + o_p, Pcol, 8 * 3 * (size_t)n3);
  for (int r = 0; r < box; ++r) memcpy(hp + o_patch + (size_t)r * 16, patch + (size_t)r * box, box);
  CU_TRY(c, cudaMemcpyAsync(c->stg_dev, hp, total - 64, cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, sl2_launch_append(d, s, reinterpret_cast<const double *>(c->stg_dev),
                              reinterpret_cast<const double *>(c->stg_dev + o_xp), c->stg_dev + o_patch,
                              Pcol ? reinterpret_cast<const double *>(c->stg_dev + o_p) : nullptr, c->stream));
  ++c->launches;
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return nf;  // index of the new feature
}

// ---- patch search -----------------------------------------------------------------------------
static int search_staged(sl2_ctx *c, int32_t s, int32_t slot, int32_t n, const int32_t *feat_index,
                         int32_t single_feat, const double *centre, const double *PuInv3,
                         int32_t *u, int32_t *v, uint8_t *found, double *best) {
  if (bad_stream(c, s) || bad_slot(c, slot) || n < 0 || !centre || !PuInv3)
    return fail(c, SL2_ERR_ARG, "patch search: bad argument");
  if (n == 0) return SL2_OK;
  int nf = 0;
  int rc = device_nfeat(c, s, &nf);
  if (rc) return rc;
  for (int i = 0; i < n; ++i) {
    const int f = feat_index ? feat_index[i] : single_feat;
    if (f < 0 || f >= nf) return fail(c, SL2_ERR_ARG, "patch search: feature index out of range");
  }
  // staging layout: centre(2n) puinv(3n) best(n) | feat(n) uv(2n) | found(n)
  const size_t o_c = 0, o_p = o_c + 16 * (size_t)n, o_b = o_p + 24 * (size_t)n,
               o_f = o_b + 8 * (size_t)n, o_uv = o_f + 4 * (size_t)n, o_fd = o_uv + 8 * (size_t)n,
               total = o_fd + n + 64;
  rc = stage_reserve(c, total);
  if (rc) return rc;
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  uint8_t *hp = c->stg_host;
  memcpy(hp + o_c, centre, 16 * (size_t)n);
  memcpy(hp + o_p, PuInv3, 24 * (size_t)n);
  int *hf = reinterpret_cast<int *>(hp + o_f);
  for (int i = 0; i < n; ++i) hf[i] = feat_index ? feat_index[i] : single_feat;
  CU_TRY(c, cudaMemcpyAsync(c->stg_dev, hp, o_uv, cudaMemcpyHostToDevice, c->stream));
  SearchLaunch L = {};
  L.job_centre = reinterpret_cast<const double *>(c->stg_dev + o_c);
  L.job_puinv = reinterpret_cast<const double *>(c->stg_dev + o_p);
  L.job_feat = reinterpret_cast<const int *>(c->stg_dev + o_f);
  L.jobs_per_stream = n;
  L.stream_lo = s;
  L.stream_cnt = 1;
  L.slot = slot;
  L.out_uv = reinterpret_cast<int *>(c->stg_dev + o_uv);
  L.out_found = c->stg_dev + o_fd;
  L.out_best = reinterpret_cast<double *>(c->stg_dev + o_b);
  L.scatter_to_features = 0;
  CU_TRY(c, sl2_launch_search(c->d, c->tmap, L, c->stream));
  ++c->launches;
  CU_TRY(c, cudaMemcpyAsync(hp + o_b, c->stg_dev + o_b, total - 64 - o_b, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  const int *huv = reinterpret_cast<const int *>(hp + o_uv);
  const double *hb = reinterpret_cast<const double *>(hp + o_b);
  for (int i = 0; i < n; ++i) {
    if (u) u[i] = huv[2 * i];
    if (v) v[i] = huv[2 * i + 1];
    if (found) found[i] = hp[o_fd + i];
    if (best) best[i] = hb[i];
  }
  return SL2_OK;
}

int sl2_patch_search(sl2_ctx *c, int32_t s, int32_t slot, int32_t n, const int32_t *feat_index,
                     const double *centre, const double *PuInv3, int32_t *u, int32_t *v,
                     uint8_t *found, double *best) {
  if (n > 0 && !feat_index) return fail(c, SL2_ERR_ARG, "sl2_patch_search: feat_index is null");
  return search_staged(c, s, slot, n, feat_index, 0, centre, PuInv3, u, v, found, best);
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

static int partial_features(sl2_ctx *c, int32_t s, int32_t slot, const PartialIO &io, const char *who) {
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
    int nf = 0;
    const int rc = device_nfeat(c, s, &nf);
    if (rc) return rc;
    for (int f = 0; f < F; ++f)
      if (io.feat_index[f] < 0 || io.feat_index[f] >= nf)
        return fail(c, SL2_ERR_ARG, std::string(who) + ": feature index out of range");
  }
  const size_t n = (size_t)F * Kmax, box = (size_t)d.box;
  // staging, inputs first: K(F) feat(F) | ypi(6F) Pxy(78F) Pyy(36F) lambda(n) prob(n) h(2n) Sinv3(3n) detS(n) |
  //          templates (F x box x 16)   then outputs: cum(n) mean_var(2F) uv(2n int) left(F int) found(n) keep(n)
  size_t o = 0;
  auto take = [&](size_t bytes) { const size_t at = o; o += (bytes + 15) & ~(size_t)15; return at; };
  const size_t o_K = take(4 * F), o_ft = take(4 * F), o_y = take(48 * F), o_xy = take(8 * 78 * F),
               o_yy = take(8 * 36 * F), o_l = take(8 * n), o_pr = take(8 * n), o_h = take(16 * n),
               o_si = take(24 * n), o_dt = take(8 * n), o_tp = take((size_t)F * box * 16), o_in_end = o,
               o_cu = take(8 * n), o_mv = take(16 * F), o_uv = take(8 * n), o_left = take(4 * F), o_fd = take(n),
               o_kp = take(n), total = o + 64;
  int rc = stage_reserve(c, total);
  if (rc) return rc;
  const size_t map_bytes = sl2_smoe_map_bytes(d, F);
  if (map_bytes > c->smoe_map_bytes) {
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    if (c->smoe_map) cudaFree(c->smoe_map);
    c->smoe_map = nullptr;
    c->smoe_map_bytes = 0;
    CU_TRY(c, cudaMalloc(&c->smoe_map, map_bytes));
    c->smoe_map_bytes = map_bytes;
  }
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  uint8_t *hp = c->stg_host;
  memset(hp, 0, o_in_end);
  memcpy(hp + o_K, io.K, 4 * (size_t)F);
  int *hf = reinterpret_cast<int *>(hp + o_ft);
  for (int f = 0; f < F; ++f) hf[f] = io.feat_index ? io.feat_index[f] : (d.B - s) * d.Nmax + f;
  if (predict) {
    memcpy(hp + o_y, io.ypi, 48 * (size_t)F);
    memcpy(hp + o_xy, io.Pxy, 8 * 78 * (size_t)F);
    memcpy(hp + o_yy, io.Pyy, 8 * 36 * (size_t)F);
  } else {
    memcpy(hp + o_h, io.h, 16 * n);
    memcpy(hp + o_si, io.Sinv3, 24 * n);
    if (io.detS) memcpy(hp + o_dt, io.detS, 8 * n);
  }
  if (io.lambda) memcpy(hp + o_l, io.lambda, 8 * n);
  if (reweight) memcpy(hp + o_pr, io.prob, 8 * n);
  if (io.patches)
    for (int f = 0; f < F; ++f)
      for (size_t r = 0; r < box; ++r)
        memcpy(hp + o_tp + ((size_t)f * box + r) * 16, io.patches + ((size_t)f * box + r) * box, box);
  CU_TRY(c, cudaMemcpyAsync(c->stg_dev, hp, o_in_end, cudaMemcpyHostToDevice, c->stream));
  if (io.patches)  // raw templates -> the scratch slots behind the map templates
    CU_TRY(c, cudaMemcpyAsync(d.patches + (size_t)d.B * d.Nmax * box * 16, c->stg_dev + o_tp, (size_t)F * box * 16,
                              cudaMemcpyDeviceToDevice, c->stream));
  uint8_t *dv = c->stg_dev;
  const int *dK = reinterpret_cast<const int *>(dv + o_K);
  double *dh = reinterpret_cast<double *>(dv + o_h), *dsi = reinterpret_cast<double *>(dv + o_si),
         *ddt = reinterpret_cast<double *>(dv + o_dt), *dl = reinterpret_cast<double *>(dv + o_l);
  if (predict) {
    CU_TRY(c, sl2_launch_particle_predict(d, s, F, Kmax, dK, reinterpret_cast<const double *>(dv + o_y),
                                          reinterpret_cast<const double *>(dv + o_xy),
                                          reinterpret_cast<const double *>(dv + o_yy), dl, dh, dsi, ddt, c->stream));
    ++c->launches;
  }
  // measure_feature_with_multiple_priors (monoslam.cpp:1408-1438): ellipses (SInv_k, h_k), one template per feature
  CU_TRY(c, sl2_launch_smoe(d, s, slot, F, Kmax, dK, reinterpret_cast<const int *>(dv + o_ft), dh, dsi, c->smoe_map,
                            reinterpret_cast<int *>(dv + o_uv), dv + o_fd, nullptr, c->stream));
  c->launches += 2;
  if (reweight) {
    CU_TRY(c, sl2_launch_particles(F, Kmax, dK, dh, dsi, ddt, dl, reinterpret_cast<const int *>(dv + o_uv), dv + o_fd,
                                   io.prune, reinterpret_cast<double *>(dv + o_pr), dv + o_kp,
                                   reinterpret_cast<double *>(dv + o_cu), reinterpret_cast<double *>(dv + o_mv),
                                   reinterpret_cast<int *>(dv + o_left), c->stream));
    ++c->launches;
  }
  // results: prob .. detS (inputs region, rewritten on the device) and the output region
  CU_TRY(c, cudaMemcpyAsync(hp + o_pr, dv + o_pr, o_tp - o_pr, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaMemcpyAsync(hp + o_cu, dv + o_cu, total - 64 - o_cu, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  if (predict) {
    memcpy(io.h, hp + o_h, 16 * n);
    memcpy(io.Sinv3, hp + o_si, 24 * n);
    memcpy(io.detS, hp + o_dt, 8 * n);
  }
  if (reweight) {
    memcpy(io.prob, hp + o_pr, 8 * n);
    if (io.cumulative) memcpy(io.cumulative, hp + o_cu, 8 * n);
    if (io.mean_var) memcpy(io.mean_var, hp + o_mv, 16 * (size_t)F);
    if (io.keep) memcpy(io.keep, hp + o_kp, n);
    if (io.left) memcpy(io.left, hp + o_left, 4 * (size_t)F);
  }
  if (io.z_uv) memcpy(io.z_uv, hp + o_uv, 8 * n);
  if (io.found) memcpy(io.found, hp + o_fd, n);
  return SL2_OK;
}

static int smoe_one(sl2_ctx *c, int32_t s, int32_t slot, const int32_t *feat_index, const uint8_t *patch, int32_t K,
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

static int measure_particles(sl2_ctx *c, int32_t s, int32_t slot, const int32_t *feat_index, const uint8_t *patch,
                             int32_t K, const double *h, const double *Sinv3, const double *detS,
                             const double *lambda, double prune_probability_threshold, double *prob,
                             int32_t *z_uv, uint8_t *found, uint8_t *keep, double *cumulative,
                             double *mean_var) {
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

int sl2_score_map(sl2_ctx *c, int32_t s, int32_t slot, int32_t feat, const double *centre,
                  const double *PuInv3, int32_t *box6, double *corr, double *sd_image,
                  uint8_t *inside, size_t cap) {
  if (bad_stream(c, s) || bad_slot(c, slot) || !centre || !PuInv3 || !box6)
    return fail(c, SL2_ERR_ARG, "sl2_score_map: bad argument");
  int nf = 0;
  int rc = device_nfeat(c, s, &nf);
  if (rc) return rc;
  if (feat < 0 || feat >= nf) return fail(c, SL2_ERR_ARG, "sl2_score_map: bad feature index");
  // staging: centre(2) puinv(3) feat(int, 8 B slot) box(6 int -> 32 B) corr(cap) sd(cap) inside(cap)
  const size_t o_box = 48, o_corr = 80, o_sd = o_corr + 8 * cap, o_in = o_sd + 8 * cap,
               total = o_in + cap + 64;
  rc = stage_reserve(c, total);
  if (rc) return rc;
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  uint8_t *hp = c->stg_host;
  memcpy(hp, centre, 16);
  memcpy(hp + 16, PuInv3, 24);
  int f = feat;
  memcpy(hp + 40, &f, sizeof(int));
  CU_TRY(c, cudaMemcpyAsync(c->stg_dev, hp, 48, cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, cudaMemsetAsync(c->stg_dev + o_box, 0xff, total - o_box, c->stream));  // NaN / 0xff fill
  CU_TRY(c, sl2_launch_score_map(c->d, c->tmap, s, slot, feat,
                                 reinterpret_cast<const double *>(c->stg_dev),
                                 reinterpret_cast<int *>(c->stg_dev + o_box),
                                 reinterpret_cast<double *>(c->stg_dev + o_corr),
                                 reinterpret_cast<double *>(c->stg_dev + o_sd), c->stg_dev + o_in,
                                 (int)cap, c->stream));
  ++c->launches;
  CU_TRY(c, cudaMemcpyAsync(hp + o_box, c->stg_dev + o_box, total - 64 - o_box, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  memcpy(box6, hp + o_box, 24);
  if (corr) memcpy(corr, hp + o_corr, 8 * cap);
  if (sd_image) memcpy(sd_image, hp + o_sd, 8 * cap);
  if (inside) memcpy(inside, hp + o_in, cap);
  return SL2_OK;
}

int sl2_find_best_patch(sl2_ctx *c, int32_t s, int32_t slot, int32_t n, const int32_t *regions,
                        int32_t *ubest, int32_t *vbest, double *evbest) {
  if (bad_stream(c, s) || bad_slot(c, slot) || n < 0 || (n && (!regions || !evbest)))
    return fail(c, SL2_ERR_ARG, "sl2_find_best_patch: bad argument");
  if (n == 0) return SL2_OK;
  const size_t o_uv = 16 * (size_t)n, o_ev = o_uv + 8 * (size_t)n, o_sc = o_ev + 8 * (size_t)n,
               total = o_sc + sl2_detect_scratch_bytes(c->d, n) + 64;
  int rc = stage_reserve(c, total);
  if (rc) return rc;
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  memcpy(c->stg_host, regions, 16 * (size_t)n);
  CU_TRY(c, cudaMemcpyAsync(c->stg_dev, c->stg_host, 16 * (size_t)n, cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, sl2_launch_detect(c->d, s, slot, n, reinterpret_cast<const int *>(c->stg_dev),
                              reinterpret_cast<int *>(c->stg_dev + o_uv),
                              reinterpret_cast<double *>(c->stg_dev + o_ev), c->stg_dev + o_sc, c->stream));
  c->launches += 2;
  CU_TRY(c, cudaMemcpyAsync(c->stg_host + o_uv, c->stg_dev + o_uv, 16 * (size_t)n, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  const int *uv = reinterpret_cast<const int *>(c->stg_host + o_uv);
  const double *ev = reinterpret_cast<const double *>(c->stg_host + o_ev);
  for (int i = 0; i < n; ++i) {
    evbest[i] = ev[i];
    if (uv[2 * i] >= 0) {
      if (ubest) ubest[i] = uv[2 * i];
      if (vbest) vbest[i] = uv[2 * i + 1];
    }
  }
  return SL2_OK;
}

// ---- EKF ----------------------------------------------------------------------------------------
int sl2_ekf_predict(sl2_ctx *c, int32_t s, const double *u3) {
  if (bad_stream(c, s)) return fail(c, SL2_ERR_ARG, "bad stream");
  const double *u_dev = nullptr;
  if (u3) {
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    memcpy(c->stg_host, u3, 24);
    CU_TRY(c, cudaMemcpyAsync(c->stg_dev, c->stg_host, 24, cudaMemcpyHostToDevice, c->stream));
    u_dev = reinterpret_cast<const double *>(c->stg_dev);
  }
  CU_TRY(c, sl2_launch_predict(c->d, s, 1, u_dev, 1, 0, c->stream));
  ++c->launches;
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return SL2_OK;
}

int sl2_predict_measurements(sl2_ctx *c, int32_t s) {
  if (bad_stream(c, s)) return fail(c, SL2_ERR_ARG, "bad stream");
  CU_TRY(c, sl2_launch_predict(c->d, s, 1, nullptr, 0, 1, c->stream));
  ++c->launches;
  int nv = 0;
  CU_TRY(c, cudaMemcpyAsync(&nv, c->d.nvisible + s, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return nv;
}

int sl2_make_measurements(sl2_ctx *c, int32_t s, int32_t slot) {
  if (bad_stream(c, s) || bad_slot(c, slot)) return fail(c, SL2_ERR_ARG, "bad stream/slot");
  const Sl2Dev &d = c->d;
  const size_t fb = (size_t)s * d.Nmax;
  SearchLaunch L = {};
  L.job_feat = d.job_feat + fb;
  L.job_centre = d.job_centre + fb * 2;
  L.job_puinv = d.job_puinv + fb * 3;
  L.jobs_per_stream = d.Nmax;
  L.stream_lo = s;
  L.stream_cnt = 1;
  L.slot = slot;
  L.scatter_to_features = 1;
  CU_TRY(c, sl2_launch_search(d, c->tmap, L, c->stream));
  ++c->launches;
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
    if (jf[r] >= 0 && jf[r] < d.Nmax && f[jf[r]]) ++cnt;
  return cnt;
}

int sl2_ekf_update(sl2_ctx *c, int32_t s, int32_t m, const int32_t *feat_index, const double *H_xv,
                   const double *H_y, const double *R, const double *nu) {
  if (bad_stream(c, s) || m < 0 || (m & 1) || m > 2 * c->cfg.max_features)
    return fail(c, SL2_ERR_ARG, "sl2_ekf_update: bad m");
  if (m == 0) return SL2_OK;
  if (!feat_index || !H_xv || !H_y || !R || !nu) return fail(c, SL2_ERR_ARG, "sl2_ekf_update: null argument");
  const int K = m / 2;
  int nf = 0;
  int rc = device_nfeat(c, s, &nf);
  if (rc) return rc;
  for (int k = 0; k < K; ++k) {
    if (feat_index[k] < 0 || feat_index[k] >= nf) return fail(c, SL2_ERR_ARG, "sl2_ekf_update: bad feature index");
    // the full 2x2 block R_k enters S (kalman.cpp:101); a covariance block has to be symmetric
    if (R[k * 4 + 1] != R[k * 4 + 2]) return fail(c, SL2_ERR_ARG, "sl2_ekf_update: R block is not symmetric");
  }
  const size_t o_hx = 0, o_hy = o_hx + 8 * 26 * (size_t)K, o_r = o_hy + 8 * 6 * (size_t)K,
               o_nu = o_r + 8 * 4 * (size_t)K, o_f = o_nu + 8 * 2 * (size_t)K,
               total = o_f + 4 * (size_t)K + 64;
  rc = stage_reserve(c, total);
  if (rc) return rc;
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  uint8_t *hp = c->stg_host;
  int nl = 0;
  memcpy(hp + o_hx, H_xv, 8 * 26 * (size_t)K);
  memcpy(hp + o_hy, H_y, 8 * 6 * (size_t)K);
  memcpy(hp + o_r, R, 8 * 4 * (size_t)K);
  memcpy(hp + o_nu, nu, 8 * 2 * (size_t)K);
  memcpy(hp + o_f, feat_index, 4 * (size_t)K);
  CU_TRY(c, cudaMemcpyAsync(c->stg_dev, hp, total - 64, cudaMemcpyHostToDevice, c->stream));
  CU_TRY(c, sl2_launch_update(c->d, s, 1, m, reinterpret_cast<const int *>(c->stg_dev + o_f),
                              reinterpret_cast<const double *>(c->stg_dev + o_hx),
                              reinterpret_cast<const double *>(c->stg_dev + o_hy),
                              reinterpret_cast<const double *>(c->stg_dev + o_r),
                              reinterpret_cast<const double *>(c->stg_dev + o_nu), 0, c->stream, nullptr, &nl));
  c->launches += nl;
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return SL2_OK;
}

int sl2_ekf_update_measured(sl2_ctx *c, int32_t s) {
  if (bad_stream(c, s)) return fail(c, SL2_ERR_ARG, "bad stream");
  int nl = 0;
  CU_TRY(c, sl2_launch_update(c->d, s, 1, -1, nullptr, nullptr, nullptr, nullptr, nullptr, 0, c->stream, nullptr, &nl));
  c->launches += nl;
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return SL2_OK;
}

int sl2_normalise_state(sl2_ctx *c, int32_t s) {
  if (bad_stream(c, s)) return fail(c, SL2_ERR_ARG, "bad stream");
  int nl = 0;
  CU_TRY(c, sl2_launch_update(c->d, s, 1, -1, nullptr, nullptr, nullptr, nullptr, nullptr, 1, c->stream, nullptr, &nl));
  c->launches += nl;
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return SL2_OK;
}

// ---- fused step ---------------------------------------------------------------------------------
static int step_group(sl2_ctx *c, int32_t slot, int lo, int cnt, cudaStream_t st, cudaEvent_t after_search,
                      bool t) {
  const Sl2Dev &d = c->d;
  if (t) CU_TRY(c, cudaEventRecord(c->ev[0], st));
  CU_TRY(c, sl2_launch_predict(d, lo, cnt, nullptr, 1, 1, st));
  if (t) CU_TRY(c, cudaEventRecord(c->ev[1], st));
  SearchLaunch L = {};
  // job arrays are indexed by the stream number local to the launch
  L.job_feat = d.job_feat + (size_t)lo * d.Nmax;
  L.job_centre = d.job_centre + (size_t)lo * d.Nmax * 2;
  L.job_puinv = d.job_puinv + (size_t)lo * d.Nmax * 3;
  L.jobs_per_stream = d.Nmax;
  L.stream_lo = lo;
  L.stream_cnt = cnt;
  L.slot = slot;
  L.scatter_to_features = 1;
  CU_TRY(c, sl2_launch_search(d, c->tmap, L, st));
  if (t) CU_TRY(c, cudaEventRecord(c->ev[2], st));
  if (after_search) CU_TRY(c, cudaEventRecord(after_search, st));
  int nl = 3;
  CU_TRY(c, sl2_launch_update(d, lo, cnt, -1, nullptr, nullptr, nullptr, nullptr, nullptr, 0, st,
                              t ? c->evu : nullptr, &nl));
  if (t) CU_TRY(c, cudaEventRecord(c->ev[3], st));
  CU_TRY(c, sl2_launch_cull(d, lo, cnt, -1, st));
  if (t) CU_TRY(c, cudaEventRecord(c->ev[4], st));
  c->launches += nl;
  return SL2_OK;
}

// number of camera streams in group A when the step runs as two staggered groups, else 0
static int split_point(const sl2_ctx *c) {
  return (c->step_groups >= 2 && !c->timing && c->d.B >= 2) ? (c->d.B + 1) / 2 : 0;
}

static int step_enqueue(sl2_ctx *c, int32_t slot, bool serial = false) {
  const Sl2Dev &d = c->d;
  const int BA = serial ? 0 : split_point(c);
  if (BA == 0) {
    enter(c);  // serial order on `stream` (timing mode, one stream, or grouping switched off)
    return step_group(c, slot, 0, d.B, c->stream, nullptr, c->timing);
  }
  // group B sees everything `stream` has done so far (uploads, staged calls, the frame copy)
  CU_TRY(c, cudaEventRecord(c->ev_main, c->stream));
  CU_TRY(c, cudaStreamWaitEvent(c->stream_b, c->ev_main, 0));
  if (c->b_search_valid) CU_TRY(c, cudaStreamWaitEvent(c->stream, c->ev_b_search, 0));
  int rc = step_group(c, slot, 0, BA, c->stream, c->ev_a_search, false);
  if (rc) return rc;
  CU_TRY(c, cudaStreamWaitEvent(c->stream_b, c->ev_a_search, 0));
  rc = step_group(c, slot, BA, d.B - BA, c->stream_b, c->ev_b_search, false);
  if (rc) return rc;
  c->b_search_valid = true;
  CU_TRY(c, cudaEventRecord(c->ev_b_done, c->stream_b));
  c->b_pending = true;
  return SL2_OK;
}

// the slot's frames are busy until everything queued so far on the step stream(s) has run
static int mark_slot_busy(sl2_ctx *c, int32_t slot) {
  CU_TRY(c, cudaEventRecord(c->ev_cmp[slot], c->stream));
  if (c->b_pending) CU_TRY(c, cudaEventRecord(c->ev_cmp_b[slot], c->stream_b));
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
  cudaStream_t cs = c->copy_stream;
  // the frame slot may still be in use by work queued earlier on it: ev_cmp[slot] / ev_cmp_b[slot] are recorded
  // behind EVERY operation that reads or writes the slot (fused steps of either stream group, sl2_set_frame(s));
  // the remaining slot users (staged searches, detector, particles) synchronise the stream before they return.
  // Work on OTHER slots is not waited for: the copy of frame t+1 overlaps the kernels of frame t.
  CU_TRY(c, cudaStreamWaitEvent(cs, c->ev_cmp[slot], 0));
  CU_TRY(c, cudaStreamWaitEvent(cs, c->ev_cmp_b[slot], 0));
  uint8_t *dst = d.frames + (size_t)slot * d.B * d.H * d.pitch;
  if (d.pitch == d.W) {
    CU_TRY(c, cudaMemcpyAsync(dst, gray, (size_t)d.B * d.H * d.W, cudaMemcpyHostToDevice, cs));
  } else {
    CU_TRY(c, cudaMemcpy2DAsync(dst, d.pitch, gray, d.W, d.W, (size_t)d.B * d.H, cudaMemcpyHostToDevice, cs));
  }
  CU_TRY(c, cudaEventRecord(c->ev_h2d[slot], cs));
  CU_TRY(c, cudaStreamWaitEvent(c->stream, c->ev_h2d[slot], 0));
  CU_TRY(c, cudaStreamWaitEvent(c->stream, c->ev_out[slot], 0));  // staging buffer of this slot is free
  int rc = step_enqueue(c, slot);
  if (rc) return rc;
  // camera states of this step -> per-slot staging (each group on its own stream) -> host
  double *stage = c->xv_stage + (size_t)slot * d.B * SL2_NXV;
  const int BA = c->b_pending ? split_point(c) : 0;
  const int nA = BA ? BA : d.B;
  CU_TRY(c, cudaMemcpy2DAsync(stage, sizeof(double) * SL2_NXV, d.x, sizeof(double) * d.ld,
                              sizeof(double) * SL2_NXV, nA, cudaMemcpyDeviceToDevice, c->stream));
  CU_TRY(c, cudaEventRecord(c->ev_cmp[slot], c->stream));
  CU_TRY(c, cudaStreamWaitEvent(c->out_stream, c->ev_cmp[slot], 0));
  if (BA) {
    CU_TRY(c, cudaMemcpy2DAsync(stage + (size_t)BA * SL2_NXV, sizeof(double) * SL2_NXV,
                                d.x + (size_t)BA * d.ld, sizeof(double) * d.ld, sizeof(double) * SL2_NXV,
                                d.B - BA, cudaMemcpyDeviceToDevice, c->stream_b));
    CU_TRY(c, cudaEventRecord(c->ev_cmp_b[slot], c->stream_b));
    CU_TRY(c, cudaEventRecord(c->ev_b_done, c->stream_b));
    CU_TRY(c, cudaStreamWaitEvent(c->out_stream, c->ev_cmp_b[slot], 0));
  }
  if (xv_out)
    CU_TRY(c, cudaMemcpyAsync(xv_out, stage, sizeof(double) * SL2_NXV * d.B, cudaMemcpyDeviceToHost,
                              c->out_stream));
  CU_TRY(c, cudaEventRecord(c->ev_out[slot], c->out_stream));
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

int sl2_set_tuning(sl2_ctx *c, int32_t key, int32_t value) {
  if (!c || key < 0 || key >= SL2_TUNE_COUNT || value < 0) return fail(c, SL2_ERR_ARG, "sl2_set_tuning: bad key / value");
  enter(c);
  c->d.tune[key] = value;  // Sl2Dev travels by value with every launch: the next launch sees it
  return SL2_OK;
}

int sl2_wait_slot(sl2_ctx *c, int32_t slot) {
  enter(c);
  if (!c || bad_slot(c, slot)) return fail(c, SL2_ERR_ARG, "sl2_wait_slot: bad slot");
  CU_TRY(c, cudaEventSynchronize(c->ev_out[slot]));
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
  CU_TRY(c, cudaEventSynchronize(c->ev[4]));
  for (int i = 0; i < 4; ++i) CU_TRY(c, cudaEventElapsedTime(&ms4[i], c->ev[i], c->ev[i + 1]));
  return SL2_OK;
}

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
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  for (int i = 0; i < nf; ++i) {
    if (dh_by_dxv)
      for (int col = 0; col < 13; ++col)
        for (int r = 0; r < 2; ++r) dh_by_dxv[i * 26 + col * 2 + r] = col < 7 ? xp[i * 14 + r * 7 + col] : 0.0;
    if (dh_by_dy)
      for (int col = 0; col < 3; ++col)
        for (int r = 0; r < 2; ++r) dh_by_dy[i * 6 + col * 2 + r] = dy[i * 6 + r * 3 + col];
    if (R) { R[i * 4 + 0] = rv[i]; R[i * 4 + 1] = 0.0; R[i * 4 + 2] = 0.0; R[i * 4 + 3] = rv[i]; }
    if (nu) { nu[i * 2] = (double)zz[i * 2] - hh[i * 2]; nu[i * 2 + 1] = (double)zz[i * 2 + 1] - hh[i * 2 + 1]; }
  }
  return nf;
}

int sl2_last_update_times(sl2_ctx *c, float *ms5) {
  enter(c);
  if (!c || !ms5) return SL2_ERR_ARG;
  if (!c->timing) return fail(c, SL2_ERR_STATE, "timing not enabled");
  CU_TRY(c, cudaEventSynchronize(c->evu[5]));
  for (int i = 0; i < 5; ++i) CU_TRY(c, cudaEventElapsedTime(&ms5[i], c->evu[i], c->evu[i + 1]));
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
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  for (int i = 0; i < nf; ++i) {
    if (h) { h[2 * i] = hh[2 * i]; h[2 * i + 1] = hh[2 * i + 1]; }
    if (z) { z[2 * i] = (double)zz[2 * i]; z[2 * i + 1] = (double)zz[2 * i + 1]; }
    if (S) for (int k = 0; k < 4; ++k) S[4 * i + k] = SS[4 * i + k];
    if (flags) flags[i] = (uint8_t)((rk[i] >= 0 ? 1 : 0) | (fd[i] ? 2 : 0));
    if (attempted) attempted[i] = at[i];
    if (successful) successful[i] = su[i];
    if (select_rank) select_rank[i] = rk[i];
  }
  return nf;
}

}  // extern "C"
