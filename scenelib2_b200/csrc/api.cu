// api.cu — context management and the extern "C" surface declared in include/sl2b200.h.
// Host side only orchestrates: every arithmetic step of the hot path runs in the sm_90a
// kernels of search.cu / ekf.cu / consensus.cu / reloc.cu / update.cu.  There is deliberately no CPU fallback.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <initializer_list>
#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "../../include/sl2b200.h"
#include "sl2_common.cuh"

namespace {

thread_local std::string g_create_error;

// Owning handles of the CUDA resources a context creates: a handle releases what it holds when it is reset, assigned
// or destroyed, so deleting the context releases everything it created, whatever point its creation reached.
struct DevFree { void operator()(void *p) const { cudaFree(p); } };
struct HostFree { void operator()(void *p) const { cudaFreeHost(p); } };
struct EventFree { void operator()(cudaEvent_t e) const { cudaEventDestroy(e); } };
struct StreamFree { void operator()(cudaStream_t s) const { cudaStreamDestroy(s); } };
template <typename T> using DevPtr = std::unique_ptr<T, DevFree>;    // device memory
template <typename T> using HostPtr = std::unique_ptr<T, HostFree>;  // pinned host memory
using Event = std::unique_ptr<CUevent_st, EventFree>;
using Stream = std::unique_ptr<CUstream_st, StreamFree>;

// each fills its handle only when the creation succeeds
template <typename T> cudaError_t cuda_malloc(DevPtr<T> &h, size_t bytes) {
  void *p = nullptr;
  const cudaError_t e = cudaMalloc(&p, bytes);
  if (e == cudaSuccess) h.reset(static_cast<T *>(p));
  return e;
}
template <typename T> cudaError_t cuda_malloc_host(HostPtr<T> &h, size_t bytes) {
  void *p = nullptr;
  const cudaError_t e = cudaMallocHost(&p, bytes);
  if (e == cudaSuccess) h.reset(static_cast<T *>(p));
  return e;
}
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

// the events of one frame slot: its frames have landed (h2d), the context's stream or group B is done with it (cmp,
// cmp_b), its camera states have been copied to the host (out)
struct SlotEvents { Event h2d, cmp, cmp_b, out; };

}  // namespace

struct sl2_ctx {
  sl2_config cfg;
  Sl2Dev d;
  std::vector<sl2_stream_config> cams;  // host mirror of d.cams, updated with it
  cudaStream_t stream = nullptr;        // cfg.cuda_stream, else owned_stream
  Stream owned_stream;                  // set only when the context created its stream
  CUtensorMap tmap;
  std::string err;
  std::vector<DevPtr<void>> allocs;  // behind the Sl2Dev arrays and xv_stage
  // staging
  DevPtr<uint8_t> stg_dev;   // device scratch for staged API calls
  size_t stg_bytes = 0;
  HostPtr<uint8_t> stg_host;
  DevPtr<double> smoe_map;   // [features of the call][W][H] score cache of the SMOE kernels (lazily sized)
  size_t smoe_map_bytes = 0;
  int64_t launches = 0;  // kernels launched: counted by sl2_launch_kernel through every Sl2Queue of the context
  bool timing = false;
  // timing mode: ev[0..4] bracket predict / search / update / cull, evu[0..5] the five update kernels
  Event ev[5], evu[6];
  // asynchronous end-to-end path: frames of step t+1 are copied while step t computes
  Stream copy_stream;  // H2D of the frames
  Stream out_stream;   // D2H of the results (own stream: must not block the next H2D)
  std::vector<SlotEvents> ev_slot;  // [slots]
  double *xv_stage = nullptr;       // [slots][B][13] device
  // Fused step as two staggered groups of camera streams: group A (first half) on `stream`, group B on
  // `stream_b`; B's predict+search wait for A's search of the same step and A's next step waits for
  // B's search, so the integer-bound search of one group runs under the FP64-bound update of the other
  // and the two update kernels are half a step out of phase.  Results are identical to the serial order
  // (the groups share nothing); every other entry point joins the two streams first (enter()).
  int step_groups = 1;  // off by default: with two streams per SM the update would lose its second CTA per SM
  Stream stream_b;
  Event ev_main, ev_a_search, ev_b_search, ev_b_done;
  bool b_pending = false, b_search_valid = false;
  DevPtr<sl2_step_record> rec;  // the ring d.rec points into
  int64_t rec_steps = 0;        // fused steps recorded since sl2_enable_records
  // raw frame sources (sl2_set_stream_source): the host mirror, the frame-set layout, and the device table of the
  // streams with a non-default source (src_rows, in stream order) with their raw frames' staging
  std::vector<sl2_stream_source> srcs;  // [B]
  std::vector<size_t> layout;           // [B + 1] byte offsets of the streams' frames in a frame set
  std::vector<Sl2Source> src_rows;
  DevPtr<Sl2Source> src_tab;    // [B]
  DevPtr<uint8_t> src_stage;    // [slots][src_slot_bytes] + 16 bytes of slack for the kernel's aligned loads
  size_t src_stage_bytes = 0, src_slot_bytes = 0;
  Event ev_src;                 // recorded on `stream` behind the last table write
  // match consensus (sl2_set_stream_consensus): the host mirror of every stream's inlier radius (0 = off) and the
  // device array of the squared radii the consensus kernel reads
  std::vector<double> cons_tau;  // [B]
  double *cons_tau2 = nullptr;   // [B] device
};

namespace {

int fail(sl2_ctx *c, int code, const std::string &msg) {
  if (code == SL2_ERR_CUDA) cudaGetLastError();  // reported once: sl2_launch_update returns the runtime's last error
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

// every entry point runs on the context's device whatever the calling thread's current device is
inline void enter(sl2_ctx *c, bool join = true) {
  if (!c) return;
  cudaSetDevice(c->cfg.device);
  if (join && c->b_pending) {  // the second stream group's step work becomes visible to `stream`
    cudaStreamWaitEvent(c->stream, c->ev_b_done.get(), 0);
    c->b_pending = false;
    c->b_search_valid = false;
  }
}
bool bad_stream(sl2_ctx *c, int s) {
  enter(c);
  return !c || s < 0 || s >= c->cfg.num_streams;
}
bool bad_slot(sl2_ctx *c, int s) { return s < 0 || s >= c->cfg.frame_slots; }

// Grows a scratch buffer, whose contents never outlive a call, to `bytes`: the old one is released once the context's
// stream is done with it (and before the new allocation, so the peak stays one buffer), then the device buffer and its
// pinned twin, if any, are allocated.  `size` is recorded only when both exist: after a failed grow the buffer is
// empty and the next call allocates again.
template <typename T>
int grow_scratch(sl2_ctx *c, size_t bytes, size_t &size, DevPtr<T> &dev, HostPtr<T> *host = nullptr) {
  if (bytes <= size) return SL2_OK;
  if (dev) CU_TRY(c, cudaStreamSynchronize(c->stream));
  size = 0;
  dev.reset();
  if (host) host->reset();
  CU_TRY(c, cuda_malloc(dev, bytes));
  if (host) CU_TRY(c, cuda_malloc_host(*host, bytes));
  size = bytes;
  return SL2_OK;
}

int stage_reserve(sl2_ctx *c, size_t bytes) {
  return grow_scratch(c, (bytes + 4095) & ~(size_t)4095, c->stg_bytes, c->stg_dev, &c->stg_host);
}

// One section of a staged call's buffers.  STAGE_IN sections go to the device before the launches (from `src`, or
// zero-filled when it is null, then whatever the caller packs through `h`), STAGE_OUT sections come back after them,
// STAGE_INOUT sections both ways; STAGE_DEV sections are device scratch and are copied neither way.
enum StageDir { STAGE_IN, STAGE_INOUT, STAGE_OUT, STAGE_DEV };
struct Stage {
  StageDir dir;
  size_t bytes;
  const void *src = nullptr;
  uint8_t *h = nullptr, *d = nullptr;  // pinned host and device address, set by staged_call
  size_t at = 0;                       // offset in the staging buffers
  template <typename T> T *host() const { return reinterpret_cast<T *>(h); }
  template <typename T> T *dev() const { return reinterpret_cast<T *>(d); }
};

// A synchronous call through the context's staging buffers: the sections are laid out 16-byte aligned in the order
// inputs, in-out, outputs, scratch.  Then: the one stream synchronise before the pinned buffer is rewritten (when
// anything goes in), the inputs filled and pack() run, one H2D copy of inputs and in-out, launch(), one D2H copy of
// in-out and outputs, and a synchronise, after which the caller reads the results through the host addresses.
template <typename Pack, typename Launch>
int staged_call(sl2_ctx *c, std::initializer_list<Stage *> secs, Pack &&pack, Launch &&launch) {
  size_t end[STAGE_DEV + 1], o = 0;  // end[k]: where the sections of direction k end
  for (int k = STAGE_IN; k <= STAGE_DEV; ++k) {
    for (Stage *x : secs)
      if (x->dir == k) {
        x->at = o;
        o += (x->bytes + 15) & ~(size_t)15;
      }
    end[k] = o;
  }
  int rc = stage_reserve(c, o);
  if (rc) return rc;
  const size_t h2d = end[STAGE_INOUT], d2h = end[STAGE_OUT] - end[STAGE_IN];
  if (h2d) CU_TRY(c, cudaStreamSynchronize(c->stream));
  for (Stage *x : secs) {
    x->h = c->stg_host.get() + x->at;
    x->d = c->stg_dev.get() + x->at;
    if (x->dir <= STAGE_INOUT) {
      if (x->src) memcpy(x->h, x->src, x->bytes);
      else memset(x->h, 0, x->bytes);
    }
  }
  pack();
  if (h2d) CU_TRY(c, cudaMemcpyAsync(c->stg_dev.get(), c->stg_host.get(), h2d, cudaMemcpyHostToDevice, c->stream));
  rc = launch();
  if (rc) return rc;
  if (d2h)
    CU_TRY(c, cudaMemcpyAsync(c->stg_host.get() + end[STAGE_IN], c->stg_dev.get() + end[STAGE_IN], d2h,
                              cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return SL2_OK;
}

// the launchers' queue on the context's stream
Sl2Queue queue(sl2_ctx *c) { return {c->stream, &c->launches}; }

// n box x box templates -> rows zero-padded to 16 bytes, the layout of Sl2Dev::patches
void pack_patch_rows(uint8_t *dst, const uint8_t *src, int n, int box) {
  memset(dst, 0, (size_t)n * box * 16);
  for (size_t r = 0; r < (size_t)n * box; ++r) memcpy(dst + r * 16, src + r * box, box);
}

// gray blocks of the streams [lo, hi), [hi - lo][H][W] packed, into the frame ring
cudaError_t copy_gray_blocks(const Sl2Dev &d, int slot, int lo, int hi, const uint8_t *src, cudaMemcpyKind kind,
                             cudaStream_t st) {
  uint8_t *dst = d.frames + ((size_t)slot * d.B + lo) * d.H * d.pitch;
  if (d.pitch == d.W) return cudaMemcpyAsync(dst, src, (size_t)(hi - lo) * d.H * d.W, kind, st);
  return cudaMemcpy2DAsync(dst, d.pitch, src, d.W, d.W, (size_t)(hi - lo) * d.H, kind, st);
}

uint8_t *source_stage(const sl2_ctx *c, int slot) { return c->src_stage.get() + (size_t)slot * c->src_slot_bytes; }

// convert the raw frames of source rows [base, base + cnt) of `slot`'s staging into the ring
cudaError_t ingest(sl2_ctx *c, int slot, int base, int cnt, Sl2Queue q) {
  int max_dh = 0, max_rb = 0;
  for (int j = base; j < base + cnt; ++j) {
    const Sl2Source &r = c->src_rows[j];
    max_dh = std::max(max_dh, r.dh);
    max_rb = std::max(max_rb, r.sw * sl2_source_bpp(r.format));
  }
  return sl2_launch_ingest(c->d, c->src_tab.get(), base, cnt, max_dh, max_rb, source_stage(c, slot), slot, q);
}

// One frame slot of every stream, a frame set (sl2_frame_set_layout), into the frame ring: each run of consecutive
// default streams in one copy to the ring (the whole set when no stream has a source), each run of streams with a
// source in one copy to the slot's staging, then one conversion launch for all of them.
cudaError_t copy_slot_frames(sl2_ctx *c, int slot, const uint8_t *src, cudaMemcpyKind kind, Sl2Queue q) {
  const Sl2Dev &d = c->d;
  if (c->src_rows.empty()) return copy_gray_blocks(d, slot, 0, d.B, src, kind, q.stream);
  for (int a = 0; a < d.B;) {
    const bool raw = c->srcs[a].format != SL2_SRC_GRAY_RING;
    int b = a + 1;
    while (b < d.B && (c->srcs[b].format != SL2_SRC_GRAY_RING) == raw) ++b;
    cudaError_t e;
    if (raw) {
      size_t at = 0;  // staging offset of stream a
      for (const Sl2Source &r : c->src_rows)
        if (r.stream == a) at = (size_t)r.off;
      e = cudaMemcpyAsync(source_stage(c, slot) + at, src + c->layout[a], c->layout[b] - c->layout[a], kind,
                          q.stream);
    } else {
      e = copy_gray_blocks(d, slot, a, b, src + c->layout[a], kind, q.stream);
    }
    if (e != cudaSuccess) return e;
    a = b;
  }
  return ingest(c, slot, 0, (int)c->src_rows.size(), q);
}

int device_nfeat(sl2_ctx *c, int s, int *out) {
  CU_TRY(c, cudaMemcpyAsync(out, c->d.nfeat + s, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return SL2_OK;
}

// A step measures at most min(max_features, SL2_MAX_MEASURED) features; below that capacity the selection is bounded
// by the map itself, so only a larger map needs the bound on the selection.
bool selection_fits(int max_features, int n_select) {
  return !(max_features > SL2_MAX_MEASURED && n_select > SL2_MAX_MEASURED);
}

Sl2StreamCam cam_row(const sl2_stream_config &sc) {
  Sl2StreamCam r = {};
  const double cam[8] = {(double)sc.width, (double)sc.height, sc.fku, sc.fkv, sc.u0, sc.v0, sc.kd1, sc.sd};
  for (int i = 0; i < 8; ++i) r.cam[i] = cam[i];
  r.dt = sc.delta_t;
  r.n_select = sc.number_of_features_to_select;
  return r;
}

// the row travels as a kernel parameter, so the write is ordered on the stream like any other launch
__global__ void write_cam_row_kernel(Sl2StreamCam *dst, const Sl2StreamCam row) { *dst = row; }
__global__ void write_double_kernel(double *dst, const double v) { *dst = v; }

// whether the symmetric 13 x 13 matrix A (column-major) is positive semi-definite: cyclic Jacobi eigenvalues, the
// smallest >= -1e-12 times the largest magnitude
bool psd13(const double *A0) {
  double A[13][13];
  double scale = 0.0;
  for (int i = 0; i < 13; ++i)
    for (int j = 0; j < 13; ++j) {
      A[i][j] = A0[i + 13 * j];
      scale += A[i][j] * A[i][j];
    }
  for (int sweep = 0; sweep < 100; ++sweep) {
    double off = 0.0;
    for (int p = 0; p < 13; ++p)
      for (int q = p + 1; q < 13; ++q) off += A[p][q] * A[p][q];
    if (off <= 1e-34 * scale) break;
    for (int p = 0; p < 13; ++p)
      for (int q = p + 1; q < 13; ++q) {
        if (A[p][q] == 0.0) continue;
        const double th = (A[q][q] - A[p][p]) / (2.0 * A[p][q]);
        const double t = (th >= 0.0 ? 1.0 : -1.0) / (std::fabs(th) + std::sqrt(th * th + 1.0));
        const double c = 1.0 / std::sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < 13; ++k) {
          const double akp = A[k][p], akq = A[k][q];
          A[k][p] = c * akp - s * akq;
          A[k][q] = s * akp + c * akq;
        }
        for (int k = 0; k < 13; ++k) {
          const double apk = A[p][k], aqk = A[q][k];
          A[p][k] = c * apk - s * aqk;
          A[q][k] = s * apk + c * aqk;
        }
      }
  }
  double lo = 0.0, hi = 0.0;
  for (int i = 0; i < 13; ++i) {
    lo = std::min(lo, A[i][i]);
    hi = std::max(hi, std::fabs(A[i][i]));
  }
  return lo >= -1e-12 * hi;
}

// whether some stream of [lo, lo + cnt) has the match consensus on
bool consensus_on(const sl2_ctx *c, int lo, int cnt) {
  for (int s = lo; s < lo + cnt; ++s)
    if (c->cons_tau[s] > 0.0) return true;
  return false;
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
  sl2_stream_config sc0 = {};
  sc0.width = cfg->width;
  sc0.height = cfg->height;
  sc0.fku = cfg->fku;
  sc0.fkv = cfg->fkv;
  sc0.u0 = cfg->u0;
  sc0.v0 = cfg->v0;
  sc0.kd1 = cfg->kd1;
  sc0.sd = cfg->sd;
  sc0.delta_t = cfg->delta_t;
  sc0.number_of_features_to_select = cfg->number_of_features_to_select;
  c->cams.assign(d.B, sc0);
  c->srcs.assign(d.B, sl2_stream_source{});
  c->layout.resize(d.B + 1);
  for (int s = 0; s <= d.B; ++s) c->layout[s] = (size_t)s * d.H * d.W;
  const std::vector<Sl2StreamCam> rows(d.B, cam_row(sc0));  // read by the copy below until the final synchronise

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
  ALLOC(c->cons_tau2, B);
  c->cons_tau.assign(B, 0.0);
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
// the camera values a stream of this context accepts (sl2_set_stream_config and the snapshot loads)
static int check_stream_config(sl2_ctx *c, const sl2_stream_config *sc, const std::string &who) {
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

static int install_sources(sl2_ctx *c, const std::vector<sl2_stream_source> &srcs);

int sl2_set_stream_config(sl2_ctx *c, int32_t s, const sl2_stream_config *sc) {
  if (bad_stream(c, s) || !sc) return fail(c, SL2_ERR_ARG, "sl2_set_stream_config: bad argument");
  const int rc = check_stream_config(c, sc, "sl2_set_stream_config");
  if (rc) return rc;
  CU_TRY(c, sl2_launch_kernel(write_cam_row_kernel, dim3(1), dim3(1), 0, queue(c), false, c->d.cams + s, cam_row(*sc)));
  const sl2_stream_config old = c->cams[s];
  c->cams[s] = *sc;
  if (c->srcs[s].format != SL2_SRC_GRAY_RING && (old.width != sc->width || old.height != sc->height))
    return install_sources(c, c->srcs);  // the resize target of the stream's next frame
  return SL2_OK;
}

// ---- raw frame sources ------------------------------------------------------------------------------
static size_t frame_bytes(const sl2_ctx *c, const sl2_stream_source &s) {
  return s.format == SL2_SRC_GRAY_RING ? (size_t)c->d.H * c->d.W
                                       : (size_t)s.width * s.height * sl2_source_bpp(s.format);
}

// Make `srcs` the context's sources (with the cameras in c->cams): layout, table rows, staging and the device table.
// The table is rewritten on `stream` after every conversion queued so far on the copy stream.
static int install_sources(sl2_ctx *c, const std::vector<sl2_stream_source> &srcs) {
  const Sl2Dev &d = c->d;
  std::vector<size_t> layout(d.B + 1, 0);
  std::vector<Sl2Source> rows;
  size_t raw = 0;
  for (int s = 0; s < d.B; ++s) {
    layout[s + 1] = layout[s] + frame_bytes(c, srcs[s]);
    if (srcs[s].format == SL2_SRC_GRAY_RING) continue;
    rows.push_back({s, srcs[s].format, srcs[s].width, srcs[s].height, c->cams[s].width, c->cams[s].height,
                    (int64_t)raw});
    raw += frame_bytes(c, srcs[s]);
  }
  const size_t slot_bytes = (raw + 15) & ~(size_t)15;
  const size_t need = rows.empty() ? 0 : (size_t)d.slots * slot_bytes + 16;
  // every allocation before anything changes: a failed one leaves the sources, the staging and the table as they were
  DevPtr<uint8_t> stage;
  if (need > c->src_stage_bytes) {  // nothing may still read or write the old staging
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    CU_TRY(c, cudaStreamSynchronize(c->copy_stream.get()));
    CU_TRY(c, cuda_malloc(stage, need));
  }
  if (!rows.empty() && !c->src_tab) CU_TRY(c, cuda_malloc(c->src_tab, sizeof(Sl2Source) * d.B));
  if (!rows.empty() && !c->ev_src) CU_TRY(c, cuda_event_create(c->ev_src, cudaEventDisableTiming));
  if (stage) {
    c->src_stage = std::move(stage);
    c->src_stage_bytes = need;
  }
  if (!rows.empty()) {
    for (const SlotEvents &e : c->ev_slot)  // conversions in flight
      CU_TRY(c, cudaStreamWaitEvent(c->stream, e.h2d.get(), 0));
    for (size_t first = 0; first < rows.size(); first += SL2_SOURCE_CHUNK) {
      Sl2SourceChunk ch = {};
      ch.first = (int)first;
      ch.n = (int)std::min(rows.size() - first, (size_t)SL2_SOURCE_CHUNK);
      for (int i = 0; i < ch.n; ++i) ch.row[i] = rows[first + i];
      CU_TRY(c, sl2_launch_source_write(c->src_tab.get(), ch, queue(c)));
    }
    CU_TRY(c, cudaEventRecord(c->ev_src.get(), c->stream));
  }
  c->srcs = srcs;
  c->layout = layout;
  c->src_rows = rows;
  c->src_slot_bytes = slot_bytes;
  return SL2_OK;
}

// A snapshot load gives streams [lo, lo + cnt) the blobs' cameras: a stream with a source then resizes to its new image
static int loaded_cameras(sl2_ctx *c, int lo, const std::vector<sl2_stream_config> &cams) {
  bool resized = false;
  for (size_t i = 0; i < cams.size(); ++i) {
    const sl2_stream_config &old = c->cams[lo + i];
    resized = resized || (c->srcs[lo + i].format != SL2_SRC_GRAY_RING &&
                          (old.width != cams[i].width || old.height != cams[i].height));
    c->cams[lo + i] = cams[i];
  }
  return resized ? install_sources(c, c->srcs) : SL2_OK;
}

int sl2_set_stream_source(sl2_ctx *c, int32_t s, const sl2_stream_source *src) {
  if (bad_stream(c, s) || !src) return fail(c, SL2_ERR_ARG, "sl2_set_stream_source: bad argument");
  const int f = src->format;
  if (f < SL2_SRC_GRAY_RING || f > SL2_SRC_UYVY || src->reserved != 0)
    return fail(c, SL2_ERR_ARG, "sl2_set_stream_source: unknown format or non-zero reserved field");
  if (f == SL2_SRC_GRAY_RING ? (src->width != 0 || src->height != 0)
                             : (src->width < 1 || src->height < 1 || src->width > SL2_MAX_SOURCE_DIM ||
                                src->height > SL2_MAX_SOURCE_DIM))
    return fail(c, SL2_ERR_ARG,
                "sl2_set_stream_source: size must be 0 x 0 for the default source, else in [1, SL2_MAX_SOURCE_DIM]");
  if (f == SL2_SRC_UYVY && (src->width & 1))
    return fail(c, SL2_ERR_ARG, "sl2_set_stream_source: a UYVY frame has an even width");
  std::vector<sl2_stream_source> srcs = c->srcs;
  srcs[s] = *src;
  return install_sources(c, srcs);
}

int sl2_get_stream_source(sl2_ctx *c, int32_t s, sl2_stream_source *src) {
  if (bad_stream(c, s) || !src) return fail(c, SL2_ERR_ARG, "sl2_get_stream_source: bad argument");
  *src = c->srcs[s];
  return SL2_OK;
}

int sl2_frame_set_layout(sl2_ctx *c, size_t *offsets) {
  enter(c);
  if (!c || !offsets) return fail(c, SL2_ERR_ARG, "sl2_frame_set_layout: bad argument");
  std::copy(c->layout.begin(), c->layout.end(), offsets);
  return SL2_OK;
}

int sl2_get_stream_config(sl2_ctx *c, int32_t s, sl2_stream_config *sc) {
  if (bad_stream(c, s) || !sc) return fail(c, SL2_ERR_ARG, "sl2_get_stream_config: bad argument");
  *sc = c->cams[s];
  return SL2_OK;
}

// ---- match consensus ----------------------------------------------------------------------------
int sl2_set_stream_consensus(sl2_ctx *c, int32_t s, double inlier_px) {
  if (bad_stream(c, s)) return fail(c, SL2_ERR_ARG, "sl2_set_stream_consensus: bad stream");
  if (!std::isfinite(inlier_px) || inlier_px < 0.0)
    return fail(c, SL2_ERR_ARG, "sl2_set_stream_consensus: the inlier radius must be finite and >= 0");
  const double tau = inlier_px == 0.0 ? 0.0 : inlier_px;  // -0 is off like +0
  CU_TRY(c, sl2_launch_kernel(write_double_kernel, dim3(1), dim3(1), 0, queue(c), false, c->cons_tau2 + s, tau * tau));
  c->cons_tau[s] = tau;
  return SL2_OK;
}

int sl2_get_stream_consensus(sl2_ctx *c, int32_t s, double *inlier_px) {
  if (bad_stream(c, s) || !inlier_px) return fail(c, SL2_ERR_ARG, "sl2_get_stream_consensus: bad argument");
  *inlier_px = c->cons_tau[s];
  return SL2_OK;
}

// ---- frames -----------------------------------------------------------------------------------
int sl2_set_frame(sl2_ctx *c, int32_t s, int32_t slot, const uint8_t *gray, size_t stride) {
  if (bad_stream(c, s) || bad_slot(c, slot) || !gray) return fail(c, SL2_ERR_ARG, "sl2_set_frame: bad argument");
  const Sl2Dev &d = c->d;
  if (c->srcs[s].format != SL2_SRC_GRAY_RING) {  // the raw frame to the slot's staging, then its conversion
    int j = 0;
    while (c->src_rows[j].stream != s) ++j;
    const Sl2Source &r = c->src_rows[j];
    const size_t rb = (size_t)r.sw * sl2_source_bpp(r.format);
    CU_TRY(c, cudaMemcpy2DAsync(source_stage(c, slot) + r.off, rb, gray, stride, rb, r.sh, cudaMemcpyHostToDevice,
                                c->stream));
    CU_TRY(c, ingest(c, slot, j, 1, queue(c)));
  } else {
    uint8_t *dst = d.frames + ((size_t)slot * d.B + s) * d.H * d.pitch;
    const sl2_stream_config &sc = c->cams[s];  // the stream's image, top-left of its block
    CU_TRY(c, cudaMemcpy2DAsync(dst, d.pitch, gray, stride, sc.width, sc.height, cudaMemcpyHostToDevice, c->stream));
  }
  CU_TRY(c, cudaEventRecord(c->ev_slot[slot].cmp.get(), c->stream));  // slot busy until the copy has landed
  return SL2_OK;
}

static int set_frames_any(sl2_ctx *c, int32_t slot, const uint8_t *gray, cudaMemcpyKind kind) {
  enter(c);
  if (!c || bad_slot(c, slot) || !gray) return fail(c, SL2_ERR_ARG, "sl2_set_frames: bad argument");
  CU_TRY(c, copy_slot_frames(c, slot, gray, kind, queue(c)));
  CU_TRY(c, cudaEventRecord(c->ev_slot[slot].cmp.get(), c->stream));  // slot busy until the copy has landed
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
  CU_TRY(c, sl2_launch_cull(c->d, s, 1, index, queue(c)));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return SL2_OK;
}

int sl2_append_feature(sl2_ctx *c, int32_t s, const double *y, const double *xp_org, const uint8_t *patch,
                       const double *Pcol) {
  if (bad_stream(c, s) || !y || !xp_org || !patch) return fail(c, SL2_ERR_ARG, "sl2_append_feature: bad argument");
  const int nf = sl2_num_features(c, s);
  if (nf < 0) return nf;
  if (nf >= c->cfg.max_features) return fail(c, SL2_ERR_STATE, "sl2_append_feature: the map is full (max_features)");
  const int box = c->d.box, n3 = SL2_NXV + 3 * nf + 3;
  Stage ys{STAGE_IN, 24, y}, xs{STAGE_IN, 56, xp_org}, pc{STAGE_IN, Pcol ? 8 * 3 * (size_t)n3 : 0, Pcol},
      rows{STAGE_IN, (size_t)box * 16};
  const int rc = staged_call(
      c, {&ys, &xs, &pc, &rows}, [&] { pack_patch_rows(rows.h, patch, 1, box); },
      [&] {
        CU_TRY(c, sl2_launch_append(c->d, s, ys.dev<double>(), xs.dev<double>(), rows.d,
                                    Pcol ? pc.dev<double>() : nullptr, queue(c)));
        return SL2_OK;
      });
  return rc ? rc : nf;  // index of the new feature
}

// ---- patch search -----------------------------------------------------------------------------
int sl2_patch_search(sl2_ctx *c, int32_t s, int32_t slot, int32_t n, const int32_t *feat_index,
                     const double *centre, const double *PuInv3, int32_t *u, int32_t *v,
                     uint8_t *found, double *best) {
  if (n > 0 && !feat_index) return fail(c, SL2_ERR_ARG, "sl2_patch_search: feat_index is null");
  if (bad_stream(c, s) || bad_slot(c, slot) || n < 0 || !centre || !PuInv3)
    return fail(c, SL2_ERR_ARG, "patch search: bad argument");
  if (n == 0) return SL2_OK;
  int nf = 0;
  int rc = device_nfeat(c, s, &nf);
  if (rc) return rc;
  for (int i = 0; i < n; ++i)
    if (feat_index[i] < 0 || feat_index[i] >= nf) return fail(c, SL2_ERR_ARG, "patch search: feature index out of range");
  const size_t N = n;
  Stage ce{STAGE_IN, 16 * N, centre}, pu{STAGE_IN, 24 * N, PuInv3}, fe{STAGE_IN, 4 * N, feat_index},
      uv{STAGE_OUT, 8 * N}, fd{STAGE_OUT, N}, be{STAGE_OUT, 8 * N};
  rc = staged_call(c, {&ce, &pu, &fe, &uv, &fd, &be}, [] {}, [&] {
    SearchLaunch L = {};
    L.job_centre = ce.dev<double>();
    L.job_puinv = pu.dev<double>();
    L.job_feat = fe.dev<int>();
    L.jobs_per_stream = n;
    L.stream_lo = s;
    L.stream_cnt = 1;
    L.slot = slot;
    L.out_uv = uv.dev<int>();
    L.out_found = fd.d;
    L.out_best = be.dev<double>();
    L.scatter_to_features = 0;
    CU_TRY(c, sl2_launch_search(c->d, c->tmap, L, queue(c)));
    return SL2_OK;
  });
  if (rc) return rc;
  for (int i = 0; i < n; ++i) {
    if (u) u[i] = uv.host<int>()[2 * i];
    if (v) v[i] = uv.host<int>()[2 * i + 1];
    if (found) found[i] = fd.h[i];
    if (best) best[i] = be.host<double>()[i];
  }
  return SL2_OK;
}

// ---- relocalisation ---------------------------------------------------------------------------------------------
int sl2_relocalise(sl2_ctx *c, const int32_t *ids, int32_t cnt, int32_t slot, const sl2_reloc_params *p,
                   const double *Pxx, sl2_reloc_result *out, int32_t *z_uv, uint8_t *flags) {
  enter(c);
  if (!c || cnt < 0 || (cnt > 0 && !ids) || bad_slot(c, slot) || !p || !Pxx || !out)
    return fail(c, SL2_ERR_ARG, "sl2_relocalise: bad argument");
  const Sl2Dev &d = c->d;
  std::vector<char> seen(d.B, 0);
  int lo = d.B, hi = -1;
  for (int i = 0; i < cnt; ++i) {
    const int s = ids[i];
    if (s < 0 || s >= d.B || seen[s]) return fail(c, SL2_ERR_ARG, "sl2_relocalise: bad or repeated stream id");
    seen[s] = 1;
    lo = std::min(lo, s);
    hi = std::max(hi, s);
  }
  if (!(p->inlier_px > 0.0) || !std::isfinite(p->inlier_px))
    return fail(c, SL2_ERR_ARG, "sl2_relocalise: inlier_px must be finite and > 0");
  if (p->min_inliers < 4 || p->reserved != 0)
    return fail(c, SL2_ERR_ARG, "sl2_relocalise: min_inliers must be >= 4 and reserved 0");
  for (int i = 0; i < 3; ++i)
    if (!std::isfinite(p->v[i]) || !std::isfinite(p->omega[i]))
      return fail(c, SL2_ERR_ARG, "sl2_relocalise: v and omega must be finite");
  if (!(std::sqrt(p->omega[0] * p->omega[0] + p->omega[1] * p->omega[1] + p->omega[2] * p->omega[2]) > 0.0))
    return fail(c, SL2_ERR_ARG, "sl2_relocalise: |omega| must be > 0");
  for (int i = 0; i < 13; ++i)
    for (int j = 0; j < 13; ++j)
      if (!std::isfinite(Pxx[i + 13 * j]) || Pxx[i + 13 * j] != Pxx[j + 13 * i])
        return fail(c, SL2_ERR_ARG, "sl2_relocalise: Pxx must be finite and symmetric");
  if (!psd13(Pxx)) return fail(c, SL2_ERR_ARG, "sl2_relocalise: Pxx is not positive semi-definite");
  if (cnt == 0) return SL2_OK;
  // one search job per feature of every listed stream over the id range [lo, hi], empty jobs elsewhere
  const int R = hi - lo + 1;
  std::vector<int> nf(R);
  CU_TRY(c, cudaMemcpyAsync(nf.data(), d.nfeat + lo, sizeof(int) * R, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  const size_t nj = (size_t)R * d.Nmax, nc = cnt, no = nc * d.Nmax;
  Stage is{STAGE_IN, 4 * nc, ids}, ps{STAGE_IN, sizeof(sl2_reloc_params), p}, px{STAGE_IN, 8 * 169, Pxx},
      jf{STAGE_IN, 4 * nj}, jc{STAGE_IN, 16 * nj}, jp{STAGE_IN, 24 * nj}, rs{STAGE_OUT, sizeof(sl2_reloc_result) * nc},
      zo{STAGE_OUT, 8 * no}, fo{STAGE_OUT, no}, su{STAGE_DEV, 8 * nj}, sf{STAGE_DEV, nj};
  auto pack = [&] {
    for (int r = 0; r < R; ++r) {
      const int s = lo + r;
      const sl2_stream_config &sc = c->cams[s];
      const double eps = 9.0 / ((double)sc.width * sc.width + (double)sc.height * sc.height);
      for (int f = 0; f < d.Nmax; ++f) {
        const size_t j = (size_t)r * d.Nmax + f;
        jf.host<int>()[j] = seen[s] && f < nf[r] ? f : -1;
        jc.host<double>()[2 * j] = 0.5 * (sc.width - 1);
        jc.host<double>()[2 * j + 1] = 0.5 * (sc.height - 1);
        jp.host<double>()[3 * j] = eps;
        jp.host<double>()[3 * j + 1] = 0.0;
        jp.host<double>()[3 * j + 2] = eps;
      }
    }
  };
  const int rc = staged_call(c, {&is, &ps, &px, &jf, &jc, &jp, &rs, &zo, &fo, &su, &sf}, pack, [&] {
    SearchLaunch L = {};
    L.job_feat = jf.dev<int>();
    L.job_centre = jc.dev<double>();
    L.job_puinv = jp.dev<double>();
    L.jobs_per_stream = d.Nmax;
    L.stream_lo = lo;
    L.stream_cnt = R;
    L.slot = slot;
    L.out_uv = su.dev<int>();
    L.out_found = sf.d;
    L.scatter_to_features = 0;
    CU_TRY(c, sl2_launch_search(d, c->tmap, L, queue(c)));
    CU_TRY(c, sl2_launch_reloc(d, cnt, is.dev<int>(), lo, su.dev<int>(), sf.d, ps.dev<sl2_reloc_params>(),
                               px.dev<double>(), rs.dev<sl2_reloc_result>(), zo.dev<int>(), fo.d, queue(c)));
    return SL2_OK;
  });
  if (rc) return rc;
  memcpy(out, rs.h, rs.bytes);
  if (z_uv) memcpy(z_uv, zo.h, zo.bytes);
  if (flags) memcpy(flags, fo.h, fo.bytes);
  return SL2_OK;
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
  if (predict) {
    memcpy(io.h, h.h, h.bytes);
    memcpy(io.Sinv3, Sinv3.h, Sinv3.bytes);
    memcpy(io.detS, detS.h, detS.bytes);
  }
  if (reweight) {
    memcpy(io.prob, prob.h, prob.bytes);
    if (io.cumulative) memcpy(io.cumulative, cum.h, cum.bytes);
    if (io.mean_var) memcpy(io.mean_var, mv.h, mv.bytes);
    if (io.keep) memcpy(io.keep, keep.h, keep.bytes);
    if (io.left) memcpy(io.left, left.h, left.bytes);
  }
  if (io.z_uv) memcpy(io.z_uv, uv.h, uv.bytes);
  if (io.found) memcpy(io.found, found.h, found.bytes);
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
  Stage ce{STAGE_IN, 16, centre}, pu{STAGE_IN, 24, PuInv3}, fe{STAGE_IN, 4, &feat}, bx{STAGE_OUT, 24},
      co{STAGE_OUT, 8 * cap}, sd{STAGE_OUT, 8 * cap}, in{STAGE_OUT, cap};
  rc = staged_call(c, {&ce, &pu, &fe, &bx, &co, &sd, &in}, [] {}, [&] {
    CU_TRY(c, cudaMemsetAsync(bx.d, 0xff, in.d + cap - bx.d, c->stream));  // NaN / 0xff fill of every output
    CU_TRY(c, sl2_launch_score_map(c->d, c->tmap, s, slot, ce.dev<double>(), pu.dev<double>(), fe.dev<int>(),
                                   bx.dev<int>(), co.dev<double>(), sd.dev<double>(), in.d, (int)cap, queue(c)));
    return SL2_OK;
  });
  if (rc) return rc;
  memcpy(box6, bx.h, 24);
  if (corr) memcpy(corr, co.h, 8 * cap);
  if (sd_image) memcpy(sd_image, sd.h, 8 * cap);
  if (inside) memcpy(inside, in.h, cap);
  return SL2_OK;
}

int sl2_find_best_patch(sl2_ctx *c, int32_t s, int32_t slot, int32_t n, const int32_t *regions,
                        int32_t *ubest, int32_t *vbest, double *evbest) {
  if (bad_stream(c, s) || bad_slot(c, slot) || n < 0 || (n && (!regions || !evbest)))
    return fail(c, SL2_ERR_ARG, "sl2_find_best_patch: bad argument");
  if (n == 0) return SL2_OK;
  Stage rg{STAGE_IN, 16 * (size_t)n, regions}, uv{STAGE_OUT, 8 * (size_t)n}, ev{STAGE_OUT, 8 * (size_t)n},
      scratch{STAGE_DEV, sl2_detect_scratch_bytes(c->d, n)};
  const int rc = staged_call(c, {&rg, &uv, &ev, &scratch}, [] {}, [&] {
    CU_TRY(c, sl2_launch_detect(c->d, s, slot, n, rg.dev<int>(), uv.dev<int>(), ev.dev<double>(), scratch.d, queue(c)));
    return SL2_OK;
  });
  if (rc) return rc;
  for (int i = 0; i < n; ++i) {
    evbest[i] = ev.host<double>()[i];
    if (uv.host<int>()[2 * i] >= 0) {
      if (ubest) ubest[i] = uv.host<int>()[2 * i];
      if (vbest) vbest[i] = uv.host<int>()[2 * i + 1];
    }
  }
  return SL2_OK;
}

// ---- EKF ----------------------------------------------------------------------------------------
int sl2_ekf_predict(sl2_ctx *c, int32_t s, const double *u3) {
  if (bad_stream(c, s)) return fail(c, SL2_ERR_ARG, "bad stream");
  Stage u{STAGE_IN, u3 ? (size_t)24 : 0, u3};
  return staged_call(c, {&u}, [] {}, [&] {
    CU_TRY(c, sl2_launch_predict(c->d, s, 1, u3 ? u.dev<double>() : nullptr, 1, 0, queue(c)));
    return SL2_OK;
  });
}

int sl2_predict_measurements(sl2_ctx *c, int32_t s) {
  if (bad_stream(c, s)) return fail(c, SL2_ERR_ARG, "bad stream");
  CU_TRY(c, sl2_launch_predict(c->d, s, 1, nullptr, 0, 1, queue(c)));
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
  CU_TRY(c, sl2_launch_search(d, c->tmap, L, queue(c)));
  if (c->cons_tau[s] > 0.0) CU_TRY(c, sl2_launch_consensus(d, s, 1, c->cons_tau2, queue(c)));
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

int sl2_ekf_update(sl2_ctx *c, int32_t s, int32_t m, const int32_t *feat_index, const double *H_xv,
                   const double *H_y, const double *R, const double *nu) {
  if (bad_stream(c, s) || m < 0 || (m & 1) || m > c->d.mmax)
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
  const size_t k = K;
  Stage hx{STAGE_IN, 8 * 26 * k, H_xv}, hy{STAGE_IN, 8 * 6 * k, H_y}, r{STAGE_IN, 8 * 4 * k, R},
      v{STAGE_IN, 8 * 2 * k, nu}, fe{STAGE_IN, 4 * k, feat_index};
  return staged_call(c, {&hx, &hy, &r, &v, &fe}, [] {}, [&] {
    CU_TRY(c, sl2_launch_update(c->d, s, 1, m, fe.dev<int>(), hx.dev<double>(), hy.dev<double>(), r.dev<double>(),
                                v.dev<double>(), 0, queue(c)));
    return SL2_OK;
  });
}

int sl2_ekf_update_measured(sl2_ctx *c, int32_t s) {
  if (bad_stream(c, s)) return fail(c, SL2_ERR_ARG, "bad stream");
  CU_TRY(c, sl2_launch_update(c->d, s, 1, -1, nullptr, nullptr, nullptr, nullptr, nullptr, 0, queue(c)));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return SL2_OK;
}

int sl2_normalise_state(sl2_ctx *c, int32_t s) {
  if (bad_stream(c, s)) return fail(c, SL2_ERR_ARG, "bad stream");
  CU_TRY(c, sl2_launch_update(c->d, s, 1, -1, nullptr, nullptr, nullptr, nullptr, nullptr, 1, queue(c)));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return SL2_OK;
}

// ---- fused step ---------------------------------------------------------------------------------
static int step_group(sl2_ctx *c, int32_t slot, int lo, int cnt, Sl2Queue q, cudaEvent_t after_search, bool t) {
  const Sl2Dev &d = c->d;
  const cudaStream_t st = q.stream;
  if (t) CU_TRY(c, cudaEventRecord(c->ev[0].get(), st));
  CU_TRY(c, sl2_launch_predict(d, lo, cnt, nullptr, 1, 1, q));
  if (t) CU_TRY(c, cudaEventRecord(c->ev[1].get(), st));
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
  CU_TRY(c, sl2_launch_search(d, c->tmap, L, q));
  if (consensus_on(c, lo, cnt))  // part of the search's time: the update times still sum to ev[2] .. ev[3]
    CU_TRY(c, sl2_launch_consensus(d, lo, cnt, c->cons_tau2, q));
  if (t) CU_TRY(c, cudaEventRecord(c->ev[2].get(), st));
  if (after_search) CU_TRY(c, cudaEventRecord(after_search, st));
  cudaEvent_t evu[6];
  for (int i = 0; i < 6; ++i) evu[i] = c->evu[i].get();
  CU_TRY(c, sl2_launch_update(d, lo, cnt, -1, nullptr, nullptr, nullptr, nullptr, nullptr, 0, q, t ? evu : nullptr));
  if (t) CU_TRY(c, cudaEventRecord(c->ev[3].get(), st));
  CU_TRY(c, sl2_launch_cull(d, lo, cnt, -1, q));
  if (t) CU_TRY(c, cudaEventRecord(c->ev[4].get(), st));
  if (d.rec_depth)  // after ev[4]: the step times keep their meaning
    CU_TRY(c, sl2_launch_records(d, lo, cnt, c->rec_steps, q));
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
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  for (int i = 0; i < nf; ++i) {
    if (h) { h[2 * i] = hh[2 * i]; h[2 * i + 1] = hh[2 * i + 1]; }
    if (z) { z[2 * i] = (double)zz[2 * i]; z[2 * i + 1] = (double)zz[2 * i + 1]; }
    if (S) for (int k = 0; k < 4; ++k) S[4 * i + k] = SS[4 * i + k];
    if (flags) flags[i] = (uint8_t)((rk[i] >= 0 ? 1 : 0) | (fd[i] == 1 ? 2 : 0) | (fd[i] == 2 ? 4 : 0));
    if (attempted) attempted[i] = at[i];
    if (successful) successful[i] = su[i];
    if (select_rank) select_rank[i] = rk[i];
  }
  return nf;
}

// ---- stream snapshots ---------------------------------------------------------------------------
static bool bad_range(sl2_ctx *c, int32_t lo, int32_t cnt) {
  enter(c);
  return !c || lo < 0 || cnt < 0 || lo > c->cfg.num_streams - cnt;
}

// Checks the header of one blob (and, with `index`, its job_feat / sel_rank) against this context; fills `q` with
// the validated counts for stream s.  `blob` is host memory of at least `avail` bytes, any alignment.
static int snap_validate(sl2_ctx *c, const uint8_t *blob, size_t stride, bool index, int s, Sl2SnapLoad *q,
                         const std::string &who) {
  sl2_snapshot_header h;
  memcpy(&h, blob, sizeof h);
  if (h.magic != SL2_SNAPSHOT_MAGIC || h.version != SL2_SNAPSHOT_VERSION || h.header_bytes != sizeof h)
    return fail(c, SL2_ERR_ARG, who + ": not a snapshot of this version and byte order");
  if (h.reserved0 != 0 || h.reserved1 != 0) return fail(c, SL2_ERR_ARG, who + ": reserved header fields are not 0");
  if (h.total_bytes > stride) return fail(c, SL2_ERR_ARG, who + ": blob larger than the stride");
  if (h.nfeat < 0 || h.nsel < 0 || h.nvisible < 0 || h.nmeas < 0 || h.ncull < 0)
    return fail(c, SL2_ERR_ARG, who + ": negative count");
  if ((int64_t)h.n != SL2_NXV + 3 * (int64_t)h.nfeat) return fail(c, SL2_ERR_ARG, who + ": n != 13 + 3 nfeat");
  if (h.boxsize != c->cfg.boxsize) return fail(c, SL2_ERR_ARG, who + ": boxsize differs from the context's");
  if (h.nfeat > c->cfg.max_features) return fail(c, SL2_ERR_STATE, who + ": map larger than max_features");
  const Sl2SnapLayout L = sl2_snap_layout(h.nfeat, h.boxsize);
  if (h.total_bytes != L.total) return fail(c, SL2_ERR_ARG, who + ": total size does not match nfeat and boxsize");
  // the counts are not renewed by a cull, sl2_delete_feature or sl2_set_features, so they are bounded by what any
  // prediction / update can produce, not by nfeat (include/sl2b200.h)
  if (h.nsel > SL2_MAX_MEASURED || h.nmeas > SL2_MAX_MEASURED || h.nvisible > SL2_MAX_FEATURES ||
      h.ncull > SL2_MAX_FEATURES)
    return fail(c, SL2_ERR_ARG, who + ": count above what a step can produce");
  const int rc = check_stream_config(c, &h.cam, who);
  if (rc) return rc;
  if (index) {
    for (int f = 0; f < h.nfeat; ++f) {
      int32_t r, j;
      memcpy(&r, blob + L.field[SL2_FIELD_sel_rank] + 4 * (size_t)f, 4);
      memcpy(&j, blob + L.field[SL2_FIELD_job_feat] + 4 * (size_t)f, 4);
      // the same rules as snap_check_kernel: a job below nsel may be empty, the cull writes job slot sel_rank
      if (!(r == -1 || (r >= 0 && r < h.nsel && r < h.nfeat)) || !(f < h.nsel ? (j >= -1 && j < h.nfeat) : j == -1))
        return fail(c, SL2_ERR_ARG, who + ": sel_rank or job_feat out of range");
    }
  }
  memset(q, 0, sizeof *q);
  q->cam = cam_row(h.cam);
  q->stream = s;
  q->nfeat = h.nfeat;
  q->nsel = h.nsel;
  q->nvisible = h.nvisible;
  q->nmeas = h.nmeas;
  q->ncull = h.ncull;
  return SL2_OK;
}

size_t sl2_snapshot_bytes(const sl2_ctx *c) { return c ? sl2_snap_layout(c->cfg.max_features, c->cfg.boxsize).total : 0; }

int sl2_snapshot_layout(int32_t nfeat, int32_t boxsize, sl2_snapshot_sections *out) {
  if (nfeat < 0 || nfeat > SL2_MAX_FEATURES || boxsize <= 0 || !out) return SL2_ERR_ARG;
  const Sl2SnapLayout L = sl2_snap_layout(nfeat, boxsize);
  out->x = L.x;
  out->P = L.P;
  for (int k = 0; k < SL2_SNAPSHOT_FIELDS; ++k) out->field[k] = L.field[k];
  out->templates = L.templates;
  out->total = L.total;
  return SL2_OK;
}

// The host forms stage groups of streams of at most this many bytes (at least one stream), so a save or load of a
// whole large context does not grow the staging buffers to the size of all its blobs.
static const size_t SL2_SNAP_STAGE_BYTES = (size_t)64 << 20;
static int snap_group(size_t sb) { return (int)std::max<size_t>(1, SL2_SNAP_STAGE_BYTES / sb); }

int sl2_save_streams(sl2_ctx *c, int32_t lo, int32_t cnt, void *buf, size_t stride, size_t *sizes) {
  if (bad_range(c, lo, cnt) || (cnt && !buf)) return fail(c, SL2_ERR_ARG, "sl2_save_streams: bad argument");
  const size_t sb = sl2_snapshot_bytes(c);
  if (stride < sb) return fail(c, SL2_ERR_ARG, "sl2_save_streams: stride below sl2_snapshot_bytes");
  if (cnt == 0) return SL2_OK;
  const int g = std::min(cnt, snap_group(sb));
  int rc = stage_reserve(c, (size_t)g * sb);
  if (rc) return rc;
  CU_TRY(c, cudaStreamSynchronize(c->stream));  // staging buffer reuse
  for (int i0 = 0; i0 < cnt; i0 += g) {
    const int k = std::min(g, cnt - i0);
    CU_TRY(c, sl2_launch_pack(c->d, lo + i0, k, c->stg_dev.get(), sb, queue(c)));
    CU_TRY(c, cudaMemcpyAsync(c->stg_host.get(), c->stg_dev.get(), (size_t)k * sb, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    for (int i = 0; i < k; ++i) {
      sl2_snapshot_header h;
      memcpy(&h, c->stg_host.get() + (size_t)i * sb, sizeof h);
      memcpy(static_cast<uint8_t *>(buf) + (size_t)(i0 + i) * stride, c->stg_host.get() + (size_t)i * sb, h.total_bytes);
      if (sizes) sizes[i0 + i] = h.total_bytes;
    }
  }
  return SL2_OK;
}

int sl2_save_streams_dev(sl2_ctx *c, int32_t lo, int32_t cnt, void *buf_dev, size_t stride) {
  if (bad_range(c, lo, cnt) || (cnt && !buf_dev) || ((uintptr_t)buf_dev & 7) || (stride & 7))
    return fail(c, SL2_ERR_ARG, "sl2_save_streams_dev: bad argument");
  if (stride < sl2_snapshot_bytes(c)) return fail(c, SL2_ERR_ARG, "sl2_save_streams_dev: stride below sl2_snapshot_bytes");
  if (cnt == 0) return SL2_OK;
  CU_TRY(c, sl2_launch_pack(c->d, lo, cnt, static_cast<uint8_t *>(buf_dev), stride, queue(c)));
  return SL2_OK;
}


int sl2_load_streams(sl2_ctx *c, int32_t lo, int32_t cnt, const void *buf, size_t stride) {
  if (bad_range(c, lo, cnt) || (cnt && !buf) || stride < sizeof(sl2_snapshot_header))
    return fail(c, SL2_ERR_ARG, "sl2_load_streams: bad argument");
  if (cnt == 0) return SL2_OK;
  const uint8_t *in = static_cast<const uint8_t *>(buf);
  std::vector<Sl2SnapLoad> q(cnt);
  std::vector<sl2_stream_config> cams(cnt);
  for (int i = 0; i < cnt; ++i) {
    const int rc = snap_validate(c, in + (size_t)i * stride, stride, true, lo + i, &q[i], "sl2_load_streams");
    if (rc) return rc;
    memcpy(&cams[i], in + (size_t)i * stride + offsetof(sl2_snapshot_header, cam), sizeof(sl2_stream_config));
  }
  // staging, one group of streams at a time: its load records, then its blobs at the context's snapshot size
  const size_t sb = sl2_snapshot_bytes(c);
  const int g = std::min(cnt, snap_group(sb));
  const size_t pb = ((size_t)g * sizeof(Sl2SnapLoad) + 255) & ~(size_t)255;
  int rc = stage_reserve(c, pb + (size_t)g * sb);
  if (rc) return rc;
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  for (int i0 = 0; i0 < cnt; i0 += g) {
    const int k = std::min(g, cnt - i0);
    CU_TRY(c, cudaStreamSynchronize(c->stream));  // the previous group's unpack has read the staging buffer
    memcpy(c->stg_host.get(), q.data() + i0, (size_t)k * sizeof(Sl2SnapLoad));
    size_t end = 0;
    for (int i = 0; i < k; ++i) {
      const size_t tb = sl2_snap_layout(q[i0 + i].nfeat, c->cfg.boxsize).total;
      memcpy(c->stg_host.get() + pb + (size_t)i * sb, in + (size_t)(i0 + i) * stride, tb);
      end = pb + (size_t)i * sb + tb;
    }
    CU_TRY(c, cudaMemcpyAsync(c->stg_dev.get(), c->stg_host.get(), end, cudaMemcpyHostToDevice, c->stream));
    CU_TRY(c, sl2_launch_unpack(c->d, k, reinterpret_cast<const Sl2SnapLoad *>(c->stg_dev.get()),
                                c->stg_dev.get() + pb, sb, queue(c)));
  }
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return loaded_cameras(c, lo, cams);
}

int sl2_load_streams_dev(sl2_ctx *c, int32_t lo, int32_t cnt, const void *buf_dev, size_t stride) {
  if (bad_range(c, lo, cnt) || (cnt && !buf_dev) || ((uintptr_t)buf_dev & 7) || (stride & 7) ||
      stride < sizeof(sl2_snapshot_header))
    return fail(c, SL2_ERR_ARG, "sl2_load_streams_dev: bad argument");
  if (cnt == 0) return SL2_OK;
  const uint8_t *in = static_cast<const uint8_t *>(buf_dev);
  const size_t hb = sizeof(sl2_snapshot_header);
  // staging: load records | verdict (int) | headers copied down
  const size_t pb = ((size_t)cnt * sizeof(Sl2SnapLoad) + 255) & ~(size_t)255, o_bad = pb, o_h = pb + 256;
  int rc = stage_reserve(c, o_h + (size_t)cnt * hb);
  if (rc) return rc;
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  CU_TRY(c, cudaMemcpy2DAsync(c->stg_host.get() + o_h, hb, in, stride, hb, cnt, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  std::vector<Sl2SnapLoad> q(cnt);
  std::vector<sl2_stream_config> cams(cnt);
  for (int i = 0; i < cnt; ++i) {
    const uint8_t *h = c->stg_host.get() + o_h + (size_t)i * hb;
    rc = snap_validate(c, h, stride, false, lo + i, &q[i], "sl2_load_streams_dev");
    if (rc) return rc;
    memcpy(&cams[i], h + offsetof(sl2_snapshot_header, cam), sizeof(sl2_stream_config));
  }
  memcpy(c->stg_host.get(), q.data(), (size_t)cnt * sizeof(Sl2SnapLoad));
  memset(c->stg_host.get() + o_bad, 0, sizeof(int));
  CU_TRY(c, cudaMemcpyAsync(c->stg_dev.get(), c->stg_host.get(), o_bad + sizeof(int), cudaMemcpyHostToDevice, c->stream));
  const Sl2SnapLoad *q_dev = reinterpret_cast<const Sl2SnapLoad *>(c->stg_dev.get());
  int *bad_dev = reinterpret_cast<int *>(c->stg_dev.get() + o_bad);
  CU_TRY(c, sl2_launch_snap_check(c->d, cnt, q_dev, in, stride, bad_dev, queue(c)));
  int bad = 0;
  CU_TRY(c, cudaMemcpyAsync(&bad, bad_dev, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  if (bad) return fail(c, SL2_ERR_ARG, "sl2_load_streams_dev: sel_rank or job_feat out of range");
  CU_TRY(c, sl2_launch_unpack(c->d, cnt, q_dev, in, stride, queue(c)));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return loaded_cameras(c, lo, cams);
}

// ---- step records -------------------------------------------------------------------------------
int sl2_enable_records(sl2_ctx *c, int32_t depth) {
  if (!c) return SL2_ERR_ARG;
  enter(c);
  if (depth < 0 || depth > SL2_MAX_RECORDS)
    return fail(c, SL2_ERR_ARG, "sl2_enable_records: depth outside [0, SL2_MAX_RECORDS]");
  // the new ring first, so that a failed allocation leaves the old one in place
  DevPtr<sl2_step_record> ring;
  cudaError_t e = cudaSuccess;
  if (depth) {
    const size_t bytes = (size_t)c->d.B * depth * sizeof(sl2_step_record);
    CU_TRY(c, cuda_malloc(ring, bytes));
    e = cudaMemsetAsync(ring.get(), 0, bytes, c->stream);
  }
  // steps queued before the call (either group: enter() joined them) have written the old ring
  if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
  if (e != cudaSuccess) return fail(c, SL2_ERR_CUDA, std::string("sl2_enable_records: ") + cudaGetErrorString(e));
  c->rec = std::move(ring);
  c->d.rec = c->rec.get();
  c->d.rec_depth = depth;
  c->rec_steps = 0;
  return SL2_OK;
}

// The most recent k records of streams [lo, lo + cnt), oldest first, as one or two 2-D copies (two when the k rows
// wrap around the end of the ring): row pitch `depth` records in the ring, `mx` records in the output.
static int get_records(sl2_ctx *c, int32_t lo, int32_t cnt, int32_t mx, void *out, cudaMemcpyKind kind,
                       const char *who) {
  if (bad_range(c, lo, cnt) || !out || mx < 1 ||
      (kind == cudaMemcpyDeviceToDevice && ((uintptr_t)out & 7)))
    return fail(c, SL2_ERR_ARG, std::string(who) + ": bad argument");
  const int64_t depth = c->d.rec_depth;
  if (!depth) return fail(c, SL2_ERR_STATE, std::string(who) + ": records are off (sl2_enable_records)");
  const int k = (int)std::min<int64_t>(std::min<int64_t>(mx, c->rec_steps), depth);
  if (k == 0 || cnt == 0) return k;
  const size_t R = sizeof(sl2_step_record);
  const int r0 = (int)((c->rec_steps - k) % depth);  // ring row of the oldest record returned
  const int k1 = (int)std::min<int64_t>(k, depth - r0);
  const sl2_step_record *src = c->d.rec + (size_t)lo * depth;
  uint8_t *dst = static_cast<uint8_t *>(out);
  CU_TRY(c, cudaMemcpy2DAsync(dst, (size_t)mx * R, src + r0, (size_t)depth * R, (size_t)k1 * R, cnt, kind, c->stream));
  if (k1 < k)
    CU_TRY(c, cudaMemcpy2DAsync(dst + (size_t)k1 * R, (size_t)mx * R, src, (size_t)depth * R, (size_t)(k - k1) * R,
                                cnt, kind, c->stream));
  if (kind == cudaMemcpyDeviceToHost) CU_TRY(c, cudaStreamSynchronize(c->stream));
  return k;
}

int sl2_get_records(sl2_ctx *c, int32_t lo, int32_t cnt, int32_t max, sl2_step_record *out) {
  return get_records(c, lo, cnt, max, out, cudaMemcpyDeviceToHost, "sl2_get_records");
}

int sl2_get_records_dev(sl2_ctx *c, int32_t lo, int32_t cnt, int32_t max, void *out_dev) {
  return get_records(c, lo, cnt, max, out_dev, cudaMemcpyDeviceToDevice, "sl2_get_records_dev");
}

}  // extern "C"
