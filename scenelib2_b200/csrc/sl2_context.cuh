// sl2_context.cuh — the context (struct sl2_ctx) and the host helpers the entry points of every file share: owning
// handles, error reporting, the staged-call path and the launch queue.  Host side only; not installed.  The entry
// points live beside the kernels they drive; api.cu keeps creation, the stream configuration, the map and state and
// the fused step.
#pragma once
#include <cstring>
#include <initializer_list>
#include <memory>
#include <string>
#include <vector>

#include "../../include/sl2b200.h"
#include "sl2_common.cuh"

// ---- raw frame sources (ingest.cu): one row per stream with a non-default sl2_stream_source, in stream order -------
struct Sl2Source {
  int stream, format;  // camera stream, SL2_SRC_*
  int sw, sh;          // raw frame size
  int dw, dh;          // the stream's image (sl2_stream_config width_s x height_s): the resize target
  int64_t off;         // byte offset of the raw frame in a slot of the staging area
};

namespace sl2 {

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
cudaError_t cuda_event_create(Event &h, unsigned flags);
cudaError_t cuda_stream_create(Stream &h);

// the events of one frame slot: its frames have landed (h2d), the context's stream or group B is done with it (cmp,
// cmp_b), its camera states have been copied to the host (out)
struct SlotEvents { Event h2d, cmp, cmp_b, out; };

// One camera stream's opt-in settings as their setters accepted them (include/sl2b200.h, the per-stream options); the
// getters read them back and the fused step decides from them which stages a step group runs.  Every stream starts
// with stream_option_defaults().
struct StreamOptions {
  double inlier_px;                // sl2_set_stream_consensus, 0 = off
  double chi2;                     // sl2_set_stream_rescue, 0 = off
  uint8_t warp, subpixel;          // sl2_set_stream_warp, sl2_set_stream_subpixel
  sl2_stream_blur blur;
  sl2_stream_selection sel;
  sl2_stream_gyro gyro;
  sl2_stream_accel accel;
  sl2_stream_iterated iter;
  sl2_stream_recovery recov;
  sl2_stream_normals nrm;
};
StreamOptions stream_option_defaults();

}  // namespace sl2

struct sl2_ctx {
  sl2_config cfg;
  Sl2Dev d;
  std::vector<sl2_stream_config> cams;  // host mirror of d.cams, updated with it
  cudaStream_t stream = nullptr;        // cfg.cuda_stream, else owned_stream
  sl2::Stream owned_stream;             // set only when the context created its stream
  CUtensorMap tmap;
  std::string err;
  std::vector<sl2::DevPtr<void>> allocs;  // behind the Sl2Dev arrays and xv_stage
  // staging
  sl2::DevPtr<uint8_t> stg_dev;   // device scratch for staged API calls
  size_t stg_bytes = 0;
  sl2::HostPtr<uint8_t> stg_host;
  sl2::DevPtr<double> smoe_map;   // [features of the call][W][H] score cache of the SMOE kernels (lazily sized)
  size_t smoe_map_bytes = 0;
  int64_t launches = 0;  // kernels launched: counted by sl2_launch_kernel through every Sl2Queue of the context
  bool timing = false;
  // timing mode: ev[0..4] bracket predict / search / update / cull, evu[0..5] the five update kernels
  sl2::Event ev[5], evu[6];
  // asynchronous end-to-end path: frames of step t+1 are copied while step t computes
  sl2::Stream copy_stream;  // H2D of the frames
  sl2::Stream out_stream;   // D2H of the results (own stream: must not block the next H2D)
  std::vector<sl2::SlotEvents> ev_slot;  // [slots]
  double *xv_stage = nullptr;            // [slots][B][13] device
  // Fused step as two staggered groups of camera streams: group A (first half) on `stream`, group B on
  // `stream_b`; B's predict+search wait for A's search of the same step and A's next step waits for
  // B's search, so the integer-bound search of one group runs under the FP64-bound update of the other
  // and the two update kernels are half a step out of phase.  Results are identical to the serial order
  // (the groups share nothing); every other entry point joins the two streams first (enter()).
  int step_groups = 1;  // off by default: with two streams per SM the update would lose its second CTA per SM
  sl2::Stream stream_b;
  sl2::Event ev_main, ev_a_search, ev_b_search, ev_b_done;
  bool b_pending = false, b_search_valid = false;
  sl2::DevPtr<sl2_step_record> rec;  // the ring d.rec points into
  int64_t rec_steps = 0;             // fused steps recorded since sl2_enable_records
  // raw frame sources (sl2_set_stream_source): the host mirror, the frame-set layout, and the device table of the
  // streams with a non-default source (src_rows, in stream order) with their raw frames' staging
  std::vector<sl2_stream_source> srcs;  // [B]
  std::vector<size_t> layout;           // [B + 1] byte offsets of the streams' frames in a frame set
  std::vector<Sl2Source> src_rows;
  sl2::DevPtr<Sl2Source> src_tab;    // [B]
  sl2::DevPtr<uint8_t> src_stage;    // [slots][src_slot_bytes] + 16 bytes of slack for the kernel's aligned loads
  size_t src_stage_bytes = 0, src_slot_bytes = 0;
  sl2::Event ev_src;                 // recorded on `stream` behind the last table write
  // the per-stream options: every stream's settings, then what the features' kernels read.  The [B] device arrays are
  // allocated with the context; each DevPtr<uint8_t> buffer is allocated by alloc_sections when a stream first turns
  // its feature on, and the pointers after it point into it.
  std::vector<sl2::StreamOptions> opt;  // [B]
  double *cons_tau2 = nullptr;          // [B] consensus: squared inlier radii
  uint8_t *warp_on_dev = nullptr;       // [B]
  sl2_stream_blur *blur_dev = nullptr;  // [B]
  // the job-indexed templates [B][Nmax][box][16] the warp and the blur write and the search reads
  sl2::DevPtr<uint8_t> warp_patches;
  size_t warp_patches_bytes = 0;
  // selection: the sources of the device arrays' copies, the device arrays predict_kernel and select_kernel read, and
  // the factor scratch [B][kmax][Nmax][4] (only when the factors cannot stay in shared memory)
  std::vector<int> sel_mode;              // [B]
  std::vector<double> sel_t;              // [B]
  int *sel_mode_dev = nullptr;            // [B] SL2_SELECT_*
  double *sel_t_dev = nullptr;            // [B] exp2(2 min_bits)
  sl2::DevPtr<double> sel_g;
  size_t sel_g_bytes = 0;
  // rescue: chi2, and the scratch nis1, logdet1, m2 [B] that the second update and the step records use
  double *resc_chi2_dev = nullptr;  // [B]
  sl2::DevPtr<uint8_t> resc_buf;
  Sl2Rescue resc_dev = {};
  // gyroscope: the on flags and settings [B], the sample ring [slots][B] of rates and valid bytes, the W scratch
  // [B][3][ld] and the results nis, status [B]
  sl2::DevPtr<uint8_t> gyro_buf;
  uint8_t *gyro_on_dev = nullptr, *gyro_valid = nullptr;
  Sl2GyroParam *gyro_prm = nullptr;
  double *gyro_rate = nullptr, *gyro_W = nullptr, *gyro_nis = nullptr;
  int *gyro_status = nullptr;
  // accelerometer: the on flags and settings [B], the sample ring [slots][B] of forces and valid bytes and the results
  // a [B][3], status [B]
  sl2::DevPtr<uint8_t> accel_buf;
  uint8_t *accel_on_dev = nullptr, *accel_valid = nullptr;
  Sl2AccelParam *accel_prm = nullptr;
  double *accel_force = nullptr, *accel_a = nullptr;
  int *accel_status = nullptr;
  // sub-pixel refinement: z [B][Nmax][2], refined [B][Nmax] and the on flags [B]
  sl2::DevPtr<uint8_t> subpix_buf;
  Sl2Subpix subpix_dev = {};
  uint8_t *subpix_on_dev = nullptr;
  // iterated update: the settings, the relinearised tables, the iterate and the per-stream results
  sl2::DevPtr<uint8_t> iter_buf;
  Sl2Iter iter_dev = {};
  // recovery: the settings [B], the states [B], the job table [B][Nmax] (feature, centre, ellipse) and the search and
  // pose kernels' outputs [B][Nmax]
  sl2::DevPtr<uint8_t> recov_buf;
  sl2_stream_recovery *recov_set = nullptr;
  sl2_recovery_result *recov_state = nullptr;
  int *recov_job_feat = nullptr, *recov_uv = nullptr, *recov_zuv = nullptr;
  double *recov_job_centre = nullptr, *recov_job_puinv = nullptr;
  uint8_t *recov_found = nullptr, *recov_flags = nullptr;
  // normals: the settings [B], theta, cov, count and status [B][Nmax]
  sl2::DevPtr<uint8_t> nrm_buf;
  Sl2Normals nrm_dev = {};
};

namespace sl2 {

// records `msg` as the context's last error (the create error without a context) and returns `code`
int fail(sl2_ctx *c, int code, const std::string &msg);

#define CU_TRY(c, expr)                                                              \
  do {                                                                               \
    cudaError_t e__ = (expr);                                                        \
    if (e__ != cudaSuccess)                                                          \
      return fail((c), SL2_ERR_CUDA,                                                 \
                  std::string(#expr) + ": " + cudaGetErrorString(e__));             \
  } while (0)

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
bool bad_stream(sl2_ctx *c, int s);         // enters; true for a null context or a stream outside it
bool bad_slot(sl2_ctx *c, int s);           // a frame slot outside the ring
bool bad_range(sl2_ctx *c, int lo, int cnt);  // enters; true for a null context or streams [lo, lo + cnt) outside it

// whether pred(c->opt[s]) holds for some stream s of [lo, lo + cnt)
template <typename Pred> bool any_stream(const sl2_ctx *c, int lo, int cnt, Pred pred) {
  for (int s = lo; s < lo + cnt; ++s)
    if (pred(c->opt[s])) return true;
  return false;
}

// One section of a feature's device buffer: alloc_sections points *ptr at its `bytes`
struct Section {
  template <typename T>
  Section(T **p, size_t n)
      : ptr(p), bytes(n), place([](void *q, uint8_t *at) { *static_cast<T **>(q) = reinterpret_cast<T *>(at); }) {}
  void *ptr;
  size_t bytes;
  void (*place)(void *ptr, uint8_t *at);
};
// A feature's buffer, allocated when a stream first turns the feature on: the sections in order, each at a 256-byte
// boundary, in one allocation zero-filled on the context's stream.  `buf` and the section pointers are set only once
// the allocation and the fill have both succeeded, so a failure (SL2_ERR_CUDA) leaves the feature unallocated.
int alloc_sections(sl2_ctx *c, DevPtr<uint8_t> &buf, std::initializer_list<Section> secs);

// One output of a results getter: `per_stream` bytes of stream s at src + s * per_stream on the device
struct ResultCopy {
  void *dst;
  const void *src;
  size_t per_stream;
};
// The results of streams [lo, lo + cnt) into every non-null dst: zeros when the feature's buffer was never allocated
// (no stream has run it), else one copy each and one synchronise
int read_results(sl2_ctx *c, bool allocated, int lo, int cnt, std::initializer_list<ResultCopy> outs);

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

int stage_reserve(sl2_ctx *c, size_t bytes);

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
inline Sl2Queue queue(sl2_ctx *c) { return {c->stream, &c->launches}; }

// n box x box templates -> rows zero-padded to 16 bytes, the layout of Sl2Dev::patches
void pack_patch_rows(uint8_t *dst, const uint8_t *src, int n, int box);

// *out = nfeat of stream s, read from the device
int device_nfeat(sl2_ctx *c, int s, int *out);
// one read of stream s's nfeat, then every idx[0 .. n) checked against it: SL2_ERR_ARG with `msg` for the first out of
// range
int check_feature_indices(sl2_ctx *c, int s, const int32_t *idx, int n, const std::string &msg);

// the camera values a stream of this context accepts (sl2_set_stream_config and the snapshot loads), api.cu
int check_stream_config(sl2_ctx *c, const sl2_stream_config *sc, const std::string &who);
// ingest.cu: make `srcs` the context's sources; a snapshot load gives streams [lo, lo + cams.size()) the blobs'
// cameras; one frame set into a ring slot
int install_sources(sl2_ctx *c, const std::vector<sl2_stream_source> &srcs);
int loaded_cameras(sl2_ctx *c, int lo, const std::vector<sl2_stream_config> &cams);
cudaError_t copy_slot_frames(sl2_ctx *c, int slot, const uint8_t *src, cudaMemcpyKind kind, Sl2Queue q);
// streams [lo, lo + cnt) start over with a new map (sl2_set_features, the snapshot loads): no refined matches,
// tracking, and every normal unestimated
int streams_restarted(sl2_ctx *c, int lo, int cnt);
// select.cu: the selection of the streams [lo, lo + cnt) on q, right after their prediction
int select_streams(sl2_ctx *c, int lo, int cnt, Sl2Queue q);
// rescue.cu: the rescue's kernel arguments; the rescue kernel and the second update of the streams [lo, lo + cnt) on
// q, right after their first update
Sl2Rescue rescue_args(const sl2_ctx *c);
int rescue_streams(sl2_ctx *c, int lo, int cnt, Sl2Queue q);
// gyro.cu: the gyro update of the streams [lo, lo + cnt) on q with the samples of ring slot `slot`, between their
// motion prediction and their feature prediction
int gyro_streams(sl2_ctx *c, int slot, int lo, int cnt, Sl2Queue q);
// gyro.cu: what the gyroscope and accelerometer settings share: every entry of v[0 .. n) finite; the checks that R
// (row-major, named rname in the message) is a rotation and C a symmetric positive definite covariance, an empty
// string when both hold; and Rc = R^T C R in the order include/sl2b200.h states
bool finite_all(const double *v, int n);
std::string sensor_frame_error(const double *R, const double *C, const std::string &rname);
void sensor_cov_in_camera(const double *R, const double *C, double Rc[9]);
// accel.cu: the accelerometers predict_kernel of the streams [lo, lo + cnt) reads with the samples of ring slot `slot`
// ({} when none of them has the accelerometer on)
Sl2Accel accel_args(const sl2_ctx *c, int slot, int lo, int cnt);
// subpixel.cu: the sub-pixel matches the kernels of the streams [lo, lo + cnt) read ({} when none of them has the
// refinement on); the refinement of those streams on q, right after their search of ring slot `slot` (job_patches: the
// search's templates); a load forgets the refinement of the streams [lo, lo + cnt): their z is the integer match until
// their next step
Sl2Subpix subpixel_args(const sl2_ctx *c, int lo, int cnt);
int subpixel_streams(sl2_ctx *c, int slot, int lo, int cnt, const uint8_t *job_patches, Sl2Queue q);
int subpixel_forget(sl2_ctx *c, int lo, int cnt);
// iterate.cu: the iteration's tables the final update of the streams [lo, lo + cnt) reads ({} when none of them has
// the iteration on); the iteration passes of those streams on q, right before their update
Sl2Iter iterate_args(const sl2_ctx *c, int lo, int cnt);
int iterate_streams(sl2_ctx *c, int lo, int cnt, Sl2Queue q);
// reloc.cu: the checks sl2_relocalise makes of its parameters and restart covariance; an empty string when accepted
std::string reloc_params_error(const sl2_reloc_params *p, const double *Pxx);
// recover.cu: the recovery states predict_kernel of the streams [lo, lo + cnt) reads (nullptr when none of them has
// recovery on); the decision, the full-image search and the pose kernel of those streams on q, at the end of their
// step of ring slot `slot`; the return of the streams [lo, lo + cnt) to tracking (the resets of include/sl2b200.h)
const sl2_recovery_result *recovery_args(const sl2_ctx *c, int lo, int cnt);
int recover_streams(sl2_ctx *c, int slot, int lo, int cnt, Sl2Queue q);
int recovery_reset(sl2_ctx *c, int lo, int cnt);
// normals.cu: the normal estimates the kernels of the streams [lo, lo + cnt) read ({} when none of them has normals
// on); features [f0, f0 + n) of stream s unestimated (nothing when the stream has normals off)
Sl2Normals normals_args(const sl2_ctx *c, int lo, int cnt);
int normals_reset(sl2_ctx *c, int s, int f0, int n);

}  // namespace sl2
