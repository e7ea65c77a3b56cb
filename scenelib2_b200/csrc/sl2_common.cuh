// sl2_common.cuh — shared device/host declarations of libsl2b200.so (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "../../include/sl2b200.h"  // SL2_MAX_FEATURES, SL2_MAX_MEASURED

#define SL2_NXV 13          // vehicle state size (motion_model.cpp:44)
#define SL2_SEARCH_WARPS 4  // features (warps) per search CTA
#define SL2_STRIP 8         // candidates per vertical strip task
#define SL2_MAX_FEAT_SMEM SL2_MAX_FEATURES  // per-feature shared arrays of the predict and cull kernels

// One camera stream's camera, frame period and selection count (the per-instance cfg values of MonoSLAM::Init,
// monoslam.cpp:1583-1602, 1853): one row per stream in Sl2Dev::cams, written by sl2_create and
// sl2_set_stream_config.  Kernels that predict, search or detect read the row of their stream.
struct Sl2StreamCam {
  double cam[8];  // width, height, fku, fkv, u0, v0, kd1, sd (the stream's image: width x height <= W x H)
  double dt;      // delta_t of the motion model
  int n_select;   // number_of_features_to_select
  int pad_;
};
static_assert(sizeof(Sl2StreamCam) % sizeof(double) == 0, "rows are copied as doubles");
__device__ __forceinline__ int stream_width(const Sl2StreamCam &c) { return (int)c.cam[0]; }
__device__ __forceinline__ int stream_height(const Sl2StreamCam &c) { return (int)c.cam[1]; }

// The per-stream arrays with one record of `per` elements of type T per map feature (SL2_BY_FEATURE) or per
// measurement job (SL2_BY_JOB), each [B][Nmax][per], in snapshot section order (include/sl2b200.h).  Everything that
// handles all of them expands this one table: the Sl2Dev members, their allocation, the snapshot sections, the cull
// (which moves the SL2_BY_FEATURE records of a kept feature) and the append.  `reset` is what the append starts a new
// feature with and what a load writes beyond the map; sl2_create zero-fills.
enum { SL2_BY_FEATURE, SL2_BY_JOB };
//      X(type,    name,       per, indexed by,     reset)
#define SL2_STREAM_ARRAYS(X)                                                                                    \
  X(double,  xp_org,      7, SL2_BY_FEATURE, 0)                                                                 \
  X(int,     attempted,   1, SL2_BY_FEATURE, 0)                                                                 \
  X(int,     successful,  1, SL2_BY_FEATURE, 0)                                                                 \
  /* per step, per feature */                                                                                   \
  X(double,  h,           2, SL2_BY_FEATURE, 0)                                                                 \
  X(double,  S,           4, SL2_BY_FEATURE, 0)  /* col-major */                                                \
  X(double,  Rvar,        1, SL2_BY_FEATURE, 0)                                                                 \
  X(double,  dh_dxp,     14, SL2_BY_FEATURE, 0)  /* [2][7] row-major */                                         \
  X(double,  dh_dy,       6, SL2_BY_FEATURE, 0)  /* [2][3] row-major */                                         \
  X(int,     sel_rank,    1, SL2_BY_FEATURE, -1) /* rank in the selected list or -1 */                          \
  X(int,     z_uv,        2, SL2_BY_FEATURE, 0)                                                                 \
  X(uint8_t, found,       1, SL2_BY_FEATURE, 0)  /* 1 = successful, 2 = matched but rejected by the consensus */ \
  X(double,  best,        1, SL2_BY_FEATURE, 0)                                                                 \
  /* per step, per job (rank order = measurement order) */                                                      \
  X(int,     job_feat,    1, SL2_BY_JOB,     -1) /* feature index of job r, -1 = none */                        \
  X(double,  job_centre,  2, SL2_BY_JOB,     0)                                                                 \
  X(double,  job_puinv,   3, SL2_BY_JOB,     0)

// the snapshot section of each array: L.field[SL2_FIELD_sel_rank]
#define SL2_FIELD_INDEX(T, name, per, by, reset) SL2_FIELD_##name,
enum { SL2_STREAM_ARRAYS(SL2_FIELD_INDEX) SL2_NUM_FIELDS };
#undef SL2_FIELD_INDEX
// a new array changes the blob format: the header's format list, SL2_SNAPSHOT_VERSION and lib.SNAPSHOT_FIELDS
static_assert(SL2_NUM_FIELDS == SL2_SNAPSHOT_FIELDS, "every per-stream array is a snapshot section");

// Device view of one context: everything the kernels need, passed by value.
struct Sl2Dev {
  // geometry / constants
  int B;       // camera streams in this context
  int Nmax;    // feature capacity per stream
  int W, H, pitch, slots;  // layout of the frame ring and of the SMOE score map; a stream's image may be smaller
  int box;     // BOXSIZE
  int ld;      // leading dimension of P (>= 13 + 3*Nmax, multiple of 8)
  int ldg;     // leading dimension of the update scratch G
  int kmax;    // features one step can measure: min(Nmax, SL2_MAX_MEASURED); sizes every measurement table
  int mmax;    // 2 * kmax: rows of S and of the update scratch G
  int tile_w, tile_h;  // TMA window tile (bytes x rows)
  int min_attempts;
  double match_fraction;
  double ovr[3];
  // resident state
  Sl2StreamCam *cams;  // [B]
  uint8_t *frames;   // [slots][B][H][pitch]  stream s's image in the top-left width_s x height_s of its block
  uint8_t *patches;  // [B][Nmax][box][16]   rows zero-padded to 16 bytes
  double *x;         // [B][ld]
  double *P;         // [B][ld][ld] col-major, both triangles kept consistent
  double *G;         // [B][mmax][ldg]  row-major scratch: [ S | H*P | nu ]
  int *nfeat;        // [B]
#define SL2_MEMBER(T, name, per, by, reset) T *name;
  SL2_STREAM_ARRAYS(SL2_MEMBER)  // [B][Nmax][per] each
#undef SL2_MEMBER
  int *nsel;           // [B]
  int *nvisible;       // [B]
  int *nmeas;          // [B]  successful measurements of the last step
  int *ncull;          // [B]  features the next cull would delete (set by the update's finish kernel)
  // EKF update pipeline (update.cu): factor -> solve -> syrk -> finish
  int *upd_m;          // [B]  measurement rows m of the running update (0: nothing to do)
  double *Wp;          // [B][SL2_MAX_PANELS][16*16]  W_pp = U_pp^-T of every 16-row Cholesky panel
  int nsm;             // SMs of the device
  // step records (records.cu): written by the fused step only, when rec_depth > 0
  sl2_step_record *rec;  // [B][rec_depth]  ring: the record of step t of stream s is rec[s][t % rec_depth]
  int rec_depth;         // 0 = records off
};
static_assert(sizeof(Sl2Dev) == 336, "Sl2Dev is every kernel's by-value parameter: a new member changes every launch");

#define SL2_MAX_PANELS 16  // 16-row panels of S: m <= 2 * SL2_MAX_MEASURED = 256
static_assert(2 * SL2_MAX_MEASURED <= 16 * SL2_MAX_PANELS, "every panel of S must fit the panel tables");

// ---- correctly-rounded, never-fused FP64 helpers: the oracle is built with
// -ffp-contract=off, so every bit-critical expression must avoid FMA contraction.
__device__ __forceinline__ double mul_(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double add_(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub_(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double div_(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ double sqrt_(double a) { return __dsqrt_rn(a); }

// never-fused FP64 scalar with natural operator syntax (bit-critical prologue math)
struct rd {
  double v;
  __device__ __forceinline__ rd() : v(0.0) {}
  __device__ __forceinline__ rd(double x) : v(x) {}
};
__device__ __forceinline__ rd operator+(rd a, rd b) { return rd(__dadd_rn(a.v, b.v)); }
__device__ __forceinline__ rd operator-(rd a, rd b) { return rd(__dsub_rn(a.v, b.v)); }
__device__ __forceinline__ rd operator*(rd a, rd b) { return rd(__dmul_rn(a.v, b.v)); }
__device__ __forceinline__ rd operator/(rd a, rd b) { return rd(__ddiv_rn(a.v, b.v)); }
__device__ __forceinline__ rd operator-(rd a) { return rd(-a.v); }
__device__ __forceinline__ rd rsqrt_(rd a) { return rd(__dsqrt_rn(a.v)); }

// ---- programmatic dependent launch (PDL): a kernel launched with the attribute may be scheduled while its
// predecessor in the stream drains; griddepcontrol.wait returns once the predecessor has completed and its
// writes are visible (without the attribute both instructions do nothing).  Every kernel of the fused step
// executes the pair FIRST, so completion is transitive along the chain of launches.
__device__ __forceinline__ void pdl_prologue() {
  // wait, THEN release the dependents: at most two kernels of the chain are resident at a time (triggering first
  // lets the whole chain of a step pile up on the SMs: measured slower at every batch size)
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

// The ordered gather of a block: the values v >= 0 of its threads, in thread order, into out[0 .. count); returns count
// and sets *at (if given) to this thread's index in out, -1 for v < 0.  wcount: scratch for the first nwarps warps,
// which hold every thread with a value.  All threads call; out is complete after the caller's next __syncthreads().
__device__ __forceinline__ int block_gather(int v, int *out, int *wcount, int nwarps, int *at = nullptr) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned bal = __ballot_sync(0xffffffffu, v >= 0);
  if (lane == 0) wcount[warp] = __popc(bal);
  __syncthreads();
  int base = 0, count = 0;
  for (int w = 0; w < nwarps; ++w) { base += w < warp ? wcount[w] : 0; count += wcount[w]; }
  const int j = base + __popc(bal & ((1u << lane) - 1u));
  if (v >= 0) out[j] = v;
  if (at) *at = v >= 0 ? j : -1;
  return count;
}

// PDL when the launch covers fewer camera streams than SL2_PDL_AUTO_STREAMS: a single camera stream is a chain of 8
// short kernels bound by launch-to-launch latency, which PDL shortens; a full batch fills the GPU and PDL only adds
// resident waiting CTAs.
#define SL2_PDL_AUTO_STREAMS 2
inline bool sl2_use_pdl(int stream_cnt) { return stream_cnt < SL2_PDL_AUTO_STREAMS; }

// Where a launcher enqueues: the stream, and the context's launch counter (sl2_launch_count)
struct Sl2Queue {
  cudaStream_t stream;
  int64_t *launches;
};

#ifdef __CUDACC__
// one launch path for every kernel: plain launch, or with the PDL attribute (only for kernels that begin with
// pdl_prologue()); a successful launch is counted
template <typename... KArgs, typename... Args>
inline cudaError_t sl2_launch_kernel(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, Sl2Queue q,
                                     bool pdl, Args &&...args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = q.stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl ? 1 : 0;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
  if (e == cudaSuccess) ++*q.launches;
  return e;
}
#endif

// The BOXSIZEs the patch kernels are built for: f(std::integral_constant<int, BOX>{}) for a supported box,
// cudaErrorInvalidValue otherwise
template <typename F>
inline cudaError_t sl2_with_box(int box, F &&f) {
  switch (box) {
    case 11: return f(std::integral_constant<int, 11>{});
    case 15: return f(std::integral_constant<int, 15>{});
    default: return cudaErrorInvalidValue;
  }
}
inline bool sl2_box_supported(int box) {
  return sl2_with_box(box, [](auto) { return cudaSuccess; }) == cudaSuccess;
}

// launchers (defined in search.cu / ekf.cu / consensus.cu / reloc.cu / update.cu), called from api.cu
struct SearchLaunch {
  // job arrays may be the context's own (fused step) or temporaries (staged API)
  const int *job_feat;       // [njobs_per_stream * B] or [n]
  const double *job_centre;  // x2
  const double *job_puinv;   // x3
  int jobs_per_stream;       // stride between streams in the job arrays
  int stream_lo, stream_cnt; // streams covered by the launch
  int slot;
  int *out_uv;               // [jobs][2] (by job) or nullptr
  uint8_t *out_found;        // by job
  double *out_best;          // by job
  int scatter_to_features;   // 1: also write d.z_uv/found/best indexed by feature
};

cudaError_t sl2_launch_search(const Sl2Dev &d, const CUtensorMap &tmap, const SearchLaunch &L, Sl2Queue q);
cudaError_t sl2_launch_score_map(const Sl2Dev &d, const CUtensorMap &tmap, int stream_id, int slot,
                                 const double *centre_dev, const double *puinv_dev, const int *feat_dev, int *box_dev,
                                 double *corr_dev, double *sd_dev, uint8_t *inside_dev, int cap, Sl2Queue q);
cudaError_t sl2_launch_predict(const Sl2Dev &d, int stream_lo, int stream_cnt, const double *u3_dev,
                               int do_predict, int do_measure, Sl2Queue q);
// match consensus of the streams [stream_lo, stream_lo + stream_cnt) between the search and the update; tau2_dev[s] =
// the squared inlier radius of stream s, 0 = off (consensus.cu)
cudaError_t sl2_launch_consensus(const Sl2Dev &d, int stream_lo, int stream_cnt, const double *tau2_dev, Sl2Queue q);
// relocalisation of the cnt streams ids_dev[] from the full-image search's results by job (job = (stream - stream_lo) *
// Nmax + feature): pose consensus, refinement and, on acceptance, the state write (reloc.cu reloc_kernel)
cudaError_t sl2_launch_reloc(const Sl2Dev &d, int cnt, const int *ids_dev, int stream_lo, const int *search_uv,
                             const uint8_t *search_found, const sl2_reloc_params *prm_dev, const double *Pxx_dev,
                             sl2_reloc_result *res_dev, int *zuv_dev, uint8_t *flags_dev, Sl2Queue q);
// EKF update = 5 kernels (hp, chol, solve, syrk, finish); ev6 (optional) = 6 events recorded around them
cudaError_t sl2_launch_update(const Sl2Dev &d, int stream_lo, int stream_cnt, int staged_m,
                              const int *st_feat, const double *st_Hxv, const double *st_Hy,
                              const double *st_R, const double *st_nu, int only_normalise,
                              Sl2Queue q, cudaEvent_t *ev6 = nullptr);
cudaError_t sl2_launch_cull(const Sl2Dev &d, int stream_lo, int stream_cnt, int force_index, Sl2Queue q);
cudaError_t sl2_launch_append(const Sl2Dev &d, int s, const double *y3_dev, const double *xp7_dev,
                              const uint8_t *patch_rows16_dev, const double *Pcol_dev, Sl2Queue q);
// one step record per stream of [stream_lo, stream_lo + stream_cnt) into ring row step % d.rec_depth; launched after
// the cull of the fused step (records.cu)
cudaError_t sl2_launch_records(const Sl2Dev &d, int stream_lo, int stream_cnt, int64_t step, Sl2Queue q);
size_t sl2_update_smem_bytes(const Sl2Dev &d);
cudaError_t sl2_configure_search(const Sl2Dev &d);  // per context: dynamic smem opt-in
cudaError_t sl2_configure_update(const Sl2Dev &d);
// partially-initialised features (ekf.cu, smoe.cu, particles.cu): F features x Kmax particle slots (K_dev[f] used)
cudaError_t sl2_launch_particle_predict(const Sl2Dev &d, int s, int F, int Kmax, const int *K_dev,
                                        const double *ypi, const double *Pxy, const double *Pyy,
                                        const double *lambda, double *h, double *sinv3, double *detS,
                                        Sl2Queue q);
size_t sl2_smoe_map_bytes(const Sl2Dev &d, int F);
cudaError_t sl2_launch_smoe(const Sl2Dev &d, int s, int slot, int F, int Kmax, const int *K_dev, const int *feat_dev,
                            const double *centre_dev, const double *puinv_dev, double *map_dev, int *out_uv_dev,
                            uint8_t *out_found_dev, double *out_best_dev, Sl2Queue q);
cudaError_t sl2_launch_particles(int F, int Kmax, const int *K_dev, const double *h, const double *sinv3,
                                 const double *detS, const double *lambda, const int *z_uv, const uint8_t *found,
                                 double prune_threshold, double *prob, uint8_t *keep, double *cumulative,
                                 double *mean_var, int *left_out, Sl2Queue q);
size_t sl2_detect_scratch_bytes(const Sl2Dev &d, int n);
cudaError_t sl2_launch_detect(const Sl2Dev &d, int stream, int slot, int n, const int *regions_dev,
                              int *out_uv_dev, double *out_ev_dev, void *scratch_dev, Sl2Queue q);

// ---- raw frame sources (ingest.cu): one row per stream with a non-default sl2_stream_source, in stream order -------
struct Sl2Source {
  int stream, format;  // camera stream, SL2_SRC_*
  int sw, sh;          // raw frame size
  int dw, dh;          // the stream's image (sl2_stream_config width_s x height_s): the resize target
  int64_t off;         // byte offset of the raw frame in a slot of the staging area
};
#define SL2_SOURCE_CHUNK 64  // rows one table write carries as its kernel parameter
struct Sl2SourceChunk {
  int first, n;
  Sl2Source row[SL2_SOURCE_CHUNK];
};
inline int sl2_source_bpp(int format) { return format == SL2_SRC_RGB24 ? 3 : format == SL2_SRC_UYVY ? 2 : 1; }
// table[first .. first + n) = the chunk's rows, ordered on the queue like any other launch
cudaError_t sl2_launch_source_write(Sl2Source *table, const Sl2SourceChunk &chunk, Sl2Queue q);
// convert (and resize) the raw frames of table rows [base, base + cnt) from one slot of the staging area into the
// ring slot `slot`; max_row_bytes = the largest sw * bpp of those rows
cudaError_t sl2_launch_ingest(const Sl2Dev &d, const Sl2Source *table, int base, int cnt, int max_dh,
                              int max_row_bytes, const uint8_t *stage_slot, int slot, Sl2Queue q);

// ---- stream snapshots (snapshot.cu): the blob format of include/sl2b200.h --------------------------------------
// Section field[k] of a blob is the stream's first nfeat records of array k of SL2_STREAM_ARRAYS (x, P and the
// templates are laid out separately).
struct Sl2SnapLayout {
  size_t x, P, field[SL2_SNAPSHOT_FIELDS], templates, total;  // byte offsets in the blob, total size
};
__host__ __device__ inline size_t sl2_snap_align8(size_t b) { return (b + 7) & ~(size_t)7; }
__host__ __device__ inline Sl2SnapLayout sl2_snap_layout(int nfeat, int box) {
  Sl2SnapLayout L;
  const size_t n = SL2_NXV + 3 * (size_t)nfeat;
  size_t o = sizeof(sl2_snapshot_header);
  L.x = o;
  o += sl2_snap_align8(8 * n);
  L.P = o;
  o += 8 * n * n;
#define SL2_SECTION(T, name, per, by, reset) \
  L.field[SL2_FIELD_##name] = o;             \
  o += sl2_snap_align8((size_t)nfeat * per * sizeof(T));
  SL2_STREAM_ARRAYS(SL2_SECTION)
#undef SL2_SECTION
  L.templates = o;
  o += sl2_snap_align8((size_t)nfeat * box * box);
  L.total = o;
  return L;
}

// what the host validated for one blob of a load: the kernels take sizes and counts from here, never from the blob
struct Sl2SnapLoad {
  Sl2StreamCam cam;
  int stream, nfeat, nsel, nvisible, nmeas, ncull;
  int pad_[2];
};
// pack the streams [lo, lo + cnt) into blobs at buf + i * stride (nfeat read on the device, header written)
cudaError_t sl2_launch_pack(const Sl2Dev &d, int lo, int cnt, uint8_t *buf, size_t stride, Sl2Queue q);
// adds the number of blobs whose job_feat / sel_rank fail the index rules (with the validated counts) to *bad
cudaError_t sl2_launch_snap_check(const Sl2Dev &d, int cnt, const Sl2SnapLoad *ld_dev, const uint8_t *buf,
                                  size_t stride, int *bad, Sl2Queue q);
// unpack blob i into stream ld_dev[i].stream and reset what the blob does not cover
cudaError_t sl2_launch_unpack(const Sl2Dev &d, int cnt, const Sl2SnapLoad *ld_dev, const uint8_t *buf, size_t stride,
                              Sl2Queue q);
