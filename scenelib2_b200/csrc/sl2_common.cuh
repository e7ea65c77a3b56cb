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
// The row of a stream's sl2_stream_config, or of an sl2_config (whose camera fields every stream starts with)
template <typename Config>
__host__ __device__ inline Sl2StreamCam sl2_cam_row(const Config &sc) {
  Sl2StreamCam r = {};
  const double cam[8] = {(double)sc.width, (double)sc.height, sc.fku, sc.fkv, sc.u0, sc.v0, sc.kd1, sc.sd};
  for (int i = 0; i < 8; ++i) r.cam[i] = cam[i];
  r.dt = sc.delta_t;
  r.n_select = sc.number_of_features_to_select;
  return r;
}
// and back: the fields are assigned one by one, so the padding of *sc keeps the bytes it had (the zeros of a
// snapshot header)
__host__ __device__ inline void sl2_cam_config(const Sl2StreamCam &r, sl2_stream_config *sc) {
  sc->width = (int32_t)r.cam[0];
  sc->height = (int32_t)r.cam[1];
  sc->fku = r.cam[2];
  sc->fkv = r.cam[3];
  sc->u0 = r.cam[4];
  sc->v0 = r.cam[5];
  sc->kd1 = r.cam[6];
  sc->sd = r.cam[7];
  sc->delta_t = r.dt;
  sc->number_of_features_to_select = r.n_select;
}
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

// found code of a match the consensus rescue took back (rescue.cu): set by rescue_kernel, turned into 1 by the second
// update's finish kernel of the same step, so it never leaves the step
#define SL2_FOUND_RESCUED 3

// NIS = w^T w and log det S = -2 sum log W_ii of the update whose m rows G and Wp hold, for stream s whose update ran
// on a state of n entries (records.cu says where the update leaves w and W_ii): thread tid < m takes row tid, then a
// pairwise tree over all 256 slots, the same order for every stream, every m and every launch shape.  A block of 256
// threads; all call; the sums are in s_nis[0] and s_ld[0] (the log det is 2 s_ld[0]) after the call.
__device__ __forceinline__ void update_sums(const Sl2Dev &d, int s, int m, int n, double *s_nis, double *s_ld) {
  const int tid = threadIdx.x;
  double q = 0.0, l = 0.0;
  if (tid < m) {
    const double w = d.G[((size_t)s * d.mmax + tid) * d.ldg + m + n];
    q = __dmul_rn(w, w);
    l = -log(d.Wp[((size_t)s * SL2_MAX_PANELS + (tid >> 4)) * 256 + (tid & 15) * 17]);
  }
  s_nis[tid] = q;
  s_ld[tid] = l;
  __syncthreads();
#pragma unroll
  for (int h = 256 / 2; h > 0; h >>= 1) {
    if (tid < h) {
      s_nis[tid] = __dadd_rn(s_nis[tid], s_nis[tid + h]);
      s_ld[tid] = __dadd_rn(s_ld[tid], s_ld[tid + h]);
    }
    __syncthreads();
  }
}

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

// launchers that files other than their own call (defined in search.cu / ekf.cu / select.cu / consensus.cu / warp.cu /
// subpixel.cu / update.cu / records.cu / particles.cu)
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
  const uint8_t *job_patches;  // [jobs][box][16] the template of job r (warp.cu), or nullptr: d.patches[feat]
};

cudaError_t sl2_launch_search(const Sl2Dev &d, const CUtensorMap &tmap, const SearchLaunch &L, Sl2Queue q);
// The patch normals (normals.cu; include/sl2b200.h, sl2_set_stream_normals) the warp, the cull and the alignment take
// as an argument, feature-indexed like Sl2Dev::xp_org: theta [B][Nmax][2], cov [B][Nmax][3] (S_aa, S_ab, S_bb), count
// and status [B][Nmax].  prm == nullptr when no stream of the launch has normals on; stream s is on when
// prm[s].max_iterations > 0.
struct Sl2Normals {
  const sl2_stream_normals *prm;  // [B]
  double *theta, *cov;
  int *count;
  uint8_t *status;
};
__device__ __forceinline__ bool normals_on(const Sl2Normals &n, int s) { return n.prm && n.prm[s].max_iterations > 0; }
// The planar patch warp (warp.cu): the template of every job of the streams [stream_lo, stream_lo + stream_cnt) at
// the pose xp, into out[job] in the row-padded layout of Sl2Dev::patches.  A stream whose on[s] is 0 gets its stored
// templates copied; a stream with normals on warps through its features' estimated normals.  With blur set (the
// exposure blur, include/sl2b200.h sl2_set_stream_blur), a stream whose blur[s].on is 1 gets its templates blurred
// over the exposure at the state xp (13 numbers: r, q, v, omega).
struct WarpLaunch {
  const int *job_feat;    // [stream_cnt * jobs_per_stream], -1 = no job
  int jobs_per_stream;    // stride between streams in job_feat and out
  int stream_lo, stream_cnt;
  const double *xp;       // the state (7, or 13 with blur) of a one-stream launch, or nullptr: each stream's own x
  const uint8_t *on;      // [B] the streams' warp settings, or nullptr: every stream warps
  uint8_t *out;           // [jobs][box][16]
  uint8_t *valid;         // [jobs] 2 = blurred, 1 = warped, 0 = the stored template (or no job); may be nullptr
  Sl2Normals nrm;         // the streams' estimated normals ({}: every stream warps with nW0)
  const sl2_stream_blur *blur;  // [B] the streams' blur settings, or nullptr: no stream of the launch blurs
  int *samples;           // [jobs] K of a blurred template, 0 otherwise; may be nullptr
};
cudaError_t sl2_launch_warp(const Sl2Dev &d, const WarpLaunch &L, Sl2Queue q);
// The accelerometer (include/sl2b200.h, sl2_set_stream_accel) that predict_kernel's motion prediction takes as an
// argument.  on == nullptr when no stream of the launch has it on.  An on stream s reads its sample at index
// s - sample_lo of force (3 doubles each) and valid, consumes it (valid = 0) and writes its result a[s], status[s].
struct Sl2AccelParam {  // one stream's setting as the kernel reads it (sl2_set_stream_accel)
  double R[9];   // R_ac, row-major
  double b[3];   // bias
  double Rc[9];  // R_ac^T C R_ac, row-major, exactly symmetric
  double g[3];   // gravity, world frame
  double sd2;    // sd_a sd_a
};
struct Sl2Accel {
  const uint8_t *on;           // [B]
  const Sl2AccelParam *prm;    // [B]
  const double *force;         // [.][3]
  uint8_t *valid;              // [.]
  int sample_lo;
  double *a;                   // [B][3]
  int *status;                 // [B] 0 none, 1 applied, 2 skipped
};
// sel_mode_dev: [B] the streams' SL2_SELECT_* settings, or nullptr: every stream selects by trace; rv_dev: [B] the
// streams' recovery states, or nullptr: no stream of the launch has recovery on; acc: the accelerometers of the
// launch's motion prediction ({}: none) (ekf.cu)
cudaError_t sl2_launch_predict(const Sl2Dev &d, int stream_lo, int stream_cnt, const double *u3_dev,
                               int do_predict, int do_measure, const int *sel_mode_dev, Sl2Queue q,
                               const sl2_recovery_result *rv_dev = nullptr, const Sl2Accel &acc = {});
// The mutual-information selection (select.cu) of the streams [stream_lo, stream_lo + stream_cnt) whose mode[s] is
// SL2_SELECT_INFORMATION, right after their predict_kernel: picks into sel_rank, the job slots and nsel
struct SelectLaunch {
  int stream_lo, stream_cnt;
  const int *mode;  // [B] SL2_SELECT_*
  const double *t;  // [B] exp2(2 min_bits)
  double *g;        // [B][gstride][Nmax][4] the factors, or nullptr: shared memory
  int gstride;      // picks per candidate in g: kmax in the scratch, else the most any stream of the launch makes
};
cudaError_t sl2_launch_select(const Sl2Dev &d, const SelectLaunch &L, Sl2Queue q);
// The sub-pixel matches (subpixel.cu) the kernels that read a match take as an argument: z [B][Nmax][2] and refined
// [B][Nmax], feature-indexed like Sl2Dev::z_uv.  z == nullptr when no stream of the launch has the refinement on; a
// stream with it off has every refined flag 0.
struct Sl2Subpix {
  double *z;
  uint8_t *refined;
};
// The match z of feature record f (s * Nmax + i), coordinate k, that the consensus, the update and the rescue use
__device__ __forceinline__ double match_z(const Sl2Dev &d, const Sl2Subpix &sp, size_t f, int k) {
  return (sp.z && sp.refined[f]) ? sp.z[f * 2 + k] : (double)d.z_uv[f * 2 + k];
}
// The refinement of the streams [stream_lo, stream_lo + stream_cnt) whose on[s] is 1, right after their search: every
// job's match into out.z / out.refined
struct SubpixelLaunch {
  int stream_lo, stream_cnt;
  int slot;                    // the frame ring slot the search read
  const uint8_t *on;           // [B]
  const uint8_t *job_patches;  // the search's SearchLaunch::job_patches: [jobs][box][16], or nullptr: d.patches[feat]
  Sl2Subpix out;
};
cudaError_t sl2_launch_subpixel(const Sl2Dev &d, const SubpixelLaunch &L, Sl2Queue q);
// match consensus of the streams [stream_lo, stream_lo + stream_cnt) between the search and the update; tau2_dev[s] =
// the squared inlier radius of stream s, 0 = off (consensus.cu)
cudaError_t sl2_launch_consensus(const Sl2Dev &d, int stream_lo, int stream_cnt, const double *tau2_dev,
                                 const Sl2Subpix &sp, Sl2Queue q);
// The iterated EKF update (iterate.cu; include/sl2b200.h, sl2_set_stream_iterated) that upd_hp / upd_hp2 and
// iterate_kernel take as an argument.  h == nullptr when no stream of the launch has the iteration on.  The
// relinearised tables h_eff [B][Nmax][2], Hxp [B][Nmax][14] and Hy [B][Nmax][6] are feature-indexed like Sl2Dev::h,
// dh_dxp and dh_dy; a stream reads them instead of those when max_it[s] > 0 and iters[s] > 0 (from pass 1 on).
struct Sl2Iter {
  int *max_it;        // [B] the settings' max_iterations, 0 = off
  double *tol;        // [B]
  double *h, *Hxp, *Hy;
  double *x;          // [B][ld] the running iterate x_i
  int *active;        // [B] 1 while stream s still iterates in this step
  int *iters, *status;  // [B] the results (sl2_get_iterated_results)
  double *delta;      // [B]
  int pass;           // the iteration pass i >= 0, or -1: the final update
};
// EKF update = 5 kernels (hp, chol, solve, syrk, finish); ev6 (optional) = 6 events recorded around them.  it: the
// iteration's tables the final update reads ({} off; pass -1)
cudaError_t sl2_launch_update(const Sl2Dev &d, int stream_lo, int stream_cnt, int staged_m,
                              const int *st_feat, const double *st_Hxv, const double *st_Hy,
                              const double *st_R, const double *st_nu, int only_normalise,
                              const Sl2Subpix &sp, Sl2Queue q, cudaEvent_t *ev6 = nullptr, const Sl2Iter &it = {});
// The factor half of iteration pass it.pass (update.cu): upd_hp / upd_hp2 and upd_chol over the measured rows of the
// streams still active, at their current linearisation; an inactive stream reads m = 0
cudaError_t sl2_launch_iterate_factor(const Sl2Dev &d, int stream_lo, int stream_cnt, const Sl2Subpix &sp,
                                      const Sl2Iter &it, Sl2Queue q);
// One whole iteration pass (iterate.cu): sl2_launch_iterate_factor, then iterate_kernel
cudaError_t sl2_launch_iterate_pass(const Sl2Dev &d, int stream_lo, int stream_cnt, const Sl2Subpix &sp,
                                    const Sl2Iter &it, Sl2Queue q);
// The second update of the consensus rescue: the five update kernels over the rows whose found is SL2_FOUND_RESCUED,
// with m2 (instead of Sl2Dev::upd_m) holding each stream's row count, 0 for a stream with nothing rescued, which the
// five kernels then leave as they found it (update.cu)
cudaError_t sl2_launch_update_rescued(const Sl2Dev &d, int stream_lo, int stream_cnt, int *m2, const Sl2Subpix &sp,
                                      Sl2Queue q);
// sp, nrm: the sub-pixel matches and the normal estimates move with their features
cudaError_t sl2_launch_cull(const Sl2Dev &d, int stream_lo, int stream_cnt, int force_index, const Sl2Subpix &sp,
                            Sl2Queue q, const Sl2Normals &nrm = {});
// The normal alignment (normals.cu) of the streams [stream_lo, stream_lo + stream_cnt) with normals on, after their
// last update, on the frame of ring slot `slot`
cudaError_t sl2_launch_normals(const Sl2Dev &d, int stream_lo, int stream_cnt, int slot, const Sl2Subpix &sp,
                               const Sl2Normals &nrm, Sl2Queue q);
// The consensus rescue (rescue.cu): chi2[s] (0 = off) and the consensus's tau2[s] of every stream, and the per-stream
// scratch the step records read: m2 = rows of the second update, nis1 / logdet1 = the first update's NIS and log det S
struct Sl2Rescue {
  const double *chi2, *tau2;  // [B]
  int *m2;                    // [B]
  double *nis1, *logdet1;     // [B]
};
// rescue_kernel then the second update of the streams [stream_lo, stream_lo + stream_cnt), after their first update
cudaError_t sl2_launch_rescue(const Sl2Dev &d, int stream_lo, int stream_cnt, const Sl2Rescue &r, const Sl2Subpix &sp,
                              Sl2Queue q);
// The gyroscope update (gyro.cu) of the streams [stream_lo, stream_lo + stream_cnt) whose on[s] is 1, between their
// motion prediction and their feature prediction: stream s reads its sample at index s - sample_lo of rate (3 doubles
// each) and valid, and consumes it (valid = 0)
struct Sl2GyroParam {  // one stream's setting as the kernels read it (sl2_set_stream_gyro)
  double R[9];   // R_gc, row-major
  double b[3];   // bias
  double Rc[9];  // R_gc^T C R_gc, row-major, exactly symmetric
};
struct GyroLaunch {
  int stream_lo, stream_cnt;
  const uint8_t *on;          // [B]
  const Sl2GyroParam *prm;    // [B]
  const double *rate;         // [.][3]
  uint8_t *valid;             // [.]
  int sample_lo;
  double *W;                  // [B][3][ld]: column c of stream s's W at W + (s * 3 + c) * ld
  double *nis;                // [B]
  int *status;                // [B] 0 none, 1 applied, 2 skipped
};
// gyro_prep_kernel then gyro_downdate_kernel
cudaError_t sl2_launch_gyro(const Sl2Dev &d, const GyroLaunch &G, Sl2Queue q);
// The relocalisation (reloc.cu) of the cnt streams ids_dev[] (stream_lo + i when nullptr) from the full-image search's
// results by job (job = (stream - stream_lo) * Nmax + feature).  Stream s reads its parameters at prm_dev and Pxx_dev
// advanced by s * prm_stride bytes.  rv: nullptr (sl2_relocalise), or the recovery states of the fused step
// (recover.cu): only streams with rv[s].attempted run, their result goes to rv[s].last and an acceptance returns them
// to tracking
cudaError_t sl2_launch_reloc(const Sl2Dev &d, int cnt, const int *ids_dev, int stream_lo, const int *search_uv,
                             const uint8_t *search_found, const sl2_reloc_params *prm_dev, const double *Pxx_dev,
                             size_t prm_stride, sl2_reloc_result *res_dev, int *zuv_dev, uint8_t *flags_dev,
                             sl2_recovery_result *rv, Sl2Queue q);
// one step record per stream of [stream_lo, stream_lo + stream_cnt) into ring row step % d.rec_depth; launched after
// the cull of the fused step (records.cu).  resc: the rescue's scratch when the streams' step ran the rescue, else
// nullptr
cudaError_t sl2_launch_records(const Sl2Dev &d, int stream_lo, int stream_cnt, int64_t step, const Sl2Rescue *resc,
                               Sl2Queue q);
cudaError_t sl2_configure_search(const Sl2Dev &d);  // per context: dynamic smem opt-in
cudaError_t sl2_configure_update(const Sl2Dev &d);
// partially-initialised features (ekf.cu, smoe.cu, particles.cu): F features x Kmax particle slots (K_dev[f] used)
cudaError_t sl2_launch_particle_predict(const Sl2Dev &d, int s, int F, int Kmax, const int *K_dev,
                                        const double *ypi, const double *Pxy, const double *Pyy,
                                        const double *lambda, double *h, double *sinv3, double *detS,
                                        Sl2Queue q);
cudaError_t sl2_launch_particles(int F, int Kmax, const int *K_dev, const double *h, const double *sinv3,
                                 const double *detS, const double *lambda, const int *z_uv, const uint8_t *found,
                                 double prune_threshold, double *prob, uint8_t *keep, double *cumulative,
                                 double *mean_var, int *left_out, Sl2Queue q);
