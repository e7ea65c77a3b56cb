// sl2_common.cuh — shared device/host declarations of libsl2b200.so (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define SL2_NXV 13          // vehicle state size (motion_model.cpp:44)
#define SL2_NB 8            // Cholesky row-panel height
#define SL2_SEARCH_WARPS 4  // features (warps) per search CTA
#define SL2_STRIP 8         // candidates per vertical strip task
#define SL2_MAX_FEAT_SMEM 128  // == SL2_MAX_FEATURES (include/sl2b200.h)

// keys of sl2_set_tuning (include/sl2b200.h: SL2_TUNE_*)
#define SL2_TUNE_PDL 0           // programmatic dependent launch between the kernels of the fused step (0 / 1 / 2 = auto)
#define SL2_TUNE_HP_PIPELINED 1  // upd_hp: 8-row blocks, S phase of block b under the loads of block b+1
#define SL2_TUNE_COUNT 4

// Device view of one context: everything the kernels need, passed by value.
struct Sl2Dev {
  // geometry / constants
  int B;       // camera streams in this context
  int Nmax;    // feature capacity per stream
  int W, H, pitch, slots;
  int box;     // BOXSIZE
  int ld;      // leading dimension of P (>= 13 + 3*Nmax, multiple of 8)
  int ldg;     // leading dimension of the update scratch G
  int mmax;    // 2 * Nmax
  int n_select;
  int tile_w, tile_h;  // TMA window tile (bytes x rows)
  int min_attempts;
  double match_fraction;
  double cam[8];  // width,height,fku,fkv,u0,v0,kd1,sd
  double dt;
  double ovr[3];
  // resident state
  uint8_t *frames;   // [slots][B][H][pitch]
  uint8_t *patches;  // [B][Nmax][box][16]   rows zero-padded to 16 bytes
  double *x;         // [B][ld]
  double *P;         // [B][ld][ld] col-major, both triangles kept consistent
  double *G;         // [B][mmax][ldg]  row-major scratch: [ S | H*P | nu ]
  int *nfeat;        // [B]
  double *xp_org;    // [B][Nmax][7]
  int *attempted;    // [B][Nmax]
  int *successful;   // [B][Nmax]
  // per-step, per-feature (indexed by feature)
  double *h;       // [B][Nmax][2]
  double *S;       // [B][Nmax][4] col-major
  double *Rvar;    // [B][Nmax]
  double *dh_dxp;  // [B][Nmax][2][7] row-major
  double *dh_dy;   // [B][Nmax][2][3] row-major
  int *sel_rank;   // [B][Nmax]  rank in the selected list or -1
  int *z_uv;       // [B][Nmax][2]
  uint8_t *found;  // [B][Nmax]  1 = successful measurement this step
  double *best;    // [B][Nmax]
  // per-step, per job (rank order = measurement order)
  int *job_feat;       // [B][Nmax]  feature index of job r, -1 = none
  double *job_centre;  // [B][Nmax][2]
  double *job_puinv;   // [B][Nmax][3]
  int *nsel;           // [B]
  int *nvisible;       // [B]
  int *nmeas;          // [B]  successful measurements of the last step
  int *ncull;          // [B]  features the next cull would delete (set by the update's finish kernel)
  // EKF update pipeline (update.cu): factor -> solve -> syrk -> finish
  int *upd_m;          // [B]  measurement rows m of the running update (0: nothing to do)
  double *Wp;          // [B][SL2_MAX_PANELS][16*16]  W_pp = U_pp^-T of every 16-row Cholesky panel
  // scheduling knobs (sl2_set_tuning; they never change a result, only when / where the work runs)
  int tune[SL2_TUNE_COUNT];
  int nsm;             // SMs of the device
};

#define SL2_MAX_PANELS 16  // 16-row panels of S: m <= 2 * SL2_MAX_FEATURES = 256

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
// SL2_TUNE_PDL: 0 never, 1 always, 2 (default) when the launch covers fewer camera streams than
// SL2_PDL_AUTO_STREAMS: a single camera stream is a chain of 8 short kernels bound by launch-to-launch latency, which
// PDL shortens; a full batch fills the GPU and PDL only adds resident waiting CTAs.
#define SL2_PDL_AUTO_STREAMS 2
inline bool sl2_use_pdl(const Sl2Dev &d, int stream_cnt) {
  const int mode = d.tune[SL2_TUNE_PDL];
  return mode == 1 || (mode == 2 && stream_cnt < SL2_PDL_AUTO_STREAMS);
}

#ifdef __CUDACC__
// one launch path for every kernel of the step: plain launch, or with the PDL attribute
template <typename... KArgs, typename... Args>
inline cudaError_t sl2_launch_kernel(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                     bool pdl, Args &&...args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}
#endif

// launchers (defined in search.cu / ekf.cu / update.cu), called from api.cu
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

cudaError_t sl2_launch_search(const Sl2Dev &d, const CUtensorMap &tmap, const SearchLaunch &L,
                              cudaStream_t st);
cudaError_t sl2_launch_score_map(const Sl2Dev &d, const CUtensorMap &tmap, int stream_id, int slot,
                                 int feat, const double *centre_puinv_dev /*5*/, int *box_dev,
                                 double *corr_dev, double *sd_dev, uint8_t *inside_dev, int cap,
                                 cudaStream_t st);
cudaError_t sl2_launch_predict(const Sl2Dev &d, int stream_lo, int stream_cnt, const double *u3_dev,
                               int do_predict, int do_measure, cudaStream_t st);
// EKF update = 4 kernels (factor, solve, syrk, finish); ev5 (optional) = 5 events recorded around them
cudaError_t sl2_launch_update(const Sl2Dev &d, int stream_lo, int stream_cnt, int staged_m,
                              const int *st_feat, const double *st_Hxv, const double *st_Hy,
                              const double *st_R, const double *st_nu, int only_normalise,
                              cudaStream_t st, cudaEvent_t *ev5 = nullptr, int *launches = nullptr);
cudaError_t sl2_launch_cull(const Sl2Dev &d, int stream_lo, int stream_cnt, int force_index,
                            cudaStream_t st);
cudaError_t sl2_launch_append(const Sl2Dev &d, int s, const double *y3_dev, const double *xp7_dev,
                              const uint8_t *patch_rows16_dev, const double *Pcol_dev, cudaStream_t st);
size_t sl2_update_smem_bytes(const Sl2Dev &d);
cudaError_t sl2_configure_search(const Sl2Dev &d);  // per context: dynamic smem opt-in
cudaError_t sl2_configure_update(const Sl2Dev &d);
// partially-initialised features (particles.cu, smoe.cu): F features x Kmax particle slots (K_dev[f] used)
cudaError_t sl2_launch_particle_predict(const Sl2Dev &d, int s, int F, int Kmax, const int *K_dev,
                                        const double *ypi, const double *Pxy, const double *Pyy,
                                        const double *lambda, double *h, double *sinv3, double *detS,
                                        cudaStream_t st);
size_t sl2_smoe_map_bytes(const Sl2Dev &d, int F);
cudaError_t sl2_launch_smoe(const Sl2Dev &d, int s, int slot, int F, int Kmax, const int *K_dev, const int *feat_dev,
                            const double *centre_dev, const double *puinv_dev, double *map_dev, int *out_uv_dev,
                            uint8_t *out_found_dev, double *out_best_dev, cudaStream_t st);
cudaError_t sl2_launch_particles(int F, int Kmax, const int *K_dev, const double *h, const double *sinv3,
                                 const double *detS, const double *lambda, const int *z_uv, const uint8_t *found,
                                 double prune_threshold, double *prob, uint8_t *keep, double *cumulative,
                                 double *mean_var, int *left_out, cudaStream_t st);
size_t sl2_detect_scratch_bytes(const Sl2Dev &d, int n);
cudaError_t sl2_launch_detect(const Sl2Dev &d, int stream, int slot, int n, const int *regions_dev,
                              int *out_uv_dev, double *out_ev_dev, void *scratch_dev, cudaStream_t st);
