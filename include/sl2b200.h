/* sl2b200.h — C ABI of libsl2b200.so: the H100-native (sm_90a) implementation of the
 * SceneLib2 per-frame EKF-MonoSLAM hot path.
 *
 * The reference (hanmekim/SceneLib2) has no plugin / FFI seam; the boundary is the set of C++
 * member functions on the hot path.  Each entry point below names the reference interface it
 * replaces (paths relative to scenelib2/ of the original repository).  The C++ host shim under
 * scenelib2_b200/host/ keeps the MonoSLAM / Kalman / Feature class surface on top of this ABI
 * (INTEGRATION.md shows the binding a maintainer would add).
 *
 * Conventions
 *   - return 0 on success, negative on error; sl2_last_error() gives the message.
 *   - all pointers are caller-owned HOST memory unless the name ends in _dev.
 *   - matrices are column-major FP64 (Eigen's default); images are row-major u8.
 *   - one context per GPU; calls on one context are serialised by the caller; work is queued
 *     on the context's CUDA stream and functions that return data synchronise that stream.
 *   - a context holds `num_streams` independent camera streams (one EKF + one frame each);
 *     stream_id selects one of them.  Batched entry points (sl2_step*) advance all of them.
 *   - NO CPU fallback: every function fails with SL2_ERR_CUDA when no sm_90 device is usable.
 */
#ifndef SL2B200_H
#define SL2B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SL2_OK 0
#define SL2_ERR_ARG (-1)
#define SL2_ERR_CUDA (-2)
#define SL2_ERR_STATE (-3)

#define SL2_MAX_FEATURES 128 /* per stream; state dimension n = 13 + 3 * features <= 397 */

typedef struct sl2_ctx sl2_ctx;

typedef struct sl2_config {
  int32_t device;      /* CUDA device ordinal */
  int32_t num_streams; /* independent camera streams resident in this context (>= 1) */
  int32_t frame_slots; /* frames kept in HBM per stream (ring, >= 1) */
  int32_t width, height;
  int32_t boxsize;      /* BOXSIZE: 11 (MonoSLAM::kBoxSize_, monoslam.cpp:48) or 15 */
  int32_t max_features; /* capacity per stream, <= SL2_MAX_FEATURES */
  int32_t number_of_features_to_select; /* params.number_of_features_to_select (cfg:60) */
  int32_t search_tile_radius; /* search half-extent served by ONE TMA window tile (default 20);
                                 larger ellipses are searched in several tiles */
  double fku, fkv, u0, v0, kd1, sd; /* Camera::SetCameraParameters (camera.cpp:58-82) */
  double delta_t;                   /* params.delta_t (cfg:59) */
  double search_override[3];        /* benchmark only: fixed (P00,P01,P11); P00 <= 0 = use S_i */
  int32_t minimum_attempted_measurements_of_feature; /* monoslam.cpp:1875 (10) */
  double successful_match_fraction;                  /* monoslam.cpp:1876 (0.5) */
  void *cuda_stream; /* optional cudaStream_t to run on (e.g. torch's current stream); NULL = own */
} sl2_config;

/* fills *cfg with the reference's defaults (data/SceneLib2.cfg:24-31,59-61; monoslam.cpp:47-49) */
void sl2_default_config(sl2_config *cfg);

int sl2_create(const sl2_config *cfg, sl2_ctx **out);
void sl2_destroy(sl2_ctx *ctx);
const char *sl2_last_error(const sl2_ctx *ctx); /* ctx may be NULL: error of the last failed create */
int sl2_sync(sl2_ctx *ctx);
/* library self-description: "sl2b200 <version> sm_90a" */
const char *sl2_version(void);

/* ---- frames (replaces the cv::Mat `frame` argument of MonoSLAM::GoOneStep, monoslam.cpp:108) */
/* one stream, one slot; `stride` = bytes between image rows */
int sl2_set_frame(sl2_ctx *ctx, int32_t stream_id, int32_t slot, const uint8_t *gray, size_t stride);
/* all streams of a slot at once: gray is [num_streams][height][width] contiguous (pinned memory
 * makes the copy asynchronous) */
int sl2_set_frames(sl2_ctx *ctx, int32_t slot, const uint8_t *gray);
/* device-resident producer: copy device -> device, same layout as sl2_set_frames */
int sl2_set_frames_dev(sl2_ctx *ctx, int32_t slot, const uint8_t *gray_dev);

/* ---- map and state (Feature::y_/xp_org_/patch_, feature.cpp:108-149; MonoSLAM::xv_/Pxx_ and the
 *      per-feature Pxy_/Pyy_/matrix_block_list_ blocks held as ONE dense P, layout of
 *      construct_total_covariance, monoslam.cpp:518-546) */
int sl2_set_features(sl2_ctx *ctx, int32_t stream_id, int32_t n, const double *y /* n x 3 */,
                     const double *xp_org /* n x 7 */, const uint8_t *patches /* n x B x B */);
int sl2_num_features(sl2_ctx *ctx, int32_t stream_id);
int sl2_state_size(sl2_ctx *ctx, int32_t stream_id); /* 13 + 3 * features */
int sl2_set_state(sl2_ctx *ctx, int32_t stream_id, const double *x, const double *P);
int sl2_get_state(sl2_ctx *ctx, int32_t stream_id, double *x, double *P);
/* MonoSLAM::delete_feature (monoslam.cpp:770-812): drop feature `index` and its rows/cols of P */
int sl2_delete_feature(sl2_ctx *ctx, int32_t stream_id, int32_t index);

/* MonoSLAM::AddNewKnownFeature (monoslam.cpp:1278-1289, Feature ctor feature.cpp:108-149): append ONE feature to the
 * map on the device -- y (3), xp_org (7: camera position state the feature was acquired from), patch (boxsize x
 * boxsize u8, row-major).  Pcol = NULL: Pxy_, Pyy_ and every matrix_block_list_ entry of the new feature are zero,
 * like the reference's known features; otherwise Pcol is the new feature's covariance column block, column-major
 * (n + 3) x 3 with n the state size before the call (rows 0..n-1: P_{x,y_new} / P_{y_j,y_new}, rows n..n+2: Pyy_,
 * whose upper triangle is taken) -- what the conversion of a partially-initialised feature produces
 * (monoslam.cpp:1262, feature.cpp:45-95).  Nothing else of the map moves (the mirror of sl2_delete_feature).
 * Returns the index of the new feature (>= 0), SL2_ERR_STATE when the map already holds max_features. */
int sl2_append_feature(sl2_ctx *ctx, int32_t stream_id, const double *y, const double *xp_org,
                       const uint8_t *patch, const double *Pcol);

/* ---- patch search --------------------------------------------------------------------------- */
/* MonoSLAM::elliptical_search (monoslam.cpp:401-477) o correlate2_warning (improc/improc.cpp:
 * 55-134), batched over n features of one stream.  feat_index[i] selects the stored template;
 * centre = h_i, PuInv3 = (P00,P01,P11) of Sinv (monoslam.cpp:371-378).  u/v are the patch-centre
 * pixel of the best match (unchanged, = -1, when nothing was accepted), found = corrmax <= 0.40,
 * best = final corrmax (1e6 when nothing was accepted).  Outputs may be NULL. */
int sl2_patch_search(sl2_ctx *ctx, int32_t stream_id, int32_t slot, int32_t n,
                     const int32_t *feat_index, const double *centre /* n x 2 */,
                     const double *PuInv3 /* n x 3 */, int32_t *u, int32_t *v, uint8_t *found,
                     double *best);
/* per-candidate scores of ONE feature over its clamped search box (urel-major, vrel-minor), for
 * bit-level parity of correlate2_warning: box6 = (urelstart, urelfinish, vrelstart, vrelfinish,
 * ucentre, vcentre); corr/sd_image/inside have (urelfinish-urelstart+1)*(vrelfinish-vrelstart+1)
 * entries (capacity given by cap); candidates outside the ellipse carry corr = NaN. */
int sl2_score_map(sl2_ctx *ctx, int32_t stream_id, int32_t slot, int32_t feat_index,
                  const double *centre, const double *PuInv3, int32_t *box6, double *corr,
                  double *sd_image, uint8_t *inside, size_t cap);
/* SearchMultipleOverlappingEllipses::search (improc/search_multiple_overlapping_ellipses.cpp:
 * 106-196): K ellipses sharing the template of feat_index. */
int sl2_smoe_search(sl2_ctx *ctx, int32_t stream_id, int32_t slot, int32_t feat_index, int32_t K,
                    const double *PuInv3 /* K x 3 */, const double *centres /* K x 2 */,
                    int32_t *res_u, int32_t *res_v, uint8_t *res_flag);

/* One partially-initialised feature represented by K depth particles:
 * MonoSLAM::measure_feature_with_multiple_priors (monoslam.cpp:1408-1438: SMOE search of the template of
 * feat_index over the K ellipses (Sinv_k, h_k)) followed by the body of
 * update_partially_initialised_feature_probabilities for that feature (monoslam.cpp:1447-1493):
 * prob_k *= N(z_k - h_k; S_k) (0 where the match failed), normalise_particle_vector_and_calculate_cumulative,
 * prune_particle_vector(prune_probability_threshold), calculate_mean_and_covariance (feature_init_info.cpp:
 * 95-172, scalar lambda).  The kernels run back to back on the device; K <= SL2_MAX_PARTICLES.
 * in: h (K x 2), Sinv3 (K x (S00,S01,S11)), detS (K), lambda (K); in/out: prob (K);
 * out (each may be NULL): z_uv (K x 2), found (K), keep (K; 1 = particle survives), cumulative (K; of the
 * survivors in order, 0 for pruned ones), mean_var (2).
 * Returns the number of surviving particles, 0 when every probability is zero (the reference then deletes the
 * feature and leaves prob un-normalised), < 0 on error. */
int sl2_measure_particles(sl2_ctx *ctx, int32_t stream_id, int32_t slot, int32_t feat_index, int32_t K,
                          const double *h, const double *Sinv3, const double *detS, const double *lambda,
                          double prune_probability_threshold, double *prob, int32_t *z_uv, uint8_t *found,
                          uint8_t *keep, double *cumulative, double *mean_var);

/* The same two entry points for a template that is not a map feature: `patch` is boxsize x boxsize u8, row-major
 * (the reference keeps the template of a partially-initialised feature in Feature::patch_, feature.cpp:45-95,
 * and hands it to SearchMultipleOverlappingEllipses, monoslam.cpp:1413). */
int sl2_smoe_search_patch(sl2_ctx *ctx, int32_t stream_id, int32_t slot, const uint8_t *patch, int32_t K,
                          const double *PuInv3 /* K x 3 */, const double *centres /* K x 2 */,
                          int32_t *res_u, int32_t *res_v, uint8_t *res_flag);
int sl2_measure_particles_patch(sl2_ctx *ctx, int32_t stream_id, int32_t slot, const uint8_t *patch, int32_t K,
                                const double *h, const double *Sinv3, const double *detS, const double *lambda,
                                double prune_probability_threshold, double *prob, int32_t *z_uv,
                                uint8_t *found, uint8_t *keep, double *cumulative, double *mean_var);

/* All partially-initialised features of one stream in ONE call (no host round trip between the stages):
 *   MonoSLAM::predict_partially_initialised_feature_measurements   monoslam.cpp:1347-1400
 *     per particle h_pi (PartFeatureModel::func_hpi_and_dhpi_by_dxp_and_dhpi_by_dyi, part_feature_model.cpp:
 *     231-265), R_i, S_i (FeatureModel::func_Si, feature_model.cpp:99-116), S_i^-1 and det S_i (Particle::set_S,
 *     feature_init_info.cpp:57-65), from the stream's CURRENT x_v / P_xx on the device;
 *   MonoSLAM::measure_feature_with_multiple_priors                 monoslam.cpp:1408-1438
 *     SearchMultipleOverlappingEllipses with the score of every image location computed once per feature;
 *   MonoSLAM::update_partially_initialised_feature_probabilities   monoslam.cpp:1447-1493 (see above).
 * F <= SL2_MAX_PARTIAL features, feature f uses K[f] <= Kmax <= SL2_MAX_PARTICLES particles; every per-particle
 * array is F x Kmax (entries k >= K[f] are ignored / left alone).
 * in : patches (F x boxsize x boxsize u8), ypi (F x 6: r, hhat), Pxy (F x 13x6 column-major: covariance between
 *      x_v and the feature's 6 states), Pyy (F x 6x6 column-major), lambda (F x Kmax), prune threshold;
 * in/out: prob (F x Kmax);
 * out (each may be NULL): h (F x Kmax x 2), Sinv3 (F x Kmax x (S00,S01,S11)), detS (F x Kmax), z_uv (F x Kmax x 2),
 *      found, keep (F x Kmax), cumulative (F x Kmax), mean_var (F x 2), left (F: survivors, 0 = the reference
 *      deletes the feature). */
#define SL2_MAX_PARTIAL 16
#define SL2_MAX_PARTICLES 256
int sl2_measure_partial_features(sl2_ctx *ctx, int32_t stream_id, int32_t slot, int32_t F, int32_t Kmax,
                                 const int32_t *K, const uint8_t *patches, const double *ypi, const double *Pxy,
                                 const double *Pyy, const double *lambda, double prune_probability_threshold,
                                 double *prob, double *h, double *Sinv3, double *detS, int32_t *z_uv,
                                 uint8_t *found, uint8_t *keep, double *cumulative, double *mean_var,
                                 int32_t *left);

/* MonoSLAM::find_best_patch_inside_region + find_eigenvalues (monoslam.cpp:1070-1205): Shi-Tomasi
 * smallest-eigenvalue detector over n regions (ustart, vstart, ufinish, vfinish) of one stream's
 * frame.  evbest[i] is always written; ubest/vbest[i] only when a position with a positive score
 * exists or the clamped region is empty (the reference leaves the caller's values otherwise). */
int sl2_find_best_patch(sl2_ctx *ctx, int32_t stream_id, int32_t slot, int32_t n,
                        const int32_t *regions /* n x 4 */, int32_t *ubest, int32_t *vbest,
                        double *evbest);

/* ---- EKF ------------------------------------------------------------------------------------ */
/* Kalman::KalmanFilterPredict (kalman.cpp:50-69) incl. MotionModel::func_fv_and_dfv_by_dxv and
 * func_Q (motion_model.cpp:84-217) evaluated on the device.  u3 = control accelerations (zero in
 * GoOneStep, monoslam.cpp:114-115); NULL = zero. */
int sl2_ekf_predict(sl2_ctx *ctx, int32_t stream_id, const double *u3);
/* MonoSLAM::auto_select_n_features (monoslam.cpp:187-254): per-feature prediction (h, dh/dxv,
 * dh/dy, R, S: monoslam.cpp:289-308), visibility (full_feature_model.cpp:103-170) and selection.
 * Returns the number of visible features (>= 0) or a negative error. */
int sl2_predict_measurements(sl2_ctx *ctx, int32_t stream_id);
/* MonoSLAM::make_measurements (monoslam.cpp:336-359) for the features selected by
 * sl2_predict_measurements; returns the number of successful measurements. */
int sl2_make_measurements(sl2_ctx *ctx, int32_t stream_id, int32_t slot);
/* Kalman::KalmanFilterUpdate (kalman.cpp:72-119) with host-supplied measurement rows, in the
 * order of construct_total_measurement_stuff (monoslam.cpp:548-572): row pair k belongs to
 * feature feat_index[k]; H_xv is (2k_meas) x 13 row-major, H_y (2k_meas) x 3 row-major,
 * R k_meas x (2x2 col-major, symmetric: SL2_ERR_ARG otherwise; the full block enters S), nu 2k_meas.
 * m = 2 * k_meas. */
int sl2_ekf_update(sl2_ctx *ctx, int32_t stream_id, int32_t m, const int32_t *feat_index,
                   const double *H_xv, const double *H_y, const double *R, const double *nu);
/* same, using the device-resident predictions/measurements of the two calls above */
int sl2_ekf_update_measured(sl2_ctx *ctx, int32_t stream_id);
/* MonoSLAM::normalise_state (monoslam.cpp:616-637) + the symmetrisation of GoOneStep
 * (monoslam.cpp:143-150).  sl2_ekf_update* already include both; exposed for the shim. */
int sl2_normalise_state(sl2_ctx *ctx, int32_t stream_id);

/* ---- fused step: MonoSLAM::GoOneStep (monoslam.cpp:108-180), tracking only, for ALL streams of
 *      the context: predict -> select -> measure -> update -> normalise -> cull -> symmetrise.
 *      Everything stays on the device; no host round trip inside the frame. */
int sl2_step(sl2_ctx *ctx, int32_t slot);
/* end-to-end form: host frames in ([num_streams][height][width]), camera states out
 * (xv_out: [num_streams][13], may be NULL).  Copies run on the context's stream. */
int sl2_step_host(sl2_ctx *ctx, int32_t slot, const uint8_t *gray, double *xv_out);
/* asynchronous end-to-end form for a frame ring: enqueues the H2D copy of `gray` into `slot` on a
 * copy stream, the fused step, and the D2H of the camera states into xv_out, then returns. gray and
 * xv_out must be pinned and stay valid until sl2_wait_slot(ctx, slot) (or sl2_sync) returns.
 * Consecutive calls should use different slots: the copy of frame t+1 then overlaps the kernels of
 * frame t (the producer side of FrameGrabber::GetFrame, framegrabber.cpp:73-104). */
int sl2_step_host_async(sl2_ctx *ctx, int32_t slot, const uint8_t *gray, double *xv_out);
int sl2_wait_slot(sl2_ctx *ctx, int32_t slot);
/* The fused step can run the camera streams of a context as `groups` (1 or 2, default 1) staggered groups
 * on internal CUDA streams: with 2, the patch search of one group is scheduled under the EKF update of
 * the other (useful when the update does not fill the GPU).  The groups share no state, so results do not depend on the setting; the reference's GoOneStep
 * order (monoslam.cpp:108-180) holds within every camera stream.  Every other entry point first makes
 * the context's stream wait for both groups; sl2_join does only that (no host synchronisation) -- call
 * it before recording your own events on the context's stream after a run of sl2_step calls. */
int sl2_set_step_groups(sl2_ctx *ctx, int32_t groups);
int sl2_join(sl2_ctx *ctx);
/* Scheduling knobs of the fused step (no reference counterpart: the reference runs one GoOneStep on one host
 * thread, monoslam.cpp:108-180).  They never change a result -- only how the kernels are launched / pipelined --
 * and every value is valid at any time (takes effect with the next launch).
 *   SL2_TUNE_PDL           the kernels of a step are launched with programmatic dependent launch (the next kernel's
 *                          CTAs are scheduled while the previous one drains): 0 never, 1 always, 2 (default) only for
 *                          a single camera stream, where the step is bound by launch-to-launch latency
 *   SL2_TUNE_HP_PIPELINED  1 (default): H*P in 8-row blocks with S of block b formed under the loads of block b+1 */
#define SL2_TUNE_PDL 0
#define SL2_TUNE_HP_PIPELINED 1
int sl2_set_tuning(sl2_ctx *ctx, int32_t key, int32_t value);

/* ---- read-back of per-feature results (Feature::h_/z_/S_/flags/counters, feature.h:96-140) */
int sl2_get_features(sl2_ctx *ctx, int32_t stream_id, double *h /* n x 2 */, double *z /* n x 2 */,
                     double *S /* n x 4 col-major */, uint8_t *flags /* bit0 selected, bit1 successful */,
                     int32_t *attempted, int32_t *successful, int32_t *select_rank);
/* Feature::dh_by_dxv_ (2x13), dh_by_dy_ (2x3), R_ (2x2), nu_ (2) of the last prediction /
 * measurement, all column-major like the Eigen members (feature.h:104-112). Arrays may be NULL. */
int sl2_get_feature_jacobians(sl2_ctx *ctx, int32_t stream_id, double *dh_by_dxv /* n x 26 */,
                              double *dh_by_dy /* n x 6 */, double *R /* n x 4 */,
                              double *nu /* n x 2 */);
/* device-time of the kernels of the last sl2_step (ms): [0] predict+select, [1] patch search,
 * [2] EKF update, [3] cull.  Valid after sl2_enable_timing(ctx, 1). */
int sl2_enable_timing(sl2_ctx *ctx, int32_t on);
int sl2_last_step_times(sl2_ctx *ctx, float *ms4);
/* the five kernels of the EKF update of the last sl2_step (ms): [0] hp (measurement list, H P, S = H P H^T + R),
 * [1] chol (Cholesky of S), [2] solve (Y = U^-T [H P | nu]), [3] syrk (P -= Y^T Y, x += Y^T w), [4] finish
 * (normalise, symmetrise, counters).  Their sum is sl2_last_step_times()[2]. */
int sl2_last_update_times(sl2_ctx *ctx, float *ms5);
/* kernels launched by this context since creation */
int64_t sl2_launch_count(const sl2_ctx *ctx);

#ifdef __cplusplus
}
#endif
#endif /* SL2B200_H */
