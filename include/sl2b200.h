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

/* Map capacity per stream: state dimension n = 13 + 3 * features <= 781.  x, P and the per-feature records live in
 * device memory and every kernel that scales with n loops over it. */
#define SL2_MAX_FEATURES 256
/* Features one step can measure: the rows of S = H P H^T + R are m = 2 * measured <= 256, because the Cholesky
 * factor and solve of the update keep all of S's factor in shared memory.  A context measures at most
 * min(max_features, SL2_MAX_MEASURED) features per step. */
#define SL2_MAX_MEASURED 128

typedef struct sl2_ctx sl2_ctx;

typedef struct sl2_config {
  int32_t device;      /* CUDA device ordinal */
  int32_t num_streams; /* independent camera streams resident in this context (>= 1) */
  int32_t frame_slots; /* frames kept in HBM per stream (ring, >= 1) */
  int32_t width, height;
  int32_t boxsize;      /* BOXSIZE: 11 (MonoSLAM::kBoxSize_, monoslam.cpp:48) or 15 */
  int32_t max_features; /* capacity per stream, 1 .. SL2_MAX_FEATURES */
  int32_t number_of_features_to_select; /* params.number_of_features_to_select (cfg:60); with max_features >
                                           SL2_MAX_MEASURED it must be <= SL2_MAX_MEASURED (a step never selects
                                           more than the map holds, so any value is valid below that) */
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

/* The per-instance cfg values of MonoSLAM::Init (monoslam.cpp:1583-1602, 1853) for ONE camera stream: each stream of
 * a context may have its own camera, image size, frame period and selection count.  sl2_create gives every stream
 * the values of its sl2_config. */
typedef struct sl2_stream_config {
  int32_t width, height;            /* cam.width / cam.height: this camera's image, <= the context's frame size */
  double fku, fkv, u0, v0, kd1, sd; /* Camera::SetCameraParameters (camera.cpp:58-82) */
  double delta_t;                   /* params.delta_t */
  int32_t number_of_features_to_select;
} sl2_stream_config;

int sl2_create(const sl2_config *cfg, sl2_ctx **out);
void sl2_destroy(sl2_ctx *ctx);
const char *sl2_last_error(const sl2_ctx *ctx); /* ctx may be NULL: error of the last failed create */
int sl2_sync(sl2_ctx *ctx);
/* library self-description: "sl2b200 <version> sm_90a" */
const char *sl2_version(void);

/* ---- per-stream camera ---------------------------------------------------------------------- */
/* Sets the camera of stream_id.  Ordered like every other entry point: work queued before the call uses the old
 * values, the next call that predicts, searches or detects (including the next fused step, also between two
 * sl2_step_host_async calls) uses the new ones.  A stream's filter state is left as it is.
 * SL2_ERR_ARG, with the stream's config unchanged, for: a bad stream_id or NULL sc; a non-finite value; fku, fkv or
 * delta_t <= 0; width or height outside [max(16, boxsize), the context's width or height];
 * number_of_features_to_select < 0, or > SL2_MAX_MEASURED when max_features > SL2_MAX_MEASURED. */
int sl2_set_stream_config(sl2_ctx *ctx, int32_t stream_id, const sl2_stream_config *sc);
int sl2_get_stream_config(sl2_ctx *ctx, int32_t stream_id, sl2_stream_config *sc);

/* ---- per-stream options ----------------------------------------------------------------------------------------
 * The sections from the match consensus to the iterated update, and the stream recovery, each give a camera stream an
 * opt-in setting: a setter, and a getter that returns the setting as the setter accepted it.  Every setter keeps this
 * contract; each section states only what is its own.
 *   Ordering like sl2_set_stream_config: work queued before the call uses the old setting, and the next call that runs
 *   the feature (including the next fused step) uses the new one.  A setter launches no kernel.
 *   The setting belongs to the stream slot, like the frame source: snapshots do not carry it and a load leaves it.
 *   Every stream starts with the feature off, and a context where no stream has it on runs exactly the path without
 *   it.
 *   When the feature has a device buffer ("Buffer:" in its section, payload sizes), the first stream turned on sizes
 *   it, each part at a 256-byte boundary, which may add padding: SL2_ERR_CUDA, with the setting left off, when that
 *   allocation fails.  Results read as zeros until a stream first turns the feature on.
 *   SL2_ERR_ARG, with the setting unchanged, for a bad stream_id, a NULL setting (get: a NULL output), and the values
 *   the section lists. */

/* ---- match consensus: keep wrong matches out of the EKF update (no reference counterpart) ----------------------
 * The reference trusts every match its patch search accepts.  A stream with an inlier radius tau > 0 px runs a
 * one-point RANSAC over the step's matches between the search and the update (Civera, Grasa, Davison, Montiel,
 * "1-Point RANSAC for EKF Filtering", J. Field Robotics 2010); its rescue stage is sl2_set_stream_rescue, below:
 *   M = the selected features whose match succeeded, in selection-rank order; k = |M|.
 *   Every i in M is a hypothesis (exhaustive, no random sampling: a stream's result never depends on its batch
 *   position, the step groups or the launch path).  Hypothesis i is the state-only partial update from i alone:
 *   w_i = S_i^-1 nu_i (nu_i = z_i - h_i, S_i^-1 as the search forms it), a_i = dh_dxp_i^T w_i, b_i = dh_dy_i^T w_i,
 *   dx_p = P[0:7, 0:7] a_i + P[0:7, y_i] b_i, dy_j = P[y_j, 0:7] a_i + P[y_j, y_i] b_i, with the predicted x and P.
 *   Match j is an inlier of i when the camera model maps y_j + dy_j, seen from x_p + dx_p (q not renormalised), to a
 *   point in front of the camera whose squared distance to z_j is <= fl(tau * tau); a NaN distance never is.  The
 *   support of i counts its inliers (i included).  The winner has the largest support, ties going to the lowest
 *   selection rank.  When its support is >= 2, every match of M outside its inlier set is rejected; otherwise (no
 *   two matches agree) nothing is.
 *   A rejected match keeps z and its score and gets found = 2 (sl2_get_features flags bit 2): it does not enter the
 *   update, and it counts as an attempted, unsuccessful measurement, so a feature that keeps matching the wrong place
 *   is culled by delete_bad_features' rule (minimum_attempted_measurements_of_feature, successful_match_fraction).
 *   A step record's nmeas, m, nis and logdet_s describe the rows that entered the update.
 * Every operation is a correctly rounded FP64 operation in the order written in the kernel (csrc/consensus.cu,
 * consensus_kernel), so decisions are reproducible bit for bit.
 * inlier_px = 0 (the default) is off.  SL2_ERR_ARG for a negative, NaN or infinite inlier_px. */
int sl2_set_stream_consensus(sl2_ctx *ctx, int32_t stream_id, double inlier_px);
int sl2_get_stream_consensus(sl2_ctx *ctx, int32_t stream_id, double *inlier_px);

/* ---- consensus rescue: take back the rejected matches the updated state agrees with (no reference counterpart) ---
 * The consensus judges every match against hypotheses built from one match each.  A feature whose own position is
 * still uncertain (a depth ray converted by sl2_append_feature, sigma of a few cm) is predicted several pixels from
 * its correct match by every other feature's hypothesis, so its match is rejected, its position never improves, and
 * the cull deletes it.  A stream with the consensus on and chi2 > 0 runs the high-innovation stage of the 1-point
 * RANSAC (Civera et al. 2010) after the update with the consensus's inliers:
 *   1. update 1: the update with the inliers, exactly as without the rescue (normalisation and symmetrisation
 *      included), giving x', P'.
 *   2. for every selected feature whose match the consensus rejected (found = 2), in selection-rank order: the
 *      prediction at x', P' (predict_kernel's code, bit for bit what a prediction of that state gives): h', dh/dxp',
 *      dh/dy', R' and S' = H' P' H'^T + R'; nu' = z - h'; (Si00, Si01, Si11) = the S'^-1 the search forms;
 *      w0 = Si00 nu0 + Si01 nu1, w1 = Si01 nu0 + Si11 nu1, q = nu0 w0 + nu1 w1.  The match is rescued when the
 *      feature lies in front of the camera at x' and q <= fl(chi2); a NaN q never is.  A rescued feature's h, S, R and
 *      Jacobians become the re-prediction, and the getters (sl2_get_features, sl2_get_feature_jacobians) show them.
 *   3. update 2: the update with the rescued rows only, in rank order, from x', P'.  Its finish normalises the
 *      quaternion's covariance again, so on such a step the normalisation Jacobian is applied twice.
 *   After the step a rescued match is successful (found = 1, sl2_get_features flags bit 1): every selected feature
 *   counts as one attempt, a rescued one as one success, and the cull sees those counters.
 * Every operation of step 2 is a correctly rounded FP64 operation in the order written in the kernel
 * (csrc/rescue.cu, rescue_kernel), so decisions are reproducible bit for bit.  A step in which the consensus rejected
 * nothing, and a step in which nothing is rescued, run no second update and leave the stream exactly as without the
 * rescue.  A step record's m and nmeas count the rows of both updates, nis = NIS_1 + NIS_2 and logdet_s =
 * log det S_1 + log det S_2, each from its own update (in the linear case the NIS and log det of one joint update).
 * Where it applies: the fused step (sl2_step, sl2_step_host, sl2_step_host_async) and sl2_ekf_update_measured;
 * sl2_ekf_update with the caller's rows never rescues.  A typical chi2 is 5.991, the 95 % point of chi^2 with two
 * degrees of freedom.  chi2 = 0 (the default) is off: a context where no stream has the consensus and the rescue on
 * runs exactly the path without it; one with such a stream adds six kernel launches per step group holding one
 * (timed with the update in sl2_last_step_times; sl2_last_update_times keeps timing update 1).  Buffer: the rescue
 * scratch, num_streams x 20 bytes.  SL2_ERR_ARG for a negative, NaN or infinite chi2. */
int sl2_set_stream_rescue(sl2_ctx *ctx, int32_t stream_id, double chi2);
int sl2_get_stream_rescue(sl2_ctx *ctx, int32_t stream_id, double *chi2);

/* ---- planar patch warp: match each template at the predicted viewpoint (no reference counterpart) ---------------
 * The reference searches every feature with the template stored when it was first seen, while the visibility test
 * admits distance ratios in [0.5, 2], 45 degrees of viewing angle and any roll.  A stream with the warp on searches
 * each selected feature with its template warped to the predicted viewpoint (Davison, Reid, Molton, Stasse, "MonoSLAM",
 * PAMI 2007; Molton, Davison, Reid, "Locally Planar Patch Features", BMVC 2004), taking the surface around the feature
 * as planar with its normal pointing at the camera that first saw it.
 * Warped template of feature i at the camera pose xp (r, q): with cam = the stream's camera, HALF = (B - 1) / 2,
 * y = the feature's state, xo = its xp_org,
 *   h = project_point(zeroed_point(y) from xp) (the prediction's h, bit for bit), ho = the same from xo (the centre of
 *   the stored template); the plane passes through y with world normal nW = xo[0:3] - y (not normalised);
 *   output pixel (row a, column b): p = h + (b - HALF, a - HALF); dW = adj(RRW) unproject_point(p), RRW = the
 *   matrix of xp (pose_RRW) and adj(RRW) = det(RRW) RRW^-1 (RRW is a rotation only when |q| = 1, and det(RRW) >= 0, so
 *   dW points along the ray that the camera at xp sees at p);
 *   t = (nW . (y - r)) / (nW . dW); X = r + t dW; zo = RRW(xo) (X - xo[0:3]); src = project_point(zo) - ho + (HALF, HALF);
 *   the pixel is valid when t is finite and > 0, zo[2] > 0 and src is finite;
 *   bilinear sampling of the stored template T: each coordinate of src clamped to [0, B - 1], x0 = min(floor(sx),
 *   B - 2), fx = sx - x0 (y0, fy likewise), v = (1 - fy)((1 - fx) T[y0][x0] + fx T[y0][x0+1]) + fy((1 - fx)
 *   T[y0+1][x0] + fx T[y0+1][x0+1]); the byte is (int)(v + 0.5).
 * Source positions outside the stored template repeat its edge pixels: a B x B template holds nothing beyond itself,
 * which a warp that shrinks it (the camera moving away, a slanted view) would need.  When any pixel of a feature is
 * invalid its warped template is its stored template (valid = 0).  Every operation is a correctly rounded FP64
 * operation in the order written in the device code (csrc/sl2_model.cuh: mat3_adj, patch_warp_setup, patch_warp_source,
 * patch_sample; dot products and matrix rows summed from 0.0 in ascending order), so the bytes are reproducible bit
 * for bit.
 * Where it applies: the search of the fused step (sl2_step, sl2_step_host, sl2_step_host_async) and of
 * sl2_make_measurements warps, for a stream with the warp on, each selected feature's template at the predicted pose
 * x[0:7]; the search's sigma >= 10 gates and scores then apply to that template, and no other rule changes.
 * sl2_patch_search, sl2_score_map, the SMOE and particle entry points and sl2_relocalise keep the stored templates.
 * on = 0 (the default) is off, 1 is on: a step group holding a stream that has it on adds one kernel launch (timed
 * with the search in sl2_last_step_times).  Buffer: the warped-template scratch, num_streams x max_features x boxsize
 * x 16 bytes.  SL2_ERR_ARG for an `on` other than 0 or 1. */
int sl2_set_stream_warp(sl2_ctx *ctx, int32_t stream_id, int32_t on);
int sl2_get_stream_warp(sl2_ctx *ctx, int32_t stream_id, int32_t *on);
/* The warped templates of features feat_index[0 .. n) of stream_id at the pose xp (7: r, q), whatever the stream's
 * setting: what the search of a warp-on stream sees at that pose.  out: n x boxsize x boxsize u8, row-major; valid (n,
 * may be NULL): 1 = warped, 0 = some pixel is invalid and out holds the stored template.  Joins both step
 * groups and synchronises.  SL2_ERR_ARG, with nothing written, for: a bad stream_id; n outside [0, max_features]; a
 * NULL feat_index, xp or out with n > 0; a feat_index outside [0, nfeat); a non-finite xp or a zero quaternion. */
int sl2_warp_templates(sl2_ctx *ctx, int32_t stream_id, int32_t n, const int32_t *feat_index, const double *xp,
                       uint8_t *out, uint8_t *valid);

/* ---- exposure blur: match each template through the motion blur the predicted motion makes (no reference
 * counterpart) ---------------------------------------------------------------------------------------------------
 * A camera that moves while its shutter is open smears every feature along the image motion: at 3 rad/s and a 1/60 s
 * exposure a 320 x 240 camera's features become ~10 px streaks, and a sharp template no longer matches them.  A stream
 * with the blur on searches each selected feature with its template averaged over the poses the predicted motion
 * (v, omega of the predicted state) passes through while the shutter is open (Jin, Favaro, Cipolla, "Visual Tracking
 * in the Presence of Motion Blur", CVPR 2005; Klein, Murray, "Improving the Agility of Keyframe-Based SLAM", ECCV 2008).
 * Blurred template of job feature i at the predicted state x (13: r, q, v, omega), with cam, HALF, y, xo, the plane's
 * nW (nW(theta) with normals on) and the bilinear sampling of the warp above, and h0 = the warp's h at x[0:7] (the
 * prediction's h, bit for bit):
 *   pose at time s: x[0:7] itself for s = 0 (not composed); otherwise r_s = r + v s, q_s = q (x) qw with qw =
 *   QuaternionFromAngularVelocity(omega s) (the motion model's: av = omega s, angle = sqrt(av . av), qw = (cos(angle /
 *   2), (sin(angle / 2) / angle) av), the identity for angle = 0; (x) the Hamilton product in the motion model's
 *   order), every component formed as in the motion model's prediction over dt = s;
 *   reference camera: with the warp on, the camera at xo with centre ho (the warp's); with it off, the pose x[0:7]
 *   with centre h0 (the blur alone, relative to the unwarped view);
 *   source of output pixel d = (b - HALF, a - HALF) at time s: the ray the pose at s sees at p = h0 + d
 *   (unproject_point(p), one for all times) cut with the plane and projected into the reference camera, src(s) =
 *   project_point(zo) - centre + (HALF, HALF), valid by the warp's rule; with the warp off and s = 0, src(0) = (b, a)
 *   with no round trip;
 *   times s- = offset - exposure * 0.5, s_c = offset, s+ = offset + exposure * 0.5;
 *   samples: L = sqrt(dx dx + dy dy) with (dx, dy) = src(s+) - src(s-) at d = (0, 0); K = min(32, max(1, ceil(L)));
 *   K = 1: v = the bilinear value (not rounded) at src(s_c);
 *   K > 1: D1 = src(s+) - src(s-), D2 = (src(s+) - 2 src(s_c)) + src(s-) per coordinate; for k = 0 .. K - 1,
 *   u = ((k + 0.5) / K) - 0.5, src_k = (src(s_c) + u D1) + ((2 u) u) D2 (the quadratic through the three, samples
 *   at most one template pixel apart up to a 32 px streak); v = (sum over ascending k from 0.0 of the bilinear value
 *   at src_k) / K;
 *   the byte is (int)(v + 0.5).
 * Every operation is a correctly rounded, never-fused FP64 operation in this order (csrc/sl2_model.cuh:
 * quat_from_angular_velocity, patch_ray_source, patch_bilinear; csrc/warp.cu: blur_job), except that sin and cos are
 * the device's, as in the motion model.  The needed sources are the centre's src(s-) and src(s+) and every pixel's
 * src(s_c) (K = 1) or its three (K > 1); when one of them is invalid or L is not finite, the job gets its unblurred
 * template: the warp's when the warp is on and valid, else the stored one.  Positions outside the stored template
 * repeat its edge pixels, as in the warp.  exposure = 0 and offset = 0 give K = 1 at s = 0: the warp's bytes, or the
 * stored template with the warp off.
 * Where it applies: the search of the fused step (sl2_step, sl2_step_host, sl2_step_host_async) and of
 * sl2_make_measurements, and the sub-pixel refinement, for a stream with the blur on, at the predicted state; the
 * search's sigma >= 10 gates and scores then apply to the blurred template (which fails them more often than a sharp
 * one), and no other rule changes.  The normal alignment still compares the stored, sharp template with the blurred
 * frame.  sl2_patch_search, sl2_score_map, the SMOE and particle entry points, sl2_relocalise and the recovery's
 * full-image search keep the stored templates.
 * on = 0 (the default) is off, 1 is on: a step group holding an on stream and no warp-on stream adds one kernel launch
 * (the warp's, timed with the search in sl2_last_step_times), and one that already warps adds none.  Buffer: the
 * warp's job-template scratch, shared with the warp (sized by the first stream turned on for either).  SL2_ERR_ARG for
 * reserved != 0, an `on` other than 0 or 1, an exposure that is not finite and >= 0, or an offset that is not
 * finite. */
typedef struct sl2_stream_blur {
  int32_t on;       /* 0 (default) or 1 */
  int32_t reserved; /* 0 */
  double exposure;  /* s, finite, >= 0: the shutter's open time */
  double offset;    /* s, finite: the exposure's middle relative to the frame's time (the predicted state's time);
                       -exposure / 2 for a camera that stamps the end of the exposure */
} sl2_stream_blur;
int sl2_set_stream_blur(sl2_ctx *ctx, int32_t stream_id, const sl2_stream_blur *b);
int sl2_get_stream_blur(sl2_ctx *ctx, int32_t stream_id, sl2_stream_blur *b);
/* The templates features feat_index[0 .. n) of stream_id get in the fused search at the state xv (13: r, q, v,
 * omega), with the stream's own blur, warp and normals settings.  out: n x boxsize x boxsize u8, row-major; valid (n,
 * may be NULL): 0 = the stored template, 1 = warped without blur, 2 = blurred; samples (n, may be NULL): K of a
 * blurred template, 0 otherwise.  Joins both step groups and synchronises.  SL2_ERR_ARG, with nothing written, for: a
 * bad stream_id; n outside [0, max_features]; a NULL feat_index, xv or out with n > 0; a feat_index outside [0, nfeat);
 * a non-finite xv or a zero quaternion. */
int sl2_blur_templates(sl2_ctx *ctx, int32_t stream_id, int32_t n, const int32_t *feat_index, const double *xv,
                       uint8_t *out, uint8_t *valid, int32_t *samples);

/* ---- patch normals: estimate the plane of each feature's patch from the images (no reference counterpart) --------
 * The warp above takes each patch as facing the camera that first saw it.  A stream with normals on estimates each
 * feature's normal by aligning its stored template with the step's frame through the homography the plane induces
 * (Molton, Davison, Reid, BMVC 2004), carries the estimate as a small Gaussian per feature, and its warp uses it.
 * Normal of feature i (y = its state, xo = its xp_org, theta = (a, b) its estimate): nW0 = xo[0:3] - y;
 *   R0 = row 0 of pose_RRW(xo) (camera o's x axis); q = R0 - ((R0 . nW0) / (nW0 . nW0)) nW0;
 *   E1 = q * (sqrt(nW0 . nW0) / sqrt(q . q)); E2 = (nW0 x E1) / sqrt(nW0 . nW0);
 *   nW(theta) = (nW0 + a E1) + b E2; theta = (0, 0) is nW0 bit for bit (it is taken as nW0, not computed).
 * a and b are the tangents of the patch's tilt away from facing camera o.  Warp: a stream with normals on warps (in
 * the fused step, sl2_make_measurements and sl2_warp_templates) with nW(theta_i) in place of nW0; no other rule changes.
 * Alignment of feature i, after the step's last update (x+ = the updated, normalised state, r+ its position; h+ =
 * project_point(zeroed_point(y) from x+); z = the match the update used, the refined one with the sub-pixel refinement
 * on), for every job of an on stream whose found is 1 after the update (consensus inliers and rescued matches):
 *   prior: theta- = theta_i, S- = Sigma_i + sigma_step^2 I; L = S-^-1 = [S-bb, -S-ab; -S-ab, S-aa] / (S-aa S-bb -
 *   S-ab S-ab);
 *   unknowns phi = (a, b, tu, tv, alpha, beta), starting at (theta-, z - h+, 1, 0);
 *   template pixel k = (row r, column c), k = r B + c: p_o = ho + (c - HALF, r - HALF); d_o = adj(RRW(xo))
 *   unproject_point(p_o); t = (nW(theta) . (y - xo[0:3])) / (nW(theta) . d_o); X = xo[0:3] + t d_o;
 *   zc = RRW(x+) (X - r+); g_k = project(zc) + (tu, tv) (with dh/dz J, csrc/sl2_model.cuh: patch_warp_forward);
 *   I(u, v) = the bilinear sample of the frame (not rounded; x0 = floor(u), fx = u - x0, same order as the warp's
 *   sample); I_u = (I(g + (1, 0)) - I(g - (1, 0))) * 0.5, I_v likewise; e_k = (alpha I(g_k) + beta) - T_k (T = the
 *   stored template);
 *   Jacobian row: w = RRW(x+) d_o, Jw = J w, t_a = ((E1 . (y - xo)) - t (E1 . d_o)) / (nW . d_o) (t_b with E2);
 *   de/da = alpha ((I_u Jw_u) + (I_v Jw_v)) t_a (b likewise), de/dtu = alpha I_u, de/dtv = alpha I_v, de/dalpha = I,
 *   de/dbeta = 1;
 *   sums over k: lane l of a warp takes k = l + 32 j in ascending j, then the xor-shuffle tree over offsets 16, 8, 4,
 *   2, 1 (v + v[l ^ o]); the 21 sums of J_p J_q (p <= q), the 6 of J_p e and sum e^2;
 *   with w2 = 1 / (sigma_i sigma_i) and dt = theta - theta-: H = (J^T J) w2 with L added to its theta block,
 *   G = (J^T e) w2 with L dt added to its theta part, cost = (sum e^2) w2 + (dt . L dt);
 *   valid: every pixel has t finite and > 0, zc[2] > 0 and g within [1, W - 2) x [1, H - 2) (W x H the stream's own
 *   image, so g +- 1 px is inside it), and nW(theta) . (xo[0:3] - y) > 0 and nW(theta) . (r+ - y) > 0;
 *   Gauss-Newton: for up to max_iterations steps: the 6 x 6 Cholesky H = L L^T (a pivot <= 0 or NaN ends the
 *   iteration), phi' = phi - H^-1 G; phi' accepted when it is valid and its cost is below phi's, else the iteration
 *   ends;
 *   posterior at the last accepted phi: Sigma+ = the theta block of H^-1 (the marginal over tu, tv, alpha, beta), from
 *   L^-1's first two columns; when at least one step was accepted and that Cholesky has positive pivots: theta_i,
 *   Sigma_i = theta, Sigma+, count_i + 1, status 1; otherwise both are left and status is 2 (no step accepted, or the
 *   final factor failed) or 3 (the start is not valid).  Status 0: not aligned by the stream's last alignment.
 * Every operation is a correctly rounded, never-fused FP64 operation in the order of the device code (csrc/normals.cu,
 * tests/normals_ref.py restates it), so the results are reproducible bit for bit whatever the batch position or the
 * step group.  Where it applies: the fused step (sl2_step, sl2_step_host, sl2_step_host_async) after its update, the
 * rescue's second update included, and before the cull: one more kernel launch per step group holding an on stream,
 * timed with the update in sl2_last_step_times; sl2_align_normals is that stage alone.  A stream with normals on and the
 * warp off still aligns, but nothing uses the estimates.
 * Lifecycle: a feature starts unestimated (theta = 0, Sigma = sigma0^2 I, count 0, status 0) when it enters through
 * sl2_append_feature, sl2_set_features or a snapshot load (which do not carry the estimates), and when the setter is
 * called for its stream; estimates move with their features through the cull and sl2_delete_feature, and
 * sl2_relocalise and the recovery keep them.
 * max_iterations = 0 (the default) is off; 1 .. SL2_MAX_NORMAL_ITERATIONS is on.  The setter synchronises.  Buffer:
 * num_streams x (32 + 45 max_features) bytes.  SL2_ERR_ARG for reserved != 0, max_iterations outside
 * [0, SL2_MAX_NORMAL_ITERATIONS], a sigma0 or sigma_i that is not finite and > 0, or a sigma_step that is not finite
 * and >= 0. */
#define SL2_MAX_NORMAL_ITERATIONS 8
typedef struct sl2_stream_normals {
  int32_t max_iterations; /* 0 (default, off) .. SL2_MAX_NORMAL_ITERATIONS Gauss-Newton steps per alignment */
  int32_t reserved;       /* 0 */
  double sigma0;          /* > 0: prior sigma of each tilt component of a feature that enters the map */
  double sigma_i;         /* > 0: grey-level noise of one pixel of the alignment */
  double sigma_step;      /* >= 0: added (squared) to each tilt variance before every alignment */
} sl2_stream_normals;
int sl2_set_stream_normals(sl2_ctx *ctx, int32_t stream_id, const sl2_stream_normals *v);
int sl2_get_stream_normals(sl2_ctx *ctx, int32_t stream_id, sl2_stream_normals *v);
/* The estimates of features feat_index[0 .. n) of stream_id: theta (n x 2), cov (n x 3: S_aa, S_ab, S_bb), normal_w
 * (n x 3, nW(theta) / |nW(theta)|), count (alignments accepted) and status (of the last alignment); any output may be
 * NULL.  Set: theta and cov (exactly symmetric by construction: S_aa > 0 and S_aa S_bb - S_ab S_ab > 0, all finite),
 * count and status 0.  Both join the step groups and synchronise.  SL2_ERR_STATE for a stream with normals off;
 * SL2_ERR_ARG, with nothing written, for a bad stream_id, n outside [0, max_features], a NULL feat_index (or, set, a
 * NULL theta or cov) with n > 0, an index outside [0, nfeat), a non-finite theta or a cov without positive pivots. */
int sl2_get_patch_normals(sl2_ctx *ctx, int32_t stream_id, int32_t n, const int32_t *feat_index, double *theta,
                          double *cov, double *normal_w, int32_t *count, uint8_t *status);
int sl2_set_patch_normals(sl2_ctx *ctx, int32_t stream_id, int32_t n, const int32_t *feat_index, const double *theta,
                          const double *cov);
/* The alignment of stream_id alone on the frame of ring slot `slot`, from its current state, match list and matches:
 * what the fused step does after its update.  Joins the step groups and synchronises.  SL2_ERR_STATE for a stream with
 * normals off; SL2_ERR_ARG for a bad stream_id or slot. */
int sl2_align_normals(sl2_ctx *ctx, int32_t stream_id, int32_t slot);

/* ---- sub-pixel refinement: fit each match's score around the search's minimum (no reference counterpart) -------
 * The reference's match is the integer position of the smallest correlation score (elliptical_search), so z carries a
 * quantisation error of sigma = 1 / sqrt(12) = 0.29 px per axis.  A stream with the refinement on fits a quadratic to
 * the search's own score at the 3 x 3 integer positions around each match and measures the fit's minimum (Shimizu,
 * Okutomi, "Sub-Pixel Estimation Error Cancellation on Area-Based Matching", IJCV 2005, on the estimate and its bias).
 * Which matches: every job of the stream's step whose search succeeded (found = 1 from the search, before the match
 * consensus), with integer match (u, v).  With HALF = (boxsize - 1) / 2 and the stream's own width W x height H:
 *   c(a, b) for a, b in {-1, 0, 1} is the search's exact score (improc.cpp:99-133, the chain of sl2_score_map) of the
 *   window centred at (u + a, v + b) against the template the search used (the warped one when the warp is on);
 *   c(0, 0) is the search's best score bit for bit.
 *   z = (u, v) (not refined) when: a window leaves the image (u - 1 - HALF < 0, u + 1 + HALF > W - 1, or the same in
 *   v); a window has sigma_g1 < 10 (the search's own gate); the fit below is not positive definite; or an offset
 *   component is not in [-0.5, 0.5].  NaN fails every test.
 *   The fit, every operation a correctly rounded FP64 operation with no contraction, in this order:
 *     g_u = (c(1,0) - c(-1,0)) * 0.5;  g_v = (c(0,1) - c(0,-1)) * 0.5;
 *     h_uu = (c(1,0) + c(-1,0)) - 2 c(0,0);  h_vv = (c(0,1) + c(0,-1)) - 2 c(0,0);
 *     h_uv = ((c(1,1) - c(1,-1)) - (c(-1,1) - c(-1,-1))) * 0.25;  det = h_uu h_vv - h_uv h_uv;
 *     refined only when h_uu > 0 and det > 0; du = (h_uv g_v - h_vv g_u) / det;  dv = (h_uv g_u - h_uu g_v) / det;
 *   z = (u + du, v + dv).
 * Where it applies: the match consensus, the EKF update (nu = z - h, both updates when the consensus rescue fires) and
 * the rescue's gate of the fused step and of sl2_make_measurements / sl2_ekf_update_measured read the refined z;
 * sl2_get_features returns it as z, with flags bit 3 set, and sl2_get_feature_jacobians forms nu from it.  Like the
 * other flags, bit 3 describes the feature's last match; it is never set for an off stream.  R stays sd-based: lower
 * the stream's sd (sl2_set_stream_config) to make the update trust the refined matches more.  sl2_patch_search,
 * sl2_score_map, the SMOE and particle entry points and sl2_relocalise stay integer.
 * on = 0 (the default) is off, 1 is on: a step group holding a stream that has it on adds one kernel launch (timed
 * with the search in sl2_last_step_times).  A loaded stream's z is its integer match (bit 3 clear) until its next
 * step; so is a stream's after the setting is made.  Buffer: num_streams x (17 max_features + 1) bytes.  SL2_ERR_ARG
 * for an `on` other than 0 or 1. */
int sl2_set_stream_subpixel(sl2_ctx *ctx, int32_t stream_id, int32_t on);
int sl2_get_stream_subpixel(sl2_ctx *ctx, int32_t stream_id, int32_t *on);

/* ---- feature selection: measure the features that carry the most information (no reference counterpart) --------
 * The reference measures the n_select visible features of largest trace(S_i) (auto_select_n_features,
 * monoslam.cpp:187-254).  Once the map has settled, most of every feature's innovation uncertainty is the camera
 * pose's, which they all share, so the top-trace features are largely redundant; and trace ignores that R_i grows
 * towards the image border.  A stream with SL2_SELECT_INFORMATION picks greedily by mutual information (Davison,
 * "Active Search for Real-Time Vision", ICCV 2005): each pick is the feature whose measurement, conditioned on the
 * features already picked, tells most about the state, and the picks stop when the next would add min_bits or less.
 *   Candidates: the features the trace rule would select if n_select were unlimited (visible, ranked before the first
 *   zero trace); rho_j is candidate j's trace rank, used only to break ties.  Per candidate, from the prediction:
 *   C_j = [[S00, S10], [S10, S11]] of the stored S_j, A_j = dh_dxp (2x7), B_j = dh_dy (2x3), R_j = Rvar_j; and
 *   t = exp2(2 min_bits), computed once on the host when the setting is made.
 *   Pick r = 0, 1, ... while r < n_select: over the unpicked candidates, q_j = (C00 C11 - C10 C10) / (R_j R_j)
 *   (the conditional information of measuring j is (1/2) log2 q_j bits).  The pick i has the largest q_j among those
 *   with C00 > 0 and q_j > t, ties going to the smallest rho; a NaN q never wins; if none qualifies the picks stop.
 *   Pick i is written exactly as the trace rule writes a selected feature: sel_rank[i] = r, and job slot r = (i, the
 *   centre h_i, the ellipse of the prior S_i or the search override): the search looks where the prediction says.
 *   Then L_i = chol(C_i): l00 = sqrt(C00), l10 = C10 / l00, l11 = sqrt(C11 - l10 l10);
 *   u = P H_i^T on rows 0..6 and every unpicked candidate's y rows: u[row][c] = ((0 + P[row][0] A_i[c][0]) + ... +
 *   P[row][6] A_i[c][6]) + P[row][y_i] B_i[c][0] + P[row][y_i+1] B_i[c][1] + P[row][y_i+2] B_i[c][2];
 *   for every unpicked j: c_j[a][b] = ((0 + A_j[a][0] u[0][b]) + ... + A_j[a][6] u[6][b]) + B_j[a][0] u[y_j][b] + ...
 *   + B_j[a][2] u[y_j+2][b], then for p = 0 .. r-1, e = 0, 1: c_j[a][b] -= g_{j,p}[a][e] g_{i,p}[b][e];
 *   g_{j,r} = c_j L_i^-T: g[a][0] = c_j[a][0] / l00, g[a][1] = (c_j[a][1] - g[a][0] l10) / l11;
 *   C00 = C00 - g00 g00 - g01 g01, C10 = C10 - g10 g00 - g11 g01, C11 = C11 - g10 g10 - g11 g11 (left to right).
 *   This is a block-pivoted Cholesky factorisation of the candidates' joint innovation covariance H P H^T + R whose
 *   pivot is the largest det(C_j) / R_j^2.  nsel = the number of picks; nvisible is the trace rule's; nmeas = 0.
 * Every operation is a correctly rounded FP64 operation (never fused) in the order written above and in the kernel
 * (csrc/select.cu, select_kernel), so decisions are reproducible bit for bit.
 * Where it applies: the fused step (sl2_step, sl2_step_host, sl2_step_host_async) and sl2_predict_measurements.  The
 * search, the consensus (whose ties go to the lowest selection rank, now the information order), the warp, the
 * update, the cull, the records and relocalisation read the job slots as with the trace rule.  A stream can end a
 * prediction with nothing selected.
 * mode SL2_SELECT_TRACE (the default) is the reference's rule and counts as off; a step group holding a stream that
 * selects by information adds one kernel launch, and so does sl2_predict_measurements of one (timed with the predict
 * in sl2_last_step_times).  Buffer: only when the factors of kmax = min(max_features, SL2_MAX_MEASURED) picks cannot
 * stay in shared memory, the factor scratch, num_streams x max_features x kmax x 32 bytes.  SL2_ERR_ARG for an unknown
 * mode; reserved != 0; a min_bits that is negative or not finite, or non-zero with SL2_SELECT_TRACE. */
#define SL2_SELECT_TRACE 0       /* the reference's rule: top n_select by trace(S_i) (default) */
#define SL2_SELECT_INFORMATION 1 /* greedy mutual information, above */
typedef struct sl2_stream_selection {
  int32_t mode;     /* SL2_SELECT_* */
  int32_t reserved; /* 0 */
  double min_bits;  /* INFORMATION: a pick must add more than min_bits bits; >= 0, finite.  TRACE: must be 0 */
} sl2_stream_selection;
int sl2_set_stream_selection(sl2_ctx *ctx, int32_t stream_id, const sl2_stream_selection *sel);
int sl2_get_stream_selection(sl2_ctx *ctx, int32_t stream_id, sl2_stream_selection *sel);

/* ---- gyroscope: an angular-rate update between the motion prediction and the feature prediction (no reference
 *      counterpart) ------------------------------------------------------------------------------------------------
 * The constant-velocity model allows an angular acceleration of sigma = 6 rad/s^2: a camera that starts or stops
 * turning faster than that has its features predicted outside their search regions.  A stream with a gyroscope takes
 * one rate sample per step and updates its state's omega, x[10:13] (camera frame: qnew = qold * q(omega dt)), right
 * after the motion prediction, so the feature prediction, the search ellipses and the selection already know how the
 * camera turned; P's q-omega cross terms carry the correction into q (Pinies, Lupton, Sukkarieh, Tardos, "Inertial
 * Aiding of Inverse Depth SLAM using a Monocular Camera", ICRA 2007).
 * Setting, in the gyro's frame: R_gc (row-major) takes camera-frame vectors into the gyro's frame; bias b; cov C, the
 * covariance of one sample, a sample being the mean angular rate over the stream's frame period delta_t.  The model is
 * z = R_gc omega + b + noise(C).  When the setting is made, Rc = R_gc^T C R_gc is formed once: M[k][j] = (C[k][0]
 * R[0][j] + C[k][1] R[1][j]) + C[k][2] R[2][j], then for i <= j Rc[i][j] = (R[0][i] M[0][j] + R[1][i] M[1][j]) +
 * R[2][i] M[2][j], mirrored to Rc[j][i].
 * Update of a sample z, with x and P the motion prediction (n = 13 + 3 nfeat, P(r, c) = the column-major entry):
 *   1. dk = z[k] - b[k]; zc[i] = (R[0][i] d0 + R[1][i] d1) + R[2][i] d2.
 *   2. S(i, j) = P(10 + i, 10 + j) + Rc[i][j] for i >= j; l00 = sqrt(S00), l10 = S10 / l00, l20 = S20 / l00,
 *      a11 = S11 - l10 l10, l11 = sqrt(a11), l21 = (S21 - l20 l10) / l11, a22 = (S22 - l20 l20) - l21 l21,
 *      l22 = sqrt(a22).
 *   3. nu[i] = zc[i] - x[10 + i]; w0 = nu0 / l00, w1 = (nu1 - l10 w0) / l11, w2 = ((nu2 - l20 w0) - l21 w1) / l22;
 *      NIS = (w0 w0 + w1 w1) + w2 w2.
 *   If S00, a11 or a22 is not > 0, or any of S, L, nu, w and NIS is not finite, the update is skipped: x and P stay
 *   exactly as they were (status 2).
 *   4. for every row r < n: W[r][0] = P(r, 10) / l00, W[r][1] = (P(r, 11) - W[r][0] l10) / l11,
 *      W[r][2] = ((P(r, 12) - W[r][0] l20) - W[r][1] l21) / l22 (W = P H^T L^-T, all from the predicted P).
 *   5. x[r] = x[r] + ((W[r][0] w0 + W[r][1] w1) + W[r][2] w2) for r < n;
 *      P(i, j) = P(i, j) - ((W[i][0] W[j][0] + W[i][1] W[j][1]) + W[i][2] W[j][2]) for i, j < n.  Entries outside the
 *      n x n block stay as they are.  Multiplication is commutative in IEEE arithmetic, so P(j, i) gets the same bits
 *      as P(i, j): P stays bit-symmetric without a mirror pass.
 * Every operation is a correctly rounded FP64 operation (never fused) in the order written above and in the kernels
 * (csrc/gyro.cu, gyro_prep_kernel and gyro_downdate_kernel).  Nothing is normalised: the step's visual update
 * normalises the quaternion and symmetrises as before, and a step that measures nothing leaves the gyro-updated state
 * un-normalised.  NIS is chi^2 with 3 degrees of freedom when R_gc, b and C are right: this is how to check them.
 * Where it applies: the fused step (sl2_step, sl2_step_host, sl2_step_host_async) of ring slot t consumes slot t's
 * sample of every gyro-on stream: the update runs when the sample is valid, and the step clears the sample's valid
 * byte, so a sample is used by exactly one step; a step without a valid sample does no gyro update.  The staged form
 * is sl2_gyro_update, between sl2_ekf_predict and sl2_predict_measurements.  The step records are unchanged: nis and
 * logdet_s stay the visual update's, xv and pxx_diag show the state after both updates.
 * on = 0 (the default; the getter then shows R_gc = I, b = 0, C = I) is off; a step group holding a gyro-on stream
 * splits its prediction in two launches and adds the update's two (three more launches, timed with the predict in
 * sl2_last_step_times).  A call that turns an off stream on clears that stream's samples in every slot; a call that
 * turns a stream on or off clears its last result (status 0, NIS 0).  Buffer: a sample ring of frame_slots x
 * num_streams, the W scratch of num_streams x (13 + 3 max_features, rounded up to 8) x 3 doubles and the per-stream
 * settings and results.  SL2_ERR_ARG for: reserved != 0 or on outside {0, 1}; a non-finite entry; an R_gc that is not
 * a rotation (|R R^T - I| > 1e-9 in some entry, or det R <= 0); a cov that is not exactly symmetric, or whose Cholesky
 * factor (step 2's formulas) has a pivot argument that is not > 0. */
typedef struct sl2_stream_gyro {
  int32_t on;       /* 0 (default) or 1 */
  int32_t reserved; /* 0 */
  double R_gc[9];   /* row-major rotation: camera frame -> gyro frame */
  double bias[3];   /* rad/s, gyro frame */
  double cov[9];    /* row-major covariance of one sample (rad/s)^2, gyro frame; symmetric positive definite */
} sl2_stream_gyro;
int sl2_set_stream_gyro(sl2_ctx *ctx, int32_t stream_id, const sl2_stream_gyro *g);
int sl2_get_stream_gyro(sl2_ctx *ctx, int32_t stream_id, sl2_stream_gyro *g);
/* The samples of streams [lo, lo + cnt) for the fused step of ring slot `slot`: rates cnt x 3 (rad/s, gyro frame),
 * valid cnt bytes (NULL: all valid; 0 = no sample).  Ordered on the context's stream like sl2_set_stream_config;
 * returns once the caller's buffers may be reused.  Samples of gyro-off streams are kept and never read.  SL2_ERR_ARG,
 * with nothing written, for a bad slot or range, a NULL rates with cnt > 0, or a valid sample with a non-finite rate;
 * SL2_ERR_STATE while no stream of the context has ever turned its gyro on. */
int sl2_set_gyro_samples(sl2_ctx *ctx, int32_t slot, int32_t lo, int32_t cnt, const double *rates,
                         const uint8_t *valid);
/* The staged update of one stream with the sample rate3 (3), using the stream's setting: the same two kernels as the
 * fused step.  SL2_ERR_ARG for a bad stream_id, a NULL or non-finite rate3; SL2_ERR_STATE when the stream's gyro is
 * off.  Synchronises. */
int sl2_gyro_update(sl2_ctx *ctx, int32_t stream_id, const double *rate3);
/* The last gyro update of streams [lo, lo + cnt): status 0 (none this step), 1 (applied) or 2 (skipped: S not positive
 * definite or not finite), and its NIS (0 unless status is 1).  Either pointer may be NULL.  Like the records, not
 * part of a snapshot.  Joins both step groups and synchronises.  SL2_ERR_ARG for a bad range. */
int sl2_get_gyro_results(sl2_ctx *ctx, int32_t lo, int32_t cnt, double *nis, int32_t *status);

/* ---- accelerometer: a measured linear acceleration drives the motion prediction (the reference's control input u,
 *      motion_model.cpp:84-146, with the position term and the noise below) ---------------------------------------
 * The constant-velocity model allows a linear acceleration of sigma = 4 m/s^2 per axis: a camera that is shoved,
 * braked or jolted harder has its features predicted where they are not.  A stream with an accelerometer takes one
 * specific-force sample per step and predicts with the acceleration it measures (Pinies, Lupton, Sukkarieh, Tardos,
 * ICRA 2007).
 * Setting: R_ac (row-major) takes camera-frame vectors into the accelerometer's frame; bias b (m/s^2) and cov C
 * ((m/s^2)^2, the covariance of one sample), both in the accelerometer's frame; gravity g, the gravity vector in the
 * world frame (m/s^2, the map's metres: about (0, 0, -9.81) when the world's z axis points up); sd_a >= 0 (m/s^2), the
 * linear acceleration the sample does not explain (vibration, lever arm, timing), which replaces the model's 4 m/s^2.
 * A sample f is the mean specific force over the frame period [t - dt, t] in the accelerometer's frame, so a device at
 * rest reads -R_ac R(q)^T g + b.  When the setting is made, Rc = R_ac^T C R_ac is formed once, by the formula of
 * sl2_set_stream_gyro, and s2 = sd_a sd_a.
 * Prediction of a step with a sample, x = (r, q, v, omega) the state before the step, dt the stream's delta_t; sums
 * written "sum" start from 0.0 and add their terms in ascending index order:
 *   1. dk = f[k] - b[k]; fc[i] = (R_ac[0][i] d0 + R_ac[1][i] d1) + R_ac[2][i] d2.
 *   2. R = R(q), the model's rotation of q (camera to world; Eigen's toRotationMatrix, also for |q| != 1);
 *      a[i] = sum_k R[i][k] fc[k] + g[i].
 *   3. D = dRq_times_a_by_dq(q, fc) (3 x 4, columns w, x, y, z; feature_model.cpp:164-185): the derivative of the
 *      homogeneous form R(q) fc + (|q|^2 - 1) fc, which equals d(R(q) fc)/dq along directions tangent to |q| = 1;
 *      column c is sum_k Mc[i][k] fc[k] with the reference's dR_by_dq0 / dqx / dqy / dqz matrices Mc.
 *   4. M[i][j] = sum_m R[i][m] Rc[m][j]; for i <= j: t = sum_m M[i][m] R[j][m], plus s2 when i = j;
 *      L[i][j] = L[j][i] = (t dt) dt.
 *   If any of a, D and L is not finite, the step runs the reference prediction (status 2, skipped).
 *   5. h = (0.5 dt) dt; r'[i] = (r[i] + v[i] dt) + a[i] h; q' and omega' as the reference; v'[i] = v[i] + a[i] dt.
 *   6. F is the reference's F with F[i][3 + j] = h D[i][j] and F[7 + i][3 + j] = dt D[i][j] (i < 3, j < 4).
 *   7. Q = Gn Pnn Gn^T with the reference's Gn and, in the kernel's order, (Gn Pnn)[i][k] =
 *      ((0 + Gn[i][0] L[0][k]) + Gn[i][1] L[1][k]) + Gn[i][2] L[2][k] for k < 3; the angular block of Pnn stays
 *      (6 6 dt) dt I.
 *   8. P' = F P F^T + Q through the prediction's own passes, for the 13 x 13 block and the 13 x 3N panel.
 * Every operation is a correctly rounded FP64 operation (never fused) in the order written above and in the kernel
 * (csrc/ekf.cu, accel_model, motion_model and predict_kernel).  A stream that is off, a step without a valid sample
 * and a skipped step run the reference prediction (u = 0) bit for bit.  Out of scope: the lever arm between the
 * accelerometer and the camera, a time offset, online bias estimation and per-sample covariances.
 * Where it applies: the fused step (sl2_step, sl2_step_host, sl2_step_host_async) of ring slot t consumes slot t's
 * sample of every accelerometer-on stream and clears its valid byte, so a sample is used by exactly one step.  The
 * staged form is sl2_accel_predict, in place of sl2_ekf_predict; sl2_ekf_predict(u3) stays the reference's.  With the
 * gyroscope also on, the accelerometer's prediction is the one the gyro update follows.  No launch is added: the work
 * is in the prediction kernel.  The step records are unchanged.
 * on = 0 (the default; the getter then shows R_ac = I, b = 0, C = I, g = 0, sd_a = 4) is off.  A call that turns an
 * off stream on clears that stream's samples in every slot; a call that turns a stream on or off clears its last
 * result (status 0, a = 0).  Buffer: a sample ring of frame_slots x num_streams and the per-stream settings and
 * results.  SL2_ERR_ARG for: reserved != 0 or on outside {0, 1}; a non-finite entry; an R_ac that is not a rotation or
 * a cov that is not symmetric positive definite (the checks of sl2_set_stream_gyro); a negative sd_a. */
typedef struct sl2_stream_accel {
  int32_t on;         /* 0 (default) or 1 */
  int32_t reserved;   /* 0 */
  double R_ac[9];     /* row-major rotation: camera frame -> accelerometer frame */
  double bias[3];     /* m/s^2, accelerometer frame */
  double cov[9];      /* row-major covariance of one sample (m/s^2)^2, accelerometer frame; symmetric positive definite */
  double gravity[3];  /* m/s^2, world frame */
  double sd_a;        /* m/s^2, >= 0: the acceleration a sample does not explain */
} sl2_stream_accel;
int sl2_set_stream_accel(sl2_ctx *ctx, int32_t stream_id, const sl2_stream_accel *a);
int sl2_get_stream_accel(sl2_ctx *ctx, int32_t stream_id, sl2_stream_accel *a);
/* The samples of streams [lo, lo + cnt) for the fused step of ring slot `slot`: forces cnt x 3 (m/s^2, accelerometer
 * frame), valid cnt bytes (NULL: all valid; 0 = no sample).  Ordered on the context's stream like
 * sl2_set_stream_config; returns once the caller's buffers may be reused.  Samples of off streams are kept and never
 * read.  SL2_ERR_ARG, with nothing written, for a bad slot or range, a NULL forces with cnt > 0, or a valid sample with
 * a non-finite force; SL2_ERR_STATE while no stream of the context has ever turned its accelerometer on. */
int sl2_set_accel_samples(sl2_ctx *ctx, int32_t slot, int32_t lo, int32_t cnt, const double *forces,
                          const uint8_t *valid);
/* The staged prediction of one stream with the sample f3 (3), in place of sl2_ekf_predict: the fused step's kernel
 * and operations.  SL2_ERR_ARG for a bad stream_id, a NULL or non-finite f3; SL2_ERR_STATE when the stream's
 * accelerometer is off.  Synchronises. */
int sl2_accel_predict(sl2_ctx *ctx, int32_t stream_id, const double *f3);
/* The last prediction of streams [lo, lo + cnt): accel (cnt x 3) the world-frame a of step 2 (0 unless status is 1;
 * about 0 at rest when R_ac, b and g are right) and status 0 (no sample this step), 1 (applied) or 2 (skipped).
 * Either pointer may be NULL.  Not part of a snapshot.  Joins both step groups and synchronises.  SL2_ERR_ARG for a
 * bad range. */
int sl2_get_accel_results(sl2_ctx *ctx, int32_t lo, int32_t cnt, double *accel, int32_t *status);

/* ---- iterated update: relinearise the EKF update at the updated state (no reference counterpart) -------------------
 * The plain update evaluates h and H once, at the prediction.  When an innovation is large against the curvature of h
 * (a feature whose depth is still uncertain along its ray) that linearisation is wrong to first order: the posterior
 * does not minimise the cost it stands for and its covariance is over-confident.  The iterated update is Gauss-Newton
 * on J(x) = |x - x0|^2_{P0^-1} + sum |z - h(x)|^2_{R^-1} (Bell & Cathey, "The iterated Kalman filter update as a
 * Gauss-Newton method", IEEE TAC 1993).
 * Definitions: x0, P0 are the state and covariance after the prediction (after the gyro update when that is on); M are
 * the step's measured rows (found == 1 after the consensus, in rank order) and z their matches (sub-pixel when
 * refined); R is the prediction's Rvar I and stays fixed; L_0 is the prediction's linearisation, h_eff = h with
 * Hxp = dh/dxp and Hy = dh/dy; N = max_iterations.
 *   for i = 0 .. N-1:
 *     pass i at L_i: S_i = H_i P0 H_i^T + R = U^T U, nu_i = z - h_eff_i (upd_hp and upd_chol, as the update forms them)
 *       t = S_i^-1 nu_i: forward, for every 16-row panel p (rows p0 .. p0 + nb - 1) in order, w_a = sum_b W_pp[a][b]
 *       r_b (b = 0 .. nb-1 in order, from the first product), then every later row j: r_j = r_j - U(p0 + a, j) w_a for
 *       a = 0 .. nb-1 in order (r starts as nu); backward, for every panel from the last, t_a = sum_b W_pp[b][a] r_b
 *       (b in order), then every earlier row j: r_j = r_j - U(j, p0 + a) t_a for a in order (r starts as w).
 *       W_pp = U_pp^-T is the panel inverse upd_chol forms.
 *       x_{i+1}[j] = x0[j] + sum_r (H_i P0)(r, j) t_r (r = 0 .. m-1 in order, from the first product), j < n.
 *     delta_i = max over j < n with P0(j, j) > 0 of |x_{i+1}[j] - x_i[j]| / sqrt(P0(j, j)), x_0 = x0; NaN when an
 *       entry of x_{i+1} is not finite.
 *     delta_i <= tol: status 1 (converged), stop; the final update uses L_i.
 *     relinearise every row of M at x_{i+1} with the prediction's model code (q not renormalised): h, Hxp, Hy;
 *       dx = x0[0:7] - x_{i+1}[0:7], dy = y0 - y_{i+1}; h_eff[r] = h[r] + (((Hxp[r][0] dx0 + Hxp[r][1] dx1) + ...
 *       + Hxp[r][6] dx6) + Hy[r][0] dy0 + ... + Hy[r][2] dy2), left to right.  Invalid when x_{i+1} has a non-finite
 *       entry, a camera-frame depth is <= 0 or any h_eff, Hxp, Hy is not finite: status 3, stop; the final update
 *       uses L_i.  Else L_{i+1}, iterations = i + 1.
 *   the loop ran out: status 2; the final update uses L_N.
 *   final update: the ordinary five-kernel update at L_final from x0, P0 (normalisation, symmetrisation, counters).
 * Every operation above is one correctly rounded, never-fused FP64 operation in the order written (csrc/iterate.cu,
 * iterate_kernel; tests/iterate_ref.py restates it).  max_iterations = 0 is off.  A stream whose pass 0 converges ends
 * byte-identical to the plain update: its final update reads L_0.
 * Where it applies: the fused step (sl2_step, sl2_step_host, sl2_step_host_async) and sl2_ekf_update_measured.
 * sl2_ekf_update with the caller's rows never iterates, and the consensus rescue's second update stays one pass (its
 * re-prediction is at the iterated posterior).  Unchanged: sl2_get_features and sl2_get_feature_jacobians show the
 * step's prediction (h, H, nu = z - h at x0); step records keep their layout, and their m, nis and logdet_s describe
 * the final update; sl2_last_update_times times the final update, sl2_last_step_times()[2] includes the passes.
 * Cost: a step group holding a stream with the iteration on runs N_g = the largest max_iterations of its streams
 * passes of three launches (upd_hp, upd_chol, iterate_kernel) before its update; a stream that has stopped costs an
 * early return per launch.
 * tol is in standard deviations of the prior: 0 always runs N relinearisations.  A call clears the stream's results.
 * Buffer: num_streams x max_features x 22 doubles of tables, num_streams x (13 + 3 max_features, rounded up to 8)
 * doubles of iterate and the settings and results.  SL2_ERR_ARG for reserved != 0, max_iterations outside
 * [0, SL2_MAX_ITERATIONS], or a tol that is not finite and >= 0. */
#define SL2_MAX_ITERATIONS 8
typedef struct sl2_stream_iterated {
  int32_t max_iterations; /* 0 (default, off) .. SL2_MAX_ITERATIONS relinearisations */
  int32_t reserved;       /* 0 */
  double tol;             /* stop when the step is at most tol prior standard deviations in every entry; >= 0 */
} sl2_stream_iterated;
int sl2_set_stream_iterated(sl2_ctx *ctx, int32_t stream_id, const sl2_stream_iterated *v);
int sl2_get_stream_iterated(sl2_ctx *ctx, int32_t stream_id, sl2_stream_iterated *v);
/* The last step of streams [lo, lo + cnt): iterations (relinearisations used by the final update), status (0: off or
 * no measured rows, 1 converged, 2 ran out, 3 invalid relinearisation) and the last delta.  Any pointer may be NULL.
 * Not part of a snapshot.  Joins both step groups and synchronises.  SL2_ERR_ARG for a bad range. */
int sl2_get_iterated_results(sl2_ctx *ctx, int32_t lo, int32_t cnt, int32_t *iterations, int32_t *status,
                             double *last_delta);

/* ---- frames (replaces the cv::Mat `frame` argument of MonoSLAM::GoOneStep, monoslam.cpp:108) */
/* The frame ring keeps the context's width x height per stream.  A stream whose image is smaller
 * (sl2_set_stream_config) occupies the top-left width_s x height_s of its block; the rest of the block
 * is never read into a result. */
/* one stream, one slot: copies the stream's width_s x height_s image, or its raw frame when the stream has a source
 * (below); `stride` = bytes between image (raw) rows */
int sl2_set_frame(sl2_ctx *ctx, int32_t stream_id, int32_t slot, const uint8_t *gray, size_t stride);
/* all streams of a slot at once: gray is the frame set of sl2_frame_set_layout, which is [num_streams][height][width]
 * contiguous, in the context's size, while every stream has the default source (pinned memory makes the copy
 * asynchronous) */
int sl2_set_frames(sl2_ctx *ctx, int32_t slot, const uint8_t *gray);
/* device-resident producer: copy device -> device, same layout as sl2_set_frames */
int sl2_set_frames_dev(sl2_ctx *ctx, int32_t slot, const uint8_t *gray_dev);

/* ---- live cameras: per-stream raw frame sources (framegrabber/usbcamgrabber.cpp:75-113) --------------------------
 * The reference's camera grabber takes a raw RGB24 or YUV422 (UYVY) frame, converts it with cv::cvtColor(CV_RGB2GRAY
 * / CV_YUV2GRAY_Y422) and, when it is not the cfg's image size, cv::resize(..., CV_INTER_LINEAR)s it.  A stream with a
 * source takes that raw frame and the device does both: the host only copies bytes.
 *   SL2_SRC_GRAY_RING (width = height = 0, the default): the stream contributes the context's width x height gray
 *     block to a frame set, exactly as without sources.  A context whose streams all have it runs no extra kernel.
 *   otherwise: the stream's raw frame is width x height x bpp bytes, rows contiguous.  The device converts it to gray
 *     and, when width x height differs from the stream's image (sl2_stream_config width_s x height_s), resizes it
 *     (OpenCV's 8-bit INTER_LINEAR, bit for bit) into the stream's block of the ring slot being written.
 * Frame sets (sl2_set_frames[_dev], sl2_step_host[_async]) hold the streams' frames back to back, in stream order;
 * sl2_frame_set_layout gives the byte offset of each (offsets[num_streams] = the total).
 * Ordering: like sl2_set_stream_config (frames copied after the call use the new source); joins both step groups and
 * synchronises when it has to grow the device staging of the raw frames (slots x the raw bytes of a frame set).
 * SL2_ERR_ARG, with the source unchanged, for: a bad stream_id or NULL src; an unknown format; reserved != 0; the
 * default format with a non-zero size; another format with a dimension outside [1, SL2_MAX_SOURCE_DIM]; an odd UYVY
 * width.  A source belongs to the stream slot, like the frame ring: snapshots do not carry it and a load leaves it. */
#define SL2_SRC_GRAY_RING 0 /* default */
#define SL2_SRC_GRAY8 1     /* 1 B/px gray at the source size */
#define SL2_SRC_RGB24 2     /* 3 B/px, R G B: cvtColor(CV_RGB2GRAY) of OpenCV 2.4 */
#define SL2_SRC_UYVY 3      /* 2 B/px, U Y0 V Y1: cvtColor(CV_YUV2GRAY_Y422) (Y422 == UYVY in OpenCV) */
#define SL2_MAX_SOURCE_DIM 4096
typedef struct sl2_stream_source {
  int32_t format, width, height, reserved;
} sl2_stream_source;
int sl2_set_stream_source(sl2_ctx *ctx, int32_t stream_id, const sl2_stream_source *src);
int sl2_get_stream_source(sl2_ctx *ctx, int32_t stream_id, sl2_stream_source *src);
/* offsets: num_streams + 1 entries */
int sl2_frame_set_layout(sl2_ctx *ctx, size_t *offsets);

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
 * Returns the index of the new feature (>= 0), SL2_ERR_STATE when the map already holds max_features
 * (<= SL2_MAX_FEATURES). */
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
 * Returns the number of surviving particles, < 0 on error.  0 has two causes: every probability is zero (the
 * reference deletes the feature; prob is left un-normalised), or every particle fell below the prune threshold (the
 * reference keeps the feature with no particles; prob holds the probabilities normalised before the prune). */
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
 * array is F x Kmax (entries k >= K[f] are ignored on input and left as the caller had them on output).
 * in : patches (F x boxsize x boxsize u8), ypi (F x 6: r, hhat), Pxy (F x 13x6 column-major: covariance between
 *      x_v and the feature's 6 states), Pyy (F x 6x6 column-major), lambda (F x Kmax), prune threshold;
 * in/out: prob (F x Kmax);
 * out (each may be NULL): h (F x Kmax x 2), Sinv3 (F x Kmax x (S00,S01,S11)), detS (F x Kmax), z_uv (F x Kmax x 2),
 *      found, keep (F x Kmax), cumulative (F x Kmax), mean_var (F x 2), left (F: survivors; 0 as for
 *      sl2_measure_particles: deleted by the reference, or kept with every particle pruned). */
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
 * sl2_predict_measurements, followed by the stream's match consensus when it is on; returns the number of
 * successful measurements after the consensus. */
int sl2_make_measurements(sl2_ctx *ctx, int32_t stream_id, int32_t slot);
/* Kalman::KalmanFilterUpdate (kalman.cpp:72-119) with host-supplied measurement rows, in the
 * order of construct_total_measurement_stuff (monoslam.cpp:548-572): row pair k belongs to
 * feature feat_index[k]; H_xv is (2k_meas) x 13 row-major, H_y (2k_meas) x 3 row-major,
 * R k_meas x (2x2 col-major, symmetric: SL2_ERR_ARG otherwise; the full block enters S), nu 2k_meas.
 * m = 2 * k_meas <= 2 * min(max_features, SL2_MAX_MEASURED); SL2_ERR_ARG above that. */
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
/* end-to-end form: host frames in (the frame set of sl2_set_frames), camera states out
 * (xv_out: [num_streams][13], may be NULL).  Copies run on the context's stream. */
int sl2_step_host(sl2_ctx *ctx, int32_t slot, const uint8_t *gray, double *xv_out);
/* asynchronous end-to-end form for a frame ring: enqueues the H2D copy of `gray` into `slot` on a
 * copy stream (with the conversion of the streams that have a source), the fused step, and the D2H of the camera states into xv_out, then returns. gray and
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

/* ---- read-back of per-feature results (Feature::h_/z_/S_/flags/counters, feature.h:96-140) */
int sl2_get_features(sl2_ctx *ctx, int32_t stream_id, double *h /* n x 2 */, double *z /* n x 2 */,
                     double *S /* n x 4 col-major */,
                     uint8_t *flags /* bit0 selected, bit1 successful, bit2 matched and rejected by the match
                                       consensus (sl2_set_stream_consensus), bit3 z is the sub-pixel match
                                       (sl2_set_stream_subpixel) */,
                     int32_t *attempted, int32_t *successful, int32_t *select_rank);
/* Feature::dh_by_dxv_ (2x13), dh_by_dy_ (2x3), R_ (2x2), nu_ (2) of the last prediction /
 * measurement, all column-major like the Eigen members (feature.h:104-112). Arrays may be NULL. */
int sl2_get_feature_jacobians(sl2_ctx *ctx, int32_t stream_id, double *dh_by_dxv /* n x 26 */,
                              double *dh_by_dy /* n x 6 */, double *R /* n x 4 */,
                              double *nu /* n x 2 */);
/* device-time of the kernels of the last sl2_step (ms): [0] predict+select (and the gyro update), [1] patch search,
 * [2] EKF update (with the consensus rescue and its second update when a stream has them on), [3] cull.  Valid after
 * sl2_enable_timing(ctx, 1). */
int sl2_enable_timing(sl2_ctx *ctx, int32_t on);
int sl2_last_step_times(sl2_ctx *ctx, float *ms4);
/* the five kernels of the EKF update of the last sl2_step (ms): [0] hp (measurement list, H P, S = H P H^T + R),
 * [1] chol (Cholesky of S), [2] solve (Y = U^-T [H P | nu]), [3] syrk (P -= Y^T Y, x += Y^T w), [4] finish
 * (normalise, symmetrise, counters).  Their sum is sl2_last_step_times()[2], less the consensus rescue's kernels on a
 * step that ran them: these times are the first update's. */
int sl2_last_update_times(sl2_ctx *ctx, float *ms5);
/* kernels launched by this context since creation */
int64_t sl2_launch_count(const sl2_ctx *ctx);

/* ---- stream snapshots: save, restore and move camera streams (no reference counterpart) ----------------------
 * A snapshot is ONE stream's blob: everything a later entry point reads of that stream, so that a stream loaded
 * into any stream id of any context (same boxsize, capacity >= its map, frame at least its image; another device
 * through the host form) continues bit for bit like the stream it was saved from.  Uses: checkpoint / resume,
 * moving a camera to another GPU or to a context of another capacity, rollback after a bad frame, cloning a stream.
 *
 * Format (version 1).  Host byte order; a blob of the other byte order fails the magic.  No checksum, no
 * compression.  The header below, then these sections, in this order, each starting 8-byte aligned (zero bytes pad
 * a section to the next multiple of 8), each sized from nfeat and boxsize only (never from the context's capacity):
 *    x          double[n]                  n = 13 + 3 nfeat
 *    P          double[n * n]              column-major, dense: what sl2_get_state returns
 *    xp_org     double[nfeat][7]           camera position state each feature was first seen from
 *    attempted  int32[nfeat]               measurement attempts (the cull of delete_bad_features reads them)
 *    successful int32[nfeat]               successful measurements
 *    h          double[nfeat][2]           last prediction
 *    S          double[nfeat][4]           column-major 2x2
 *    Rvar       double[nfeat]              measurement noise variance
 *    dh_dxp     double[nfeat][2][7]        row-major
 *    dh_dy      double[nfeat][2][3]        row-major
 *    sel_rank   int32[nfeat]               rank in the selected list, -1 = not selected
 *    z_uv       int32[nfeat][2]            last match
 *    found      uint8[nfeat]               1 = the last measurement of the feature succeeded, 2 = it matched and the
 *                                          match consensus rejected it, 0 = it failed
 *    best       double[nfeat]              last correlation score
 *    job_feat   int32[nfeat]               feature of measurement job r (-1 = none): only jobs r < nsel hold one
 *    job_centre double[nfeat][2]           search centre of job r
 *    job_puinv  double[nfeat][3]           search ellipse (P00, P01, P11) of job r
 *    templates  uint8[nfeat][box][box]     row-major, without the device's row padding
 * The rule for what goes in: every per-stream array of the device state that an entry point reads before a later
 * kernel overwrites it.  Out: scratch of one update, the frame ring, and the context-wide settings (boxsize, search
 * tile radius, minimum_attempted_measurements_of_feature, successful_match_fraction, search_override), which belong
 * to the receiving context; the stream's frame source (sl2_set_stream_source) stays with the stream slot, like the
 * frame ring, and a load leaves the slot's source as it was (the loaded camera's image becomes its resize target, as
 * with sl2_set_stream_config).  The format is canonical: a blob saved, loaded anywhere and saved again is
 * byte-identical. */
#define SL2_SNAPSHOT_MAGIC 0x53324C53u /* the bytes "SL2S" on a little-endian host */
#define SL2_SNAPSHOT_VERSION 1

typedef struct sl2_snapshot_header {
  uint32_t magic;         /* SL2_SNAPSHOT_MAGIC */
  uint32_t version;       /* SL2_SNAPSHOT_VERSION */
  uint32_t header_bytes;  /* sizeof(sl2_snapshot_header) = 128 */
  uint32_t reserved0;     /* 0 (a load refuses anything else) */
  uint64_t total_bytes;   /* the whole blob, header included */
  int32_t boxsize;        /* template size; must equal the receiving context's */
  int32_t nfeat;          /* map features */
  int32_t n;              /* state size 13 + 3 nfeat */
  int32_t reserved1;      /* 0 (a load refuses anything else) */
  sl2_stream_config cam;  /* the stream's camera (sl2_set_stream_config), padding bytes zero */
  int32_t nsel;           /* job slots of the last prediction (<= SL2_MAX_MEASURED) */
  int32_t nvisible;       /* visible features of the last prediction (<= SL2_MAX_FEATURES) */
  int32_t nmeas;          /* successful measurements of the last update (<= SL2_MAX_MEASURED) */
  int32_t ncull;          /* features the cull of the last update found (<= SL2_MAX_FEATURES) */
} sl2_snapshot_header;
/* The four counts describe the last prediction / update and are not renewed by every call that changes the map: a
 * cull, sl2_delete_feature and sl2_set_features leave nvisible, ncull and (sl2_set_features) nsel as they were, so a
 * saved stream may hold nvisible, ncull or nsel above nfeat, and job slots below nsel that hold -1.  Loads accept
 * these states, which the library produces itself: no kernel indexes with nvisible, nmeas or ncull, and nsel only
 * bounds a walk over the job slots, which a load fills with -1 beyond nfeat. */

/* Byte offsets of the sections of a blob of nfeat features with boxsize x boxsize templates, in the order above
 * (field[0] = xp_org ... field[14] = job_puinv), and the blob's total size.  SL2_ERR_ARG unless
 * 0 <= nfeat <= SL2_MAX_FEATURES and boxsize > 0. */
#define SL2_SNAPSHOT_FIELDS 15
typedef struct sl2_snapshot_sections {
  uint64_t x, P, field[SL2_SNAPSHOT_FIELDS], templates, total;
} sl2_snapshot_sections;
int sl2_snapshot_layout(int32_t nfeat, int32_t boxsize, sl2_snapshot_sections *out);

/* Upper bound of one stream's blob in this context: the size of a map of max_features features. */
size_t sl2_snapshot_bytes(const sl2_ctx *ctx);
/* Blob i belongs to stream lo + i and lies at buf + i * stride.
 * Ordering: like every other entry point, these join both step groups first.  A save captures the state after
 * everything queued before it (an sl2_step_host_async that has not been waited for included); a load is seen by
 * the next call (the next fused step and an sl2_step_host_async queued after it included).
 * sl2_save_streams synchronises and writes each blob's size to sizes[i] (sizes may be NULL);
 * sl2_save_streams_dev is asynchronous on the context's stream, like sl2_set_frames_dev.  The host forms stage the
 * batch through the context's pinned staging buffer in groups of streams of at most 64 MB (at least one stream), so
 * the buffer stays bounded whatever the batch.  Saves need
 * stride >= the context's snapshot size; the device forms need buf_dev and stride to be multiples of 8.
 * Loads are all or nothing: every header of the batch (for the device form: copied down first) and the index
 * fields later kernels index with (job_feat, sel_rank; the device form checks them with a kernel) are validated
 * before anything is written, and the kernels use the validated sizes.  Both loads synchronise.  SL2_ERR_ARG for a
 * bad range, NULL pointer or short stride; a wrong magic, version or header size, non-zero reserved fields, a total
 * size above the stride or different from the one nfeat and boxsize give; n != 13 + 3 nfeat; a negative count;
 * nsel or nmeas above SL2_MAX_MEASURED, nvisible or ncull above SL2_MAX_FEATURES; a boxsize other than the
 * context's; a job_feat that is neither -1 nor in [0, nfeat) for r < nsel, or not -1 for r >= nsel; a sel_rank that
 * is neither -1 nor in [0, min(nsel, nfeat)) (the cull writes job slot sel_rank); a camera sl2_set_stream_config
 * would refuse in this context.  SL2_ERR_STATE when nfeat exceeds the context's max_features.  On an error no
 * stream of the batch changes.
 * A load resets what the blob does not cover to the values sl2_create / sl2_set_features leave: x and P outside
 * n x n, the per-feature records, job slots and templates beyond nfeat are zero, sel_rank and job_feat -1.  A
 * stream's results therefore never depend on what it held before the load. */
int sl2_save_streams(sl2_ctx *ctx, int32_t lo, int32_t cnt, void *buf, size_t stride, size_t *sizes);
int sl2_load_streams(sl2_ctx *ctx, int32_t lo, int32_t cnt, const void *buf, size_t stride);
int sl2_save_streams_dev(sl2_ctx *ctx, int32_t lo, int32_t cnt, void *buf_dev, size_t stride);
int sl2_load_streams_dev(sl2_ctx *ctx, int32_t lo, int32_t cnt, const void *buf_dev, size_t stride);

/* ---- step records: every camera stream's trajectory and filter health, kept on the device --------------------
 * MonoSLAM::GoOneStep(frame, save_trajectory, ...) appends the camera position to trajectory_store_ (capped at 1000
 * entries, monoslam.cpp:172-177).  With records on, the fused step (sl2_step, sl2_step_host, sl2_step_host_async)
 * writes one record per camera stream per step into a ring of `depth` records per stream, so the trajectory and the
 * health of hundreds of streams come back in one call instead of one synchronising call per stream and quantity.
 * The staged entry points, snapshots, sl2_set_*, sl2_append_feature and sl2_delete_feature write no record and alter
 * none; a snapshot load does not rewrite a stream's past records (the snapshot format is unchanged).
 *
 * nis and logdet_s are the two standard consistency checks of the step's EKF update, S = H P H^T + R of the m
 * measured rows: nis = nu^T S^-1 nu (chi-square with m degrees of freedom when the filter is consistent) and
 * log det S.  Both are reduced on the device in a fixed order, so a stream's record does not depend on its position in
 * the batch or on the step groups. */
#define SL2_MAX_RECORDS 4096
typedef struct sl2_step_record { /* 256 bytes, no padding */
  int64_t step;         /* index of the fused step since records were (re-)enabled: 0, 1, 2, ... */
  int32_t nfeat;        /* map features after the step's cull */
  int32_t nvisible;     /* visible features of the step's prediction */
  int32_t nsel;         /* features of the step's selection still in the map after the cull (the reference's
                           selected_feature_list_ after GoOneStep) */
  int32_t nmeas;        /* successful measurements (= rows m / 2 of the update; after the match consensus) */
  int32_t nculled;      /* features the step's cull deleted */
  int32_t m;            /* rows of S; 0 when nothing was measured */
  double nis;           /* nu^T S^-1 nu of the step's update; 0 when m == 0 */
  double logdet_s;      /* log det S; 0 when m == 0 */
  double xv[13];        /* camera state after the step (xv[0..2] = the trajectory point of trajectory_store_) */
  double pxx_diag[13];  /* diagonal of Pxx after the step */
} sl2_step_record;

/* depth 0 = off (the default; frees the ring), 1 .. SL2_MAX_RECORDS = records per stream kept.  Joins both step groups
 * like every entry point, (re)allocates the ring (num_streams x depth x 256 bytes) and restarts `step` at 0; calling
 * it with the current depth also clears the ring.  SL2_ERR_ARG for a depth outside [0, SL2_MAX_RECORDS]. */
int sl2_enable_records(sl2_ctx *ctx, int32_t depth);
/* The most recent k = min(max, steps recorded, depth) records of each stream lo + i, oldest first, at
 * out[i * max + j], j < k.  All streams step together, so k is the same for every stream; returns k.
 * sl2_get_records synchronises; sl2_get_records_dev is asynchronous on the context's stream and needs out_dev to be
 * 8-byte aligned.  SL2_ERR_ARG for a bad range, a NULL pointer or max < 1; SL2_ERR_STATE while records are off.
 * On an error nothing changes. */
int sl2_get_records(sl2_ctx *ctx, int32_t lo, int32_t cnt, int32_t max, sl2_step_record *out);
int sl2_get_records_dev(sl2_ctx *ctx, int32_t lo, int32_t cnt, int32_t max, void *out_dev);

/* ---- relocalisation: put a lost camera stream back on its own map (no reference counterpart) --------------------
 * Williams, Klein, Reid, "Real-Time SLAM Relocalisation", ICCV 2007: find the map's features anywhere in the frame,
 * estimate the camera pose from those 2-D / 3-D matches with a three-point consensus, and restart the filter there.
 * For each listed stream s, in the frame of ring slot `slot`:
 *   1. Full-image search.  Every map feature i < nfeat is searched with the rules of sl2_patch_search (search box,
 *      ellipse test, sigma gates, scan-order arg-min, corrmax <= 0.40) with one job centred on ((w - 1) / 2,
 *      (h - 1) / 2) with PuInv = diag(eps, eps), eps = 9 / (w^2 + h^2) of the stream's w x h image: an ellipse that
 *      holds every window position.  M = the features whose search succeeded, in feature-index order; k = |M|.
 *   2. Bearings.  z_j (the match pixel) -> Camera::Unproject (camera.cpp:133-157) -> divided by its norm.
 *   3. Hypotheses.  Hypothesis h in [0, SL2_RELOC_HYPOTHESES) takes the matches (M[i0], M[i1], M[i2]) with
 *      a = g(3h), b = g(3h + 1), c = g(3h + 2), g(x) = splitmix64 (Steele, Lea, Flood 2014) of state x, i.e. the
 *      finaliser applied to x + 0x9E3779B97F4A7C15:  i0 = a mod k;  i1 = b mod (k - 1), then + 1 if >= i0;
 *      i2 = c mod (k - 2), then + 1 if >= min(i0, i1), then + 1 if >= max(i0, i1).  k < 3: no hypothesis.
 *      Each triple goes through Kneip, Scaramuzza, Siegwart's P3P (CVPR 2011): up to 4 poses, in the order of the
 *      real roots of its quartic.  Collinear or coincident points or bearings, and any non-finite pose, give none.
 *   4. Support of a pose xp = (r, q): match j is an inlier when the camera model (pose_RRW, zeroed_point,
 *      project_point in csrc/sl2_model.cuh) maps y_j to a point in front of the camera whose squared distance to z_j is
 *      <= fl(tau * tau); a NaN distance never is.  The winner has the largest support; ties go to the lowest
 *      (hypothesis, pose) index.
 *   5. Refinement: SL2_RELOC_GN_ITERS Gauss-Newton steps over the position and a body-frame rotation increment on the
 *      winner's inliers (stopping early when the 6 x 6 normal matrix is not positive definite); the inliers are then
 *      counted again with the refined pose.
 *   6. Acceptance iff that count >= min_inliers.  Then and only then the stream's state is written: x[0:3] = r,
 *      x[3:7] = q, x[7:10] = v, x[10:13] = omega, P[0:13, 0:13] = Pxx, P[0:13, 13:n] = P[13:n, 0:13] = 0.  Nothing
 *      else of the stream changes (Pyy, templates, counters, per-feature results, job slots, records).
 * A stream's results and writes depend only on its state, its frame and the arguments (not on the list, its order,
 * the stream id, the capacity or the step groups).  Unlisted streams are not touched.  Joins both step groups like
 * every entry point, is ordered with queued work and synchronises; writes no step record.  Two kernel launches per
 * call with cnt >= 1 (the search and the pose kernel); cnt = 0 does nothing.
 * out[i] describes stream_ids[i]; z_uv[i][f] is the search's best position of feature f ((-1, -1) when no candidate
 * was scored or f >= nfeat), flags[i][f] bit0 = matched (f in M), bit1 = inlier of the refined pose.
 * SL2_ERR_ARG, with nothing changed, for: cnt < 0; a NULL stream_ids (cnt > 0), p, Pxx or out; a bad or repeated
 * stream id; a bad slot; tau <= 0 or not finite; min_inliers < 4; reserved != 0; a non-finite v or omega, or
 * |omega| = 0; a Pxx that is not finite, not exactly symmetric, or has an eigenvalue below -1e-12 times its largest
 * eigenvalue magnitude (not positive semi-definite). */
#define SL2_RELOC_HYPOTHESES 1024 /* three-point hypotheses per stream and call */
#define SL2_RELOC_GN_ITERS 5      /* Gauss-Newton steps of the refinement */
typedef struct sl2_reloc_params {
  double inlier_px;      /* tau > 0: a match agrees with a pose when its reprojection is within tau px */
  int32_t min_inliers;   /* >= 4: inliers the refined pose needs to be accepted */
  int32_t reserved;      /* 0 */
  double v[3], omega[3]; /* velocity state written on acceptance; |omega| > 0 (omega = 0 makes the motion model's F
                            NaN) */
} sl2_reloc_params;
typedef struct sl2_reloc_result {
  int32_t status;  /* 1 = accepted and written, 0 = the stream is unchanged */
  int32_t matches; /* k: features whose full-image search succeeded */
  int32_t support; /* inliers of the winning hypothesis (0 when no hypothesis exists) */
  int32_t inliers; /* inliers of the refined pose (0 when no hypothesis exists) */
  double rms_px;   /* RMS reprojection error over those inliers (NaN when there are none) */
  double pose[7];  /* r (3), q (w, x, y, z; unit, w >= 0) of the refined pose; NaN when no hypothesis exists */
} sl2_reloc_result;
int sl2_relocalise(sl2_ctx *ctx, const int32_t *stream_ids, int32_t cnt, int32_t slot, const sl2_reloc_params *p,
                   const double *Pxx /* 13 x 13 column-major */, sl2_reloc_result *out /* cnt */,
                   int32_t *z_uv /* cnt x max_features x 2, may be NULL */,
                   uint8_t *flags /* cnt x max_features, may be NULL */);

/* ---- stream recovery: detect a lost stream inside the fused step and relocalise it there (no reference counterpart)
 * A stream that has lost its camera keeps adding failed attempts to every feature it selects, and the cull then
 * deletes the map a relocalisation needs; a host that notices the loss from the step records must synchronise first.
 * With recovery on, the fused step itself notices the loss, stops selecting features (so the map is kept) and tries
 * sl2_relocalise on its own frame.  For every stream with lost_after > 0, at the end of the fused step of ring slot
 * `slot` (after the cull and the step record, so the record keeps its meaning), with n = the step's nmeas (the count
 * its record shows):
 *   1. A stream that entered the step tracking: failed_steps = n < min_matches ? failed_steps + 1 : 0.  When
 *      failed_steps >= lost_after the stream becomes lost (lost = 1, lost_steps = 0; failed_steps keeps its value) and
 *      tries on this step.
 *   2. A stream that entered the step lost: lost_steps = lost_steps + 1; it tries when lost_steps % retry_period == 0.
 *   3. A try is exactly sl2_relocalise of that one stream on `slot` with the setting's reloc and Pxx: the same
 *      full-image jobs (centre ((w - 1) / 2, (h - 1) / 2), eps = 9 / (w^2 + h^2) of the stream's own image, formed
 *      with the same correctly rounded operations), the same hypotheses, decision and state write.  attempted = 1 and
 *      `last` = its result.  Accepted: recoveries + 1, and the stream is tracking again with lost = failed_steps =
 *      lost_steps = 0.  Rejected: nothing else changes and the stream stays lost.  A step without a try sets
 *      attempted = 0 and keeps `last`.
 *   4. A step that a stream enters lost selects no feature, under SL2_SELECT_TRACE and SL2_SELECT_INFORMATION alike,
 *      exactly as that step would with number_of_features_to_select = 0; everything else of the step runs as usual
 *      (motion prediction, gyro update, visibility, record).  No selection means no attempt, so the cull keeps the map.
 * Resets: the setter, a snapshot load into the stream, sl2_set_state, sl2_set_features and an accepted sl2_relocalise
 * of the stream return it to tracking (lost = failed_steps = lost_steps = 0); the setter also clears attempted,
 * recoveries and last.  Turning the setting off (lost_after = 0) therefore also resumes selection.
 * Where it applies: sl2_step, sl2_step_host and sl2_step_host_async (whose xv_out shows the state after the whole step,
 * an accepted try included).  The staged entry points and the C++ shim never run it.  The recovery state belongs to the
 * stream slot like the setting (one of the per-stream options, above): snapshots do not carry it (the format is
 * unchanged).
 * Cost: a step group holding a stream with recovery on launches three more kernels per step, after the step's timing
 * events (recover_kernel, the full-image search over the streams that try, reloc_kernel); a stream that does not try
 * costs an early return in each.
 * Buffer: the settings and states, a job table and search results of num_streams x max_features entries.  SL2_ERR_ARG
 * for: reserved != 0; lost_after < 0; with lost_after > 0, min_matches < 1 or retry_period < 1, or a reloc or Pxx that
 * sl2_relocalise refuses. */
typedef struct sl2_stream_recovery {
  int32_t lost_after;     /* 0 (default) = off; K >= 1: K consecutive failed steps declare the stream lost */
  int32_t min_matches;    /* >= 1: a step fails when its nmeas is < min_matches */
  int32_t retry_period;   /* >= 1: a lost stream tries on the step it is declared lost, then every retry_period-th */
  int32_t reserved;       /* 0 */
  sl2_reloc_params reloc; /* as for sl2_relocalise */
  double Pxx[169];        /* restart covariance, 13 x 13 column-major: as for sl2_relocalise */
} sl2_stream_recovery;
int sl2_set_stream_recovery(sl2_ctx *ctx, int32_t stream_id, const sl2_stream_recovery *r);
int sl2_get_stream_recovery(sl2_ctx *ctx, int32_t stream_id, sl2_stream_recovery *r);
typedef struct sl2_recovery_result {
  int32_t lost;          /* 1 while the stream is lost after the last step */
  int32_t failed_steps;  /* consecutive failed steps while tracking */
  int32_t lost_steps;    /* steps since the stream was declared lost */
  int32_t attempted;     /* 1 when the last step tried a relocalisation */
  int64_t recoveries;    /* accepted tries since the setting was made */
  sl2_reloc_result last; /* the last try's result, as sl2_relocalise reports it (zero before the first) */
} sl2_recovery_result;
/* The recovery state of streams [lo, lo + cnt) after the last step (zero for streams never turned on).  Joins both
 * step groups and synchronises.  SL2_ERR_ARG for a bad range or a NULL out with cnt > 0. */
int sl2_get_recovery_results(sl2_ctx *ctx, int32_t lo, int32_t cnt, sl2_recovery_result *out);

#ifdef __cplusplus
}
#endif
#endif /* SL2B200_H */
