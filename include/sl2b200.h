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
 * inlier_px = 0 (the default) is off: a context where no stream has it on runs exactly the path without it.
 * Ordering like sl2_set_stream_config.  The setting belongs to the stream slot, like the frame source: snapshots do
 * not carry it and a load leaves it.  SL2_ERR_ARG, with the setting unchanged, for a bad stream_id, a negative, NaN
 * or infinite inlier_px, or (get) a NULL inlier_px. */
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
 * (timed with the update in sl2_last_step_times; sl2_last_update_times keeps timing update 1).  Ordering like
 * sl2_set_stream_config.  The setting belongs to the stream slot, like the match consensus: snapshots do not carry it
 * and a load leaves it.  The first stream turned on sizes the context's rescue scratch (num_streams x 20 bytes):
 * SL2_ERR_CUDA, with the setting unchanged, when that allocation fails.  SL2_ERR_ARG, with the setting unchanged, for
 * a bad stream_id, a negative, NaN or infinite chi2, or (get) a NULL chi2. */
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
 * on = 0 (the default) is off, 1 is on: a context where no stream has it on runs exactly the path without it; one with
 * a stream that has it on adds one kernel launch per step group holding such a stream (timed with the search in
 * sl2_last_step_times).  Ordering like sl2_set_stream_config.  The setting belongs to the stream slot, like the match
 * consensus and the frame source: snapshots do not carry it and a load leaves it.  The first stream turned on sizes
 * the context's warped-template scratch (num_streams x max_features x boxsize x 16 bytes): SL2_ERR_CUDA, with the
 * setting left off, when that allocation fails.  SL2_ERR_ARG, with the setting unchanged, for a bad stream_id, an
 * `on` other than 0 or 1, or (get) a NULL on. */
int sl2_set_stream_warp(sl2_ctx *ctx, int32_t stream_id, int32_t on);
int sl2_get_stream_warp(sl2_ctx *ctx, int32_t stream_id, int32_t *on);
/* The warped templates of features feat_index[0 .. n) of stream_id at the pose xp (7: r, q), whatever the stream's
 * setting: what the search of a warp-on stream sees at that pose.  out: n x boxsize x boxsize u8, row-major; valid (n,
 * may be NULL): 1 = warped, 0 = some pixel is invalid and out holds the stored template.  Joins both step
 * groups and synchronises.  SL2_ERR_ARG, with nothing written, for: a bad stream_id; n outside [0, max_features]; a
 * NULL feat_index, xp or out with n > 0; a feat_index outside [0, nfeat); a non-finite xp or a zero quaternion. */
int sl2_warp_templates(sl2_ctx *ctx, int32_t stream_id, int32_t n, const int32_t *feat_index, const double *xp,
                       uint8_t *out, uint8_t *valid);

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
 * on = 0 (the default) is off, 1 is on: a context where no stream has it on runs exactly the path without it; one with
 * a stream that has it on adds one kernel launch per step group holding such a stream (timed with the search in
 * sl2_last_step_times).  Ordering like sl2_set_stream_config.  The setting belongs to the stream slot, like the warp:
 * snapshots do not carry it and a load leaves it.  A loaded stream's z is its integer match (bit 3 clear) until its
 * next step; so is a stream's after the setting is made.  The first stream turned on sizes the context's scratch
 * (num_streams x (17 max_features + 1) bytes): SL2_ERR_CUDA, with the setting left off, when that allocation fails.
 * SL2_ERR_ARG, with the setting unchanged, for a bad stream_id, an `on` other than 0 or 1, or (get) a NULL on. */
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
 * mode SL2_SELECT_TRACE (the default) is the reference's rule: a context where no stream selects by information runs
 * exactly the path without it; one where some stream does adds one kernel launch per step group holding such a
 * stream and per sl2_predict_measurements of one (timed with the predict in sl2_last_step_times).  Ordering like
 * sl2_set_stream_config.  The setting belongs to the stream slot, like the match consensus: snapshots do not carry it
 * and a load leaves it.  When a stream first turns the information rule on and the factors of
 * kmax = min(max_features, SL2_MAX_MEASURED) picks cannot stay in shared memory, the context sizes its factor scratch
 * (num_streams x max_features x kmax x 32 bytes): SL2_ERR_CUDA, with the setting unchanged, when that allocation
 * fails.  SL2_ERR_ARG, with the setting unchanged, for: a bad stream_id or NULL sel; an unknown mode; reserved != 0;
 * a min_bits that is negative or not finite, or non-zero with SL2_SELECT_TRACE. */
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
 * on = 0 (the default; the getter then shows R_gc = I, b = 0, C = I) is off: a context where no stream has it on runs
 * exactly the path without it; a step group holding a gyro-on stream splits its prediction in two launches and adds
 * the update's two (three more launches, timed with the predict in sl2_last_step_times).  Ordering like
 * sl2_set_stream_config.  The setting belongs to the stream slot, like the match consensus: snapshots do not carry it
 * and a load leaves it.  A call that turns an off stream on clears that stream's samples in every slot; a call that
 * turns a stream on or off clears its last result (status 0, NIS 0).  The first stream turned on allocates the
 * context's gyro buffers (a sample ring of frame_slots x num_streams, the W scratch of num_streams x (13 + 3 max_features, rounded up to 8) x 3 doubles and the per-stream
 * results): SL2_ERR_CUDA, with the setting left off, when that allocation fails.  SL2_ERR_ARG, with the setting
 * unchanged, for: a bad stream_id or NULL g; reserved != 0 or on outside {0, 1}; a non-finite entry; an R_gc that is
 * not a rotation (|R R^T - I| > 1e-9 in some entry, or det R <= 0); a cov that is not exactly symmetric, or whose
 * Cholesky factor (step 2's formulas) has a pivot argument that is not > 0. */
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

#ifdef __cplusplus
}
#endif
#endif /* SL2B200_H */
