/* deepi2p_b200 -- C ABI of the H100-native inverse-camera-projection registration path.
 *
 * Plain C, no torch / pybind types: every pointer marked [dev] is a CUDA device pointer owned
 * by the caller, every launch goes to the cudaStream_t the caller passes (0 = legacy default
 * stream), nothing is retained between calls, no call throws.  Return value: 0 on success or a
 * negative DIB_E* code; dib_last_error() gives a thread-local message.
 *
 * Each entry point replaces one interface of the reference (lijx10/DeepI2P @ cd21389):
 *
 *   frustum_solve_batch_*   FrustumRegistration.solvePGivenK          evaluation/frustum_reg/src/registration.cpp:9-186,190-206
 *                           + the multi-start loop around it          evaluation/registration_lsq.py:127-186
 *   frustum_register_batch_f32  the per-sample body of the driver     evaluation/registration_lsq.py:329-343
 *   frustum_residuals_*     the residual vector solvePGivenK returns  registration.cpp:150-155
 *   frustum_evaluate_*      (test hook: one cost/gradient/JtJ pass)   registration_{2d,3d}.hpp:34-68,105-127
 *   frustum_prepare_batch   get_initial_guess + init perturbation     evaluation/registration_lsq.py:196-220,163-164
 *   frustum_inside_mask_f32 get_inside_img_mask                        evaluation/registration_lsq.py:67-84
 *   pose_error_batch        get_P_diff + success criterion             evaluation/registration_lsq.py:87-95, registration_result_analysis.py:37-38
 *   index_max_forward       index_max.forward_cuda[_shared_mem]       models/index_max_ext/index_max_cuda.cu:30-62,84-100
 *   ball_query_forward      ball_query.forward_cuda_shared_mem        models/ball_query_ext/ball_query_cuda.cu:11-50,54-71
 *
 * INTEGRATION.md shows the binding a maintainer of the reference would add for each.
 */
#ifndef DEEPI2P_B200_H_
#define DEEPI2P_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DIB_OK 0
#define DIB_EINVAL (-22)   /* bad argument (shape, alignment, NULL)            */
#define DIB_ENOMEM (-12)   /* workspace too small                              */
#define DIB_ECUDA (-5)     /* a CUDA runtime call failed; see dib_last_error() */
#define DIB_ENODEV (-19)   /* no sm_90 device                                  */

typedef void* dib_stream_t; /* cudaStream_t */

/* ABI version (bumped on any signature change) and last error text of the calling thread. */
int dib_abi_version(void);
const char* dib_last_error(void);
/* Number of SMs of the current device, or a negative error code. */
int dib_device_sm_count(void);
/* Measurement hook: two cudaEvent_t (created by the caller with timing enabled) that every following solve launch of
 * the CALLING THREAD records on its stream right before and right after the solver kernel; (NULL, NULL) switches it
 * off.  bench.py uses it to time the dominant kernel inside its timed steps. */
void dib_profile_solve_events(void* start_event, void* stop_event);

/* ------------------------------------------------------------------------------------------
 * Registration solver.
 *
 * Device record of a cloud (13 B / point, or 25 B / point for the f64 variant):
 *   xyz    [S][3][n_stride]  coordinates, struct-of-arrays per sample   (f32 or f64)
 *   label  [S][n_stride]     int8: 1 = predicted inside the image, 0 = outside, else ignored
 *   n_pts  [S]               int32 valid prefix length per sample (NULL = n_stride everywhere)
 * n_stride must be a multiple of 16 and the base pointers 16-byte aligned.
 *
 * One problem = (sample s, init i).  Parameter vector as in registration.cpp:24-50:
 *   is_2d: x = [ry, tx, ty, tz];   else: x = [ax, ay, az, tx, ty, tz] started at [0, ry, 0, T].
 *   init   [S][I][4]  f64  (init_y_angle, Tx, Ty, Tz) per problem
 *   K9     [S][9]     f64  row-major intrinsics; fx=K[0], fy=K[4], cx=K[2], cy=K[5]
 *   lb3/ub3 HOST pointers to 3 doubles: box bounds on the translation (registration.cpp:128-135)
 * Outputs per sample (arg-min of final cost over the I inits, lowest index wins ties):
 *   P16_out [S][16] f64 row-major 4x4 pose, cost_out [S] f64, best_out [S] int32 (may be NULL)
 * Optional per-problem outputs (each may be NULL):
 *   params_all [S][I][6] f64, cost_all [S][I] f64,
 *   stats_all  [S][I][4] int32 = (LM iterations, cloud passes (evaluations), line-search
 *                                 contractions, termination code)
 * Termination codes: 0 gradient tol, 1 parameter tol, 2 function tol, 3 max iterations,
 *   4 min trust-region radius, 5 too many invalid steps, 6 infeasible start (init returned; its cost is the
 *   cost evaluated at the init, as registration.cpp:150-155 does after the failed solve; 0 LM iterations, 0 passes
 *   counted).
 * workspace: [dev] 256-byte aligned scratch of at least frustum_solve_workspace_bytes(S, I, n_stride) bytes:
 *   per-problem results, the per-group bounding-box table (1 B/point) and the packed {x,y,z,label} copy of the
 *   clouds (sized for the f64 record: 32 B/point) that the solver builds from the cloud at every call, i.e.
 *   about 35 B per point of the batch (366 MB for 512 clouds x 20480 points).  Calls that may overlap on
 *   different streams need separate workspaces.
 * ------------------------------------------------------------------------------------------ */
size_t frustum_solve_workspace_bytes(int S, int I, int n_stride);

int frustum_solve_batch_f32(const float* xyz, const int8_t* label, const int32_t* n_pts, int n_stride,
                            const double* K9, const double* init, const double* lb3, const double* ub3,
                            double H, double W, int max_iter, int is_2d, int S, int I,
                            double* P16_out, double* cost_out, int32_t* best_out,
                            double* params_all, double* cost_all, int32_t* stats_all,
                            void* workspace, size_t workspace_bytes, dib_stream_t stream);

int frustum_solve_batch_f64(const double* xyz, const int8_t* label, const int32_t* n_pts, int n_stride,
                            const double* K9, const double* init, const double* lb3, const double* ub3,
                            double H, double W, int max_iter, int is_2d, int S, int I,
                            double* P16_out, double* cost_out, int32_t* best_out,
                            double* params_all, double* cost_all, int32_t* stats_all,
                            void* workspace, size_t workspace_bytes, dib_stream_t stream);

/* Same solve with a per-evaluation trace (parity tooling: tests/tools/trace_divergence.py compares it with the
 * oracle's trace to find the first evaluation at which two trajectories part).
 *   trace [S][I][trace_cap][16] f64 [dev], zero-filled by the call; record e of a problem is written when the
 *   solver consumes its e-th cloud pass:  [0..5] evaluated point x_t (P entries), [6] cost at x_t, [7] cost of the
 *   current iterate, [8] trust-region radius, [9] LM iteration, [10] phase (0 initial, 1 line-search sample,
 *   2 candidate after a failed line search, 3 cost at an infeasible start), [11] 1 if x_t became the iterate,
 *   [12] termination code after this evaluation (-1 = still running), [13] line-search step size, [14] model cost
 *   change of the step, [15] 1 (record written).  Evaluations beyond trace_cap are not recorded. */
int frustum_solve_traced_f32(const float* xyz, const int8_t* label, const int32_t* n_pts, int n_stride,
                             const double* K9, const double* init, const double* lb3, const double* ub3,
                             double H, double W, int max_iter, int is_2d, int S, int I,
                             double* P16_out, double* cost_out, int32_t* best_out,
                             double* params_all, double* cost_all, int32_t* stats_all,
                             double* trace, int trace_cap,
                             void* workspace, size_t workspace_bytes, dib_stream_t stream);

/* Slicing policy (parity tooling).  The solver forms the sums of a pass either in one piece or as a fixed sequence of
 * slices (frustum_solve_slice_rounds x 1024 points each) added in slice order, so that idle warps can help; the
 * variants differ at rounding level, each is deterministic.  A batch of fewer than ~4 waves of problems slices every
 * pass into short slices (slice_after 0, 2 rounds); a larger one slices only from a problem's 48th pass on, 4 rounds
 * per slice -- except for the problems at the last queue positions (one resident grid's worth), which start while the
 * batch drains and use the small-batch slicing from their first pass.  dib_evaluate_sliced(r) (thread-local; r = rounds per slice, 0 = one piece; default 4) selects which of
 * them frustum_evaluate_* reproduces bit for bit. */
int frustum_solve_slice_after(int S, int I, int is_2d, int f64_record);
int frustum_solve_slice_rounds(int S, int I, int is_2d, int f64_record);
void dib_evaluate_sliced(int rounds_per_slice);

/* One evaluation pass per sample at explicit parameters x [S][6] f64:
 * cost_out [S], grad_out [S][6] (J^T r), JtJ_out [S][36] (row-major P x P in the top-left).
 * workspace: [dev] at least frustum_evaluate_workspace_bytes(S, n_stride) bytes. */
size_t frustum_evaluate_workspace_bytes(int S, int n_stride);
int frustum_evaluate_f32(const float* xyz, const int8_t* label, const int32_t* n_pts, int n_stride,
                         const double* K9, const double* x, double H, double W, int is_2d, int S,
                         double* cost_out, double* grad_out, double* JtJ_out, void* workspace,
                         size_t workspace_bytes, dib_stream_t stream);
int frustum_evaluate_f64(const double* xyz, const int8_t* label, const int32_t* n_pts, int n_stride,
                         const double* K9, const double* x, double H, double W, int is_2d, int S,
                         double* cost_out, double* grad_out, double* JtJ_out, void* workspace,
                         size_t workspace_bytes, dib_stream_t stream);

/* Loss-corrected residual vector at x (single cloud), in point order, one row per label-0 point
 * and three per label-1 point (registration.cpp:150-155).  row_offset [n] int32 [dev] = exclusive
 * prefix of rows per point (caller-computed); residuals [rows] f64 [dev]. */
int frustum_residuals_f32(const float* xyz, const int8_t* label, int n, int n_stride, const double* K9,
                          const double* x, double H, double W, int is_2d, const int32_t* row_offset,
                          double* residuals, dib_stream_t stream);
int frustum_residuals_f64(const double* xyz, const int8_t* label, int n, int n_stride, const double* K9,
                          const double* x, double H, double W, int is_2d, const int32_t* row_offset,
                          double* residuals, dib_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Front end of the multi-start driver, on device (registration_lsq.py:196-220 get_initial_guess,
 * :163-164 perturbed inits, :329-332 degenerate-sample flag).
 *   xyz_in [S][3][n_in_stride] f32, pred [S][n_in_stride] int8 (1 = predicted inside), n_in valid.
 * Outputs (n_out_stride = round_up(n_in, 16)):
 *   xyz_out [S][3][n_out_stride] f32, label_out [S][n_out_stride] int8 : front-filtered cloud, tail
 *       padded with ignored points; n_pts [S] int32 = points kept.  sort == 0 keeps the original
 *       point order; sort != 0 (and n_in <= 32768) orders the kept points by (label, 12-bit Morton
 *       cell of (x,z), original index): the solver's sums do not depend on the order beyond
 *       rounding, and its per-group bounding-box culling becomes ~3x more selective
 *   init [S][I][4] f64 : (init_y_angle + N(0, ry_sigma), 0, 0, U(-t_amp, t_amp)), Philox4x32-10
 *       counter (init, sample, 0, 0), key = seed
 *   init_y_angle [S] f64, degenerate [S] int32 (1 = no predicted-inside point)
 * ------------------------------------------------------------------------------------------ */
size_t frustum_prepare_workspace_bytes(int S, int I);
int frustum_prepare_batch_f32(const float* xyz_in, const int8_t* pred, int n_in, int n_in_stride, int S, int I,
                              uint64_t seed, double ry_sigma, double t_amp, int sort, float* xyz_out,
                              int8_t* label_out,
                              int32_t* n_pts, double* init, double* init_y_angle, int32_t* degenerate,
                              void* workspace, size_t workspace_bytes, dib_stream_t stream);

/* Reorder clouds by (label, Morton cell of (x,z), original index) WITHOUT filtering: every point is kept, labels other
 * than 0 / 1 become -1 (ignored) and sort last; clouds of more than 32768 points keep their order.  For callers that
 * hand the solver an already filtered cloud -- the drop-in solvePGivenK (registration.cpp:190-206) sorts its cloud with
 * this before frustum_solve_batch_f32 (the residual vector is still formed in the caller's point order).
 * xyz_in [S][3][n_in_stride] f32, label [S][n_in_stride] int8; xyz_out [S][3][round_up(n_in,16)], label_out, n_pts [S]. */
int frustum_sort_batch_f32(const float* xyz_in, const int8_t* label, int n_in, int n_in_stride, int S, float* xyz_out,
                           int8_t* label_out, int32_t* n_pts, dib_stream_t stream);

/* The whole per-sample body of evaluation/registration_lsq.py:329-343 in ONE call -- the batched entry point that
 * replaces the reference's fork-per-solve loop (registration_lsq.py:142-186): frustum_prepare_batch_f32 (sort on) +
 * frustum_solve_batch_f32 + arg-min + the degenerate-sample rule (no predicted-inside point: P = I, cost = 1e4,
 * best = 0; :329-332).  Inputs as frustum_prepare_batch_f32 / frustum_solve_batch_f32.  Optional outputs (each may
 * be NULL): init_y_angle_out [S] f64, n_pts_out [S] i32 (points kept by the front filter), degenerate_out [S] i32,
 * init_out [S][I][4] f64, params_all / cost_all / stats_all as above.
 * workspace: [dev] 256-byte aligned, >= frustum_register_workspace_bytes(S, I, n_in) (front-filtered clouds + the
 * solver's workspace). */
size_t frustum_register_workspace_bytes(int S, int I, int n_in);
int frustum_register_batch_f32(const float* xyz_in, const int8_t* pred, int n_in, int n_in_stride, int S, int I,
                               uint64_t seed, double ry_sigma, double t_amp, const double* K9, const double* lb3,
                               const double* ub3, double H, double W, int max_iter, int is_2d, double* P16_out,
                               double* cost_out, int32_t* best_out, double* init_y_angle_out, int32_t* n_pts_out,
                               int32_t* degenerate_out, double* init_out, double* params_all, double* cost_all,
                               int32_t* stats_all, void* workspace, size_t workspace_bytes, dib_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Evaluation-side ops (SURVEY.md 8f N3).
 *   frustum_inside_mask_f32: label rule of evaluation/registration_lsq.py:67-84 /
 *       models/multimodal_classifier.py:136-148: mask[s][i] = 1 if 0<=u<=W-1, 0<=v<=H-1, z>0.1 for
 *       [u v 1] ~ K (P p), else 0; -1 beyond n_pts[s].  P16 [S][16] row-major 4x4 (or 3x4 padded).
 *   pose_error_batch: get_P_diff (registration_lsq.py:87-95) per sample: P_diff = P_pred^-1 P_gt,
 *       t_err = |P_diff[:3,3]|, r_err_deg = sum |euler 'xzy'| in degrees; success (may be NULL) =
 *       t_err < t_thresh_m and r_err_deg < r_thresh_deg (registration_result_analysis.py:37-38: 2 m, 5 deg).
 * ------------------------------------------------------------------------------------------ */
int frustum_inside_mask_f32(const float* xyz, const int32_t* n_pts, int n_stride, const double* P16,
                            const double* K9, double H, double W, int S, int8_t* mask_out, dib_stream_t stream);
int pose_error_batch(const double* P_pred16, const double* P_gt16, int S, double t_thresh_m, double r_thresh_deg,
                     double* t_err, double* r_err_deg, int32_t* success, dib_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Segmented arg-max (index_max) and first-K-in-radius (ball_query).  Bit-exact index outputs.
 *   data  [B][C][N] f32, index [B][N] int32 in [0,K), out [B][C][K] int32
 *   dist  [B][M][N] f32, out [B][M][K] int32
 * ------------------------------------------------------------------------------------------ */
int index_max_forward(const float* data, const int32_t* index, int32_t* out,
                      int B, int C, int N, int K, dib_stream_t stream);
int ball_query_forward(const float* dist, float radius, int32_t* out,
                       int B, int M, int N, int K, dib_stream_t stream);

/* Coordinate-based variant (SURVEY.md 8f N4): same output contract as ball_query_forward, computed with a
 * uniform grid hash from  points [B][3][N] f32  and  nodes [B][3][M] f32  (channel-first, as
 * models/networks_pc.py:47-65 holds them) -- the dense B x M x N distance matrix is never built.
 * hit <=> ((dx*dx + dy*dy) + dz*dz) <= radius*radius in float32 without fma -- a contract on SQUARED distances (the
 * reference thresholds the rounded square root; they can differ within one ulp of the radius).  N <= 65536.
 * workspace: [dev], 16-byte aligned, >= ball_query_xyz_workspace_bytes(B, N). */
size_t ball_query_xyz_workspace_bytes(int B, int N);
int ball_query_xyz_forward(const float* points, const float* nodes, float radius, int32_t* out, int B, int M, int N,
                           int K, void* workspace, size_t workspace_bytes, dib_stream_t stream);

/* ---- clustering front-end of the point-cloud encoder (SURVEY.md 8f N4; replaces the B x N x Ma
 * intermediates of models/networks_pc.py:60-85) -------------------------------------------------
 * pc [B][3][N] f32, node [B][3][M] f32 [dev].  Outputs [dev]:
 *   min_k_idx [B][N][k] i32  k nearest nodes of each point, nearest first (torch.topk(diff, k, largest=False), :63-64);
 *                            key ((dx*dx + dy*dy) + dz*dz) in float32 without fma, ties -> lower node index
 *   min_idx   [B][N]    i32  = min_k_idx[..][0], the `index` argument of index_max (:65,:88-90)
 *   count     [B][M]    i32  points per node (mask_row_sum, :69-72; mask_row_max = count > 0)
 *   cluster_mean [B][3][M] f32 = float(sum_fixed * 2^-24) / (float(count) + 1e-5f), sum_fixed = exact int64 sum
 *                            of rint(x * 2^24) -- order independent (:74-76); points with a non-finite coordinate are
 *                            left out of count and sums (they still get min_idx 0)
 *   pc_centers, pc_decentered [B][3][N] f32 (each may be NULL): cluster_mean gathered by min_idx, pc - centers (:78-82)
 * 1 <= k <= min(8, M), M <= 2048.  workspace: [dev], 8-byte aligned, >= cluster_assign_workspace_bytes(B, M). */
size_t cluster_assign_workspace_bytes(int B, int M);
int cluster_assign_forward(const float* pc, const float* node, int B, int N, int M, int k, int32_t* min_k_idx,
                           int32_t* min_idx, int32_t* count, float* cluster_mean, float* pc_centers,
                           float* pc_decentered, void* workspace, size_t workspace_bytes, dib_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * PnP-RANSAC registration from grid classifications (evaluation/registration_pnp.py:95-148: cv2.solvePnPRansac with
 * SOLVEPNP_EPNP, iterationsCount, reprojectionError), batched over S frames.  DESIGN.md "PnP-RANSAC" states the
 * contract.  Per frame: points with coarse_pred == 1 are kept (n_sel of them, input order); fine cell f -> pixel
 * CORNER py = floor(f / Wf), px = f - py * Wf, Wf = W * scale, float64; K_f = scale * K (K[0][1] ignored);
 * hypothesis h samples 5 distinct indices with Philox4x32-10, counter (h, s, draw, 0), key = seed, solves EPnP and
 * counts inliers ((u-px)^2 + (v-py)^2 <= reproj_err^2); sequential adaptive stop (niters = min(niters,
 * ceil(log(1-confidence) / log(1-w^5))) on each strictly better hypothesis with >= 5 inliers); EPnP refit on the
 * winner's inliers.  P = I and outlier_ratio = 1 when n_sel < 4, no hypothesis wins, EPnP fails or |t| >= 14.14;
 * else outlier_ratio = 1 - inliers / n_sel.  4 <= n_sel <= 5: EPnP on all points, inliers counted under that pose.
 *   xyz [S][3][n_stride] f32, coarse_pred [S][n_stride] int8, fine_pred [S][n_stride] int32, n_pts [S] (NULL =
 *   n_stride), K9 [S][9] f64 unscaled row-major -- all [dev].  0 <= S <= 65535 (larger batches: split them).
 *   Outputs [dev]: P16_out [S][16], outlier_ratio_out [S], inliers_out [S] (the winner's count); may be NULL:
 *   n_sel_out [S], hyp_used_out [S] (hypotheses the sequential rule evaluated), inlier_mask_out [S][n_stride] (1 =
 *   selected point that is an inlier of the winner), hyp_pose_out [S][iterations][12] (R row-major | t; zeros for an
 *   invalid hypothesis) and hyp_inliers_out [S][iterations] (0 for invalid); entries at h >= hyp_used are unspecified.
 * workspace: [dev] 256-byte aligned, >= pnp_ransac_workspace_bytes(S, n_stride, iterations).
 * epnp_batch_f64 (test hook): EPnP on B point sets, set b = rows offsets[b] .. offsets[b+1]-1 of xyz [N][3] f64 and
 * uv [N][2] f64 pixels, intrinsics K9 [B][9] used as given; pose12_out [B][12], ok_out [B] int32 (0 = degenerate).
 * ------------------------------------------------------------------------------------------ */
size_t pnp_ransac_workspace_bytes(int S, int n_stride, int iterations);
int pnp_ransac_batch_f32(const float* xyz, const int8_t* coarse_pred, const int32_t* fine_pred, const int32_t* n_pts,
                         int n_stride, int S, const double* K9, double H, double W, double scale, int iterations,
                         double reproj_err, double confidence, uint64_t seed, double* P16_out,
                         double* outlier_ratio_out, int32_t* inliers_out, int32_t* n_sel_out, int32_t* hyp_used_out,
                         uint8_t* inlier_mask_out, double* hyp_pose_out, int32_t* hyp_inliers_out, void* workspace,
                         size_t workspace_bytes, dib_stream_t stream);
int epnp_batch_f64(const double* xyz, const double* uv, const int32_t* offsets, int B, const double* K9,
                   double* pose12_out, int32_t* ok_out, dib_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Multi-start point-to-point ICP of a LiDAR cloud against a monocular-depth cloud (evaluation/icp/registration_icp.py:
 * 115-162: Open3D registration_icp with TransformationEstimationPointToPoint, default convergence criteria, the best
 * of I random inits), batched over S frames.  DESIGN.md "ICP" states the contract.  One problem = (frame s, init i):
 *   pass(T): q = T p for every source point (fp64, no FMA); its exact nearest target point (d2 = (dx*dx + dy*dy) +
 *   dz*dz, ties -> lowest target index) is a correspondence iff d2 < max_corr_dist^2; fitness = n_corr / n_pts,
 *   rmse = sqrt(sum d2 / n_corr) (0 without correspondences).  result = pass(init); then up to max_iteration times:
 *   T = umeyama(correspondences) * T (rigid, no scaling; identity without correspondences), result = pass(T), stop
 *   when |d fitness| < relative_fitness and |d rmse| < relative_rmse.
 * Per frame: the first init whose fitness is strictly above the best so far (starting at 0.001) wins; none -> P = I,
 * fitness 0.001, best -1.  force_2d != 0 sets P[0][1] = P[1][0] = P[1][2] = P[2][1] = 0, P[1][1] = 1 on the winner
 * (registration_icp.py:127-133; not re-scored, the 3x3 block is then not orthonormal).
 *   src [S][3][n_stride] f32, n_pts [S] i32 (NULL = n_stride), tgt [S][3][m_stride] f32, m_pts [S] (NULL = m_stride),
 *   init16 [S][I][16] f64 row-major 4x4 -- all [dev].  Strides are multiples of 16; 0 <= S <= 65535,
 *   1 <= I <= 4096, S * m_stride < 2^31; max_corr_dist > 0; max_iteration >= 0.
 *   Outputs [dev]: P16_out [S][16], fitness_out [S]; may be NULL: best_out [S] (-1 = none), T_all [S][I][16],
 *   fitness_all [S][I], rmse_all [S][I], stats_all [S][I][2] = (update steps, n_corr of the last pass).
 * workspace: [dev] 256-byte aligned, >= icp_workspace_bytes(S, I, n_stride, m_stride) (the per-frame nearest-neighbour
 *   index over the target, about 60 B per target point, and the per-problem results).
 *   The target index holds up to 2^27 leaves of 16 points; every m_stride the S * m_stride < 2^31 rule admits fits.
 * icp_register_batch_counted_f32 (measurement): the same call, which also adds (nearest-neighbour queries, point
 *   distance evaluations) of its problems to counters [dev] (two unsigned 64-bit words, not cleared by the call).
 * icp_build_index_f32 (measurement): only the per-frame index build of a call (target layout as above), into a
 *   workspace of >= icp_workspace_bytes(S, 1, 16, m_stride) bytes; it computes nothing a caller can read.
 * ------------------------------------------------------------------------------------------ */
size_t icp_workspace_bytes(int S, int I, int n_stride, int m_stride);
int icp_register_batch_f32(const float* src, const int32_t* n_pts, int n_stride, const float* tgt,
                           const int32_t* m_pts, int m_stride, int S, const double* init16, int I,
                           double max_corr_dist, int max_iteration, double relative_fitness, double relative_rmse,
                           int force_2d, double* P16_out, double* fitness_out, int32_t* best_out, double* T_all,
                           double* fitness_all, double* rmse_all, int32_t* stats_all, void* workspace,
                           size_t workspace_bytes, dib_stream_t stream);
int icp_register_batch_counted_f32(const float* src, const int32_t* n_pts, int n_stride, const float* tgt,
                                   const int32_t* m_pts, int m_stride, int S, const double* init16, int I,
                                   double max_corr_dist, int max_iteration, double relative_fitness,
                                   double relative_rmse, int force_2d, double* P16_out, double* fitness_out,
                                   int32_t* best_out, double* T_all, double* fitness_all, double* rmse_all,
                                   int32_t* stats_all, unsigned long long* counters, void* workspace,
                                   size_t workspace_bytes, dib_stream_t stream);
int icp_build_index_f32(const float* tgt, const int32_t* m_pts, int m_stride, int S, void* workspace,
                        size_t workspace_bytes, dib_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * LiDAR scan preparation (data/kitti/kitti_pc_bin_to_npy_with_downsample_sn.py:48-74 and the loaders'
 * downsample_with_intensity_sn / downsample_with_reflectance: Open3D voxel_down_sample, estimate_normals with
 * KDTreeSearchParamHybrid, orient_normals_to_align_with_direction, and the 1-NN intensity transfer), batched over S
 * clouds.  DESIGN.md "Scan preparation" states the contract.  All arithmetic is fp64 without FMA.
 * Common rules: [dev] pointers, strides are multiples of 16, 0 <= S <= 65535, S * stride < 2^31, coordinates finite;
 * count arrays (n_pts, m_pts, q_pts) may be NULL (= the stride); entries past a cloud's count are not written.
 *
 * voxel_downsample_batch_f32: xyz [S][3][n_stride] f32, optional attr [S][C][n_stride] f64 (0 <= C <= 64; NULL when
 *   C = 0).  Per cloud: min_bound = min(p) - 0.5 v, voxel = floor((p - min_bound) / v); per occupied voxel, in ascending
 *   (ix, iy, iz) order, the mean of its points and attributes (sums in ascending point index, then / count) into
 *   xyz_out [S][3][n_stride] f64, attr_out [S][C][n_stride] f64, and the voxel count into m_pts_out [S] i32.
 *   Returns DIB_EINVAL when a cloud spans 2^21 or more voxels along an axis.  The call reads the clouds' boxes back
 *   to the host, so it waits for the work queued on the stream before it.
 *   workspace >= voxel_downsample_workspace_bytes(S, n_stride, C), 256-byte aligned (about 44 B per point).
 * estimate_normals_batch_f32: xyz [S][3][m_stride] f32.  Per point i: the min(max_nn, c) nearest points of the cloud
 *   with d2 < radius^2 (itself included, ties -> lower index; 1 <= max_nn <= 64); fewer than 3 -> (0, 0, 1); else the
 *   unit eigenvector of the smallest eigenvalue of the covariance about p_i (zero covariance -> 0); then a zero normal
 *   becomes orient3 [host, 3 f64] and n . orient3 < 0 flips n.  normals_out [S][3][m_stride] f64; count_out
 *   [S][m_stride] i32 (may be NULL) = neighbours used.
 *   workspace >= estimate_normals_workspace_bytes(S, m_stride), 256-byte aligned (the Morton index of icp.cu).
 * nearest_batch_f32: for each query q [S][3][q_stride] f64 (q_pts [S]), the index of the nearest point of xyz
 *   [S][3][m_stride] f32 (d2 as above, ties -> lowest index; -1 for an empty cloud or d2 >= DBL_MAX / 2) into idx_out
 *   [S][q_stride] i32.
 *   workspace >= estimate_normals_workspace_bytes(S, m_stride).
 * ------------------------------------------------------------------------------------------ */
size_t voxel_downsample_workspace_bytes(int S, int n_stride, int C);
int voxel_downsample_batch_f32(const float* xyz, const int32_t* n_pts, int n_stride, int S, const double* attr, int C,
                               double voxel_size, double* xyz_out, double* attr_out, int32_t* m_pts_out,
                               void* workspace, size_t workspace_bytes, dib_stream_t stream);
size_t estimate_normals_workspace_bytes(int S, int m_stride);
int estimate_normals_batch_f32(const float* xyz, const int32_t* m_pts, int m_stride, int S, double radius, int max_nn,
                               const double* orient3, double* normals_out, int32_t* count_out, void* workspace,
                               size_t workspace_bytes, dib_stream_t stream);
int nearest_batch_f32(const double* q, const int32_t* q_pts, int q_stride, const float* xyz, const int32_t* m_pts,
                      int m_stride, int S, int32_t* idx_out, void* workspace, size_t workspace_bytes,
                      dib_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Batch assembly of the classifier's point inputs (the loaders' __getitem__ after the scan records are read:
 * data/kitti_pc_img_pose_loader.py:199-446, data/oxford_pc_img_pose_loader.py:262-352).  DESIGN.md "Batch assembly"
 * states the contract.  [dev] pointers; 0 <= S <= 65535; fp64 arithmetic without FMA, rounded once to float32.
 * Random draws are Philox4x32-10 with key = seed and counter (position, sample, stream id, 0); stream ids: 1 resample
 * key, 2 pc jitter, 3 sn jitter, 4 node_a candidates, 5 node_b candidates, 6 intensity jitter.
 *
 * assemble_accumulate_f32: T frames xyz [T][3][n_stride] f32, intensity [T][n_stride] f32, sn [T][3][n_stride] f32
 *   (may be NULL), n_pts [T] i32 (NULL = n_stride); frame_sample [T] i32 non-decreasing in [0, S); frame_T16 [T][16]
 *   f64 row-major.  p' = ((T00 x + T01 y) + T02 z) + T03 per row, normals get the rotation only; range_max > 0 keeps
 *   points with x'^2 + z'^2 < range_max^2 in float32.  Each sample's kept points are written in (frame, index) order to
 *   xyz_out [S][3][out_stride], intensity_out [S][out_stride], sn_out [S][3][out_stride] (with sn); count_out [S] i32.
 *   workspace >= assemble_accumulate_workspace_bytes(T, n_stride, S), 256-byte aligned.
 * assemble_resample_f32: S clouds as above (stride n_stride, counts n_pts [S]) to input_pt_num = N points each
 *   (data/kitti_pc_img_pose_loader.py:158-171): with n >= N points, the N smallest (key, index); otherwise index o < r n
 *   takes o mod n (r >= 1 the smallest with (r + 1) n >= N) and the rest the N - r n smallest keys, in ascending key
 *   order.  jitter mask 1 = pc, 2 = sn, 4 = intensity: + (float)clip(sigma z, -clip, clip), z from Box-Muller; then
 *   M16 [S][16] f64 (pc affine, sn rotation only).  xyz_out [S][3][N], intensity_out [S][N], sn_out [S][3][N] (may be
 *   NULL; zeros without sn), src_out [S][N] i32 (index into the input cloud; -1 for an empty cloud).
 *   workspace >= assemble_resample_workspace_bytes(S, n_stride), 256-byte aligned.
 * assemble_candidates_f32: per sample of pc [S][3][N] f32, the m smallest-key points (node_set 0 = node_a, 1 = node_b),
 *   in ascending key order: idx_out [S][m] i32, xyz_out [S][3][m] f32.  1 <= m <= N.
 *   workspace >= assemble_candidates_workspace_bytes(S, N), 256-byte aligned.
 * fps_batch_f32 / fps_batch_f64: farthest-point sampling (data/kitti_helper.py:224-243) of k points from each of S sets
 *   xyz [S][3][n_stride] (n_pts [S] i32, NULL = n_stride), starting at start [S] i32 (NULL, or outside [0, n): 0).
 *   d2 = (dx dx + dy dy) + dz dz in fp64; each round takes the point of largest running minimum, lowest index on ties.
 *   1 <= k <= n_stride <= 65536; idx_out [S][k] i32, nodes_out [S][3][k] (-1 and zeros for an empty set).  No
 *   workspace.  Sets above 8192 points run on a thread-block cluster.
 * ------------------------------------------------------------------------------------------ */
size_t assemble_accumulate_workspace_bytes(int T, int n_stride, int S);
int assemble_accumulate_f32(const float* xyz, const float* intensity, const float* sn, const int32_t* n_pts,
                            int n_stride, int T, const int32_t* frame_sample, const double* frame_T16, int S,
                            double range_max, float* xyz_out, float* intensity_out, float* sn_out, int out_stride,
                            int32_t* count_out, void* workspace, size_t workspace_bytes, dib_stream_t stream);
size_t assemble_resample_workspace_bytes(int S, int n_stride);
int assemble_resample_f32(const float* xyz, const float* intensity, const float* sn, const int32_t* n_pts,
                          int n_stride, int S, int input_pt_num, uint64_t seed, const double* M16, double sigma,
                          double clip, int jitter, float* xyz_out, float* intensity_out, float* sn_out,
                          int32_t* src_out, void* workspace, size_t workspace_bytes, dib_stream_t stream);
size_t assemble_candidates_workspace_bytes(int S, int N);
int assemble_candidates_f32(const float* pc, int N, int S, uint64_t seed, int node_set, int m, int32_t* idx_out,
                            float* xyz_out, void* workspace, size_t workspace_bytes, dib_stream_t stream);
int fps_batch_f32(const float* xyz, const int32_t* n_pts, int n_stride, int S, int k, const int32_t* start,
                  int32_t* idx_out, float* nodes_out, dib_stream_t stream);
int fps_batch_f64(const double* xyz, const int32_t* n_pts, int n_stride, int S, int k, const int32_t* start,
                  int32_t* idx_out, double* nodes_out, dib_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Inverse-distance feature interpolation of the classifier's decoder (models/networks_united.py:76-103,
 * KeypointDetector.upsample_by_interpolation; SURVEY.md 8f N9).  DESIGN.md 4.12 states the contract.  [dev] pointers;
 * 0 <= B <= 65535, 1 <= M <= 2048, 1 <= k <= 8; float32 arithmetic without FMA, IEEE sqrt and division.
 *
 * interp_weights_f32: topk_idx [B][Nq][k] int32 (idx_bytes 4) or int64 (idx_bytes 8), query [B][3][Nq] f32, node
 *   [B][3][M] f32.  Per query point d_j = sqrt((dx*dx + dy*dy) + dz*dz), dx = query - node[idx_j]; S = ((d_0 + d_1) +
 *   ...) + d_{k-1}; w_j = 1 - d_j / S into w_out [B][Nq][k] f32, the index into idx_out [B][Nq][k] int32.  A point with
 *   any index outside [0, M) reads no node and gets w = NaN, idx = -1 in all k slots.
 * interp_forward_f32: out [B][C][Nq] = ((w_0 F[c][i_0] + w_1 F[c][i_1]) + ...) from features [B][C][M] f32 and the
 *   weights call's w / idx; a point with idx = -1 gets NaN in all C channels.
 * interp_backward_f32: grad_features [B][C][M] f32 = sum over (n, j) with idx[b][n][j] = m of w[b][n][j] *
 *   grad_out[b][c][n], for grad_out with element (b, c, n) at b * grad_batch_stride + c * Nq + n (grad_batch_stride >=
 *   0; a channel slice of a larger [B][C'][Nq] tensor passes C' * Nq).  The fp32 products are added exactly in fp64, in ascending (n, j) within fixed slices of n and the slices
 *   in order, then rounded once: deterministic for a given shape, no atomics.  Points with idx = -1 contribute nothing.
 *   workspace: [dev] 8-byte aligned, >= interp_backward_workspace_bytes(B, C, Nq, M) (fp64 slice partials).
 * ------------------------------------------------------------------------------------------ */
int interp_weights_f32(const void* topk_idx, int idx_bytes, const float* query, const float* node, int B, int Nq,
                       int M, int k, float* w_out, int32_t* idx_out, dib_stream_t stream);
int interp_forward_f32(const float* features, const float* w, const int32_t* idx, int B, int C, int Nq, int M, int k,
                       float* out, dib_stream_t stream);
size_t interp_backward_workspace_bytes(int B, int C, int Nq, int M);
int interp_backward_f32(const float* grad_out, int64_t grad_batch_stride, const float* w, const int32_t* idx, int B,
                        int C, int Nq, int M, int k, float* grad_features, void* workspace, size_t workspace_bytes,
                        dib_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * The image side of classifier batches (data/kitti_pc_img_pose_loader.py:326-349,360-362,439-440,
 * data/oxford_pc_img_pose_loader.py:238-259,300-301,368; SURVEY.md 8f N10).  DESIGN.md 4.13 states the contract.
 * For each of S samples: rows [row0, row0 + rows) of an h x w x 3 uint8 frame (HWC, packed at src + offsets[s]),
 * cv2.resize(INTER_LINEAR) to dh x dw (1 <= dh <= rows, 1 <= dw <= w; OpenCV's fixed-point arithmetic), the
 * img_H x img_W window at (dy, dx) of the resized image, with jitter torchvision's ColorJitter steps on a PIL image in
 * the given order (0 brightness, 1 contrast, 2 saturation, 3 hue; Pillow's arithmetic), with flip a column flip, and
 * the CHW write into img_out [S][3][img_H][img_W] (float32 holding the integer values, or uint8).
 *
 * src: [dev] packed frames of src_bytes bytes.  offsets [host] int64 [S]; params [host] int32 [S][DIB_IMAGE_PARAMS]
 * indexed by the DIB_IMG_* constants (flip, jitter 0 or 1; shift is the hue step's uint8 shift,
 * (uint8)(int32)(hue * 255)); factors [host] float32 [S][3] = (brightness, contrast, saturation).  Every field is
 * checked on the host (DIB_EINVAL).  workspace: [dev] 256-byte aligned, >= image_assemble_workspace_bytes(S, img_H,
 * img_W) (DIB_ENOMEM); the parameters are uploaded into it on `stream`.  Deterministic: the contrast mean is an exact
 * integer sum.
 * ------------------------------------------------------------------------------------------ */
#define DIB_IMAGE_PARAMS 16
#define DIB_IMG_H 0
#define DIB_IMG_W 1
#define DIB_IMG_ROW0 2
#define DIB_IMG_ROWS 3
#define DIB_IMG_DH 4
#define DIB_IMG_DW 5
#define DIB_IMG_DY 6
#define DIB_IMG_DX 7
#define DIB_IMG_FLIP 8
#define DIB_IMG_JITTER 9
#define DIB_IMG_ORDER 10 /* 4 entries */
#define DIB_IMG_SHIFT 14
size_t image_assemble_workspace_bytes(int S, int img_H, int img_W);
int image_assemble_f32(const uint8_t* src, size_t src_bytes, const int64_t* offsets, const int32_t* params,
                       const float* factors, int S, int img_H, int img_W, float* img_out, void* workspace,
                       size_t workspace_bytes, dib_stream_t stream);
int image_assemble_u8(const uint8_t* src, size_t src_bytes, const int64_t* offsets, const int32_t* params,
                      const float* factors, int S, int img_H, int img_W, uint8_t* img_out, void* workspace,
                      size_t workspace_bytes, dib_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* DEEPI2P_B200_H_ */
