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

/* Test hooks of the solver's control step, T independent cases, one warp each, all arrays [dev].
 * frustum_poly_roots_f64: real parts of the roots of the monic polynomial coeffs [T][5] (highest power first,
 *   coeffs[t][0] = 1) of degree deg [T] in {3, 4} (other degrees give NaN) -> roots [T][4] (the first deg are used).
 * frustum_interp_step_f64: line-search step minimising the polynomial through samples [T][3][5] (lower, previous,
 *   current; each x, value, gradient, value_valid, gradient_valid, validity as 0 / 1) over bounds [T][2]
 *   (xmin, xmax) -> step [T].
 * frustum_lm_next_step_f64: the damped Levenberg-Marquardt step from one state, P in {4, 6}, NA = P (P + 1) / 2.
 *   in [T][6P + NA + 2] = x[P] g[P] A[NA] (packed upper triangle of J^T J, row by row) scale[P] diag[P] lb[P] ub[P]
 *   radius dec; in_flags [T][2] = reuse_diag, invalid (count of invalid steps so far).
 *   out [T][4P + 3] = step[P] (scaled space) delta[P] xt[P] diag[P] mcc radius dec (step, delta, xt and mcc hold a
 *   step when the return code is 1); out_flags [T][4] = return code (0 done, 1 evaluate xt), termination (-1 running, 4
 *   radius, 5 five invalid steps), invalid, iteration. */
int frustum_poly_roots_f64(const double* coeffs, const int32_t* deg, int T, double* roots, dib_stream_t stream);
int frustum_interp_step_f64(const double* samples, const double* bounds, int T, double* step, dib_stream_t stream);
int frustum_lm_next_step_f64(int P, int T, const double* in, const int32_t* in_flags, double* out,
                             int32_t* out_flags, dib_stream_t stream);

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
 *                            key ((dx*dx + dy*dy) + dz*dz) in float32 without fma, ties -> lower node index,
 *                            +inf after every finite key and NaN after +inf (k distinct nodes always)
 *   min_idx   [B][N]    i32  = min_k_idx[..][0], the `index` argument of index_max (:65,:88-90)
 *   count     [B][M]    i32  points per node (mask_row_sum, :69-72; mask_row_max = count > 0)
 *   cluster_mean [B][3][M] f32 = round_f32(sum_fixed * 2^-24) / (float(count) + 1e-5f), sum_fixed = the exact
 *                            (two-word) sum of rint(x * 2^24) -- order independent (:74-76), at most 2^-25 per point
 *                            from the exact sum; points with a coordinate of magnitude >= 2^39 or a non-finite one
 *                            are left out of count and sums (they keep their min_k_idx / min_idx)
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
 * voxel_downsample_batch_f64: the same with fp64 coordinates xyz [S][3][n_stride] f64 (min_bound from the fp64 box).
 *   Same workspace.
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
 * sym3_eig_batch_f64 (test hook): the 3x3 symmetric eigensolver that the normals and EPnP share, on n matrices C
 *   [n][9] f64 row-major (read as given, not symmetrised) -> eigenvalues lam [n][3] in descending order and
 *   eigenvectors E [n][9] (row-major, column k belongs to lam[k]), all [dev].
 * ------------------------------------------------------------------------------------------ */
size_t voxel_downsample_workspace_bytes(int S, int n_stride, int C);
int voxel_downsample_batch_f32(const float* xyz, const int32_t* n_pts, int n_stride, int S, const double* attr, int C,
                               double voxel_size, double* xyz_out, double* attr_out, int32_t* m_pts_out,
                               void* workspace, size_t workspace_bytes, dib_stream_t stream);
int voxel_downsample_batch_f64(const double* xyz, const int32_t* n_pts, int n_stride, int S, const double* attr, int C,
                               double voxel_size, double* xyz_out, double* attr_out, int32_t* m_pts_out,
                               void* workspace, size_t workspace_bytes, dib_stream_t stream);
size_t estimate_normals_workspace_bytes(int S, int m_stride);
int estimate_normals_batch_f32(const float* xyz, const int32_t* m_pts, int m_stride, int S, double radius, int max_nn,
                               const double* orient3, double* normals_out, int32_t* count_out, void* workspace,
                               size_t workspace_bytes, dib_stream_t stream);
int nearest_batch_f32(const double* q, const int32_t* q_pts, int q_stride, const float* xyz, const int32_t* m_pts,
                      int m_stride, int S, int32_t* idx_out, void* workspace, size_t workspace_bytes,
                      dib_stream_t stream);
int sym3_eig_batch_f64(const double* C, int n, double* lam, double* E, dib_stream_t stream);

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
 * assemble_accumulate_gather_f32: assemble_accumulate_f32 on frames gathered from a ragged scan store: SoA planes
 *   xyz [3][plane_stride], intensity [plane_stride], sn [3][plane_stride] (may be NULL) f32, in device memory or in
 *   pinned host memory (read through its mapped device address; other host memory is an error).  Frame t is store
 *   points [frame_offset[t], frame_offset[t] + frame_n[t]) (frame_offset [T] i64, frame_n [T] i32 clamped to
 *   [0, n_max], both device; the caller keeps every range inside the store).  A store range may back several frames,
 *   in any order.  The outputs equal assemble_accumulate_f32's bit for bit on the same frames padded into
 *   [T][3][n_max] with n_pts = frame_n.  workspace >= assemble_accumulate_gather_workspace_bytes(T, n_max, S).
 * assemble_accumulate_f64 (data/nuscenes_pc_img_pose_loader.py:194-267): as assemble_accumulate_f32 without sn, with
 *   the coordinates kept in fp64, xyz_out [S][3][out_stride] f64.  exclude_box [host, 4 f32] (x_lo, x_hi, y_lo, y_hi)
 *   or NULL drops points with x_lo < x < x_hi and y_lo < y < y_hi, compared in float32 on the frame's own (source)
 *   coordinates before the transform.  workspace >= assemble_accumulate_f64_workspace_bytes(T, n_stride, S).
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
size_t assemble_accumulate_gather_workspace_bytes(int T, int n_max, int S);
int assemble_accumulate_gather_f32(const float* xyz, const float* intensity, const float* sn, int64_t plane_stride,
                                   const int64_t* frame_offset, const int32_t* frame_n, int n_max, int T,
                                   const int32_t* frame_sample, const double* frame_T16, int S, double range_max,
                                   float* xyz_out, float* intensity_out, float* sn_out, int out_stride,
                                   int32_t* count_out, void* workspace, size_t workspace_bytes, dib_stream_t stream);
size_t assemble_accumulate_f64_workspace_bytes(int T, int n_stride, int S);
int assemble_accumulate_f64(const float* xyz, const float* intensity, const int32_t* n_pts, int n_stride, int T,
                            const int32_t* frame_sample, const double* frame_T16, int S, double range_max,
                            const float* exclude_box, double* xyz_out, float* intensity_out, int out_stride,
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
 * The point encoder's SO-Net cluster max-pool and node kNN grouping (models/networks_pc.py:88-111,
 * models/layers_pc.py:793-807; SURVEY.md 8f N12).  DESIGN.md 4.16 states the contract.  [dev] pointers; 0 <= B <= 65535.
 * Backwards: fp64 sums in an order fixed by the shape, rounded once to f32; no float atomics.
 *
 * cluster_pool_forward_f32: features [B][C][N] f32, min_idx [B][N] int32 (cluster_assign_forward's), N >= 1, M >= 1.
 *   sel [B][C][M] int32 = index_max_forward(features, min_idx, M) (the same kernel); mask [B][M] f32 = 1.0f where some
 *   point has min_idx == m, else 0.0f; pooled [B][C][M] = features[b][c][sel] * mask (one f32 multiply: an empty
 *   segment gives features[b][c][0] * 0.0f); scattered [B][C][N] (NULL: not written) = pooled[b][c][min_idx[b][n]],
 *   NaN for a point whose min_idx is outside [0, M) (it joins no segment).
 * cluster_pool_backward_f32: grad_features [B][C][N] f32 = sum over m with sel[b][c][m] = n of mask[b][m] *
 *   (grad_pooled[b][c][m] + sum over n' with min_idx[b][n'] = m of grad_scattered[b][c][n']), the inner sum in
 *   ascending n' within fixed slices of n' and the slices in order, then the terms in ascending m.  grad_pooled
 *   [B][C][M] contiguous and grad_scattered (element (b, c, n) at b * grad_scattered_batch_stride + c * N + n) may each
 *   be NULL (a zero gradient).  sel and mask are the forward's.  workspace: [dev] 8-byte aligned, >=
 *   cluster_pool_backward_workspace_bytes(B, C, N, M) when grad_scattered is given (fp64 slice partials), else unused.
 * knn_group_forward_f32: query [B][3][M], database [B][3][N], features [B][C][N] f32; 1 <= N <= 2048, 1 <= K <= min(32,
 *   N).  knn_idx [B][M][K] int32: the K nearest database nodes of each query, nearest first, by cluster_assign's key
 *   (((dx*dx + dy*dy) + dz*dz) in f32 without fma, ties -> lower index, +inf after finite keys, NaN after +inf).
 *   grouped [B][3 + C][M][K] f32: rows 0..2 database[idx] - query, rows 3.. features[idx].
 * knn_group_backward_f32: grad_features [B][C][N] f32 = sum over (m, j) with knn_idx[b][m][j] = n of
 *   grad_grouped[b][3 + c][m][j], in ascending (m, j) within fixed slices and the slices in order.  grad_grouped element
 *   (b, r, m, j) at b * grad_batch_stride + (r * M + m) * K + j; rows 0..2 (the coordinates) are not read.  workspace:
 *   [dev] 8-byte aligned, >= knn_group_backward_workspace_bytes(B, C, M, N, K) (fp64 slice partials).
 * ------------------------------------------------------------------------------------------ */
int cluster_pool_forward_f32(const float* features, const int32_t* min_idx, int B, int C, int N, int M, int32_t* sel,
                             float* mask, float* pooled, float* scattered, dib_stream_t stream);
size_t cluster_pool_backward_workspace_bytes(int B, int C, int N, int M);
int cluster_pool_backward_f32(const float* grad_pooled, const float* grad_scattered, int64_t grad_scattered_batch_stride,
                              const int32_t* min_idx, const int32_t* sel, const float* mask, int B, int C, int N, int M,
                              float* grad_features, void* workspace, size_t workspace_bytes, dib_stream_t stream);
int knn_group_forward_f32(const float* query, const float* database, const float* features, int B, int C, int M,
                          int N, int K, int32_t* knn_idx, float* grouped, dib_stream_t stream);
size_t knn_group_backward_workspace_bytes(int B, int C, int M, int N, int K);
int knn_group_backward_f32(const float* grad_grouped, int64_t grad_batch_stride, const int32_t* knn_idx, int B, int C,
                           int M, int N, int K, float* grad_features, void* workspace, size_t workspace_bytes,
                           dib_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * The classifier's attention-weighted image-feature fusion (models/networks_united.py:149-150,172-174,
 * torch.mean(F.unsqueeze(3) * A.unsqueeze(1), dim=2); SURVEY.md 8f N13).  DESIGN.md 4.17 states the contract.  [dev]
 * pointers; 1 <= B <= 65535, C, P, M >= 1, C and P <= 2097120.  Every sum has one fp64 accumulator starting at +0.0
 * and adds the exact products of f32 operands in ascending order; the sum divided by P in fp64 is rounded once to
 * f32.  No atomics, no workspace: bit-identical across runs, streams and batch compositions.
 *
 * attn_fusion_forward_f32: img_features F [B][C][P] and attention A [B][P][M] f32, contiguous.  out [B][C][M] =
 *   float((sum over p ascending of F[b][c][p] * A[b][p][m]) / P).
 * attn_fusion_backward_f32: grad_out gO element (b, c, m) at b * grad_batch_stride + c * M + m (grad_batch_stride >= 0;
 *   a channel slice of a larger [B][C'][M] tensor passes C' * M).  grad_img_features [B][C][P] = float((sum over m
 *   ascending of gO[b][c][m] * A[b][p][m]) / P) and grad_attention [B][P][M] = float((sum over c ascending of
 *   F[b][c][p] * gO[b][c][m]) / P); either may be NULL (not computed), and then the operand only it reads (attention
 *   for grad_img_features, img_features for grad_attention) may be NULL too.
 * ------------------------------------------------------------------------------------------ */
int attn_fusion_forward_f32(const float* img_features, const float* attention, int B, int C, int P, int M, float* out,
                            dib_stream_t stream);
int attn_fusion_backward_f32(const float* grad_out, int64_t grad_batch_stride, const float* img_features,
                             const float* attention, int B, int C, int P, int M, float* grad_img_features,
                             float* grad_attention, dib_stream_t stream);

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

/* ------------------------------------------------------------------------------------------
 * Training targets, losses, accuracies and predictions of the classifier (models/multimodal_classifier.py:135-191,
 * coarse-only :482-508; SURVEY.md 8f N11).  DESIGN.md 4.15 states the contract.  [dev] pointers; 1 <= B <= 65535,
 * N >= 1, B * N < 2^31, focal_gamma >= 0.  Scores: element (b, c, n) at b * batch_stride + c * N + n.  fine = NULL is
 * the coarse-only classifier (the fine outputs are then not written and may be NULL).  No synchronous call.
 *
 * classifier_loss_forward_f32: pc [B][3][N] f32, P12 [B][12] f64 (rows 0..2 of P), K9 [B][9] f64.  Coarse label:
 *   the rule of frustum_inside_mask_f32, bit for bit; fine label floor(u / s) + floor(v / s) * W_f for inside points,
 *   -1 otherwise (L == H_f * W_f, floor((W-1)/s) < W_f and floor((H-1)/s) < H_f are checked on the host).  Writes
 *   coarse_labels / coarse_pred int8 [B][N], fine_labels / fine_pred int32 [B][N], lse f32 [2][B][N] (each fine
 *   row's max m and log sum exp(z - m), read by the backward), the f32 scalars loss = coarse_loss + fine_loss, coarse_loss (kornia focal
 *   mean times coarse_loss_alpha) and fine_loss (cross-entropy mean over inside points, 0 if there is none), accuracy
 *   [2] f32 (coarse over all points, fine over inside points; NaN when there is none), and int32 n_inside [B],
 *   coarse_correct [B], fine_correct [B], n_inside_total [1].  Sums are fp64 in an order fixed by the shape.
 *   workspace: [dev] 8-byte aligned, >= classifier_loss_workspace_bytes(B, N) (per-CTA partials).
 * classifier_loss_backward_f32: grad_coarse [B][2][N] and grad_fine [B][L][N] f32 (either may be NULL), contiguous,
 *   for the upstream gradients grad_loss, grad_coarse_loss, grad_fine_loss (each a [dev] f32 scalar) of the
 *   forward's three losses, from its labels, lse and n_inside_total.
 * ------------------------------------------------------------------------------------------ */
size_t classifier_loss_workspace_bytes(int B, int N);
int classifier_loss_forward_f32(const float* coarse, int64_t coarse_batch_stride, const float* fine,
                                int64_t fine_batch_stride, int L, const float* pc, const double* P12, const double* K9,
                                int B, int N, double H, double W, double fine_scale, int H_f, int W_f,
                                double coarse_loss_alpha, double focal_alpha, int focal_gamma, double eps,
                                int8_t* coarse_labels, int32_t* fine_labels, int8_t* coarse_pred, int32_t* fine_pred,
                                float* lse, float* loss, float* coarse_loss, float* fine_loss, float* accuracy,
                                int32_t* n_inside, int32_t* coarse_correct, int32_t* fine_correct,
                                int32_t* n_inside_total, void* workspace, size_t workspace_bytes, dib_stream_t stream);
int classifier_loss_backward_f32(const float* coarse, int64_t coarse_batch_stride, const float* fine,
                                 int64_t fine_batch_stride, int L, int B, int N, const int8_t* coarse_labels,
                                 const int32_t* fine_labels, const float* lse, const int32_t* n_inside_total,
                                 const float* grad_loss, const float* grad_coarse_loss, const float* grad_fine_loss,
                                 double coarse_loss_alpha, double focal_alpha, int focal_gamma, double eps,
                                 float* grad_coarse, float* grad_fine, dib_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Batched JPEG decoding (the Oxford and nuScenes loaders' Image.open(<frame>.jpg)).  DESIGN.md 4.19 states the
 * contract: 8-bit sequential Huffman streams with one scan of 1 or 3 components, decoded bit for bit as libjpeg-turbo
 * does with its defaults (ISLOW IDCT, fancy upsampling) into HWC uint8 RGB, grey replicated to three channels.
 * deepi2p_b200/jpeg.py parses the headers and fills the inputs.
 *
 * data: [dev] data_bytes bytes holding each image's entropy-coded data (from the byte after its SOS segment to
 *   the end of the file).  desc: [host] int64 [S][DIB_JPEG_DESC]: slots 0..39 as csrc/jpeg.cu lists them (offsets
 *   into data and out, size, restart interval, MCU grid and per-component sampling, block grid, downsampled size
 *   and first block; slot 45 the component of each MCU block, 4 bits each); the other slots are the library's and are
 *   ignored.  huff: [dev] int32 [S][6][DIB_JPEG_HUFF_WORDS] (DC, AC table of each component; jpeg.py
 *   device_huff_table); quant: [dev] int32 [S][3][64] quantisers in natural order, as int16 values.
 *   window_bits: the bit length, in [32, 2^20], of the windows the Huffman decoder synchronises (8192 is the
 *   default; smaller values force more synchronisation work and exist for tests).  out: [dev] out_bytes bytes, image s at desc offset.
 *   status: [dev] int32 [S][2]: DIB_JPEG_* code of image s, then the synchronisation rounds its decode took.  An image
 *   with a non-zero code has no pixels written.  workspace: [dev] 256-byte aligned, >=
 *   jpeg_decode_workspace_bytes(desc, S, data_bytes, window_bits) (0 for invalid descriptors).  Deterministic: no
 *   atomics touch the output.
 * ------------------------------------------------------------------------------------------ */
#define DIB_JPEG_DESC 48
#define DIB_JPEG_HUFF_WORDS 356
#define DIB_JPEG_OK 0
#define DIB_JPEG_TRUNCATED 1 /* the entropy-coded data has no ending marker                   */
#define DIB_JPEG_MARKER 2    /* the data ends in a marker other than EOI (e.g. a second scan)  */
#define DIB_JPEG_RESTARTS 3  /* the restart-marker count does not match the DRI               */
#define DIB_JPEG_HUFFMAN 4   /* an invalid Huffman code                                       */
#define DIB_JPEG_MCUS 5      /* an interval's data does not hold exactly its MCUs (truncated) */
size_t jpeg_decode_workspace_bytes(const int64_t* desc, int S, size_t data_bytes, int window_bits);
int jpeg_decode_batch_u8(const uint8_t* data, size_t data_bytes, const int64_t* desc, const int32_t* huff,
                         const int32_t* quant, int S, int window_bits, uint8_t* out, size_t out_bytes,
                         int32_t* status, void* workspace, size_t workspace_bytes, dib_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Fused inference of the classifier's per-point layers (the PointNets of models/layers_pc.py:345-408 applied per
 * point in models/networks_united.py:193-197 and networks_pc.py:86-103; SURVEY.md 8f N16).  DESIGN.md 4.21 states the
 * contract.  A chain of 1..3 layers y = act(W x + b) over the N points of each of B samples, inference only, with
 * BatchNorm already folded into W and b by the caller.  The rows of layer 1's input are the concatenation, in order,
 * of 1..4 sources that is never written to memory; the total is at most 1024 rows, every C_out is in [1, 256].
 *
 * sources: [host] int64 [n_sources][DIB_MLP_SRC]; pointers are [dev] addresses stored as integers.
 *   dense source (NODES = 0): DATA f32, element (b, c, n) at b * BSTRIDE + c * N + n (BSTRIDE >= CHANNELS * N: a
 *     channel slice of a wider tensor passes the wider tensor's batch stride).
 *   interpolated source (NODES = M in [1, 2048]): DATA node features f32, element (b, c, m) at b * BSTRIDE + c * M + m;
 *     W f32 [B][N][K] and IDX int32 [B][N][K] as interp_weights_f32 writes them, 1 <= K <= 8.  Its rows are
 *     sum_j w_j F[c][idx_j]; a point with an index outside [0, M) has NaN in all of them.
 * layers: [host] int64 [n_layers][DIB_MLP_LAYER]: W [dev] f32 [C_out][C_in] contiguous, B [dev] f32 [C_out] or 0 (no
 *   bias), COUT, RELU (1: ReLU that keeps NaN, 0: identity).  pointwise_mlp_f32 reads only COUT and RELU.
 *
 * pointwise_mlp_pack_f32 writes the layers in the kernel's order into packed ([dev] 16-byte aligned, >=
 *   pointwise_mlp_packed_bytes): every weight rounded to TF32 (nearest, ties away from zero) once.  It depends on the
 *   sources' CHANNELS, NODES and K only.
 * pointwise_mlp_f32 evaluates the chain.  The products run on the tensor cores in TF32 with f32 accumulation; source
 *   values and the activations fed to the next layer are rounded to TF32 like the weights; bias, ReLU and the
 *   arg-max are f32.  An interpolated source's block of W1 is applied to its node features first (a TF32 product
 *   per node, kept in f32 in the workspace) and the projected rows are interpolated per point in f32.
 *   c_split = 0: out [B][C_out][N] f32, the last layer's activations.
 *   1 <= c_split <= min(C_out, 128): pred_a int8 [B][N] = arg-max over channels [0, c_split) and pred_b int32 [B][N]
 *     = arg-max over [c_split, C_out) minus c_split (not written, and may be NULL, when c_split = C_out), both by
 *     torch.max's rule (NaN is maximal, the first maximal index wins); out, when not NULL, also receives the scores.
 *   workspace: [dev] 16-byte aligned, >= pointwise_mlp_workspace_bytes (0 without interpolated sources).
 *   Deterministic: no atomics; 0 <= B <= 65535, N >= 0.
 * ------------------------------------------------------------------------------------------ */
#define DIB_MLP_SRC 8
#define DIB_MLP_SRC_DATA 0
#define DIB_MLP_SRC_BSTRIDE 1
#define DIB_MLP_SRC_CHANNELS 2
#define DIB_MLP_SRC_NODES 3
#define DIB_MLP_SRC_W 4
#define DIB_MLP_SRC_IDX 5
#define DIB_MLP_SRC_K 6
#define DIB_MLP_SRC_BCAST 7
#define DIB_MLP_LAYER 4
#define DIB_MLP_LAYER_W 0
#define DIB_MLP_LAYER_B 1
#define DIB_MLP_LAYER_COUT 2
#define DIB_MLP_LAYER_RELU 3
size_t pointwise_mlp_packed_bytes(const int64_t* sources, int n_sources, const int64_t* layers, int n_layers);
int pointwise_mlp_pack_f32(const int64_t* sources, int n_sources, const int64_t* layers, int n_layers, void* packed,
                           size_t packed_bytes, dib_stream_t stream);
size_t pointwise_mlp_workspace_bytes(const int64_t* sources, int n_sources, const int64_t* layers, int n_layers,
                                     int B);
int pointwise_mlp_f32(const int64_t* sources, int n_sources, const int64_t* layers, int n_layers, const void* packed,
                      size_t packed_bytes, int B, int N, int c_split, float* out, int8_t* pred_a, int32_t* pred_b,
                      void* workspace, size_t workspace_bytes, dib_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Fused inference of the point encoder's node kNN module (GeneralKNNFusionModule.forward, models/layers_pc.py:793-818)
 * and of its global feature (final_pointnet + torch.max over the nodes, models/networks_pc.py:107-115; SURVEY.md 8f
 * N21).  DESIGN.md 4.26 states the contract.  Inference only, BatchNorm folded into W and b by the caller; layers use
 * pointwise_mlp's DIB_MLP_LAYER table, every C_out in [1, 512].  The products run on the tensor cores in TF32 with f32
 * accumulation; weights (once, when packed), staged inputs and the activations fed to the next layer are rounded to
 * TF32 (nearest, ties away from zero); bias, ReLU (NaN stays NaN) and every max are f32, a NaN in a group giving NaN.
 * Deterministic: no atomics.  [dev] pointers; 0 <= B <= 65535.
 *
 * knn_fusion_*: layers holds n_before (1..3) then n_after (1..3) layers.  Layer 1 takes C_in = 3 + C rows (<= 512);
 *   the first after layer takes 2 C_b rows, C_b the last before layer's width: columns [0, C_b) multiply the per-node
 *   max and [C_b, 2 C_b) the columns themselves (torch.cat((max, x), dim=1)).
 * knn_fusion_pack_f32 writes the layers in the kernel's order into packed ([dev] 16-byte aligned, >=
 *   knn_fusion_packed_bytes).
 * knn_fusion_f32: query [B][3][M], database [B][3][N], features [B][C][N] f32 contiguous; 1 <= N <= 2048, 1 <= K <=
 *   min(32, N).  knn_idx [B][M][K] int32 receives knn_group_forward_f32's indices; out [B][C_out][M] f32 = the max
 *   over the K neighbours of the after layers over the columns [database[idx] - query; features[idx]] extended by
 *   the max over the K neighbours of the before layers.
 * pointwise_mlp_max_*: a chain of 1..3 layers over the concatenation of 1..4 dense sources (pointwise_mlp's
 *   DIB_MLP_SRC table with NODES = 0, C_in <= 512 rows in all), then the max over the N >= 1 columns of each sample:
 *   out [B][C_out] f32.  workspace: [dev] 16-byte aligned, >= pointwise_mlp_max_workspace_bytes(C_out, B, N) (the
 *   per-tile maxes, reduced in ascending tile order).
 * ------------------------------------------------------------------------------------------ */
size_t knn_fusion_packed_bytes(int C_in, const int64_t* layers, int n_before, int n_after);
int knn_fusion_pack_f32(int C_in, const int64_t* layers, int n_before, int n_after, void* packed, size_t packed_bytes,
                        dib_stream_t stream);
int knn_fusion_f32(const float* query, const float* database, const float* features, int B, int C, int M, int N,
                   int K, const int64_t* layers, int n_before, int n_after, const void* packed, size_t packed_bytes,
                   int32_t* knn_idx, float* out, dib_stream_t stream);
size_t pointwise_mlp_max_packed_bytes(int C_in, const int64_t* layers, int n_layers);
int pointwise_mlp_max_pack_f32(int C_in, const int64_t* layers, int n_layers, void* packed, size_t packed_bytes,
                               dib_stream_t stream);
size_t pointwise_mlp_max_workspace_bytes(int C_out, int B, int N);
int pointwise_mlp_max_f32(const int64_t* sources, int n_sources, const int64_t* layers, int n_layers,
                          const void* packed, size_t packed_bytes, int B, int N, float* out, void* workspace,
                          size_t workspace_bytes, dib_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Fused inference of the decoder's node-level PointNets (node_b_attention_pn, node_b_pn, node_a_attention_pn and
 * node_a_pn of models/networks_united.py:147-189; SURVEY.md 8f N22).  DESIGN.md 4.27 states the contract.  A chain of
 * 1..3 layers y = act(W x + b) over the M columns of each of B samples, inference only, BatchNorm folded into W and b
 * by the caller; every C_out in [1, 1024].  Layer 1's input rows are the concatenation, in order, of the sources
 * (pointwise_mlp's DIB_MLP_SRC table, NODES = 0), which is never written to memory:
 *   dense source (BCAST = 0, at most 4 with at most 1024 rows in all): DATA f32, element (b, c, m) at b * BSTRIDE + c * M + m (BSTRIDE >=
 *     CHANNELS * M, so a channel slice of a wider tensor passes the wider tensor's batch stride).
 *   broadcast source (BCAST = 1, any number with at most 65536 rows in all): DATA f32 [B][C] (or [B][C][1]), element (b, c) at b * BSTRIDE + c
 *     (BSTRIDE >= CHANNELS), the same for every column of sample b.
 * The dense rows' block of W1 runs on the tensor cores in TF32 with f32 accumulation.  The broadcast rows' block is
 * applied once per (sample, output row) as an f32 fma chain in ascending input row (TF32 weights times TF32 values,
 * each product exact in f32) and added to every column of the sample before the bias.  Weights (once, when packed),
 * source values and the activations fed to the next layer are rounded to TF32 (nearest, ties away from zero); bias and
 * ReLU (NaN stays NaN) are f32.  Deterministic: no atomics.  [dev] pointers; 0 <= B <= 65535, M >= 0.
 *
 * node_mlp_pack_f32 writes the layers in the kernel's order into packed ([dev] 16-byte aligned, >=
 *   node_mlp_packed_bytes); it depends on the sources' CHANNELS and BCAST only.
 * node_mlp_f32: out [B][C_out][M] f32, the last layer.  workspace: [dev] 16-byte aligned, >= node_mlp_workspace_bytes
 *   (the per-sample projections, [B][C1 rounded up to 16]; 0 bytes, and may be NULL, without broadcast sources).
 * ------------------------------------------------------------------------------------------ */
size_t node_mlp_packed_bytes(const int64_t* sources, int n_sources, const int64_t* layers, int n_layers);
int node_mlp_pack_f32(const int64_t* sources, int n_sources, const int64_t* layers, int n_layers, void* packed,
                      size_t packed_bytes, dib_stream_t stream);
size_t node_mlp_workspace_bytes(const int64_t* sources, int n_sources, const int64_t* layers, int n_layers, int B);
int node_mlp_f32(const int64_t* sources, int n_sources, const int64_t* layers, int n_layers, const void* packed,
                 size_t packed_bytes, int B, int M, float* out, void* workspace, size_t workspace_bytes,
                 dib_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Batched PNG decoding (KITTI's official odometry colour frames).  DESIGN.md 4.23 states the contract: 8-bit
 * truecolour, not interlaced, decoded bit for bit as OpenCV 4.13's cv2.imdecode(..., IMREAD_COLOR)[:, :, ::-1]
 * (HWC uint8 RGB).  deepi2p_b200/png.py walks the chunks, checks IHDR / PLTE / IEND and the zlib header, and fills
 * the inputs.
 *
 * data: [dev] data_bytes bytes holding each image's IDAT payloads, each starting 16-byte aligned (no padding is
 *   needed after the last).
 *   desc: [host] int64 [S][DIB_PNG_DESC]: 0 data offset, 1 IDAT bytes, 2 out offset, 3 w, 4 h, 5 first chunk,
 *   6 log2 of the zlib window, 7 skip (1: no work and no output for this image), 9 chunk count, 10 bytes per pixel
 *   (0 or 3: RGB; 1: 8-bit grey, h x w output bytes); slot 8 is the library's.  chunks: [host] int64 [n_chunks][4]:
 *   image, data offset, payload length, stored CRC-32 of each IDAT chunk, an image's chunks consecutive and covering
 *   its data.  out: [dev] out_bytes bytes, image s at its offset.
 *   status: [dev] int32 [S][4]: the inflate code, the chunk CRC code, the Adler-32 code and the filter code of image s
 *   (DIB_PNG_*, 0 = fine); the pixels of an image with any non-zero code are unspecified.  workspace: [dev] 256-byte
 *   aligned, >= png_decode_workspace_bytes(desc, S, chunks, n_chunks, data_bytes) (0 for invalid descriptors).
 *   Deterministic: no atomics touch the data.
 * ------------------------------------------------------------------------------------------ */
#define DIB_PNG_DESC 12
#define DIB_PNG_OK 0
#define DIB_PNG_TRUNCATED 1   /* the zlib stream needs more data than the IDAT chunks hold            */
#define DIB_PNG_BLOCK_TYPE 2  /* Deflate block type 3                                                 */
#define DIB_PNG_STORED 3      /* stored block LEN != ~NLEN                                            */
#define DIB_PNG_LENGTHS 4     /* over-subscribed or incomplete code set                               */
#define DIB_PNG_NO_EOB 5      /* the literal/length code has no end-of-block code                     */
#define DIB_PNG_REPEAT 6      /* code-length repeat 16 with no previous length                        */
#define DIB_PNG_OVERRUN 7     /* code lengths run past HLIT + HDIST                                   */
#define DIB_PNG_SYMBOLS 8     /* HLIT > 286 or HDIST > 30                                             */
#define DIB_PNG_LITLEN 9      /* an invalid literal/length code or symbol 286-287                     */
#define DIB_PNG_DISTANCE 10   /* an invalid distance code or symbol 30-31                             */
#define DIB_PNG_FAR 11        /* a distance before the start of the output                            */
#define DIB_PNG_WINDOW 12     /* a distance beyond the window the zlib header declares                */
#define DIB_PNG_TOO_MUCH 13   /* more inflated data than h x (1 + 3 w)                                */
#define DIB_PNG_SHORT 14      /* the zlib stream ends before the image is complete                    */
#define DIB_PNG_NO_ADLER 15   /* the Adler-32 trailer is missing                                      */
#define DIB_PNG_ADLER 16      /* the Adler-32 of the inflated data does not match                     */
#define DIB_PNG_CRC 17        /* an IDAT chunk's CRC-32 does not match                                */
#define DIB_PNG_FILTER 18     /* a row filter byte above 4                                            */
size_t png_decode_workspace_bytes(const int64_t* desc, int S, const int64_t* chunks, int n_chunks, size_t data_bytes);
int png_decode_batch_u8(const uint8_t* data, size_t data_bytes, const int64_t* desc, int S, const int64_t* chunks,
                        int n_chunks, uint8_t* out, size_t out_bytes, int32_t* status, void* workspace,
                        size_t workspace_bytes, dib_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Oxford RobotCar point-cloud build (data/oxford/build_dataset.py: my_build_pointcloud, downsample and the output
 * transform), S clouds of one traversal per call.  DESIGN.md 4.24 states the contract; deepi2p_b200/oxford_build.py
 * plans the windows and chains the calls with voxel_downsample_batch_f64 (C = 1) between scatter and pack.  All
 * arithmetic is fp64 without FMA, each sum in the association stated; all pointers [dev] unless marked [host].
 *
 * oxford_build_plan_f64: lms_poses [n_lms][16] row-major absolute poses, present [n_lms] u8 (0: no scan file),
 *   windows [S][2] i64 LMS index range [lo, hi), centre_inv [S][16] the inverse of each centre's absolute pose,
 *   G [host, 16] G_posesource_laser.  Per cloud, for i in [lo, hi) with present[i]: rel = M_c P_i (each entry
 *   ((a0 b0 + a1 b1) + a2 b2) + a3 b3); unless it is the first kept scan, d = rows 0-2 of inv(prev) rel[:, 3] and
 *   the scan is skipped when sqrt((d0 d0 + d1 d1) + d2 d2) < skip_threshold, prev being the last kept rel and inv a
 *   Gauss-Jordan inverse with partial pivoting (first largest |pivot|; all eight columns of [A | I] updated, rows in
 *   ascending order).  A kept scan writes kept_scan [S][w_stride] i32 = i and kept_T [S][w_stride][12] = rows 0-2
 *   of rel G.  n_kept [S], n_skipped [S] i32.  A window outside [0, n_lms] or longer than w_stride gives n_kept = 0,
 *   n_skipped = -1.
 * oxford_build_count_f64: x, r [store] f64 planes, offsets [n_lms + 1] i64 (scan i = [offsets[i], offsets[i+1])).
 *   A point is kept when use_mask is 0 or x < threshold.  pos [S][w_stride] i32 = first output index of each kept
 *   scan, n_pts [S] i32 = kept points of the cloud, rmax [S] f64 = their largest reflectance (-inf when none).
 *   workspace >= oxford_build_count_workspace_bytes(S, w_stride), 256-byte aligned.
 * oxford_build_scatter_f64: the kept points in scan order, then point order: xyz_out [S][3][n_stride] =
 *   ((T0 x + T1 y) + T2 0) + T3 per row, attr_out [S][n_stride] = r / rmax.  Entries past n_pts are not written;
 *   n_stride % 16 == 0 and n_stride >= max n_pts.
 * oxford_build_pack_f32: xyz [S][3][n_stride], attr [S][n_stride] (voxel_downsample_batch_f64's outputs), m_pts
 *   [S] i32 <= m_stride, O [host, 16]: out [S][4][m_stride] f32 = (float)(((O0 x + O1 y) + O2 z) + O3) for rows
 *   0-2 and (float)(attr * rmax) for row 3, zeros past m_pts.
 * ------------------------------------------------------------------------------------------ */
int oxford_build_plan_f64(const double* lms_poses, const uint8_t* present, int64_t n_lms, const int64_t* windows,
                          const double* centre_inv, int S, const double* G, double skip_threshold, int w_stride,
                          int32_t* kept_scan, double* kept_T, int32_t* n_kept, int32_t* n_skipped,
                          dib_stream_t stream);
size_t oxford_build_count_workspace_bytes(int S, int w_stride);
int oxford_build_count_f64(const double* x, const double* r, const int64_t* offsets, const int32_t* kept_scan,
                           const int32_t* n_kept, int S, int w_stride, int use_mask, double threshold, int32_t* pos,
                           int32_t* n_pts, double* rmax, void* workspace, size_t workspace_bytes,
                           dib_stream_t stream);
int oxford_build_scatter_f64(const double* x, const double* y, const double* r, const int64_t* offsets,
                             const int32_t* kept_scan, const double* kept_T, const int32_t* n_kept,
                             const int32_t* pos, const double* rmax, int S, int w_stride, int use_mask,
                             double threshold, int n_stride, double* xyz_out, double* attr_out,
                             dib_stream_t stream);
int oxford_build_pack_f32(const double* xyz, const double* attr, const int32_t* m_pts, const double* rmax,
                          const double* O, int S, int n_stride, int m_stride, float* out, dib_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Oxford RobotCar stereo-centre frames (the SDK's load_image for the stereo camera).  DESIGN.md 4.25 states the
 * contract: GBRG bilinear demosaicing (colour_demosaicing, float64, scipy 'reflect' borders) and the undistortion LUT
 * through scipy's map_coordinates(order=1, mode 'constant'), then numpy's uint8 cast, bit for bit.
 *
 * oxford_debayer_undistort_u8: grey [dev] grey_bytes bytes, image s an h x w mosaic at desc offset 0; lut [dev]
 *   16-byte aligned float64 (x, y) pairs, lut_pairs of them, image s reading the h w pairs from desc slot 4; desc
 *   [host] int64 [S][DIB_OXIMG_DESC]: 0 mosaic offset, 1 output offset, 2 h, 3 w, 4 first LUT pair (h, w in
 *   2..65536); out [dev] HWC RGB uint8, image s at its offset.  workspace [dev] >= oxford_debayer_workspace_bytes(S).
 *
 * Batched baseline JPEG encoding (4:2:0, quality tables given, Annex K Huffman tables, no restart markers), bit for
 * bit with OpenCV 4.13's cv2.imencode(".jpg") on libjpeg-turbo 3.1; deepi2p_b200/jpeg_encode.py builds the tables
 * and the markers around the entropy-coded data.
 *
 * jpeg_encode_entropy_u8: rgb [dev] HWC uint8; desc [host] int64 [S][DIB_JPEGE_DESC]: 0 input offset, 1 h, 2 w
 *   (1..65500), the other slots the library's; quant [host] int32 [2][64] luma and chroma quantisers in natural order
 *   (1..255); huff [host] int32 [4][256] (length << 16) | code per symbol of the DC luma, AC luma, DC chroma and AC
 *   chroma tables.  Codes every image into the workspace and writes counts [dev] int64 [S][2]: the entropy-coded
 *   bytes before stuffing (padded with 1 bits) and their number of 0xFF bytes.
 * jpeg_encode_stuff_u8: the same desc and workspace, after jpeg_encode_entropy_u8 on the same stream: writes image s's
 *   bytes, each 0xFF followed by 0x00, to out [dev] at out_off[s] [host] (its bytes + 0xFF count long).
 *   workspace [dev] 256-byte aligned, >= jpeg_encode_workspace_bytes(desc, S) (0 for invalid descriptors).
 * ------------------------------------------------------------------------------------------ */
#define DIB_OXIMG_DESC 8
size_t oxford_debayer_workspace_bytes(int S);
int oxford_debayer_undistort_u8(const uint8_t* grey, size_t grey_bytes, const double* lut, int64_t lut_pairs,
                                const int64_t* desc, int S, uint8_t* out, size_t out_bytes, void* workspace,
                                size_t workspace_bytes, dib_stream_t stream);
#define DIB_JPEGE_DESC 8
size_t jpeg_encode_workspace_bytes(const int64_t* desc, int S);
int jpeg_encode_entropy_u8(const uint8_t* rgb, size_t rgb_bytes, const int64_t* desc, int S, const int32_t* quant,
                           const int32_t* huff, int64_t* counts, void* workspace, size_t workspace_bytes,
                           dib_stream_t stream);
int jpeg_encode_stuff_u8(const int64_t* desc, int S, const int64_t* out_off, uint8_t* out, size_t out_bytes,
                         void* workspace, size_t workspace_bytes, dib_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* DEEPI2P_B200_H_ */
