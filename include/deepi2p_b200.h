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

#ifdef __cplusplus
}
#endif
#endif /* DEEPI2P_B200_H_ */
