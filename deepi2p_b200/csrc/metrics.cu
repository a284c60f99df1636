// Batched evaluation-side ops next to the solver (SURVEY.md 8f, row N3):
//   frustum_inside_mask_f32 : the ground-truth / prediction-check label rule
//        0 <= u <= W-1  and  0 <= v <= H-1  and  z > 0.1      with  [u v 1]^T ~ K (P p)
//        (evaluation/registration_lsq.py:67-84, models/multimodal_classifier.py:136-148)
//   pose_error_batch        : get_P_diff (evaluation/registration_lsq.py:87-95): P_diff = P_pred^-1 P_gt with a
//        general inverse (P_pred need not be rigid), translation error |P_diff[:3,3]|, rotation error = sum |euler
//        'xzy' angles| in degrees as scipy computes them (gimbal lock included), and the authors' success flag
//        t < 2 m and r < 5 deg (evaluation/registration_result_analysis.py:37-38).
// The file is compiled with --fmad=false (build.py NOFMA_SOURCES): oracle.pose_diff_restated restates
// pose_error_kernel bit for bit.  inside_mask_kernel's decisions do not depend on rounding away from the boundaries.
#include <cmath>

#include "common.cuh"

namespace dib {

__global__ void inside_mask_kernel(const float* __restrict__ xyz, const int32_t* __restrict__ n_pts, int n_stride,
                                   const double* __restrict__ P16, const double* __restrict__ K9, double H, double W,
                                   int8_t* __restrict__ mask) {
  const int s = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_stride) return;
  const int n = n_pts ? n_pts[s] : n_stride;
  int8_t out = -1;
  if (i < n) {
    const double* P = P16 + (size_t)s * 16;
    const double* K = K9 + (size_t)s * 9;
    const float* b = xyz + (size_t)s * 3 * n_stride;
    const double x = b[i], y = b[n_stride + i], z = b[2 * (size_t)n_stride + i];
    // P_points = (P [x y z 1]^T)[0:3]
    const double X = P[0] * x + P[1] * y + P[2] * z + P[3];
    const double Y = P[4] * x + P[5] * y + P[6] * z + P[7];
    const double Z = P[8] * x + P[9] * y + P[10] * z + P[11];
    // K_pc = K P_points ; pxpy = K_pc[0:2] / K_pc[2]
    const double kx = K[0] * X + K[1] * Y + K[2] * Z;
    const double ky = K[3] * X + K[4] * Y + K[5] * Z;
    const double kz = K[6] * X + K[7] * Y + K[8] * Z;
    const double u = kx / kz, v = ky / kz;
    out = (u >= 0.0 && u <= W - 1.0 && v >= 0.0 && v <= H - 1.0 && Z > 0.1) ? 1 : 0;
  }
  mask[(size_t)s * n_stride + i] = out;
}

// ---- pose_error_kernel: get_P_diff restated operation for operation (DESIGN.md 4.14) ---------------------------------
// The reference inverts P_pred with np.linalg.inv and hands P_diff's rotation block to scipy's
// Rotation.from_matrix(...).as_euler('xzy').  The kernel follows both steps rather than assuming a rigid P_pred:
//   1. the general cofactor inverse of the 4x4 P_pred (one fp64 division per entry), P_diff = inv(P_pred) P_gt;
//   2. from_matrix: det(M) <= 0 is no rotation (scipy raises; here r_err = NaN, success = 0); M is used as it is when
//      |M M^T - I| <= 1e-12 + 1e-5 I elementwise, else replaced by its orthogonal polar factor (scipy's U V^T, here by
//      Newton's iteration X <- (X + X^-T) / 2); the quaternion comes from the largest of m00, m11, m22, trace;
//   3. as_euler('xzy') by the quaternion route: with (a, b, c, d) = (w - z, x - y, z + w, -y - x),
//      middle = 2 atan2(|(c, d)|, |(a, b)|) - pi/2, half_sum = atan2(b, a), half_diff = atan2(d, c); within 1e-7 rad
//      of gimbal lock (middle = -pi/2 or +pi/2) the third angle is 0 and the first 2 half_sum or -2 half_diff,
//      otherwise first = half_sum - half_diff, third = -(half_sum + half_diff); each angle wrapped to [-pi, pi).
// atan2 is built from +, -, *, /, sqrt (two argument halvings, then a 12-term series), so with the file compiled
// without FMA contraction every result is the one oracle.pose_diff_restated computes in numpy, bit for bit.
constexpr double kPi = 3.141592653589793115997963468544185161590576171875;
__device__ constexpr double kAtanC[12] = {1.0,        -1.0 / 3.0,  1.0 / 5.0,  -1.0 / 7.0,  1.0 / 9.0,  -1.0 / 11.0,
                                          1.0 / 13.0, -1.0 / 15.0, 1.0 / 17.0, -1.0 / 19.0, 1.0 / 21.0, -1.0 / 23.0};

__device__ double atan2_restated(double y, double x) {
  const double ax = fabs(x), ay = fabs(y);
  const bool swap = ay > ax;
  const double num = swap ? ax : ay, den = swap ? ay : ax;
  double t = den == 0.0 ? 0.0 : num / den;
  t = t / (1.0 + sqrt(1.0 + t * t));                  // atan(t) = 2 atan(t / (1 + sqrt(1 + t^2))), twice:
  t = t / (1.0 + sqrt(1.0 + t * t));                  // |t| <= tan(pi/16)
  const double z = t * t;
  double p = kAtanC[11];
#pragma unroll
  for (int k = 10; k >= 0; --k) p = p * z + kAtanC[k];
  double r = 4.0 * (t * p);
  if (swap) r = kPi / 2 - r;
  if (signbit(x)) r = kPi - r;
  return signbit(y) ? -r : r;
}

__device__ double wrap_pi(double a) {              // numpy's (a + pi) % (2 pi) - pi
  double m = fmod(a + kPi, 2 * kPi);
  m = m == 0.0 ? 0.0 : (m < 0.0 ? m + 2 * kPi : m);
  return m - kPi;
}

__device__ double cof3(const double m[3][3], double C[3][3]) {   // cofactor matrix; returns the determinant
  C[0][0] = m[1][1] * m[2][2] - m[1][2] * m[2][1];
  C[0][1] = m[1][2] * m[2][0] - m[1][0] * m[2][2];
  C[0][2] = m[1][0] * m[2][1] - m[1][1] * m[2][0];
  C[1][0] = m[0][2] * m[2][1] - m[0][1] * m[2][2];
  C[1][1] = m[0][0] * m[2][2] - m[0][2] * m[2][0];
  C[1][2] = m[0][1] * m[2][0] - m[0][0] * m[2][1];
  C[2][0] = m[0][1] * m[1][2] - m[0][2] * m[1][1];
  C[2][1] = m[0][2] * m[1][0] - m[0][0] * m[1][2];
  C[2][2] = m[0][0] * m[1][1] - m[0][1] * m[1][0];
  return m[0][0] * C[0][0] + m[0][1] * C[0][1] + m[0][2] * C[0][2];
}

constexpr int kPolarMaxIter = 64;

__global__ void pose_error_kernel(const double* __restrict__ Pp, const double* __restrict__ Pg, int S,
                                  double t_thresh, double r_thresh, double* __restrict__ t_err,
                                  double* __restrict__ r_err_deg, int32_t* __restrict__ success) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= S) return;
  double a[4][4], B[4][4];
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) { a[r][c] = Pp[(size_t)s * 16 + 4 * r + c]; B[r][c] = Pg[(size_t)s * 16 + 4 * r + c]; }
  // rows 0..2 of inv(P_pred) by 2x2 sub-determinants of the top (s) and bottom (c) row pairs
  const double s0 = a[0][0] * a[1][1] - a[1][0] * a[0][1], s1 = a[0][0] * a[1][2] - a[1][0] * a[0][2];
  const double s2 = a[0][0] * a[1][3] - a[1][0] * a[0][3], s3 = a[0][1] * a[1][2] - a[1][1] * a[0][2];
  const double s4 = a[0][1] * a[1][3] - a[1][1] * a[0][3], s5 = a[0][2] * a[1][3] - a[1][2] * a[0][3];
  const double c5 = a[2][2] * a[3][3] - a[3][2] * a[2][3], c4 = a[2][1] * a[3][3] - a[3][1] * a[2][3];
  const double c3 = a[2][1] * a[3][2] - a[3][1] * a[2][2], c2 = a[2][0] * a[3][3] - a[3][0] * a[2][3];
  const double c1 = a[2][0] * a[3][2] - a[3][0] * a[2][2], c0 = a[2][0] * a[3][1] - a[3][0] * a[2][1];
  const double det = s0 * c5 - s1 * c4 + s2 * c3 + s3 * c2 - s4 * c1 + s5 * c0;
  const double inv[3][4] = {
      {(a[1][1] * c5 - a[1][2] * c4 + a[1][3] * c3) / det, (-a[0][1] * c5 + a[0][2] * c4 - a[0][3] * c3) / det,
       (a[3][1] * s5 - a[3][2] * s4 + a[3][3] * s3) / det, (-a[2][1] * s5 + a[2][2] * s4 - a[2][3] * s3) / det},
      {(-a[1][0] * c5 + a[1][2] * c2 - a[1][3] * c1) / det, (a[0][0] * c5 - a[0][2] * c2 + a[0][3] * c1) / det,
       (-a[3][0] * s5 + a[3][2] * s2 - a[3][3] * s1) / det, (a[2][0] * s5 - a[2][2] * s2 + a[2][3] * s1) / det},
      {(a[1][0] * c4 - a[1][1] * c2 + a[1][3] * c0) / det, (-a[0][0] * c4 + a[0][1] * c2 - a[0][3] * c0) / det,
       (a[3][0] * s4 - a[3][1] * s2 + a[3][3] * s0) / det, (-a[2][0] * s4 + a[2][1] * s2 - a[2][3] * s0) / det}};
  double M[3][3], t[3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 4; ++j) {
      const double v = ((inv[i][0] * B[0][j] + inv[i][1] * B[1][j]) + inv[i][2] * B[2][j]) + inv[i][3] * B[3][j];
      if (j < 3) M[i][j] = v; else t[i] = v;
    }
  const double te = sqrt((t[0] * t[0] + t[1] * t[1]) + t[2] * t[2]);

  double C[3][3];
  const bool valid = cof3(M, C) > 0.0;
  bool ortho = true;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      const double g = (M[i][0] * M[j][0] + M[i][1] * M[j][1]) + M[i][2] * M[j][2];
      ortho &= i == j ? fabs(g - 1.0) <= 1e-12 + 1e-5 : fabs(g) <= 1e-12;
    }
  if (valid && !ortho) {
    for (int it = 0; it < kPolarMaxIter; ++it) {
      const double dX = cof3(M, C);
      bool done = true;
      for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
          const double x = 0.5 * (M[i][j] + C[i][j] / dX);
          done &= fabs(x - M[i][j]) < 1e-10;                 // quadratic convergence: x is now exact
          M[i][j] = x;
        }
      if (done) break;
    }
  }
  // quaternion (x, y, z, w) from the largest of m00, m11, m22, trace (the first on ties)
  const double tr = (M[0][0] + M[1][1]) + M[2][2];
  int choice = 0;
  double best = M[0][0];
  if (M[1][1] > best) { choice = 1; best = M[1][1]; }
  if (M[2][2] > best) { choice = 2; best = M[2][2]; }
  if (tr > best) choice = 3;
  double q[4];
  if (choice == 3) {
    q[0] = M[2][1] - M[1][2]; q[1] = M[0][2] - M[2][0]; q[2] = M[1][0] - M[0][1]; q[3] = 1.0 + tr;
  } else {
    const int i = choice, j = (i + 1) % 3, k = (i + 2) % 3;
    q[i] = (1.0 - tr) + 2.0 * M[i][i];
    q[j] = M[j][i] + M[i][j];
    q[k] = M[k][i] + M[i][k];
    q[3] = M[k][j] - M[j][k];
  }
  const double qn = sqrt(((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3]);
  const double qx = q[0] / qn, qy = q[1] / qn, qz = q[2] / qn, qw = q[3] / qn;
  // extrinsic 'xzy': axes (i, j, k) = (0, 2, 1), sign -1, lambda = pi/2
  const double ea = qw - qz, eb = qx - qy, ec = qz + qw, ed = -qy - qx;
  const double half_sum = atan2_restated(eb, ea), half_diff = atan2_restated(ed, ec);
  const double mid = 2.0 * atan2_restated(sqrt(ec * ec + ed * ed), sqrt(ea * ea + eb * eb));
  const bool lock0 = fabs(mid) <= 1e-7;                    // middle angle -pi/2
  const bool lock1 = !lock0 && fabs(mid - kPi) <= 1e-7;   // middle angle +pi/2
  const double first = lock0 ? 2.0 * half_sum : (lock1 ? -2.0 * half_diff : half_sum - half_diff);
  const double third = (lock0 || lock1) ? 0.0 : -(half_sum + half_diff);
  constexpr double kDeg = 180.0 / kPi;
  double re = (fabs(wrap_pi(first) * kDeg) + fabs(wrap_pi(mid - kPi / 2) * kDeg)) + fabs(wrap_pi(third) * kDeg);
  if (!valid) re = nan("");
  t_err[s] = te;
  r_err_deg[s] = re;
  if (success) success[s] = (te < t_thresh && re < r_thresh) ? 1 : 0;
}

}  // namespace dib

extern "C" {

int frustum_inside_mask_f32(const float* xyz, const int32_t* n_pts, int n_stride, const double* P16, const double* K9,
                            double H, double W, int S, int8_t* mask_out, dib_stream_t stream) {
  using namespace dib;
  DIB_REQUIRE(xyz && P16 && K9 && mask_out, "NULL argument");
  DIB_REQUIRE(S >= 0 && n_stride >= 0 && S <= 65535, "bad sizes");
  if (S == 0 || n_stride == 0) return DIB_OK;
  dim3 grid((n_stride + 255) / 256, S);
  inside_mask_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(xyz, n_pts, n_stride, P16, K9, H, W, mask_out);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

int pose_error_batch(const double* P_pred16, const double* P_gt16, int S, double t_thresh_m, double r_thresh_deg,
                     double* t_err, double* r_err_deg, int32_t* success, dib_stream_t stream) {
  using namespace dib;
  DIB_REQUIRE(P_pred16 && P_gt16 && t_err && r_err_deg, "NULL argument");
  DIB_REQUIRE(S >= 0, "bad sizes");
  if (S == 0) return DIB_OK;
  pose_error_kernel<<<(S + 127) / 128, 128, 0, (cudaStream_t)stream>>>(P_pred16, P_gt16, S, t_thresh_m, r_thresh_deg,
                                                                         t_err, r_err_deg, success);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

}  // extern "C"
