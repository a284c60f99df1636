// The classifier's label rule (models/multimodal_classifier.py:136-148, evaluation/registration_lsq.py:67-84):
//   [u v 1]^T ~ K (P [x y z 1]^T),  inside  <=>  0 <= u <= W-1  and  0 <= v <= H-1  and  Z > 0.1
// evaluated in fp64 from float32 coordinates.  metrics.cu (frustum_inside_mask_f32) and classifier_loss.cu both call
// this one function and are both compiled without FMA contraction (build.py NOFMA_SOURCES), so their labels agree bit
// for bit.  NaN coordinates or Z <= 0.1 give "outside".
#pragma once

namespace dib {

// P: rows 0..2 of the pose, row-major (the first 12 entries of a 3x4 or 4x4 matrix); K: 3x3 row-major.
// Writes the projected pixel (u, v) and returns the inside decision.
__device__ __forceinline__ bool project_inside(const double* __restrict__ P, const double* __restrict__ K, double x,
                                               double y, double z, double H, double W, double* u_out, double* v_out) {
  // P_points = (P [x y z 1]^T)[0:3]
  const double X = P[0] * x + P[1] * y + P[2] * z + P[3];
  const double Y = P[4] * x + P[5] * y + P[6] * z + P[7];
  const double Z = P[8] * x + P[9] * y + P[10] * z + P[11];
  // K_pc = K P_points ; pxpy = K_pc[0:2] / K_pc[2]
  const double kx = K[0] * X + K[1] * Y + K[2] * Z;
  const double ky = K[3] * X + K[4] * Y + K[5] * Z;
  const double kz = K[6] * X + K[7] * Y + K[8] * Z;
  const double u = kx / kz, v = ky / kz;
  *u_out = u;
  *v_out = v;
  return u >= 0.0 && u <= W - 1.0 && v >= 0.0 && v <= H - 1.0 && Z > 0.1;
}

}  // namespace dib
