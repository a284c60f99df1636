// Serial cyclic Jacobi eigensolver for small symmetric matrices (+ - * / sqrt only), shared by pnp_ransac.cu (EPnP's
// 3x3 problems) and pointprep.cu (surface normals).  oracle_pnp/pnp_oracle.cpp and oracle_prep/prep_oracle.cpp restate
// it line for line; the including files are compiled with --fmad=false, so every operation rounds as theirs do.
#pragma once
#include <cmath>

namespace dib {

// Cyclic Jacobi for small n (the 3x3 problems): eigenvalues on the diagonal, V = eigenvectors in columns.
static __device__ void jacobi_serial(double* A, double* V, int n) {
  for (int i = 0; i < n * n; ++i) V[i] = (i / n == i % n) ? 1.0 : 0.0;
  double fro = 0.0;
  for (int i = 0; i < n * n; ++i) fro += A[i] * A[i];
  for (int sweep = 0; sweep < 30; ++sweep) {
    double off = 0.0;
    for (int i = 0; i < n; ++i)
      for (int j = 0; j < n; ++j)
        if (i != j) off += A[i * n + j] * A[i * n + j];
    if (off <= 1e-32 * fro) break;
    bool rotated = false;
    for (int p = 0; p < n - 1; ++p)
      for (int q = p + 1; q < n; ++q) {
        const double apq = A[p * n + q], app = A[p * n + p], aqq = A[q * n + q];
        if (apq == 0.0 || fabs(apq) <= 1e-17 * sqrt(fabs(app) * fabs(aqq))) continue;
        const double theta = (aqq - app) / (2.0 * apq);
        const double t = fabs(theta) > 1e150 ? 0.5 / theta
                                             : (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < n; ++k) {
          const double x = A[p * n + k], y = A[q * n + k];
          A[p * n + k] = c * x - s * y;
          A[q * n + k] = s * x + c * y;
        }
        for (int k = 0; k < n; ++k) {
          const double x = A[k * n + p], y = A[k * n + q];
          A[k * n + p] = c * x - s * y;
          A[k * n + q] = s * x + c * y;
        }
        A[p * n + q] = A[q * n + p] = 0.0;
        for (int k = 0; k < n; ++k) {
          const double x = V[k * n + p], y = V[k * n + q];
          V[k * n + p] = c * x - s * y;
          V[k * n + q] = s * x + c * y;
        }
        rotated = true;
      }
    if (!rotated) break;
  }
}

static __device__ void sym3_eig_desc(const double C[9], double lam[3], double E[9]) {
  double A[9], V[9];
  for (int i = 0; i < 9; ++i) A[i] = C[i];
  jacobi_serial(A, V, 3);
  int o[3] = {0, 1, 2};
  for (int i = 0; i < 3; ++i)
    for (int j = i + 1; j < 3; ++j)
      if (A[o[j] * 4] > A[o[i] * 4]) { const int t = o[i]; o[i] = o[j]; o[j] = t; }
  for (int k = 0; k < 3; ++k) {
    lam[k] = A[o[k] * 4];
    for (int r = 0; r < 3; ++r) E[r * 3 + k] = V[r * 3 + o[k]];
  }
}

}  // namespace dib
