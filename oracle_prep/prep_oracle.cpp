// CPU oracle of the scan-preparation path (DESIGN.md "Scan preparation") -- TEST INFRASTRUCTURE ONLY.
// Serial restatement of csrc/pointprep.cu per cloud: the voxel grouping by a stable sort of (ix, iy, iz) tuples, the
// radius search by a uniform grid of 2r cells (not the kernels' Morton tree), the covariance sums and Jacobi
// eigensolver in the kernels' order.  Built with -ffp-contract=off, so every operation rounds as the kernels' do.
#include <algorithm>
#include <array>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <numeric>
#include <unordered_map>
#include <vector>

namespace {

// csrc/sym3_eig.cuh line for line.
void jacobi_serial(double* A, double* V, int n) {
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
        if (apq == 0.0 || std::fabs(apq) <= 1e-17 * std::sqrt(std::fabs(app) * std::fabs(aqq))) continue;
        const double theta = (aqq - app) / (2.0 * apq);
        const double t = std::fabs(theta) > 1e150
                             ? 0.5 / theta
                             : (theta >= 0.0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
        const double c = 1.0 / std::sqrt(t * t + 1.0), s = t * c;
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

void sym3_eig_desc(const double C[9], double lam[3], double E[9]) {
  double A[9], V[9];
  std::memcpy(A, C, sizeof(A));
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

struct CellHash {
  size_t operator()(const std::array<long long, 3>& c) const {
    return (size_t)(c[0] * 73856093LL) ^ (size_t)(c[1] * 19349663LL) ^ (size_t)(c[2] * 83492791LL);
  }
};

}  // namespace

extern "C" {

// One cloud: xyz [3][stride] f32 (n points), attr [C][stride] f64.  Outputs [3][stride], [C][stride]; *m_out voxels.
// Returns 0, or -22 when the cloud spans 2^21 or more voxels along an axis.
int prep_oracle_voxel(const float* xyz, int n, int stride, const double* attr, int C, double v, double* xyz_out,
                      double* attr_out, int* m_out) {
  *m_out = 0;
  if (n <= 0) return 0;
  float lo[3], hi[3];
  for (int a = 0; a < 3; ++a) {
    lo[a] = hi[a] = xyz[(size_t)a * stride];
    for (int j = 1; j < n; ++j) {
      lo[a] = std::min(lo[a], xyz[(size_t)a * stride + j]);
      hi[a] = std::max(hi[a], xyz[(size_t)a * stride + j]);
    }
  }
  double mb[3];
  for (int a = 0; a < 3; ++a) {
    mb[a] = (double)lo[a] - 0.5 * v;
    if (!(std::floor(((double)hi[a] - mb[a]) / v) < (double)(1 << 21))) return -22;
  }
  std::vector<std::array<long long, 3>> key(n);
  for (int j = 0; j < n; ++j)
    for (int a = 0; a < 3; ++a) key[j][a] = (long long)std::floor(((double)xyz[(size_t)a * stride + j] - mb[a]) / v);
  std::vector<int> ord(n);
  std::iota(ord.begin(), ord.end(), 0);
  std::stable_sort(ord.begin(), ord.end(), [&](int p, int q) { return key[p] < key[q]; });
  int m = 0;
  for (int b = 0; b < n;) {
    int e = b + 1;
    while (e < n && key[ord[e]] == key[ord[b]]) ++e;
    const double cnt = (double)(e - b);
    for (int a = 0; a < 3; ++a) {
      double s = 0.0;
      for (int t = b; t < e; ++t) s += (double)xyz[(size_t)a * stride + ord[t]];
      xyz_out[(size_t)a * stride + m] = s / cnt;
    }
    for (int c = 0; c < C; ++c) {
      double s = 0.0;
      for (int t = b; t < e; ++t) s += attr[(size_t)c * stride + ord[t]];
      attr_out[(size_t)c * stride + m] = s / cnt;
    }
    ++m;
    b = e;
  }
  *m_out = m;
  return 0;
}

// One cloud: xyz [3][stride] f32 (m points).  normals [3][stride] f64, count [m] i32, nbr [m][max_nn] i32 (-1 padded;
// may be NULL) = the neighbours in ascending (d2, index) order.
void prep_oracle_normals(const float* xyz, int m, int stride, double r, int max_nn, const double* o, double* normals,
                         int* count, int* nbr) {
  if (m <= 0) return;
  const double r2 = r * r, cell = 2.0 * r;
  const float* X = xyz;
  const float* Y = xyz + stride;
  const float* Z = xyz + (size_t)2 * stride;
  double lo[3] = {DBL_MAX, DBL_MAX, DBL_MAX};
  for (int j = 0; j < m; ++j) {
    lo[0] = std::min(lo[0], (double)X[j]);
    lo[1] = std::min(lo[1], (double)Y[j]);
    lo[2] = std::min(lo[2], (double)Z[j]);
  }
  auto cell_of = [&](int j) {
    return std::array<long long, 3>{(long long)std::floor(((double)X[j] - lo[0]) / cell),
                                    (long long)std::floor(((double)Y[j] - lo[1]) / cell),
                                    (long long)std::floor(((double)Z[j] - lo[2]) / cell)};
  };
  std::unordered_map<std::array<long long, 3>, std::vector<int>, CellHash> grid;
  for (int j = 0; j < m; ++j) grid[cell_of(j)].push_back(j);
#pragma omp parallel for schedule(dynamic, 256)
  for (int i = 0; i < m; ++i) {
    const double qx = X[i], qy = Y[i], qz = Z[i];
    const std::array<long long, 3> ci = cell_of(i);
    std::vector<std::pair<double, int>> cand;
    for (long long a = -1; a <= 1; ++a)
      for (long long b = -1; b <= 1; ++b)
        for (long long c = -1; c <= 1; ++c) {
          const auto it = grid.find({ci[0] + a, ci[1] + b, ci[2] + c});
          if (it == grid.end()) continue;
          for (const int j : it->second) {
            const double dx = qx - (double)X[j], dy = qy - (double)Y[j], dz = qz - (double)Z[j];
            const double d2 = (dx * dx + dy * dy) + dz * dz;
            if (d2 < r2) cand.emplace_back(d2, j);
          }
        }
    std::sort(cand.begin(), cand.end());
    const int cnt = std::min((int)cand.size(), max_nn);
    double n[3] = {0.0, 0.0, 1.0};
    if (cnt >= 3) {
      double s[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
      for (int t = 0; t < cnt; ++t) {
        const int j = cand[t].second;
        const double dx = (double)X[j] - qx, dy = (double)Y[j] - qy, dz = (double)Z[j] - qz;
        s[0] += dx; s[1] += dy; s[2] += dz;
        s[3] += dx * dx; s[4] += dx * dy; s[5] += dx * dz;
        s[6] += dy * dy; s[7] += dy * dz; s[8] += dz * dz;
      }
      for (int q = 0; q < 9; ++q) s[q] = s[q] / (double)cnt;
      double C[9];
      C[0] = s[3] - s[0] * s[0];
      C[4] = s[6] - s[1] * s[1];
      C[8] = s[8] - s[2] * s[2];
      C[1] = C[3] = s[4] - s[0] * s[1];
      C[2] = C[6] = s[5] - s[0] * s[2];
      C[5] = C[7] = s[7] - s[1] * s[2];
      if (C[0] == 0.0 && C[4] == 0.0 && C[8] == 0.0 && C[1] == 0.0 && C[2] == 0.0 && C[5] == 0.0) {
        n[0] = n[1] = n[2] = 0.0;
      } else {
        double lam[3], E[9];
        sym3_eig_desc(C, lam, E);
        const double e0 = E[2], e1 = E[5], e2 = E[8];
        const double nn = std::sqrt((e0 * e0 + e1 * e1) + e2 * e2);
        n[0] = e0 / nn; n[1] = e1 / nn; n[2] = e2 / nn;
      }
    }
    if (n[0] == 0.0 && n[1] == 0.0 && n[2] == 0.0) {
      n[0] = o[0]; n[1] = o[1]; n[2] = o[2];
    } else if ((n[0] * o[0] + n[1] * o[1]) + n[2] * o[2] < 0.0) {
      n[0] = -n[0]; n[1] = -n[1]; n[2] = -n[2];
    }
    for (int q = 0; q < 3; ++q) normals[(size_t)q * stride + i] = n[q];
    count[i] = cnt;
    if (nbr)
      for (int t = 0; t < max_nn; ++t) nbr[(size_t)i * max_nn + t] = t < cnt ? cand[t].second : -1;
  }
}

}  // extern "C"
