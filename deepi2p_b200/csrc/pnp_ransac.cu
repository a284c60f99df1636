// Batched PnP-RANSAC registration from grid classifications: the contract of evaluation/registration_pnp.py:95-148
// (cv2.solvePnPRansac(..., SOLVEPNP_EPNP)) restated for many frames at once.  DESIGN.md "PnP-RANSAC" states the
// contract; oracle_pnp/pnp_oracle.cpp is its serial CPU restatement.
//
// Per frame s:
//   select    (one CTA)   order-preserving compaction of the points with coarse_pred == 1; fine cell f -> pixel
//                         corner (px, py) = (f - floor(f / Wf) * Wf, floor(f / Wf)) in float64, Wf = W * scale
//   hyp       (one warp per hypothesis)  5 distinct Philox4x32-10 indices (counter (h, s, draw, 0), key = seed),
//                         minimal EPnP; the 12x12 eigenproblem of M^T M is a parallel-ordered cyclic Jacobi shared by
//                         the lanes (6 disjoint rotations per step)
//   score     (one CTA per frame and block of kBlockH hypotheses)  the frame's correspondences are staged through
//                         shared memory in tiles; counts by ballot + popc
//   replay    (one thread per frame)  the sequential adaptive stopping rule over the block, in hypothesis order
//   refit     (one warp per frame)  EPnP on the winner's inliers, then the reference's final rules
// hyp / score / replay run once per block of kBlockH hypotheses; a frame whose replay has stopped does no more work.
// All sums have a fixed order (lane-strided partial sums, xor-butterfly across lanes), so results are bit-identical
// run to run.  The inlier test is written with __dmul_rn / __dadd_rn so no FMA is contracted into it.
#include <cfloat>
#include <cmath>

#include "common.cuh"
#include "sym3_eig.cuh"

namespace dib {
namespace pnp {

constexpr int kBlockH = 64;           // hypotheses per replay block
constexpr int kHypWarps = 4;          // warps (= hypotheses) per CTA of the hypothesis kernel
constexpr int kScoreThreads = 256;    // 8 warps x 8 hypotheses
constexpr int kScoreTile = 512;       // correspondences staged per tile
constexpr int kSelThreads = 256;
enum { ST_NSEL = 0, ST_NITERS, ST_BEST, ST_BESTCNT, ST_USED, ST_STOPPED, ST_WORDS = 8 };

struct Cam {
  double fu, fv, cu, cv;
};

__device__ __forceinline__ Cam scaled_cam(const double* K9, double scale) {
  return Cam{__dmul_rn(scale, K9[0]), __dmul_rn(scale, K9[4]), __dmul_rn(scale, K9[2]), __dmul_rn(scale, K9[5])};
}

// The inlier rule: ((u - px)^2 + (v - py)^2 <= thr^2), (u, v) = projection of (X, Y, Z) by pose p = R | t.
__device__ __forceinline__ bool is_inlier(const double* p, double X, double Y, double Z, double U, double V,
                                          const Cam& c, double thr2) {
  const double x = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(p[0], X), __dmul_rn(p[1], Y)), __dmul_rn(p[2], Z)), p[9]);
  const double y = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(p[3], X), __dmul_rn(p[4], Y)), __dmul_rn(p[5], Z)), p[10]);
  const double z = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(p[6], X), __dmul_rn(p[7], Y)), __dmul_rn(p[8], Z)), p[11]);
  const double du = __dsub_rn(__dadd_rn(__dmul_rn(c.fu, __ddiv_rn(x, z)), c.cu), U);
  const double dv = __dsub_rn(__dadd_rn(__dmul_rn(c.fv, __ddiv_rn(y, z)), c.cv), V);
  return __dadd_rn(__dmul_rn(du, du), __dmul_rn(dv, dv)) <= thr2;
}

template <int N>
__device__ __forceinline__ void warp_sum(double (&v)[N]) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
#pragma unroll
    for (int k = 0; k < N; ++k) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
}

// Correspondences of one EPnP problem: point k of the problem is element i = idx ? idx[k] : k of the arrays,
// coordinates at X[i * sx] ..., pixels at U[i * su], V[i * su].
template <typename T>
struct Pts {
  const T *X, *Y, *Z;
  const double *U, *V;
  int sx, su;
  const int* idx;
  int n;
  __device__ __forceinline__ int at(int k) const { return idx ? idx[k] : k; }
};

struct Scratch {          // per-warp shared memory of warp_epnp
  double A[144], V[144];
  double cs[12], cp[12];
  double betas[3][4];
  int partner[12];
  int order[4];
  int bvalid[3];
  int idx[5];
};

// ---- serial pieces (identical on every lane that runs them) ----

// Proper rotation R = U V^T maximising tr(R^T H).  False when H has rank < 2.
__device__ bool kabsch(const double H[9], double R[9]) {
  double HtH[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) HtH[i * 3 + j] = H[i] * H[j] + H[3 + i] * H[3 + j] + H[6 + i] * H[6 + j];
  double lam[3], Vm[9];
  sym3_eig_desc(HtH, lam, Vm);
  const double det = Vm[0] * (Vm[4] * Vm[8] - Vm[5] * Vm[7]) - Vm[1] * (Vm[3] * Vm[8] - Vm[5] * Vm[6]) +
                     Vm[2] * (Vm[3] * Vm[7] - Vm[4] * Vm[6]);
  if (det < 0.0)
    for (int r = 0; r < 3; ++r) Vm[r * 3 + 2] = -Vm[r * 3 + 2];
  double u0[3], u1[3], u2[3];
  for (int r = 0; r < 3; ++r) {
    u0[r] = H[r * 3] * Vm[0] + H[r * 3 + 1] * Vm[3] + H[r * 3 + 2] * Vm[6];
    u1[r] = H[r * 3] * Vm[1] + H[r * 3 + 1] * Vm[4] + H[r * 3 + 2] * Vm[7];
  }
  const double n0 = sqrt(u0[0] * u0[0] + u0[1] * u0[1] + u0[2] * u0[2]);
  if (!(n0 > 0.0)) return false;
  for (int r = 0; r < 3; ++r) u0[r] /= n0;
  const double d = u0[0] * u1[0] + u0[1] * u1[1] + u0[2] * u1[2];
  for (int r = 0; r < 3; ++r) u1[r] -= d * u0[r];
  const double n1 = sqrt(u1[0] * u1[0] + u1[1] * u1[1] + u1[2] * u1[2]);
  if (!(n1 > 1e-12 * n0)) return false;
  for (int r = 0; r < 3; ++r) u1[r] /= n1;
  u2[0] = u0[1] * u1[2] - u0[2] * u1[1];
  u2[1] = u0[2] * u1[0] - u0[0] * u1[2];
  u2[2] = u0[0] * u1[1] - u0[1] * u1[0];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) R[i * 3 + j] = u0[i] * Vm[j * 3] + u1[i] * Vm[j * 3 + 1] + u2[i] * Vm[j * 3 + 2];
  return true;
}

// min |A x - b| for A [6][m] row-major (m <= 5), Householder QR.  False on a zero pivot.
__device__ bool ls6(const double* Ain, int m, const double* bin, double* x) {
  double A[6][5], b[6];
  for (int i = 0; i < 6; ++i) {
    b[i] = bin[i];
    for (int j = 0; j < m; ++j) A[i][j] = Ain[i * m + j];
  }
  for (int k = 0; k < m; ++k) {
    double nrm = 0.0;
    for (int i = k; i < 6; ++i) nrm += A[i][k] * A[i][k];
    nrm = sqrt(nrm);
    if (!(nrm > 0.0)) return false;
    const double alpha = A[k][k] > 0.0 ? -nrm : nrm;
    double v[6];
    for (int i = 0; i < 6; ++i) v[i] = i < k ? 0.0 : A[i][k];
    v[k] -= alpha;
    double vv = 0.0;
    for (int i = k; i < 6; ++i) vv += v[i] * v[i];
    if (!(vv > 0.0)) return false;
    for (int j = k; j < m; ++j) {
      double d = 0.0;
      for (int i = k; i < 6; ++i) d += v[i] * A[i][j];
      d = 2.0 * d / vv;
      for (int i = k; i < 6; ++i) A[i][j] -= d * v[i];
    }
    double d = 0.0;
    for (int i = k; i < 6; ++i) d += v[i] * b[i];
    d = 2.0 * d / vv;
    for (int i = k; i < 6; ++i) b[i] -= d * v[i];
  }
  for (int k = m - 1; k >= 0; --k) {
    double r = b[k];
    for (int j = k + 1; j < m; ++j) r -= A[k][j] * x[j];
    x[k] = r / A[k][k];
  }
  return true;
}

// Betas of the three EPnP approximations (N = 4, 2, 3 null vectors), each refined by 5 Gauss-Newton steps on the
// 6 control-point distance constraints.  v[k] = k-th smallest eigenvector of M^T M, cw = world control points.
__device__ void epnp_betas(const double (&v)[4][12], const double (&cw)[4][3], double (&betas)[3][4], int (&ok)[3]) {
  const int pairs[6][2] = {{0, 1}, {0, 2}, {0, 3}, {1, 2}, {1, 3}, {2, 3}};
  double L[6][10], rho[6];
  for (int e = 0; e < 6; ++e) {
    const int a = pairs[e][0], b = pairs[e][1];
    double dv[4][3];
    for (int k = 0; k < 4; ++k)
      for (int d = 0; d < 3; ++d) dv[k][d] = v[k][3 * a + d] - v[k][3 * b + d];
#define DOT(x, y) (dv[x][0] * dv[y][0] + dv[x][1] * dv[y][1] + dv[x][2] * dv[y][2])
    L[e][0] = DOT(0, 0); L[e][1] = 2 * DOT(0, 1); L[e][2] = DOT(1, 1); L[e][3] = 2 * DOT(0, 2);
    L[e][4] = 2 * DOT(1, 2); L[e][5] = DOT(2, 2); L[e][6] = 2 * DOT(0, 3); L[e][7] = 2 * DOT(1, 3);
    L[e][8] = 2 * DOT(2, 3); L[e][9] = DOT(3, 3);
#undef DOT
    double r2 = 0.0;
    for (int d = 0; d < 3; ++d) r2 += (cw[a][d] - cw[b][d]) * (cw[a][d] - cw[b][d]);
    rho[e] = r2;
  }
  const int cols[3][5] = {{0, 1, 3, 6, -1}, {0, 1, 2, -1, -1}, {0, 1, 2, 3, 4}};
  for (int cand = 0; cand < 3; ++cand) {
    const int m = cand == 0 ? 4 : (cand == 1 ? 3 : 5);
    double A[30], x[5], bt[4] = {0.0, 0.0, 0.0, 0.0};
    for (int e = 0; e < 6; ++e)
      for (int j = 0; j < m; ++j) A[e * m + j] = L[e][cols[cand][j]];
    ok[cand] = ls6(A, m, rho, x) ? 1 : 0;
    if (!ok[cand]) continue;
    if (cand == 0) {
      const double s = x[0] < 0.0 ? -1.0 : 1.0;
      bt[0] = sqrt(s * x[0]);
      for (int k = 1; k < 4; ++k) bt[k] = s * x[k] / bt[0];
    } else {
      if (x[0] < 0.0) { bt[0] = sqrt(-x[0]); bt[1] = x[2] < 0.0 ? sqrt(-x[2]) : 0.0; }
      else { bt[0] = sqrt(x[0]); bt[1] = x[2] > 0.0 ? sqrt(x[2]) : 0.0; }
      if (x[1] < 0.0) bt[0] = -bt[0];
      if (cand == 2) bt[2] = x[3] / bt[0];
    }
    for (int it = 0; it < 5; ++it) {
      const double b0 = bt[0], b1 = bt[1], b2 = bt[2], b3 = bt[3];
      const double B[10] = {b0 * b0, b0 * b1, b1 * b1, b0 * b2, b1 * b2, b2 * b2, b0 * b3, b1 * b3, b2 * b3, b3 * b3};
      const double dB[4][10] = {{2 * b0, b1, 0, b2, 0, 0, b3, 0, 0, 0},
                                {0, b0, 2 * b1, 0, b2, 0, 0, b3, 0, 0},
                                {0, 0, 0, b0, b1, 2 * b2, 0, 0, b3, 0},
                                {0, 0, 0, 0, 0, 0, b0, b1, b2, 2 * b3}};
      double J[24], r[6], dx[4];
      for (int e = 0; e < 6; ++e) {
        double lb = 0.0;
        for (int q = 0; q < 10; ++q) lb += L[e][q] * B[q];
        r[e] = rho[e] - lb;
        for (int k = 0; k < 4; ++k) {
          double g = 0.0;
          for (int q = 0; q < 10; ++q) g += L[e][q] * dB[k][q];
          J[e * 4 + k] = g;
        }
      }
      if (!ls6(J, 4, r, dx)) break;
      for (int k = 0; k < 4; ++k) bt[k] += dx[k];
    }
    for (int k = 0; k < 4; ++k) betas[cand][k] = bt[k];
  }
}

// ---- warp-parallel pieces ----

// Eigen-decomposition of the symmetric 12x12 w->A (eigenvalues end on its diagonal, w->V = eigenvectors in columns)
// by cyclic Jacobi with the round-robin parallel ordering: 11 steps of 6 disjoint rotations per sweep, each step
// applied as one A <- J^T A J, V <- V J by all lanes.  Stops when off(A)^2 <= 1e-32 |A|_F^2, after a sweep without
// rotation, or after 30 sweeps.
__device__ void warp_jacobi12(Scratch* w) {
  const int lane = threadIdx.x & 31;
  double fro = 0.0;
  for (int e = lane; e < 144; e += 32) {
    w->V[e] = (e / 12 == e % 12) ? 1.0 : 0.0;
    fro += w->A[e] * w->A[e];
  }
  {
    double t[1] = {fro};
    warp_sum(t);
    fro = t[0];
  }
  __syncwarp();
  for (int sweep = 0; sweep < 30; ++sweep) {
    double off = 0.0;
    for (int e = lane; e < 144; e += 32)
      if (e / 12 != e % 12) off += w->A[e] * w->A[e];
    double t[1] = {off};
    warp_sum(t);
    if (t[0] <= 1e-32 * fro) break;
    bool any_rot = false;
    for (int step = 0; step < 11; ++step) {
      int p = 0, q = 0;
      bool rot = false;
      if (lane < 6) {
        p = lane == 0 ? 0 : ((lane - 1 + step) % 11) + 1;
        q = ((10 - lane + step) % 11) + 1;
        if (p > q) { const int x = p; p = q; q = x; }
        const double apq = w->A[p * 12 + q], app = w->A[p * 13], aqq = w->A[q * 13];
        double c = 1.0, s = 0.0;
        if (!(apq == 0.0 || fabs(apq) <= 1e-17 * sqrt(fabs(app) * fabs(aqq)))) {
          const double theta = (aqq - app) / (2.0 * apq);
          const double tt = fabs(theta) > 1e150 ? 0.5 / theta
                                                : (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
          c = 1.0 / sqrt(tt * tt + 1.0);
          s = tt * c;
          rot = true;
        }
        w->partner[p] = q; w->partner[q] = p;
        w->cs[p] = c; w->cp[p] = -s;
        w->cs[q] = c; w->cp[q] = s;
      }
      const bool step_rot = __any_sync(0xffffffffu, rot);
      __syncwarp();
      if (!step_rot) continue;
      any_rot = true;
      double na[5], nv[5];
#pragma unroll
      for (int m = 0; m < 5; ++m) {
        const int e = lane + 32 * m;
        if (e < 144) {
          const int i = e / 12, j = e % 12, pi = w->partner[i], pj = w->partner[j];
          const double ci = w->cs[i], si = w->cp[i], cj = w->cs[j], sj = w->cp[j];
          na[m] = ci * cj * w->A[i * 12 + j] + ci * sj * w->A[i * 12 + pj] + si * cj * w->A[pi * 12 + j] +
                  si * sj * w->A[pi * 12 + pj];
          nv[m] = cj * w->V[i * 12 + j] + sj * w->V[i * 12 + pj];
        }
      }
      __syncwarp();
#pragma unroll
      for (int m = 0; m < 5; ++m) {
        const int e = lane + 32 * m;
        if (e < 144) { w->A[e] = na[m]; w->V[e] = nv[m]; }
      }
      __syncwarp();
      if (rot) { w->A[p * 12 + q] = 0.0; w->A[q * 12 + p] = 0.0; }
      __syncwarp();
    }
    if (!any_rot) break;
  }
}

// EPnP (Lepetit, Moreno-Noguer, Fua, IJCV 2009) on the correspondences P, run by one full warp.  out = R row-major |
// t.  Returns false (on every lane) for a degenerate set.
template <typename T>
__device__ bool warp_epnp(const Pts<T>& P, const Cam& c, Scratch* w, double out[12]) {
  const int lane = threadIdx.x & 31;
  const int n = P.n;
  if (n < 4) return false;
  // control points: centroid + scaled principal axes
  double c0[3] = {0.0, 0.0, 0.0};
  for (int k = lane; k < n; k += 32) {
    const int i = P.at(k);
    c0[0] += (double)P.X[i * P.sx]; c0[1] += (double)P.Y[i * P.sx]; c0[2] += (double)P.Z[i * P.sx];
  }
  warp_sum(c0);
  for (int d = 0; d < 3; ++d) c0[d] /= n;
  double cov[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int k = lane; k < n; k += 32) {
    const int i = P.at(k);
    const double dx = (double)P.X[i * P.sx] - c0[0], dy = (double)P.Y[i * P.sx] - c0[1],
                 dz = (double)P.Z[i * P.sx] - c0[2];
    cov[0] += dx * dx; cov[1] += dx * dy; cov[2] += dx * dz; cov[3] += dy * dy; cov[4] += dy * dz; cov[5] += dz * dz;
  }
  warp_sum(cov);
  const double C[9] = {cov[0], cov[1], cov[2], cov[1], cov[3], cov[4], cov[2], cov[4], cov[5]};
  double lam[3], E[9], sc[3];
  sym3_eig_desc(C, lam, E);
  // A coplanar or collinear set has lam[2] = 0, so the computed lam[2] is rounding noise and the fourth control point
  // has an arbitrary depth: EPnP then returns wrong poses as valid.  Each entry of C is a sum of
  // m + 5 additions (m = ceil(n / 32) terms per lane, then the 5-level butterfly) of terms dx dy carrying 3 roundings,
  // so |dC_ij| <= gamma_{m+8} sum |dx_i dx_j| and ||dC||_2 <= 9 gamma_{m+8} lam[0]; the Jacobi eigenvalues of C add
  // at most 52 u lam[0] (30 u ||C||_F, ||C||_F <= sqrt(3) lam[0]).  By Weyl's inequality a computed lam[2] at or
  // below that sum cannot be told from 0, and the set is rejected (DESIGN.md 4.8).  u = 2^-53.  lam[0] >= 1e75 (a
  // spread above about 1e37) is rejected too: the Jacobi sweeps on C and on kabsch()'s H^T H (of the order of C^2)
  // sum the squares of their entries, which would overflow and end the sweeps before the first rotation.
  const double tol = (9.0 * (double)((n + 31) / 32 + 8) + 52.0) * 0x1p-53;
  if (!(lam[2] > tol * lam[0]) || !(lam[0] < 1e75)) return false;
  for (int k = 0; k < 3; ++k) {
    sc[k] = sqrt(lam[k] / n);
    if (!(sc[k] > 0.0) || !isfinite(sc[k])) return false;
  }
  double cw[4][3];
  for (int d = 0; d < 3; ++d) cw[0][d] = c0[d];
  for (int k = 0; k < 3; ++k)
    for (int d = 0; d < 3; ++d) cw[k + 1][d] = c0[d] + sc[k] * E[d * 3 + k];
  auto alphas = [&](int i, double a[4]) {
    const double dx = (double)P.X[i * P.sx] - c0[0], dy = (double)P.Y[i * P.sx] - c0[1],
                 dz = (double)P.Z[i * P.sx] - c0[2];
    for (int k = 0; k < 3; ++k) a[k + 1] = (E[k] * dx + E[3 + k] * dy + E[6 + k] * dz) / sc[k];
    a[0] = 1.0 - a[1] - a[2] - a[3];
  };
  // M^T M = sum_i (a a^T) (x) [[fu^2, 0, fu du], [0, fv^2, fv dv], [fu du, fv dv, du^2 + dv^2]], du = cu - u
  double acc[40];
#pragma unroll
  for (int k = 0; k < 40; ++k) acc[k] = 0.0;
  for (int k = lane; k < n; k += 32) {
    const int i = P.at(k);
    double a[4];
    alphas(i, a);
    const double du = c.cu - P.U[i * P.su], dv = c.cv - P.V[i * P.su], dd = du * du + dv * dv;
    int p = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int l = j; l < 4; ++l, ++p) {
        const double aa = a[j] * a[l];
        acc[4 * p] += aa; acc[4 * p + 1] += aa * du; acc[4 * p + 2] += aa * dv; acc[4 * p + 3] += aa * dd;
      }
  }
  warp_sum(acc);
  {
    const int off4[4] = {0, 4, 7, 9};
#pragma unroll
    for (int m = 0; m < 5; ++m) {
      const int e = lane + 32 * m;
      if (e < 144) {
        const int row = e / 12, col = e % 12, j = row / 3, l = col / 3, r = row % 3, q = col % 3;
        const int p = j <= l ? off4[j] + l - j : off4[l] + j - l;
        const double* s = acc + 4 * p;
        double val;
        if (r == 2 && q == 2) val = s[3];
        else if (r == q) val = (r == 0 ? c.fu * c.fu : c.fv * c.fv) * s[0];
        else if (r == 2 || q == 2) val = (r == 0 || q == 0) ? c.fu * s[1] : c.fv * s[2];
        else val = 0.0;
        w->A[e] = val;
      }
    }
  }
  __syncwarp();
  warp_jacobi12(w);
  if (lane == 0) {
    int o[12];
    for (int i = 0; i < 12; ++i) o[i] = i;
    for (int i = 0; i < 4; ++i)
      for (int j = i + 1; j < 12; ++j)
        if (w->A[o[j] * 13] < w->A[o[i] * 13]) { const int t = o[i]; o[i] = o[j]; o[j] = t; }
    double v[4][12];
    for (int k = 0; k < 4; ++k)
      for (int r = 0; r < 12; ++r) v[k][r] = w->V[r * 12 + o[k]];
    epnp_betas(v, cw, w->betas, w->bvalid);
    for (int k = 0; k < 4; ++k) w->order[k] = o[k];
  }
  __syncwarp();
  double best_err = INFINITY;
  bool found = false;
  for (int cand = 0; cand < 3; ++cand) {
    if (!w->bvalid[cand]) continue;
    double cc[4][3];
    for (int j = 0; j < 4; ++j)
      for (int d = 0; d < 3; ++d) {
        double x = 0.0;
        for (int k = 0; k < 4; ++k) x += w->betas[cand][k] * w->V[(3 * j + d) * 12 + w->order[k]];
        cc[j][d] = x;
      }
    {
      double a[4];
      alphas(P.at(0), a);
      if (a[0] * cc[0][2] + a[1] * cc[1][2] + a[2] * cc[2][2] + a[3] * cc[3][2] < 0.0)
        for (int j = 0; j < 4; ++j)
          for (int d = 0; d < 3; ++d) cc[j][d] = -cc[j][d];
    }
    double pc0[3] = {0.0, 0.0, 0.0};
    for (int k = lane; k < n; k += 32) {
      double a[4];
      alphas(P.at(k), a);
      for (int d = 0; d < 3; ++d) pc0[d] += a[0] * cc[0][d] + a[1] * cc[1][d] + a[2] * cc[2][d] + a[3] * cc[3][d];
    }
    warp_sum(pc0);
    for (int d = 0; d < 3; ++d) pc0[d] /= n;
    double H[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int k = lane; k < n; k += 32) {
      const int i = P.at(k);
      double a[4], pc[3];
      alphas(i, a);
      for (int d = 0; d < 3; ++d) pc[d] = a[0] * cc[0][d] + a[1] * cc[1][d] + a[2] * cc[2][d] + a[3] * cc[3][d];
      const double dw[3] = {(double)P.X[i * P.sx] - c0[0], (double)P.Y[i * P.sx] - c0[1],
                            (double)P.Z[i * P.sx] - c0[2]};
      for (int r = 0; r < 3; ++r)
        for (int q = 0; q < 3; ++q) H[r * 3 + q] += (pc[r] - pc0[r]) * dw[q];
    }
    warp_sum(H);
    double R[9];
    if (!kabsch(H, R)) continue;
    double t[3];
    for (int d = 0; d < 3; ++d) t[d] = pc0[d] - (R[d * 3] * c0[0] + R[d * 3 + 1] * c0[1] + R[d * 3 + 2] * c0[2]);
    double err[1] = {0.0};
    for (int k = lane; k < n; k += 32) {
      const int i = P.at(k);
      const double X = P.X[i * P.sx], Y = P.Y[i * P.sx], Z = P.Z[i * P.sx];
      const double x = R[0] * X + R[1] * Y + R[2] * Z + t[0];
      const double y = R[3] * X + R[4] * Y + R[5] * Z + t[1];
      const double z = R[6] * X + R[7] * Y + R[8] * Z + t[2];
      const double eu = P.U[i * P.su] - (c.cu + c.fu * x / z), ev = P.V[i * P.su] - (c.cv + c.fv * y / z);
      err[0] += sqrt(eu * eu + ev * ev);
    }
    warp_sum(err);
    const double e = err[0] / n;
    if (e < best_err) {
      best_err = e;
      found = true;
      for (int k = 0; k < 9; ++k) out[k] = R[k];
      for (int k = 0; k < 3; ++k) out[9 + k] = t[k];
    }
  }
  if (!found) return false;
  for (int k = 0; k < 12; ++k)
    if (!isfinite(out[k])) return false;
  return true;
}

// ---- kernels ----

struct Work {
  float *X, *Y, *Z;
  double *U, *V;
  int32_t *orig, *list, *state;
  double* hyp_pose;       // [S][iterations][12]
  int32_t* hyp_cnt;       // [S][iterations]: -1 invalid (before scoring), else inliers
};

__global__ void __launch_bounds__(kSelThreads) select_kernel(const float* __restrict__ xyz,
                                                             const int8_t* __restrict__ coarse,
                                                             const int32_t* __restrict__ fine,
                                                             const int32_t* __restrict__ n_pts, int n_stride,
                                                             double Wf, int iterations, Work wk) {
  __shared__ int warp_tot[kSelThreads / 32];
  __shared__ int base;
  const int s = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int n = n_pts ? min(max(n_pts[s], 0), n_stride) : n_stride;
  const size_t row = (size_t)s * n_stride;
  if (tid == 0) base = 0;
  __syncthreads();
  for (int t0 = 0; t0 < n; t0 += kSelThreads) {
    const int i = t0 + tid;
    const bool sel = i < n && coarse[row + i] == 1;
    const unsigned b = __ballot_sync(0xffffffffu, sel);
    if (lane == 0) warp_tot[wid] = __popc(b);
    __syncthreads();
    int off = base;
    for (int q = 0; q < wid; ++q) off += warp_tot[q];
    if (sel) {
      const int o = off + __popc(b & ((1u << lane) - 1u));
      const double f = (double)fine[row + i];
      const double py = floor(__ddiv_rn(f, Wf));
      wk.X[row + o] = xyz[(size_t)s * 3 * n_stride + i];
      wk.Y[row + o] = xyz[(size_t)s * 3 * n_stride + n_stride + i];
      wk.Z[row + o] = xyz[(size_t)s * 3 * n_stride + 2 * n_stride + i];
      wk.U[row + o] = __dsub_rn(f, __dmul_rn(py, Wf));
      wk.V[row + o] = py;
      wk.orig[row + o] = i;
    }
    __syncthreads();
    if (tid == 0)
      for (int q = 0; q < kSelThreads / 32; ++q) base += warp_tot[q];
    __syncthreads();
  }
  if (tid == 0) {
    int32_t* st = wk.state + s * ST_WORDS;
    st[ST_NSEL] = base;
    st[ST_NITERS] = iterations;
    st[ST_BEST] = -1;
    st[ST_BESTCNT] = 0;
    st[ST_USED] = 0;
    st[ST_STOPPED] = base < 6 ? 1 : 0;     // n <= 5 skips sampling
  }
}

__global__ void __launch_bounds__(kHypWarps * 32) hyp_kernel(const double* __restrict__ K9, double scale, int n_stride,
                                                             int iterations, int h0, uint64_t seed, Work wk) {
  __shared__ Scratch scr[kHypWarps];
  const int s = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = h0 + blockIdx.x * kHypWarps + warp;
  const int32_t* st = wk.state + s * ST_WORDS;
  if (st[ST_STOPPED] || h >= iterations || h >= st[ST_NITERS]) return;
  const int n = st[ST_NSEL];
  Scratch* w = &scr[warp];
  if (lane == 0) {
    int d = 0;
    for (int k = 0; k < 5; ++k) {
      for (;;) {
        uint32_t c[4] = {(uint32_t)h, (uint32_t)s, (uint32_t)d++, 0u};
        philox4x32_10(c, (uint32_t)(seed & 0xffffffffull), (uint32_t)(seed >> 32));
        const int idx = (int)(((uint64_t)c[0] * (uint64_t)n) >> 32);
        bool dup = false;
        for (int j = 0; j < k; ++j) dup |= w->idx[j] == idx;
        if (!dup) { w->idx[k] = idx; break; }
      }
    }
  }
  __syncwarp();
  const size_t row = (size_t)s * n_stride;
  Pts<float> P{wk.X + row, wk.Y + row, wk.Z + row, wk.U + row, wk.V + row, 1, 1, w->idx, 5};
  double pose[12];
  const bool ok = warp_epnp(P, scaled_cam(K9 + 9 * s, scale), w, pose);
  if (lane == 0) {
    double* o = wk.hyp_pose + ((size_t)s * iterations + h) * 12;
    for (int k = 0; k < 12; ++k) o[k] = ok ? pose[k] : 0.0;
    wk.hyp_cnt[(size_t)s * iterations + h] = ok ? 0 : -1;
  }
}

__global__ void __launch_bounds__(kScoreThreads) score_kernel(const double* __restrict__ K9, double scale, int n_stride,
                                                              int iterations, int h0, double thr2, Work wk) {
  __shared__ double pose[kBlockH][12];
  __shared__ int valid[kBlockH];
  __shared__ float tx[kScoreTile], ty[kScoreTile], tz[kScoreTile];
  __shared__ double tu[kScoreTile], tv[kScoreTile];
  const int s = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int32_t* st = wk.state + s * ST_WORDS;
  if (st[ST_STOPPED]) return;
  const int nh = min(min(h0 + kBlockH, iterations), st[ST_NITERS]) - h0;
  if (nh <= 0) return;
  const int n = st[ST_NSEL];
  const size_t row = (size_t)s * n_stride;
  for (int e = tid; e < nh * 12; e += kScoreThreads) pose[e / 12][e % 12] = wk.hyp_pose[((size_t)s * iterations + h0) * 12 + e];
  for (int e = tid; e < nh; e += kScoreThreads) valid[e] = wk.hyp_cnt[(size_t)s * iterations + h0 + e] >= 0;
  const Cam c = scaled_cam(K9 + 9 * s, scale);
  int cnt[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int b = 0; b < n; b += kScoreTile) {
    const int tn = min(kScoreTile, n - b);
    __syncthreads();
    for (int i = tid; i < tn; i += kScoreThreads) {
      tx[i] = wk.X[row + b + i]; ty[i] = wk.Y[row + b + i]; tz[i] = wk.Z[row + b + i];
      tu[i] = wk.U[row + b + i]; tv[i] = wk.V[row + b + i];
    }
    __syncthreads();
    for (int i = lane; i < ((tn + 31) & ~31); i += 32) {
      const bool pt = i < tn;
      const double X = pt ? tx[i] : 0.0, Y = pt ? ty[i] : 0.0, Z = pt ? tz[i] : 0.0;
      const double U = pt ? tu[i] : 0.0, V = pt ? tv[i] : 0.0;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int hk = warp * 8 + k;
        const bool in = pt && hk < nh && is_inlier(pose[hk], X, Y, Z, U, V, c, thr2);
        cnt[k] += __popc(__ballot_sync(0xffffffffu, in));
      }
    }
  }
  if (lane == 0)
    for (int k = 0; k < 8; ++k) {
      const int hk = warp * 8 + k;
      if (hk < nh) wk.hyp_cnt[(size_t)s * iterations + h0 + hk] = valid[hk] ? cnt[k] : 0;
    }
}

// niters after a new best with cnt inliers out of n: min(niters, ceil(log(1 - conf) / log(1 - w^5))), w = cnt / n;
// no bound while 1 - w^5 rounds to 1.
__device__ __forceinline__ int update_niters(int niters, int cnt, int n, double confidence) {
  const double w = (double)cnt / (double)n;
  const double den = log(1.0 - w * w * w * w * w);
  if (!(den < 0.0)) return niters;
  const double k = ceil(log(1.0 - confidence) / den);
  return k < (double)niters ? (int)k : niters;
}

__global__ void replay_kernel(int S, int iterations, int h0, double confidence, Work wk) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= S) return;
  int32_t* st = wk.state + s * ST_WORDS;
  if (st[ST_STOPPED]) return;
  const int n = st[ST_NSEL];
  int niters = st[ST_NITERS], best = st[ST_BEST], best_cnt = st[ST_BESTCNT];
  int h = h0;
  const int hend = min(h0 + kBlockH, iterations);
  for (; h < hend && h < niters; ++h) {
    const int cnt = wk.hyp_cnt[(size_t)s * iterations + h];
    if (cnt >= 5 && cnt > best_cnt) {
      best = h;
      best_cnt = cnt;
      niters = update_niters(niters, cnt, n, confidence);
    }
  }
  st[ST_NITERS] = niters;
  st[ST_BEST] = best;
  st[ST_BESTCNT] = best_cnt;
  st[ST_USED] = h;
  if (h >= niters || h >= iterations) st[ST_STOPPED] = 1;
}

struct Out {
  double *P16, *ratio;
  int32_t *inliers, *n_sel, *hyp_used;
  uint8_t* mask;
};

__global__ void __launch_bounds__(32) refit_kernel(const double* __restrict__ K9, double scale, int n_stride,
                                                   int iterations, double thr2, Work wk, Out out) {
  __shared__ Scratch scr;
  const int s = blockIdx.x, lane = threadIdx.x;
  const int32_t* st = wk.state + s * ST_WORDS;
  const int n = st[ST_NSEL];
  const size_t row = (size_t)s * n_stride;
  const Cam c = scaled_cam(K9 + 9 * s, scale);
  int32_t* list = wk.list + row;
  if (out.mask)
    for (int i = lane; i < n_stride; i += 32) out.mask[row + i] = 0;
  double pose[12];
  bool ok = false;
  int cnt = 0;
  // inliers of `p` -> list (ascending), count
  auto collect = [&](const double* p) {
    int m = 0;
    for (int b = 0; b < n; b += 32) {
      const int i = b + lane;
      const bool in = i < n && is_inlier(p, wk.X[row + i], wk.Y[row + i], wk.Z[row + i], wk.U[row + i],
                                         wk.V[row + i], c, thr2);
      const unsigned bal = __ballot_sync(0xffffffffu, in);
      if (in) list[m + __popc(bal & ((1u << lane) - 1u))] = i;
      m += __popc(bal);
    }
    __syncwarp();
    return m;
  };
  if (n >= 4 && n <= 5) {
    Pts<float> P{wk.X + row, wk.Y + row, wk.Z + row, wk.U + row, wk.V + row, 1, 1, nullptr, n};
    ok = warp_epnp(P, c, &scr, pose);
    if (ok) cnt = collect(pose);
  } else if (n >= 6 && st[ST_BEST] >= 0) {
    double hp[12];
    for (int k = 0; k < 12; ++k) hp[k] = wk.hyp_pose[((size_t)s * iterations + st[ST_BEST]) * 12 + k];
    cnt = collect(hp);
    Pts<float> P{wk.X + row, wk.Y + row, wk.Z + row, wk.U + row, wk.V + row, 1, 1, list, cnt};
    ok = warp_epnp(P, c, &scr, pose);
  }
  const bool good = ok && sqrt(pose[9] * pose[9] + pose[10] * pose[10] + pose[11] * pose[11]) < 14.14;
  if (ok && out.mask) {
    __syncwarp();
    for (int k = lane; k < cnt; k += 32) out.mask[row + wk.orig[row + list[k]]] = 1;
  }
  if (lane < 16) {
    const int r = lane >> 2, q = lane & 3;
    double v = r == q ? 1.0 : 0.0;
    if (good && r < 3) v = q < 3 ? pose[r * 3 + q] : pose[9 + r];
    out.P16[(size_t)s * 16 + lane] = v;
  }
  if (lane == 0) {
    out.ratio[s] = good ? 1.0 - (double)cnt / (double)n : 1.0;
    out.inliers[s] = ok ? cnt : 0;
    if (out.n_sel) out.n_sel[s] = n;
    if (out.hyp_used) out.hyp_used[s] = st[ST_USED];
  }
}

__global__ void __launch_bounds__(32) epnp_kernel(const double* __restrict__ xyz, const double* __restrict__ uv,
                                                  const int32_t* __restrict__ offsets, const double* __restrict__ K9,
                                                  double* __restrict__ out12, int32_t* __restrict__ ok_out) {
  __shared__ Scratch scr;
  const int b = blockIdx.x;
  const int o = offsets[b], n = offsets[b + 1] - o;
  Pts<double> P{xyz + 3 * (size_t)o, xyz + 3 * (size_t)o + 1, xyz + 3 * (size_t)o + 2, uv + 2 * (size_t)o,
                uv + 2 * (size_t)o + 1, 3, 2, nullptr, n};
  const Cam c{K9[9 * b], K9[9 * b + 4], K9[9 * b + 2], K9[9 * b + 5]};
  double pose[12];
  const bool ok = warp_epnp(P, c, &scr, pose);
  if (threadIdx.x < 12) out12[(size_t)b * 12 + threadIdx.x] = ok ? pose[threadIdx.x] : 0.0;
  if (threadIdx.x == 0) ok_out[b] = ok ? 1 : 0;
}

inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

// Workspace carve-up; returns the bytes needed (base may be NULL).
size_t carve(char* base, int S, int n_stride, int iterations, Work* wk) {
  const size_t np = (size_t)S * n_stride;
  size_t off = 0;
  auto take = [&](size_t bytes) { char* p = base ? base + off : nullptr; off += align256(bytes); return p; };
  Work w;
  w.X = (float*)take(np * 4); w.Y = (float*)take(np * 4); w.Z = (float*)take(np * 4);
  w.U = (double*)take(np * 8); w.V = (double*)take(np * 8);
  w.orig = (int32_t*)take(np * 4); w.list = (int32_t*)take(np * 4);
  w.state = (int32_t*)take((size_t)S * ST_WORDS * 4);
  w.hyp_pose = (double*)take((size_t)S * iterations * 12 * 8);
  w.hyp_cnt = (int32_t*)take((size_t)S * iterations * 4);
  if (wk) *wk = w;
  return off;
}

}  // namespace pnp
}  // namespace dib

extern "C" {

size_t pnp_ransac_workspace_bytes(int S, int n_stride, int iterations) {
  if (S < 0 || n_stride < 0 || iterations < 1) return 0;
  return dib::pnp::carve(nullptr, S, n_stride, iterations, nullptr);
}

int pnp_ransac_batch_f32(const float* xyz, const int8_t* coarse_pred, const int32_t* fine_pred, const int32_t* n_pts,
                         int n_stride, int S, const double* K9, double H, double W, double scale, int iterations,
                         double reproj_err, double confidence, uint64_t seed, double* P16_out,
                         double* outlier_ratio_out, int32_t* inliers_out, int32_t* n_sel_out, int32_t* hyp_used_out,
                         uint8_t* inlier_mask_out, double* hyp_pose_out, int32_t* hyp_inliers_out, void* workspace,
                         size_t workspace_bytes, dib_stream_t stream) {
  using namespace dib;
  using namespace dib::pnp;
  (void)H;
  DIB_REQUIRE(xyz && coarse_pred && fine_pred && K9 && P16_out && outlier_ratio_out && inliers_out, "NULL argument");
  DIB_REQUIRE(S >= 0 && S <= 65535 && n_stride >= 1, "bad sizes (S=%d must be in [0, 65535], n_stride=%d)", S,
              n_stride);      // the hypothesis kernel puts frames on grid y
  DIB_REQUIRE(iterations >= 1, "iterations must be >= 1 (got %d)", iterations);
  DIB_REQUIRE(std::isfinite(W) && std::isfinite(scale) && W > 0.0 && scale > 0.0 && W * scale > 0.0,
              "W and scale must be positive");
  DIB_REQUIRE(std::isfinite(reproj_err) && reproj_err > 0.0, "reproj_err must be positive");
  DIB_REQUIRE(confidence > 0.0 && confidence < 1.0, "confidence must be in (0, 1)");
  const size_t need = carve(nullptr, S, n_stride, iterations, nullptr);
  DIB_REQUIRE(workspace && workspace_bytes >= need, "workspace too small (%zu < %zu)", workspace_bytes, need);
  DIB_REQUIRE(((uintptr_t)workspace & 255) == 0, "workspace must be 256-byte aligned");
  if (S == 0) return DIB_OK;
  Work wk;
  carve((char*)workspace, S, n_stride, iterations, &wk);
  if (hyp_pose_out) wk.hyp_pose = hyp_pose_out;
  if (hyp_inliers_out) wk.hyp_cnt = hyp_inliers_out;
  cudaStream_t st = (cudaStream_t)stream;
  const double thr2 = reproj_err * reproj_err;
  select_kernel<<<S, kSelThreads, 0, st>>>(xyz, coarse_pred, fine_pred, n_pts, n_stride, W * scale, iterations, wk);
  DIB_CHECK_CUDA(cudaGetLastError());
  for (int h0 = 0; h0 < iterations; h0 += kBlockH) {
    hyp_kernel<<<dim3(kBlockH / kHypWarps, S), kHypWarps * 32, 0, st>>>(K9, scale, n_stride, iterations, h0, seed, wk);
    score_kernel<<<S, kScoreThreads, 0, st>>>(K9, scale, n_stride, iterations, h0, thr2, wk);
    replay_kernel<<<(S + 127) / 128, 128, 0, st>>>(S, iterations, h0, confidence, wk);
  }
  DIB_CHECK_CUDA(cudaGetLastError());
  Out out{P16_out, outlier_ratio_out, inliers_out, n_sel_out, hyp_used_out, inlier_mask_out};
  refit_kernel<<<S, 32, 0, st>>>(K9, scale, n_stride, iterations, thr2, wk, out);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

int epnp_batch_f64(const double* xyz, const double* uv, const int32_t* offsets, int B, const double* K9,
                   double* pose12_out, int32_t* ok_out, dib_stream_t stream) {
  using namespace dib;
  DIB_REQUIRE(xyz && uv && offsets && K9 && pose12_out && ok_out, "NULL argument");
  DIB_REQUIRE(B >= 0, "bad sizes (B=%d)", B);
  if (B == 0) return DIB_OK;
  pnp::epnp_kernel<<<B, 32, 0, (cudaStream_t)stream>>>(xyz, uv, offsets, K9, pose12_out, ok_out);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

}  // extern "C"
