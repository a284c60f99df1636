// CPU oracle of the PnP-RANSAC registration path (deepi2p_b200/csrc/pnp_ransac.cu) -- TEST INFRASTRUCTURE ONLY.
//
// A serial restatement of the whole contract of evaluation/registration_pnp.py:95-148 as DESIGN.md "PnP-RANSAC"
// states it: selection of the predicted-inside points, fine cell -> pixel decoding, Philox4x32-10 minimal samples,
// EPnP (Lepetit, Moreno-Noguer, Fua, IJCV 2009), the inlier rule, the sequential adaptive stopping rule, the refit on
// the winner's inliers and the reference's final rules.  Compiled with -ffp-contract=off so the inlier test rounds
// exactly as the kernel's, and it restates the kernel's arithmetic order too: every sum over points is accumulated in
// the warp's order (WarpSum) and the 12x12 eigenproblem uses the kernel's parallel Jacobi ordering.  The kernel is
// compiled without FMA contraction, so the two agree bit for bit as long as the math libraries do (sqrt and division
// are correctly rounded on both sides; only the stopping rule's log can differ by an ulp).
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

namespace {

void philox4x32_10(uint32_t c[4], uint32_t k0, uint32_t k1) {
  for (int r = 0; r < 10; ++r) {
    const uint64_t p0 = (uint64_t)0xD2511F53u * c[0], p1 = (uint64_t)0xCD9E8D57u * c[2];
    const uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0, hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
    const uint32_t n0 = hi1 ^ c[1] ^ k0, n2 = hi0 ^ c[3] ^ k1;
    c[0] = n0; c[1] = lo1; c[2] = n2; c[3] = lo0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
}

struct Cam { double fu, fv, cu, cv; };

struct Frame {          // the selected correspondences of one frame
  std::vector<double> X, Y, Z, U, V;
  std::vector<int> orig;
};

// Cyclic Jacobi on a symmetric n x n matrix (row-major, destroyed: eigenvalues end on the diagonal), V = eigenvectors
// in columns.  Stops when off(A)^2 <= 1e-32 * |A|_F^2, after a sweep without rotation, or after 30 sweeps.
void jacobi(double* A, double* V, int n) {
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
        double t;
        if (std::fabs(theta) > 1e150) t = 0.5 / theta;
        else t = (theta >= 0.0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
        const double c = 1.0 / std::sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < n; ++k) {   // rows p, q
          const double x = A[p * n + k], y = A[q * n + k];
          A[p * n + k] = c * x - s * y;
          A[q * n + k] = s * x + c * y;
        }
        for (int k = 0; k < n; ++k) {   // columns p, q
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

// The kernel's reduction order: point k goes to lane k % 32 (lanes sum in point order), then an xor butterfly
// (offsets 16, 8, 4, 2, 1) combines the 32 partial sums.
template <int N>
struct WarpSum {
  double part[32][N];
  WarpSum() { std::memset(part, 0, sizeof(part)); }
  double* lane(int k) { return part[k & 31]; }
  void reduce(double* out) {
    for (int o = 16; o > 0; o >>= 1) {
      double nxt[32][N];
      for (int i = 0; i < 32; ++i)
        for (int j = 0; j < N; ++j) nxt[i][j] = part[i][j] + part[i ^ o][j];
      std::memcpy(part, nxt, sizeof(part));
    }
    for (int j = 0; j < N; ++j) out[j] = part[0][j];
  }
};

// Jacobi on the symmetric 12x12 A with the kernel's round-robin parallel ordering: 11 steps of 6 disjoint rotations
// per sweep, each step applied at once as A <- J^T A J, V <- V J.  Same stopping rule as jacobi().
void jacobi12_parallel(double* A, double* V) {
  for (int i = 0; i < 144; ++i) V[i] = (i / 12 == i % 12) ? 1.0 : 0.0;
  double fro;
  {
    WarpSum<1> w;
    for (int e = 0; e < 144; ++e) w.lane(e)[0] += A[e] * A[e];
    w.reduce(&fro);
  }
  for (int sweep = 0; sweep < 30; ++sweep) {
    double off;
    {
      WarpSum<1> w;
      for (int e = 0; e < 144; ++e)
        if (e / 12 != e % 12) w.lane(e)[0] += A[e] * A[e];
      w.reduce(&off);
    }
    if (off <= 1e-32 * fro) break;
    bool any_rot = false;
    for (int step = 0; step < 11; ++step) {
      double cs[12], cp[12];
      int partner[12], pp[6], qq[6];
      bool rot[6], step_rot = false;
      for (int l = 0; l < 6; ++l) {
        int p = l == 0 ? 0 : ((l - 1 + step) % 11) + 1;
        int q = ((10 - l + step) % 11) + 1;
        if (p > q) { const int x = p; p = q; q = x; }
        const double apq = A[p * 12 + q], app = A[p * 13], aqq = A[q * 13];
        double c = 1.0, s = 0.0;
        rot[l] = false;
        if (!(apq == 0.0 || std::fabs(apq) <= 1e-17 * std::sqrt(std::fabs(app) * std::fabs(aqq)))) {
          const double theta = (aqq - app) / (2.0 * apq);
          const double tt = std::fabs(theta) > 1e150
                                ? 0.5 / theta
                                : (theta >= 0.0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
          c = 1.0 / std::sqrt(tt * tt + 1.0);
          s = tt * c;
          rot[l] = true;
        }
        step_rot |= rot[l];
        pp[l] = p; qq[l] = q;
        partner[p] = q; partner[q] = p;
        cs[p] = c; cp[p] = -s;
        cs[q] = c; cp[q] = s;
      }
      if (!step_rot) continue;
      any_rot = true;
      double na[144], nv[144];
      for (int e = 0; e < 144; ++e) {
        const int i = e / 12, j = e % 12, pi = partner[i], pj = partner[j];
        const double ci = cs[i], si = cp[i], cj = cs[j], sj = cp[j];
        na[e] = ci * cj * A[i * 12 + j] + ci * sj * A[i * 12 + pj] + si * cj * A[pi * 12 + j] + si * sj * A[pi * 12 + pj];
        nv[e] = cj * V[i * 12 + j] + sj * V[i * 12 + pj];
      }
      std::memcpy(A, na, sizeof(na));
      std::memcpy(V, nv, sizeof(nv));
      for (int l = 0; l < 6; ++l)
        if (rot[l]) { A[pp[l] * 12 + qq[l]] = 0.0; A[qq[l] * 12 + pp[l]] = 0.0; }
    }
    if (!any_rot) break;
  }
}

// min |A x - b| for A [6][m] (row-major, m <= 5) by Householder QR.  Returns false on a zero pivot.
bool ls6(const double* Ain, int m, const double* bin, double* x) {
  double A[6][5], b[6];
  for (int i = 0; i < 6; ++i) {
    b[i] = bin[i];
    for (int j = 0; j < m; ++j) A[i][j] = Ain[i * m + j];
  }
  for (int k = 0; k < m; ++k) {
    double nrm = 0.0;
    for (int i = k; i < 6; ++i) nrm += A[i][k] * A[i][k];
    nrm = std::sqrt(nrm);
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

void sym3_eig_desc(const double C[9], double lam[3], double E[9]) {   // E columns = eigenvectors, descending
  double A[9], V[9];
  std::memcpy(A, C, sizeof(A));
  jacobi(A, V, 3);
  int o[3] = {0, 1, 2};
  for (int i = 0; i < 3; ++i)
    for (int j = i + 1; j < 3; ++j)
      if (A[o[j] * 4] > A[o[i] * 4]) { int t = o[i]; o[i] = o[j]; o[j] = t; }
  for (int k = 0; k < 3; ++k) {
    lam[k] = A[o[k] * 4];
    for (int r = 0; r < 3; ++r) E[r * 3 + k] = V[r * 3 + o[k]];
  }
}

// R = U V^T from H = sum (pc - pc0)(pw - pw0)^T (proper rotation).  False when H has rank < 2.
bool kabsch(const double H[9], double R[9]) {
  double HtH[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) HtH[i * 3 + j] = H[0 * 3 + i] * H[0 * 3 + j] + H[1 * 3 + i] * H[1 * 3 + j] + H[2 * 3 + i] * H[2 * 3 + j];
  double lam[3], Vm[9];
  sym3_eig_desc(HtH, lam, Vm);
  const double det = Vm[0] * (Vm[4] * Vm[8] - Vm[5] * Vm[7]) - Vm[1] * (Vm[3] * Vm[8] - Vm[5] * Vm[6]) +
                     Vm[2] * (Vm[3] * Vm[7] - Vm[4] * Vm[6]);
  if (det < 0.0) for (int r = 0; r < 3; ++r) Vm[r * 3 + 2] = -Vm[r * 3 + 2];
  double u0[3], u1[3], u2[3];
  for (int r = 0; r < 3; ++r) {
    u0[r] = H[r * 3 + 0] * Vm[0] + H[r * 3 + 1] * Vm[3] + H[r * 3 + 2] * Vm[6];
    u1[r] = H[r * 3 + 0] * Vm[1] + H[r * 3 + 1] * Vm[4] + H[r * 3 + 2] * Vm[7];
  }
  const double n0 = std::sqrt(u0[0] * u0[0] + u0[1] * u0[1] + u0[2] * u0[2]);
  if (!(n0 > 0.0)) return false;
  for (int r = 0; r < 3; ++r) u0[r] /= n0;
  const double d = u0[0] * u1[0] + u0[1] * u1[1] + u0[2] * u1[2];
  for (int r = 0; r < 3; ++r) u1[r] -= d * u0[r];
  const double n1 = std::sqrt(u1[0] * u1[0] + u1[1] * u1[1] + u1[2] * u1[2]);
  if (!(n1 > 1e-12 * n0)) return false;
  for (int r = 0; r < 3; ++r) u1[r] /= n1;
  u2[0] = u0[1] * u1[2] - u0[2] * u1[1];
  u2[1] = u0[2] * u1[0] - u0[0] * u1[2];
  u2[2] = u0[0] * u1[1] - u0[1] * u1[0];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) R[i * 3 + j] = u0[i] * Vm[j * 3 + 0] + u1[i] * Vm[j * 3 + 1] + u2[i] * Vm[j * 3 + 2];
  return true;
}

const int kPairs[6][2] = {{0, 1}, {0, 2}, {0, 3}, {1, 2}, {1, 3}, {2, 3}};

// EPnP on the points idx[0..n) of f.  out = R (row-major 9) | t (3).  Returns false for a degenerate set.
bool epnp(const Frame& f, const int* idx, int n, const Cam& c, double out[12]) {
  if (n < 4) return false;
  double c0[3];
  {
    WarpSum<3> w;
    for (int k = 0; k < n; ++k) {
      const int i = idx[k];
      double* l = w.lane(k);
      l[0] += f.X[i]; l[1] += f.Y[i]; l[2] += f.Z[i];
    }
    w.reduce(c0);
  }
  for (int d = 0; d < 3; ++d) c0[d] /= n;
  double C[9];
  {
    WarpSum<6> w;
    for (int k = 0; k < n; ++k) {
      const int i = idx[k];
      const double dx = f.X[i] - c0[0], dy = f.Y[i] - c0[1], dz = f.Z[i] - c0[2];
      double* l = w.lane(k);
      l[0] += dx * dx; l[1] += dx * dy; l[2] += dx * dz; l[3] += dy * dy; l[4] += dy * dz; l[5] += dz * dz;
    }
    double cv[6];
    w.reduce(cv);
    const double full[9] = {cv[0], cv[1], cv[2], cv[1], cv[3], cv[4], cv[2], cv[4], cv[5]};
    std::memcpy(C, full, sizeof(C));
  }
  double lam[3], E[9];
  sym3_eig_desc(C, lam, E);
  // Coplanar (and collinear) sets: lam[2] within the rounding bound of lam[0] -> degenerate; a spread whose squares
  // would overflow the Jacobi sweeps -> rejected (DESIGN.md 4.8).
  const double tol = (9.0 * (double)((n + 31) / 32 + 8) + 52.0) * 0x1p-53;
  if (!(lam[2] > tol * lam[0]) || !(lam[0] < 1e75)) return false;
  double sc[3];
  for (int k = 0; k < 3; ++k) {
    sc[k] = std::sqrt(lam[k] / n);
    if (!(sc[k] > 0.0) || !std::isfinite(sc[k])) return false;
  }
  double cw[4][3];
  for (int d = 0; d < 3; ++d) cw[0][d] = c0[d];
  for (int k = 0; k < 3; ++k)
    for (int d = 0; d < 3; ++d) cw[k + 1][d] = c0[d] + sc[k] * E[d * 3 + k];
  auto alphas = [&](int i, double a[4]) {
    const double d[3] = {f.X[i] - c0[0], f.Y[i] - c0[1], f.Z[i] - c0[2]};
    for (int k = 0; k < 3; ++k) a[k + 1] = (E[0 * 3 + k] * d[0] + E[1 * 3 + k] * d[1] + E[2 * 3 + k] * d[2]) / sc[k];
    a[0] = 1.0 - a[1] - a[2] - a[3];
  };
  // M^T M = sum_i (a a^T) (x) B_i with B_i = [[fu^2,0,fu du],[0,fv^2,fv dv],[fu du,fv dv,du^2+dv^2]], du = cu - u.
  double acc[10][4];
  {
    WarpSum<40> w;
    for (int k = 0; k < n; ++k) {
      const int i = idx[k];
      double a[4];
      alphas(i, a);
      const double du = c.cu - f.U[i], dv = c.cv - f.V[i], dd = du * du + dv * dv;
      double* l4 = w.lane(k);
      int p = 0;
      for (int j = 0; j < 4; ++j)
        for (int l = j; l < 4; ++l, ++p) {
          const double aa = a[j] * a[l];
          l4[4 * p] += aa; l4[4 * p + 1] += aa * du; l4[4 * p + 2] += aa * dv; l4[4 * p + 3] += aa * dd;
        }
    }
    w.reduce(&acc[0][0]);
  }
  double MtM[144], Vv[144];
  {
    int p = 0;
    for (int j = 0; j < 4; ++j)
      for (int l = j; l < 4; ++l, ++p) {
        const double blk[9] = {c.fu * c.fu * acc[p][0], 0.0, c.fu * acc[p][1],
                               0.0, c.fv * c.fv * acc[p][0], c.fv * acc[p][2],
                               c.fu * acc[p][1], c.fv * acc[p][2], acc[p][3]};
        for (int r = 0; r < 3; ++r)
          for (int q = 0; q < 3; ++q) {
            MtM[(3 * j + r) * 12 + 3 * l + q] = blk[r * 3 + q];
            MtM[(3 * l + q) * 12 + 3 * j + r] = blk[r * 3 + q];
          }
      }
  }
  jacobi12_parallel(MtM, Vv);
  int o[12];
  for (int i = 0; i < 12; ++i) o[i] = i;
  for (int i = 0; i < 4; ++i)
    for (int j = i + 1; j < 12; ++j)
      if (MtM[o[j] * 13] < MtM[o[i] * 13]) { int t = o[i]; o[i] = o[j]; o[j] = t; }
  double v[4][12];
  for (int k = 0; k < 4; ++k)
    for (int r = 0; r < 12; ++r) v[k][r] = Vv[r * 12 + o[k]];
  double L[6][10], rho[6];
  for (int e = 0; e < 6; ++e) {
    const int a = kPairs[e][0], b = kPairs[e][1];
    double dv[4][3];
    for (int k = 0; k < 4; ++k)
      for (int d = 0; d < 3; ++d) dv[k][d] = v[k][3 * a + d] - v[k][3 * b + d];
    auto dot = [&](int x, int y) { return dv[x][0] * dv[y][0] + dv[x][1] * dv[y][1] + dv[x][2] * dv[y][2]; };
    L[e][0] = dot(0, 0); L[e][1] = 2 * dot(0, 1); L[e][2] = dot(1, 1); L[e][3] = 2 * dot(0, 2); L[e][4] = 2 * dot(1, 2);
    L[e][5] = dot(2, 2); L[e][6] = 2 * dot(0, 3); L[e][7] = 2 * dot(1, 3); L[e][8] = 2 * dot(2, 3); L[e][9] = dot(3, 3);
    double r2 = 0.0;
    for (int d = 0; d < 3; ++d) r2 += (cw[a][d] - cw[b][d]) * (cw[a][d] - cw[b][d]);
    rho[e] = r2;
  }
  double best_err = INFINITY;
  bool found = false;
  for (int cand = 0; cand < 3; ++cand) {
    static const int cols[3][5] = {{0, 1, 3, 6, -1}, {0, 1, 2, -1, -1}, {0, 1, 2, 3, 4}};
    const int m = cand == 0 ? 4 : (cand == 1 ? 3 : 5);
    double A[30], x[5], bt[4] = {0, 0, 0, 0};
    for (int e = 0; e < 6; ++e)
      for (int j = 0; j < m; ++j) A[e * m + j] = L[e][cols[cand][j]];
    if (!ls6(A, m, rho, x)) continue;
    if (cand == 0) {          // B11 B12 B13 B14
      const double s = x[0] < 0.0 ? -1.0 : 1.0;
      bt[0] = std::sqrt(s * x[0]);
      for (int k = 1; k < 4; ++k) bt[k] = s * x[k] / bt[0];
    } else {                  // B11 B12 B22 [B13 B23]
      if (x[0] < 0.0) { bt[0] = std::sqrt(-x[0]); bt[1] = x[2] < 0.0 ? std::sqrt(-x[2]) : 0.0; }
      else { bt[0] = std::sqrt(x[0]); bt[1] = x[2] > 0.0 ? std::sqrt(x[2]) : 0.0; }
      if (x[1] < 0.0) bt[0] = -bt[0];
      if (cand == 2) bt[2] = x[3] / bt[0];
    }
    for (int it = 0; it < 5; ++it) {   // Gauss-Newton on the 6 distance constraints, all four betas
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
    // camera-frame control points, sign, Procrustes, reprojection error
    double cc[4][3];
    for (int j = 0; j < 4; ++j)
      for (int d = 0; d < 3; ++d)
        {
          double x = 0.0;
          for (int k = 0; k < 4; ++k) x += bt[k] * v[k][3 * j + d];
          cc[j][d] = x;
        }
    {
      double a[4];
      alphas(idx[0], a);
      const double z0 = a[0] * cc[0][2] + a[1] * cc[1][2] + a[2] * cc[2][2] + a[3] * cc[3][2];
      if (z0 < 0.0)
        for (int j = 0; j < 4; ++j)
          for (int d = 0; d < 3; ++d) cc[j][d] = -cc[j][d];
    }
    auto pcam = [&](int i, double pc[3]) {
      double a[4];
      alphas(i, a);
      for (int d = 0; d < 3; ++d) pc[d] = a[0] * cc[0][d] + a[1] * cc[1][d] + a[2] * cc[2][d] + a[3] * cc[3][d];
    };
    double pc0[3];
    {
      WarpSum<3> w;
      for (int k = 0; k < n; ++k) {
        double pc[3];
        pcam(idx[k], pc);
        for (int d = 0; d < 3; ++d) w.lane(k)[d] += pc[d];
      }
      w.reduce(pc0);
    }
    for (int d = 0; d < 3; ++d) pc0[d] /= n;
    double H[9];
    {
      WarpSum<9> w;
      for (int k = 0; k < n; ++k) {
        const int i = idx[k];
        double pc[3];
        pcam(i, pc);
        const double dw[3] = {f.X[i] - c0[0], f.Y[i] - c0[1], f.Z[i] - c0[2]};
        for (int a = 0; a < 3; ++a)
          for (int b = 0; b < 3; ++b) w.lane(k)[a * 3 + b] += (pc[a] - pc0[a]) * dw[b];
      }
      w.reduce(H);
    }
    double R[9];
    if (!kabsch(H, R)) continue;
    double t[3];
    for (int d = 0; d < 3; ++d) t[d] = pc0[d] - (R[d * 3 + 0] * c0[0] + R[d * 3 + 1] * c0[1] + R[d * 3 + 2] * c0[2]);
    WarpSum<1> werr;
    for (int k = 0; k < n; ++k) {
      const int i = idx[k];
      const double x = R[0] * f.X[i] + R[1] * f.Y[i] + R[2] * f.Z[i] + t[0];
      const double y = R[3] * f.X[i] + R[4] * f.Y[i] + R[5] * f.Z[i] + t[1];
      const double z = R[6] * f.X[i] + R[7] * f.Y[i] + R[8] * f.Z[i] + t[2];
      const double eu = f.U[i] - (c.cu + c.fu * x / z), ev = f.V[i] - (c.cv + c.fv * y / z);
      werr.lane(k)[0] += std::sqrt(eu * eu + ev * ev);
    }
    double err;
    werr.reduce(&err);
    err /= n;
    if (err < best_err) {     // NaN never wins
      best_err = err;
      found = true;
      for (int k = 0; k < 9; ++k) out[k] = R[k];
      for (int k = 0; k < 3; ++k) out[9 + k] = t[k];
    }
  }
  if (!found) return false;
  for (int k = 0; k < 12; ++k)
    if (!std::isfinite(out[k])) return false;
  return true;
}

// The inlier rule, evaluation order fixed (this file is compiled with -ffp-contract=off).
inline bool is_inlier(const double* p, double X, double Y, double Z, double U, double V, const Cam& c, double thr2) {
  const double x = ((p[0] * X + p[1] * Y) + p[2] * Z) + p[9];
  const double y = ((p[3] * X + p[4] * Y) + p[5] * Z) + p[10];
  const double z = ((p[6] * X + p[7] * Y) + p[8] * Z) + p[11];
  const double du = (c.fu * (x / z) + c.cu) - U;
  const double dv = (c.fv * (y / z) + c.cv) - V;
  return du * du + dv * dv <= thr2;
}

int count_inliers(const Frame& f, const double* p, const Cam& c, double thr2, std::vector<int>* list) {
  int cnt = 0;
  for (size_t i = 0; i < f.X.size(); ++i)
    if (is_inlier(p, f.X[i], f.Y[i], f.Z[i], f.U[i], f.V[i], c, thr2)) {
      ++cnt;
      if (list) list->push_back((int)i);
    }
  return cnt;
}

}  // namespace

extern "C" {

// Sample draw of hypothesis h of frame s: 5 distinct indices in [0, n) (n >= 5).
void pnp_oracle_sample(int h, int s, int n, uint64_t seed, int32_t* out5) {
  int d = 0;
  for (int k = 0; k < 5; ++k) {
    for (;;) {
      uint32_t c[4] = {(uint32_t)h, (uint32_t)s, (uint32_t)d++, 0u};
      philox4x32_10(c, (uint32_t)(seed & 0xffffffffull), (uint32_t)(seed >> 32));
      const int idx = (int)(((uint64_t)c[0] * (uint64_t)n) >> 32);
      bool dup = false;
      for (int j = 0; j < k; ++j) dup |= out5[j] == idx;
      if (!dup) { out5[k] = idx; break; }
    }
  }
}

// niters after a new best with `cnt` inliers out of n.
int pnp_oracle_update_niters(int niters, int cnt, int n, double confidence) {
  const double w = (double)cnt / (double)n;
  const double den = std::log(1.0 - w * w * w * w * w);
  if (!(den < 0.0)) return niters;                      // 1 - w^5 rounds to 1: no bound
  const double k = std::ceil(std::log(1.0 - confidence) / den);
  return k < (double)niters ? (int)k : niters;
}

// sym3_eig_desc on n matrices C [n][9] -> lam [n][3], E [n][9] (the kernels' sym3_eig_batch_f64).
void pnp_oracle_sym3_eig(const double* C, int n, double* lam, double* E) {
  for (int t = 0; t < n; ++t) sym3_eig_desc(C + 9 * (size_t)t, lam + 3 * (size_t)t, E + 9 * (size_t)t);
}

// EPnP on n packed correspondences (xyz [n][3], uv [n][2], K9 unscaled row-major). Returns 1 on success.
int pnp_oracle_epnp(const double* xyz, const double* uv, int n, const double* K9, double* out12) {
  Frame f;
  std::vector<int> idx(n);
  for (int i = 0; i < n; ++i) {
    f.X.push_back(xyz[3 * i]); f.Y.push_back(xyz[3 * i + 1]); f.Z.push_back(xyz[3 * i + 2]);
    f.U.push_back(uv[2 * i]); f.V.push_back(uv[2 * i + 1]);
    idx[i] = i;
  }
  const Cam c{K9[0], K9[4], K9[2], K9[5]};
  return epnp(f, idx.data(), n, c, out12) ? 1 : 0;
}

// One frame of the whole contract.  xyz [3][n_pts] f32, coarse [n_pts] int8, fine [n_pts] int32, K9 row-major.
// Outputs: P16, outlier_ratio, inliers, n_sel, hyp_used, winner (-1 = none), mask [n_pts] (may be NULL),
// hyp_pose [iterations][12], hyp_inliers [iterations] (may be NULL; entries beyond hyp_used are untouched).
int pnp_oracle_frame(const float* xyz, const int8_t* coarse, const int32_t* fine, int n_pts, int s, const double* K9,
                     double H, double W, double scale, int iterations, double thr, double confidence, uint64_t seed,
                     double* P16, double* outlier_ratio, int32_t* inliers, int32_t* n_sel_out, int32_t* hyp_used_out,
                     int32_t* winner_out, uint8_t* mask, double* hyp_pose, int32_t* hyp_inliers) {
  (void)H;
  Frame f;
  const double Wf = W * scale;
  for (int i = 0; i < n_pts; ++i) {
    if (coarse[i] != 1) continue;
    const double fi = (double)fine[i];
    const double py = std::floor(fi / Wf);
    const double px = fi - py * Wf;
    f.X.push_back(xyz[i]); f.Y.push_back(xyz[n_pts + i]); f.Z.push_back(xyz[2 * n_pts + i]);
    f.U.push_back(px); f.V.push_back(py);
    f.orig.push_back(i);
  }
  const int n = (int)f.X.size();
  const Cam c{scale * K9[0], scale * K9[4], scale * K9[2], scale * K9[5]};
  const double thr2 = thr * thr;
  for (int k = 0; k < 16; ++k) P16[k] = (k % 5 == 0) ? 1.0 : 0.0;
  *outlier_ratio = 1.0;
  *inliers = 0;
  *n_sel_out = n;
  *hyp_used_out = 0;
  *winner_out = -1;
  if (mask) std::memset(mask, 0, (size_t)n_pts);
  if (n < 4) return 0;
  double pose[12];
  std::vector<int> list;
  bool ok;
  if (n <= 5) {
    std::vector<int> all(n);
    for (int i = 0; i < n; ++i) all[i] = i;
    ok = epnp(f, all.data(), n, c, pose);
    if (ok) count_inliers(f, pose, c, thr2, &list);
  } else {
    int niters = iterations, best = -1, best_cnt = 0, h = 0;
    std::vector<double> poses((size_t)iterations * 12);
    for (; h < niters; ++h) {
      int smp[5];
      pnp_oracle_sample(h, s, n, seed, smp);
      double* p = &poses[(size_t)h * 12];
      int cnt = 0;
      if (epnp(f, smp, 5, c, p)) cnt = count_inliers(f, p, c, thr2, nullptr);
      else for (int k = 0; k < 12; ++k) p[k] = 0.0;
      if (hyp_pose) std::memcpy(hyp_pose + (size_t)h * 12, p, sizeof(double) * 12);
      if (hyp_inliers) hyp_inliers[h] = cnt;
      if (cnt >= 5 && cnt > best_cnt) {
        best = h;
        best_cnt = cnt;
        niters = pnp_oracle_update_niters(niters, cnt, n, confidence);
      }
    }
    *hyp_used_out = h;
    *winner_out = best;
    if (best < 0) return 0;
    count_inliers(f, &poses[(size_t)best * 12], c, thr2, &list);
    ok = epnp(f, list.data(), (int)list.size(), c, pose);
  }
  if (!ok) return 0;
  *inliers = (int)list.size();
  if (mask)
    for (int i : list) mask[f.orig[i]] = 1;
  const double tn = std::sqrt(pose[9] * pose[9] + pose[10] * pose[10] + pose[11] * pose[11]);
  if (!(tn < 14.14)) return 0;
  for (int r = 0; r < 3; ++r) {
    for (int q = 0; q < 3; ++q) P16[r * 4 + q] = pose[r * 3 + q];
    P16[r * 4 + 3] = pose[9 + r];
  }
  *outlier_ratio = 1.0 - (double)*inliers / (double)n;
  return 0;
}

}  // extern "C"
