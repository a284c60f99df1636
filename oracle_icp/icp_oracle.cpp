// CPU oracle of the batched ICP path (deepi2p_b200/csrc/icp.cu) -- test infrastructure only.
//
// Restates the contract of DESIGN.md "ICP" serially: Open3D-style point-to-point ICP (registration_icp.py:115-162)
// with an exact nearest-neighbour search of its own (a median-split k-d tree with bounding boxes, unrelated to the
// kernels' Morton-order tree), and the kernels' summation order: the partial sums of 256 threads that take points
// t, t + 256, ... in order, an xor butterfly inside each warp of 32, then the 8 warp sums added in warp order.
// Compiled with -ffp-contract=off, as icp.cu is with --fmad=false, so both sides round every operation alike.
#include <algorithm>
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kSweeps = 8;
constexpr int kMoments = 16;
constexpr int kLeaf = 8;

inline double dot3(const double* a, const double* b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }

void kabsch(const double* A, double* R) {
  double B[3][3], V[3][3];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) { B[c][r] = A[r * 3 + c]; V[c][r] = r == c ? 1.0 : 0.0; }
  for (int sw = 0; sw < kSweeps; ++sw)
    for (int pr = 0; pr < 3; ++pr) {
      const int p = pr == 2 ? 1 : 0, q = pr == 0 ? 1 : 2;
      const double alpha = dot3(B[p], B[p]), beta = dot3(B[q], B[q]), gamma = dot3(B[p], B[q]);
      if (gamma == 0.0) continue;
      const double zeta = (beta - alpha) / (2.0 * gamma);
      const double t = (zeta >= 0.0 ? 1.0 : -1.0) / (std::fabs(zeta) + std::sqrt(1.0 + zeta * zeta));
      const double cs = 1.0 / std::sqrt(1.0 + t * t), sn = cs * t;
      for (int r = 0; r < 3; ++r) {
        const double bp = B[p][r], bq = B[q][r];
        B[p][r] = cs * bp - sn * bq;
        B[q][r] = sn * bp + cs * bq;
        const double vp = V[p][r], vq = V[q][r];
        V[p][r] = cs * vp - sn * vq;
        V[q][r] = sn * vp + cs * vq;
      }
    }
  double sg[3];
  for (int k = 0; k < 3; ++k) sg[k] = std::sqrt(dot3(B[k], B[k]));
  int o[3] = {0, 1, 2};
  if (sg[o[1]] > sg[o[0]]) std::swap(o[0], o[1]);
  if (sg[o[2]] > sg[o[1]]) std::swap(o[1], o[2]);
  if (sg[o[1]] > sg[o[0]]) std::swap(o[0], o[1]);
  double u1[3], u2[3], u3[3];
  if (sg[o[0]] > 0.0) {
    for (int r = 0; r < 3; ++r) u1[r] = B[o[0]][r] / sg[o[0]];
  } else {
    u1[0] = 1.0; u1[1] = 0.0; u1[2] = 0.0;
  }
  const double pj = dot3(u1, B[o[1]]);
  double w[3];
  for (int r = 0; r < 3; ++r) w[r] = B[o[1]][r] - pj * u1[r];
  double nw = std::sqrt(dot3(w, w));
  if (!(nw > 1e-14 * sg[o[0]]) || nw == 0.0) {
    int e = 0;
    for (int r = 1; r < 3; ++r)
      if (std::fabs(u1[r]) < std::fabs(u1[e])) e = r;
    for (int r = 0; r < 3; ++r) w[r] = (r == e ? 1.0 : 0.0) - u1[e] * u1[r];
    nw = std::sqrt(dot3(w, w));
  }
  for (int r = 0; r < 3; ++r) u2[r] = w[r] / nw;
  u3[0] = u1[1] * u2[2] - u1[2] * u2[1];
  u3[1] = u1[2] * u2[0] - u1[0] * u2[2];
  u3[2] = u1[0] * u2[1] - u1[1] * u2[0];
  const double* v1 = V[o[0]];
  const double* v2 = V[o[1]];
  const double* v3 = V[o[2]];
  const double c23[3] = {v2[1] * v3[2] - v2[2] * v3[1], v2[2] * v3[0] - v2[0] * v3[2], v2[0] * v3[1] - v2[1] * v3[0]};
  if (dot3(v1, c23) < 0.0)
    for (int r = 0; r < 3; ++r) u3[r] = -u3[r];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) R[r * 3 + c] = (u1[r] * v1[c] + u2[r] * v2[c]) + u3[r] * v3[c];
}

// U from the moments about c (nc correspondences); U = I when nc == 0.  Writes U [12] (3x4 row-major).
void umeyama_moments(const double* M, int nc, const double* c, double* U, double* mut) {
  for (int k = 0; k < 12; ++k) U[k] = (k % 5) == 0 ? 1.0 : 0.0;
  if (nc <= 0) {
    for (int a = 0; a < 3; ++a) mut[a] = c[a];
    return;
  }
  const double n = (double)nc;
  double mq[3], mt[3], A[9], R[9], muq[3];
  for (int a = 0; a < 3; ++a) { mq[a] = M[1 + a] / n; mt[a] = M[4 + a] / n; }
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) A[a * 3 + b] = M[7 + a * 3 + b] / n - mt[a] * mq[b];
  kabsch(A, R);
  for (int a = 0; a < 3; ++a) { muq[a] = c[a] + mq[a]; mut[a] = c[a] + mt[a]; }
  for (int a = 0; a < 3; ++a) {
    for (int b = 0; b < 3; ++b) U[a * 4 + b] = R[a * 3 + b];
    U[a * 4 + 3] = mut[a] - ((R[a * 3] * muq[0] + R[a * 3 + 1] * muq[1]) + R[a * 3 + 2] * muq[2]);
  }
}

void compose(const double* U, double* T) {       // T <- U T (rows 0-2)
  double Tn[12];
  for (int a = 0; a < 3; ++a)
    for (int k = 0; k < 4; ++k)
      Tn[a * 4 + k] = ((U[a * 4] * T[k] + U[a * 4 + 1] * T[4 + k]) + U[a * 4 + 2] * T[8 + k]) + U[a * 4 + 3] * T[12 + k];
  std::memcpy(T, Tn, sizeof(Tn));
}

// ---- exact nearest neighbour: median-split k-d tree, each node with the bounding box of its points
struct KdTree {
  const float* X;
  int m, stride;
  std::vector<int> idx;
  struct Node { float lo[3], hi[3]; int begin, end, left, right; };
  std::vector<Node> nodes;

  float coord(int j, int a) const { return X[(size_t)a * stride + j]; }
  int build(int b, int e) {
    Node nd;
    for (int a = 0; a < 3; ++a) { nd.lo[a] = FLT_MAX; nd.hi[a] = -FLT_MAX; }
    for (int k = b; k < e; ++k)
      for (int a = 0; a < 3; ++a) {
        nd.lo[a] = std::min(nd.lo[a], coord(idx[k], a));
        nd.hi[a] = std::max(nd.hi[a], coord(idx[k], a));
      }
    nd.begin = b; nd.end = e; nd.left = nd.right = -1;
    const int id = (int)nodes.size();
    nodes.push_back(nd);
    if (e - b > kLeaf) {
      int ax = 0;
      for (int a = 1; a < 3; ++a)
        if (nd.hi[a] - nd.lo[a] > nd.hi[ax] - nd.lo[ax]) ax = a;
      const int mid = (b + e) / 2;
      std::nth_element(idx.begin() + b, idx.begin() + mid, idx.begin() + e,
                       [&](int p, int q) { return coord(p, ax) < coord(q, ax); });
      const int l = build(b, mid), r = build(mid, e);
      nodes[id].left = l;
      nodes[id].right = r;
    }
    return id;
  }
  KdTree(const float* X_, int m_, int stride_) : X(X_), m(m_), stride(stride_), idx(m_) {
    for (int j = 0; j < m; ++j) idx[j] = j;
    if (m > 0) build(0, m);
  }
  static double lb(const Node& n, const double* q) {
    double d[3];
    for (int a = 0; a < 3; ++a) d[a] = std::max(std::max((double)n.lo[a] - q[a], q[a] - (double)n.hi[a]), 0.0);
    return (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2];
  }
  // best (d2, j) by (d2, then lowest j) among points with d2 <= bound; j = INT_MAX if none
  void query(int id, const double* q, double& bd2, int& bj) const {
    const Node& n = nodes[id];
    if (lb(n, q) > bd2) return;
    if (n.left < 0) {
      for (int k = n.begin; k < n.end; ++k) {
        const int j = idx[k];
        const double dx = q[0] - (double)coord(j, 0), dy = q[1] - (double)coord(j, 1), dz = q[2] - (double)coord(j, 2);
        const double d2 = (dx * dx + dy * dy) + dz * dz;
        if (d2 < bd2 || (d2 == bd2 && j < bj)) { bd2 = d2; bj = j; }
      }
      return;
    }
    const double l0 = lb(nodes[n.left], q), l1 = lb(nodes[n.right], q);
    if (l1 < l0) { query(n.right, q, bd2, bj); query(n.left, q, bd2, bj); }
    else { query(n.left, q, bd2, bj); query(n.right, q, bd2, bj); }
  }
  void nearest(const double* q, double r2, double& d2, int& j) const {
    d2 = r2;
    j = INT_MAX;
    if (m > 0) query(0, q, d2, j);
  }
};

struct PassResult { int nc; double M[kMoments]; double fit, rmse; };

PassResult pass(const float* src, int n, int n_stride, const KdTree& kd, const float* tgt, int m_stride,
                const double* T, const double* c, double r2) {
  std::vector<double> part((size_t)kThreads * kMoments, 0.0);
  int nc = 0;
  for (int t = 0; t < kThreads; ++t) {
    double* acc = &part[(size_t)t * kMoments];
    for (int i = t; i < n; i += kThreads) {
      const double px = src[i], py = src[(size_t)n_stride + i], pz = src[(size_t)2 * n_stride + i];
      const double q[3] = {((T[0] * px + T[1] * py) + T[2] * pz) + T[3], ((T[4] * px + T[5] * py) + T[6] * pz) + T[7],
                           ((T[8] * px + T[9] * py) + T[10] * pz) + T[11]};
      double d2;
      int j;
      kd.nearest(q, r2, d2, j);
      if (j != INT_MAX && d2 < r2) {
        const double dq[3] = {q[0] - c[0], q[1] - c[1], q[2] - c[2]};
        const double dt[3] = {(double)tgt[j] - c[0], (double)tgt[(size_t)m_stride + j] - c[1],
                              (double)tgt[(size_t)2 * m_stride + j] - c[2]};
        ++nc;
        acc[0] += d2;
        for (int a = 0; a < 3; ++a) { acc[1 + a] += dq[a]; acc[4 + a] += dt[a]; }
        for (int u = 0; u < 3; ++u)
          for (int v = 0; v < 3; ++v) acc[7 + u * 3 + v] += dt[u] * dq[v];
      }
    }
  }
  PassResult r;
  r.nc = nc;
  double wsum[kWarps][kMoments];
  for (int w = 0; w < kWarps; ++w) {
    double v[32][kMoments], nv[32][kMoments];
    for (int l = 0; l < 32; ++l) std::memcpy(v[l], &part[(size_t)(w * 32 + l) * kMoments], sizeof(v[l]));
    for (int o = 16; o > 0; o >>= 1) {
      for (int l = 0; l < 32; ++l)
        for (int q = 0; q < kMoments; ++q) nv[l][q] = v[l][q] + v[l ^ o][q];
      std::memcpy(v, nv, sizeof(v));
    }
    std::memcpy(wsum[w], v[0], sizeof(wsum[w]));
  }
  for (int q = 0; q < kMoments; ++q) r.M[q] = wsum[0][q];
  for (int w = 1; w < kWarps; ++w)
    for (int q = 0; q < kMoments; ++q) r.M[q] = r.M[q] + wsum[w][q];
  r.fit = n > 0 ? (double)nc / (double)n : 0.0;
  r.rmse = nc > 0 ? std::sqrt(r.M[0] / (double)nc) : 0.0;
  return r;
}

}  // namespace

extern "C" {

// One frame, I inits.  src [3][n_stride] f32 (first n valid), tgt [3][m_stride] f32 (first m valid), init16 [I][16].
// Per init: T_all [I][16], fit_all [I], rmse_all [I], stats [I][2] (update steps, n_corr), trace_nc [I][max_it + 1]
// (n_corr of every pass, -1 after the last; may be NULL).  Per frame: P16, fitness, best.
void icp_oracle_frame(const float* src, int n, int n_stride, const float* tgt, int m, int m_stride,
                      const double* init16, int I, double r, int max_it, double rel_fit, double rel_rmse, int force_2d,
                      double* T_all, double* fit_all, double* rmse_all, int32_t* stats, int32_t* trace_nc,
                      double* P16, double* fitness, int32_t* best) {
  const KdTree kd(tgt, m, m_stride);
  const double r2 = r * r;
#pragma omp parallel for schedule(dynamic, 1)
  for (int i = 0; i < I; ++i) {
    double T[16], c[3] = {0.0, 0.0, 0.0};
    std::memcpy(T, init16 + (size_t)i * 16, sizeof(T));
    int32_t* tr = trace_nc ? trace_nc + (size_t)i * (max_it + 1) : nullptr;
    if (tr)
      for (int k = 0; k <= max_it; ++k) tr[k] = -1;
    PassResult res = pass(src, n, n_stride, kd, tgt, m_stride, T, c, r2);
    if (tr) tr[0] = res.nc;
    int k = 0;
    while (k < max_it) {
      double U[12], mut[3];
      umeyama_moments(res.M, res.nc, c, U, mut);
      if (res.nc > 0) {
        compose(U, T);
        std::memcpy(c, mut, sizeof(c));
      }
      ++k;
      const PassResult prev = res;
      res = pass(src, n, n_stride, kd, tgt, m_stride, T, c, r2);
      if (tr) tr[k] = res.nc;
      if (std::fabs(prev.fit - res.fit) < rel_fit && std::fabs(prev.rmse - res.rmse) < rel_rmse) break;
    }
    std::memcpy(T_all + (size_t)i * 16, T, sizeof(T));
    fit_all[i] = res.fit;
    rmse_all[i] = res.rmse;
    stats[2 * i] = k;
    stats[2 * i + 1] = res.nc;
  }
  double bf = 0.001;
  int b = -1;
  for (int i = 0; i < I; ++i)
    if (fit_all[i] > bf) { bf = fit_all[i]; b = i; }
  for (int q = 0; q < 16; ++q) P16[q] = b >= 0 ? T_all[(size_t)b * 16 + q] : ((q % 5) == 0 ? 1.0 : 0.0);
  if (force_2d) { P16[1] = 0.0; P16[4] = 0.0; P16[5] = 1.0; P16[6] = 0.0; P16[9] = 0.0; }
  *fitness = bf;
  *best = b;
}

// Umeyama (no scaling) of n pairs src [n][3] -> dst [n][3] with moments about c [3], in point order (test hook).
void icp_oracle_umeyama(const double* src, const double* dst, int n, const double* c, double* U12) {
  double M[kMoments] = {0.0};
  for (int i = 0; i < n; ++i) {
    const double dq[3] = {src[3 * i] - c[0], src[3 * i + 1] - c[1], src[3 * i + 2] - c[2]};
    const double dt[3] = {dst[3 * i] - c[0], dst[3 * i + 1] - c[1], dst[3 * i + 2] - c[2]};
    for (int a = 0; a < 3; ++a) { M[1 + a] += dq[a]; M[4 + a] += dt[a]; }
    for (int u = 0; u < 3; ++u)
      for (int v = 0; v < 3; ++v) M[7 + u * 3 + v] += dt[u] * dq[v];
  }
  double mut[3];
  umeyama_moments(M, n, c, U12, mut);
}

// Nearest target point of each query q [k][3] f64 within d2 < r^2 (j = -1 otherwise); tgt [3][m_stride] (test hook).
void icp_oracle_nearest(const float* tgt, int m, int m_stride, const double* q, int k, double r, int32_t* j_out,
                        double* d2_out) {
  const KdTree kd(tgt, m, m_stride);
  for (int i = 0; i < k; ++i) {
    double d2;
    int j;
    kd.nearest(q + 3 * i, r * r, d2, j);
    const bool hit = j != INT_MAX && d2 < r * r;
    j_out[i] = hit ? j : -1;
    d2_out[i] = hit ? d2 : INFINITY;
  }
}

}  // extern "C"
