// Batched multi-start point-to-point ICP of a LiDAR cloud against a monocular-depth cloud: the contract of
// evaluation/icp/registration_icp.py:115-162 (Open3D registration_icp, TransformationEstimationPointToPoint, default
// ICPConvergenceCriteria, 60 random inits, best fitness kept) restated for many frames at once.  DESIGN.md "ICP"
// states the contract; oracle_icp/icp_oracle.cpp is its serial CPU restatement.
//
// Per frame s (index build, once per call):
//   bbox      (one CTA per frame)  bounding box of the target cloud
//   morton    48-bit Morton code of every target point in its frame's box, key = (s << 48) | code
//   sort      cub::DeviceRadixSort of (key, point index); the order only affects speed, never a result
//   gather    sorted points as float4 (x, y, z, original index)
//   leaves / levels   an implicit binary tree of boxes: leaf k holds sorted points [16k, 16k + 16), node k of level l
//             covers nodes 2k and 2k + 1 of level l - 1.  Counts follow from m alone: ceil(m / (16 << l)).
// Per problem (frame s, init i), one CTA of kThreads runs the whole ICP loop:
//   pass      every thread takes source points tid, tid + kThreads, ... in order: q = T p (fp64, no FMA), exact nearest
//             target point by a depth-first descent pruned by the running best d2 (ties -> lowest target index),
//             correspondence iff d2 < r^2; partial sums of (count, sum d2, sum (q - c), sum (t - c),
//             sum (t - c)(q - c)^T) in point order, an xor butterfly per warp, then warp 0 .. 7 in order
//   update    thread 0: Umeyama without scaling (one-sided Jacobi SVD of the 3x3 cross-covariance), T = U T, the
//             reference point c becomes the mean of the matched targets, convergence test
//   select    (one thread per frame)  the first init with fitness strictly above the best so far (from 0.001),
//             identity if none, then the 2-D forcing of registration_icp.py:127-133
// The file is compiled with --fmad=false (build.py NOFMA_SOURCES), so every operation rounds as the oracle's does.
#include <cfloat>
#include <climits>
#include <cmath>

#include <cub/device/device_radix_sort.cuh>

#include "morton_index.cuh"

namespace dib {
namespace icp {

constexpr int kThreads = 256;         // threads of one ICP problem (8 warps)
constexpr int kWarps = kThreads / 32;
constexpr int kSweeps = 8;            // one-sided Jacobi sweeps of the 3x3 SVD
constexpr int kMoments = 16;          // sum d2, sum dq[3], sum dt[3], sum dt dq^T [9]

struct Work : Index {       // the target index and the per-problem results
  double* T;                // [S][I][16]
  double* fit;              // [S][I]
  double* rmse;             // [S][I]
};

// ---------------------------------------------------------------------------------------------------------------
// Index build.

__global__ void __launch_bounds__(256) bbox_kernel(const float* __restrict__ tgt, const int32_t* __restrict__ m_pts,
                                                    int m_stride, float* __restrict__ bbox) {
  const int s = blockIdx.x;
  const int m = clamp_n(m_pts, s, m_stride);
  const float* X = tgt + (size_t)s * 3 * m_stride;
  float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  for (int j = threadIdx.x; j < m; j += blockDim.x)
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const float v = X[(size_t)a * m_stride + j];
      lo[a] = fminf(lo[a], v);
      hi[a] = fmaxf(hi[a], v);
    }
  __shared__ float red[6][8];
#pragma unroll
  for (int a = 0; a < 3; ++a)
    for (int o = 16; o > 0; o >>= 1) {
      lo[a] = fminf(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
      hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
    }
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0)
    for (int a = 0; a < 3; ++a) red[a][w] = lo[a], red[3 + a][w] = hi[a];
  __syncthreads();
  if (threadIdx.x < 6) {
    float v = red[threadIdx.x][0];
    for (int k = 1; k < (int)(blockDim.x >> 5); ++k)
      v = threadIdx.x < 3 ? fminf(v, red[threadIdx.x][k]) : fmaxf(v, red[threadIdx.x][k]);
    bbox[s * 6 + threadIdx.x] = v;
  }
}

__device__ __forceinline__ unsigned long long morton48(unsigned x, unsigned y, unsigned z) {
  unsigned long long c = 0;
#pragma unroll
  for (int b = 0; b < 16; ++b)
    c |= ((unsigned long long)((x >> b) & 1u) << (3 * b)) | ((unsigned long long)((y >> b) & 1u) << (3 * b + 1)) |
         ((unsigned long long)((z >> b) & 1u) << (3 * b + 2));
  return c;
}

__device__ __forceinline__ unsigned quant16(float v, float lo, float hi) {
  const float ext = hi - lo;
  if (!(ext > 0.f)) return 0u;
  const float f = (v - lo) / ext * 65535.f;
  return f <= 0.f ? 0u : (f >= 65535.f ? 65535u : (unsigned)f);
}

__global__ void morton_kernel(const float* __restrict__ tgt, const int32_t* __restrict__ m_pts, int m_stride, int S,
                              const float* __restrict__ bbox, unsigned long long* __restrict__ key,
                              int32_t* __restrict__ val) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)S * m_stride) return;
  const int s = (int)(g / m_stride), j = (int)(g - (long long)s * m_stride);
  const int m = clamp_n(m_pts, s, m_stride);
  unsigned long long code = 0xFFFFFFFFFFFFull;                       // padding sorts to the end of its frame
  if (j < m) {
    const float* X = tgt + (size_t)s * 3 * m_stride;
    const float* b = bbox + s * 6;
    code = morton48(quant16(X[j], b[0], b[3]), quant16(X[(size_t)m_stride + j], b[1], b[4]),
                    quant16(X[(size_t)2 * m_stride + j], b[2], b[5]));
  }
  key[g] = ((unsigned long long)s << 48) | code;
  val[g] = j;
}

__global__ void gather_kernel(const float* __restrict__ tgt, const int32_t* __restrict__ m_pts, int m_stride, int S,
                              const int32_t* __restrict__ val, float4* __restrict__ pts) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)S * m_stride) return;
  const int s = (int)(g / m_stride), k = (int)(g - (long long)s * m_stride);
  if (k >= clamp_n(m_pts, s, m_stride)) return;
  const int j = val[g];
  const float* X = tgt + (size_t)s * 3 * m_stride;
  pts[g] = make_float4(X[j], X[(size_t)m_stride + j], X[(size_t)2 * m_stride + j], __int_as_float(j));
}

// Level l of the tree (l = 0: leaves over the sorted points).
__global__ void level_kernel(const int32_t* __restrict__ m_pts, int m_stride, int S, int l, Levels L,
                             const float4* __restrict__ pts, float4* __restrict__ lo, float4* __restrict__ hi) {
  const int cap = level_count(m_stride, l);
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)S * cap) return;
  const int s = (int)(g / cap), k = (int)(g - (long long)s * cap);
  const int m = clamp_n(m_pts, s, m_stride);
  if (k >= level_count(m, l)) return;
  float4 a = make_float4(FLT_MAX, FLT_MAX, FLT_MAX, 0.f), b = make_float4(-FLT_MAX, -FLT_MAX, -FLT_MAX, 0.f);
  const size_t base = (size_t)s * L.per_frame;
  if (l == 0) {
    const float4* p = pts + (size_t)s * m_stride;
    const int e = k * kLeaf + min(kLeaf, m - k * kLeaf);
    for (int j = k * kLeaf; j < e; ++j) {
      const float4 v = p[j];
      a.x = fminf(a.x, v.x); a.y = fminf(a.y, v.y); a.z = fminf(a.z, v.z);
      b.x = fmaxf(b.x, v.x); b.y = fmaxf(b.y, v.y); b.z = fmaxf(b.z, v.z);
    }
  } else {
    const int nc = level_count(m, l - 1);
    for (int c = 2 * k; c < min(2 * k + 2, nc); ++c) {
      const float4 u = lo[base + L.off[l - 1] + c], v = hi[base + L.off[l - 1] + c];
      a.x = fminf(a.x, u.x); a.y = fminf(a.y, u.y); a.z = fminf(a.z, u.z);
      b.x = fmaxf(b.x, v.x); b.y = fmaxf(b.y, v.y); b.z = fmaxf(b.z, v.z);
    }
  }
  lo[base + L.off[l] + k] = a;
  hi[base + L.off[l] + k] = b;
}

// ---------------------------------------------------------------------------------------------------------------
// Umeyama without scaling from the pass moments (shared with the oracle line by line).

__host__ __device__ inline double dot3(const double* a, const double* b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }

// R (row-major 3x3) maximising tr(R^T A), A = cross-covariance dst x src: R = U diag(1, 1, det V) V^T with the
// columns of A V orthogonalised by a cyclic one-sided Jacobi of kSweeps sweeps, u1, u2 from its two largest columns and
// u3 = u1 x u2.  This is Eigen's umeyama rotation (S = diag(1, 1, -1) when det U det V < 0) written so that rank
// deficient A stays finite and deterministic (A = 0 gives R = I).
__host__ __device__ inline void kabsch(const double* A, double* R) {
  double B[3][3], V[3][3];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) { B[c][r] = A[r * 3 + c]; V[c][r] = r == c ? 1.0 : 0.0; }   // B[c] = column c
  for (int sw = 0; sw < kSweeps; ++sw)
    for (int pr = 0; pr < 3; ++pr) {
      const int p = pr == 2 ? 1 : 0, q = pr == 0 ? 1 : 2;
      const double alpha = dot3(B[p], B[p]), beta = dot3(B[q], B[q]), gamma = dot3(B[p], B[q]);
      if (gamma == 0.0) continue;
      const double zeta = (beta - alpha) / (2.0 * gamma);
      const double t = (zeta >= 0.0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
      const double cs = 1.0 / sqrt(1.0 + t * t), sn = cs * t;
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
  for (int k = 0; k < 3; ++k) sg[k] = sqrt(dot3(B[k], B[k]));
  int o[3] = {0, 1, 2};
  if (sg[o[1]] > sg[o[0]]) { const int x = o[0]; o[0] = o[1]; o[1] = x; }
  if (sg[o[2]] > sg[o[1]]) { const int x = o[1]; o[1] = o[2]; o[2] = x; }
  if (sg[o[1]] > sg[o[0]]) { const int x = o[0]; o[0] = o[1]; o[1] = x; }
  double u1[3], u2[3], u3[3];
  if (sg[o[0]] > 0.0) {
    for (int r = 0; r < 3; ++r) u1[r] = B[o[0]][r] / sg[o[0]];
  } else {
    u1[0] = 1.0; u1[1] = 0.0; u1[2] = 0.0;
  }
  const double pj = dot3(u1, B[o[1]]);
  double w[3];
  for (int r = 0; r < 3; ++r) w[r] = B[o[1]][r] - pj * u1[r];
  double nw = sqrt(dot3(w, w));
  if (!(nw > 1e-14 * sg[o[0]]) || nw == 0.0) {       // rank <= 1: any unit vector orthogonal to u1
    int e = 0;
    for (int r = 1; r < 3; ++r)
      if (fabs(u1[r]) < fabs(u1[e])) e = r;
    for (int r = 0; r < 3; ++r) w[r] = (r == e ? 1.0 : 0.0) - u1[e] * u1[r];
    nw = sqrt(dot3(w, w));
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

// One update: U from the moments M (about the reference point c) of nc correspondences, T <- U T, c <- mean of the
// matched targets.  nc == 0: U = I (Open3D returns the identity for an empty correspondence set).
__host__ __device__ inline void icp_update(const double* M, int nc, double* c, double* T) {
  if (nc <= 0) return;
  const double n = (double)nc;
  double mq[3], mt[3], A[9], R[9], muq[3], mut[3], U[12];
  for (int a = 0; a < 3; ++a) { mq[a] = M[1 + a] / n; mt[a] = M[4 + a] / n; }
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) A[a * 3 + b] = M[7 + a * 3 + b] / n - mt[a] * mq[b];
  kabsch(A, R);
  for (int a = 0; a < 3; ++a) { muq[a] = c[a] + mq[a]; mut[a] = c[a] + mt[a]; }
  for (int a = 0; a < 3; ++a) {
    for (int b = 0; b < 3; ++b) U[a * 4 + b] = R[a * 3 + b];
    U[a * 4 + 3] = mut[a] - ((R[a * 3] * muq[0] + R[a * 3 + 1] * muq[1]) + R[a * 3 + 2] * muq[2]);
  }
  double Tn[12];
  for (int a = 0; a < 3; ++a)
    for (int k = 0; k < 4; ++k)
      Tn[a * 4 + k] = ((U[a * 4] * T[k] + U[a * 4 + 1] * T[4 + k]) + U[a * 4 + 2] * T[8 + k]) + U[a * 4 + 3] * T[12 + k];
  for (int k = 0; k < 12; ++k) T[k] = Tn[k];
  for (int a = 0; a < 3; ++a) c[a] = mut[a];
}

// ---------------------------------------------------------------------------------------------------------------
// The ICP loop: one CTA per (frame, init), frame-major.

struct Args {
  const float* src;
  const int32_t* n_pts;
  int n_stride;
  const int32_t* m_pts;
  int m_stride;
  const double* init16;
  int I;
  double r2;
  int max_iteration;
  double rel_fit, rel_rmse;
  int32_t* stats;           // [S][I][2] or NULL
  unsigned long long* counters;   // (queries, distance evaluations) or NULL
};

__global__ void __launch_bounds__(kThreads, 2) icp_kernel(Args a, Levels L, Work wk) {
  const int prob = blockIdx.x;
  const int s = prob / a.I;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n = clamp_n(a.n_pts, s, a.n_stride), m = clamp_n(a.m_pts, s, a.m_stride);
  __shared__ double T[16], c[3], red[kWarps][kMoments];
  __shared__ int red_n[kWarps], done, ncorr;
  __shared__ double fit_s, rmse_s;
  if (tid < 16) T[tid] = a.init16[(size_t)prob * 16 + tid];
  if (tid < 3) c[tid] = 0.0;
  if (tid == 0) done = 0;
  int root = 0;
  while (level_count(m, root) > 1) ++root;
  const float4* pts = wk.pts + (size_t)s * a.m_stride;
  const float4* lo = wk.lo + (size_t)s * L.per_frame;
  const float4* hi = wk.hi + (size_t)s * L.per_frame;
  const float* X = a.src + (size_t)s * 3 * a.n_stride;
  unsigned long long evals = 0, queries = 0;
  double prev_fit = 0.0, prev_rmse = 0.0;
  int k = 0;
  __syncthreads();
  for (int pass = 0;; ++pass) {
    // ---- one correspondence pass at T
    double acc[kMoments];
#pragma unroll
    for (int q = 0; q < kMoments; ++q) acc[q] = 0.0;
    int cnt = 0;
    const double t0 = T[0], t1 = T[1], t2 = T[2], t3 = T[3], t4 = T[4], t5 = T[5], t6 = T[6], t7 = T[7];
    const double t8 = T[8], t9 = T[9], t10 = T[10], t11 = T[11], cx = c[0], cy = c[1], cz = c[2];
    for (int i = tid; i < n; i += kThreads) {
      const double px = X[i], py = X[(size_t)a.n_stride + i], pz = X[(size_t)2 * a.n_stride + i];
      const double qx = ((t0 * px + t1 * py) + t2 * pz) + t3;
      const double qy = ((t4 * px + t5 * py) + t6 * pz) + t7;
      const double qz = ((t8 * px + t9 * py) + t10 * pz) + t11;
      Hit h;
      h.d2 = a.r2;
      nearest(pts, lo, hi, L, m, root, qx, qy, qz, h, evals);
      ++queries;
      if (h.j != INT_MAX && h.d2 < a.r2) {
        const double dq[3] = {qx - cx, qy - cy, qz - cz};
        const double dt[3] = {(double)h.x - cx, (double)h.y - cy, (double)h.z - cz};
        ++cnt;
        acc[0] += h.d2;
#pragma unroll
        for (int q = 0; q < 3; ++q) { acc[1 + q] += dq[q]; acc[4 + q] += dt[q]; }
#pragma unroll
        for (int u = 0; u < 3; ++u)
#pragma unroll
          for (int v = 0; v < 3; ++v) acc[7 + u * 3 + v] += dt[u] * dq[v];
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
      for (int q = 0; q < kMoments; ++q) acc[q] = acc[q] + __shfl_xor_sync(0xffffffffu, acc[q], o);
      cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    }
    if (lane == 0) {
#pragma unroll
      for (int q = 0; q < kMoments; ++q) red[warp][q] = acc[q];
      red_n[warp] = cnt;
    }
    __syncthreads();
    if (tid == 0) {
      double M[kMoments];
      int nc = red_n[0];
      for (int q = 0; q < kMoments; ++q) M[q] = red[0][q];
      for (int w = 1; w < kWarps; ++w) {
        nc += red_n[w];
        for (int q = 0; q < kMoments; ++q) M[q] = M[q] + red[w][q];
      }
      const double fit = n > 0 ? (double)nc / (double)n : 0.0;
      const double rmse = nc > 0 ? sqrt(M[0] / (double)nc) : 0.0;
      int stop = 0;
      if (pass > 0 && fabs(prev_fit - fit) < a.rel_fit && fabs(prev_rmse - rmse) < a.rel_rmse) stop = 1;
      if (k >= a.max_iteration) stop = 1;
      prev_fit = fit;
      prev_rmse = rmse;
      fit_s = fit;
      rmse_s = rmse;
      ncorr = nc;
      if (!stop) {
        double Tl[16], cl[3] = {c[0], c[1], c[2]};
        for (int q = 0; q < 16; ++q) Tl[q] = T[q];
        icp_update(M, nc, cl, Tl);
        for (int q = 0; q < 12; ++q) T[q] = Tl[q];
        for (int q = 0; q < 3; ++q) c[q] = cl[q];
        ++k;
      }
      done = stop;
    }
    __syncthreads();
    if (done) break;
  }
  if (tid < 16) wk.T[(size_t)prob * 16 + tid] = T[tid];
  if (tid == 0) {
    wk.fit[prob] = fit_s;
    wk.rmse[prob] = rmse_s;
    if (a.stats) { a.stats[(size_t)prob * 2] = k; a.stats[(size_t)prob * 2 + 1] = ncorr; }
  }
  if (a.counters) {
    atomicAdd(a.counters, queries);
    atomicAdd(a.counters + 1, evals);
  }
}

__global__ void select_kernel(int S, int I, int force_2d, const double* __restrict__ T, const double* __restrict__ fit,
                              double* __restrict__ P16, double* __restrict__ fit_out, int32_t* __restrict__ best_out) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= S) return;
  double best = 0.001;
  int b = -1;
  for (int i = 0; i < I; ++i) {
    const double f = fit[(size_t)s * I + i];
    if (f > best) { best = f; b = i; }
  }
  double P[16];
  for (int q = 0; q < 16; ++q) P[q] = b >= 0 ? T[((size_t)s * I + b) * 16 + q] : ((q % 5) == 0 ? 1.0 : 0.0);
  if (force_2d) { P[1] = 0.0; P[4] = 0.0; P[5] = 1.0; P[6] = 0.0; P[9] = 0.0; }
  for (int q = 0; q < 16; ++q) P16[(size_t)s * 16 + q] = P[q];
  fit_out[s] = best;
  if (best_out) best_out[s] = b;
}

inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

Levels make_levels(int m_stride) {
  Levels L{};
  int off = 0, l = 0;
  for (;; ++l) {
    L.off[l] = off;
    const int c = level_count(m_stride, l);
    off += c;
    if (c <= 1) break;
  }
  L.n = l + 1;
  L.per_frame = off;
  return L;
}

// Radix-sort scratch reserved in the workspace: cub's need (queried at run time, when a device exists) is a few
// hundred bytes per 3840-item tile; 8 B per item plus 4 MiB is far above it at every batch size.
inline size_t sort_reserve(size_t N) { return 8 * N + ((size_t)4 << 20); }

size_t carve_index(char* base, size_t off, int S, int m_stride, Index* ix) {
  const size_t N = (size_t)S * m_stride;
  const Levels L = make_levels(m_stride);
  auto take = [&](size_t bytes) { char* p = base ? base + off : nullptr; off += align256(bytes); return p; };
  Index w;
  w.bbox = (float*)take((size_t)S * 6 * 4);
  w.key0 = (unsigned long long*)take(N * 8); w.key1 = (unsigned long long*)take(N * 8);
  w.val0 = (int32_t*)take(N * 4); w.val1 = (int32_t*)take(N * 4);
  w.pts = (float4*)take(N * 16);
  w.lo = (float4*)take((size_t)S * L.per_frame * 16); w.hi = (float4*)take((size_t)S * L.per_frame * 16);
  w.sort_tmp_bytes = sort_reserve(N);
  w.sort_tmp = take(w.sort_tmp_bytes);
  if (ix) *ix = w;
  return off;
}

// Workspace carve-up; returns the bytes needed (base may be NULL).
size_t carve(char* base, int S, int I, int m_stride, Work* wk) {
  Work w;
  size_t off = carve_index(base, 0, S, m_stride, &w);
  auto take = [&](size_t bytes) { char* p = base ? base + off : nullptr; off += align256(bytes); return p; };
  w.T = (double*)take((size_t)S * I * 16 * 8);
  w.fit = (double*)take((size_t)S * I * 8);
  w.rmse = (double*)take((size_t)S * I * 8);
  if (wk) *wk = w;
  return off;
}

constexpr int kMaxS = 65535;     // frames: 16 bits of the sort key
constexpr int kMaxI = 4096;

// Host-side checks shared by the entry points that build the index.
int check_index_args(const float* tgt, int m_stride, int S, int I, void* workspace, size_t workspace_bytes) {
  DIB_REQUIRE(tgt, "NULL argument (tgt)");
  DIB_REQUIRE(S >= 0 && S <= kMaxS, "S=%d must be in [0, %d] (larger batches: split them)", S, kMaxS);
  DIB_REQUIRE(I >= 1 && I <= kMaxI, "I=%d must be in [1, %d]", I, kMaxI);
  DIB_REQUIRE(m_stride >= 16 && m_stride % 16 == 0, "m_stride=%d must be a positive multiple of 16", m_stride);
  DIB_REQUIRE((long long)S * m_stride < (1LL << 31), "S * m_stride must be below 2^31");
  DIB_REQUIRE(make_levels(m_stride).n <= kMaxLevels, "m_stride=%d is too large for the index", m_stride);
  const size_t need = carve(nullptr, S, I, m_stride, nullptr);
  DIB_REQUIRE(workspace && workspace_bytes >= need, "workspace too small (%zu < %zu)", workspace_bytes, need);
  DIB_REQUIRE(((uintptr_t)workspace & 255) == 0, "workspace must be 256-byte aligned");
  return DIB_OK;
}

void cloud_bbox(const float* X, const int32_t* n_pts, int stride, int S, float* bbox, cudaStream_t st) {
  bbox_kernel<<<S, 256, 0, st>>>(X, n_pts, stride, bbox);
}

int build_index(const float* tgt, const int32_t* m_pts, int m_stride, int S, const Levels& L, Index& wk,
                cudaStream_t st) {
  const long long N = (long long)S * m_stride;
  const int nb = (int)((N + 255) / 256);
  bbox_kernel<<<S, 256, 0, st>>>(tgt, m_pts, m_stride, wk.bbox);
  morton_kernel<<<nb, 256, 0, st>>>(tgt, m_pts, m_stride, S, wk.bbox, wk.key0, wk.val0);
  DIB_CHECK_CUDA(cudaGetLastError());
  int fb = 0;
  while ((1 << fb) < S) ++fb;
  cub::DoubleBuffer<unsigned long long> keys(wk.key0, wk.key1);
  cub::DoubleBuffer<int32_t> vals(wk.val0, wk.val1);
  size_t tmp = 0;
  DIB_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp, keys, vals, (int)N, 0, 48 + fb, st));
  if (tmp > wk.sort_tmp_bytes) {
    set_error("index: the radix sort needs %zu bytes of scratch, %zu reserved", tmp, wk.sort_tmp_bytes);
    return DIB_ENOMEM;
  }
  DIB_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(wk.sort_tmp, tmp, keys, vals, (int)N, 0, 48 + fb, st));
  gather_kernel<<<nb, 256, 0, st>>>(tgt, m_pts, m_stride, S, vals.Current(), wk.pts);
  for (int l = 0; l < L.n; ++l) {
    const long long cnt = (long long)S * level_count(m_stride, l);
    level_kernel<<<(int)((cnt + 255) / 256), 256, 0, st>>>(m_pts, m_stride, S, l, L, wk.pts, wk.lo, wk.hi);
  }
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

int register_batch(const float* src, const int32_t* n_pts, int n_stride, const float* tgt, const int32_t* m_pts,
                   int m_stride, int S, const double* init16, int I, double max_corr_dist, int max_iteration,
                   double relative_fitness, double relative_rmse, int force_2d, double* P16_out, double* fitness_out,
                   int32_t* best_out, double* T_all, double* fitness_all, double* rmse_all, int32_t* stats_all,
                   unsigned long long* counters, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  DIB_REQUIRE(src && tgt && init16 && P16_out && fitness_out, "NULL argument (src, tgt, init16, P16_out, fitness_out)");
  DIB_REQUIRE(n_stride >= 16 && n_stride % 16 == 0, "n_stride=%d must be a positive multiple of 16", n_stride);
  DIB_REQUIRE(std::isfinite(max_corr_dist) && max_corr_dist > 0.0, "max_corr_dist must be positive (got %g)",
              max_corr_dist);
  DIB_REQUIRE(max_iteration >= 0, "max_iteration must be >= 0 (got %d)", max_iteration);
  DIB_REQUIRE(!std::isnan(relative_fitness) && !std::isnan(relative_rmse), "convergence criteria must not be NaN");
  const int rc = check_index_args(tgt, m_stride, S, I, workspace, workspace_bytes);
  if (rc != DIB_OK) return rc;
  if (S == 0) return DIB_OK;
  Work wk;
  carve((char*)workspace, S, I, m_stride, &wk);
  if (T_all) wk.T = T_all;
  if (fitness_all) wk.fit = fitness_all;
  if (rmse_all) wk.rmse = rmse_all;
  const Levels L = make_levels(m_stride);
  const int rb = build_index(tgt, m_pts, m_stride, S, L, wk, st);
  if (rb != DIB_OK) return rb;
  const double r2 = max_corr_dist * max_corr_dist;
  Args a{src, n_pts, n_stride, m_pts, m_stride, init16, I, r2, max_iteration, relative_fitness, relative_rmse,
         stats_all, counters};
  icp_kernel<<<S * I, kThreads, 0, st>>>(a, L, wk);
  DIB_CHECK_CUDA(cudaGetLastError());
  select_kernel<<<(S + 127) / 128, 128, 0, st>>>(S, I, force_2d, wk.T, wk.fit, P16_out, fitness_out, best_out);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

}  // namespace icp
}  // namespace dib

extern "C" {

size_t icp_workspace_bytes(int S, int I, int n_stride, int m_stride) {
  (void)n_stride;
  if (S < 0 || I < 1 || m_stride < 16 || S > dib::icp::kMaxS || I > dib::icp::kMaxI) return 0;
  return dib::icp::carve(nullptr, S, I, m_stride, nullptr);
}

int icp_register_batch_f32(const float* src, const int32_t* n_pts, int n_stride, const float* tgt,
                           const int32_t* m_pts, int m_stride, int S, const double* init16, int I,
                           double max_corr_dist, int max_iteration, double relative_fitness, double relative_rmse,
                           int force_2d, double* P16_out, double* fitness_out, int32_t* best_out, double* T_all,
                           double* fitness_all, double* rmse_all, int32_t* stats_all, void* workspace,
                           size_t workspace_bytes, dib_stream_t stream) {
  return dib::icp::register_batch(src, n_pts, n_stride, tgt, m_pts, m_stride, S, init16, I, max_corr_dist,
                                  max_iteration, relative_fitness, relative_rmse, force_2d, P16_out, fitness_out,
                                  best_out, T_all, fitness_all, rmse_all, stats_all, nullptr, workspace,
                                  workspace_bytes, (cudaStream_t)stream);
}

int icp_register_batch_counted_f32(const float* src, const int32_t* n_pts, int n_stride, const float* tgt,
                                   const int32_t* m_pts, int m_stride, int S, const double* init16, int I,
                                   double max_corr_dist, int max_iteration, double relative_fitness,
                                   double relative_rmse, int force_2d, double* P16_out, double* fitness_out,
                                   int32_t* best_out, double* T_all, double* fitness_all, double* rmse_all,
                                   int32_t* stats_all, unsigned long long* counters, void* workspace,
                                   size_t workspace_bytes, dib_stream_t stream) {
  using namespace dib;
  DIB_REQUIRE(counters, "NULL argument (counters)");
  return icp::register_batch(src, n_pts, n_stride, tgt, m_pts, m_stride, S, init16, I, max_corr_dist, max_iteration,
                             relative_fitness, relative_rmse, force_2d, P16_out, fitness_out, best_out, T_all,
                             fitness_all, rmse_all, stats_all, counters, workspace, workspace_bytes,
                             (cudaStream_t)stream);
}

int icp_build_index_f32(const float* tgt, const int32_t* m_pts, int m_stride, int S, void* workspace,
                        size_t workspace_bytes, dib_stream_t stream) {
  using namespace dib::icp;
  const int rc = check_index_args(tgt, m_stride, S, 1, workspace, workspace_bytes);
  if (rc != DIB_OK || S == 0) return rc;
  Work wk;
  carve((char*)workspace, S, 1, m_stride, &wk);
  return build_index(tgt, m_pts, m_stride, S, make_levels(m_stride), wk, (cudaStream_t)stream);
}

}  // extern "C"
