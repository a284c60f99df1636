// The point encoder's SO-Net cluster max-pool and its node kNN grouping (SURVEY.md 8f row N12):
// PCEncoder.forward (models/networks_pc.py:88-111) and GeneralKNNFusionModule.forward (models/layers_pc.py:793-807)
// without their expanded int64 index tensors, with deterministic backwards with respect to the features.
//
//   cluster max-pool, forward (cluster_pool_forward_f32):
//     index_max_kernel        sel [B][C][M] = index_max_forward(features, min_idx, M): the existing arg-max, launched
//                             through its C entry point.
//     pool_mask_kernel        mask [B][M] = 1.0f where some point has min_idx == m (plain stores of one value).
//     pool_gather_kernel      pooled [b][c][m] = features[b][c][sel] * mask[b][m], one thread per element.
//     pool_scatter_kernel     scattered [b][c][n] = pooled[b][c][min_idx[b][n]] (NaN for an index outside [0, M)),
//                             one point per thread, a chunk of channels per CTA row, coalesced along n.
//   node kNN grouping, forward (knn_group_forward_f32):
//     knn_search_kernel<KK>   one thread per query; the batch item's database [3][N] sits in shared memory and
//                             nearest_k<KK> (cluster_assign's key, nearest_k.cuh) keeps the KK best; KK is the
//                             smallest instantiated width >= K, and the first K slots are written (a sorted prefix).
//     knn_group_kernel        grouped [b][r][m][j]: r < 3 database[idx] - query, r >= 3 features[idx]; one (m, j)
//                             per thread, a chunk of rows per CTA row, coalesced along (m, j).
//   backwards (cluster_pool_backward_f32, knn_group_backward_f32):
//     segment_sum_kernel      CTA (one warp) per (slice x segment range, 32-channel chunk, b): the g tile [32][32]
//                             is staged coalesced and read transposed; lane c owns the fp64 accumulators of channel c
//                             over the segment range in padded shared memory and adds g in ascending element order.
//                             Partials [B][slices][C][S] f64.  This is interp_backward_kernel (interp.cu) with one
//                             index per element and no weight.
//     pool_finish_kernel      warp per (b, c): t_m = (gP + ((p_0 + p_1) + ...)) * mask in fp64; gF[sel] = float(t_m)
//                             where sel != 0 (one m per point), and gF[0] = float(sum of the t_m with sel == 0 in
//                             ascending m); every other gF is zero.
//     knn_reduce_kernel       gF[b][c][n] = float(((p_0 + p_1) + ...) + p_{S-1}) over the slice partials.
// Each accumulator has one owner and a fixed order: no float atomics, bit-identical across runs and streams.
// Single-precision arithmetic is written with explicit-rounding intrinsics, so FMA contraction cannot change it.
#include <math.h>

#include "common.cuh"
#include "nearest_k.cuh"

namespace dib {

constexpr int kKnnMaxK = 32;
constexpr int kKnnMaxNodes = 2048;
constexpr int kKnnThreads = 64;                // queries per search CTA
constexpr int kGroupThreads = 256;             // (m, j) elements per grouping CTA
constexpr int kGroupRows = 16;                 // rows of grouped per grouping CTA
constexpr int kScatterThreads = 256;           // points per scatter CTA
constexpr int kScatterChannels = 16;           // channels per scatter CTA
constexpr int kSegChannels = 32;               // channels per segment-sum CTA = its one warp
constexpr int kSegTile = 32;                   // elements staged per step
constexpr int kSegRange = 128;                 // segments per segment-sum CTA (accumulators per lane)
constexpr int kSegTargetCtas = 1024;           // slices are added until the grid has about this many CTAs ...
constexpr int kSegMinTiles = 16;               // ... while every slice keeps at least this many tiles

__global__ void pool_mask_kernel(const int32_t* __restrict__ min_idx, int N, int M, float* __restrict__ mask) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (n >= N) return;
  const int m = min_idx[(size_t)b * N + n];
  if (m >= 0 && m < M) mask[(size_t)b * M + m] = 1.0f;      // every writer stores the same value
}

// one thread per (b, c, m)
__global__ void pool_gather_kernel(const float* __restrict__ features, const int32_t* __restrict__ sel,
                                   const float* __restrict__ mask, int C, int N, int M, size_t total,
                                   float* __restrict__ pooled) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const size_t bc = i / M;
  const int m = (int)(i % M), b = (int)(bc / C);
  pooled[i] = __fmul_rn(features[bc * N + sel[i]], mask[(size_t)b * M + m]);
}

// grid (ceil(N / 256), ceil(C / 16), B)
__global__ void __launch_bounds__(kScatterThreads)
    pool_scatter_kernel(const float* __restrict__ pooled, const int32_t* __restrict__ min_idx, int C, int N, int M,
                        float* __restrict__ scattered) {
  const int n = blockIdx.x * kScatterThreads + threadIdx.x, b = blockIdx.z, c0 = blockIdx.y * kScatterChannels;
  if (n >= N) return;
  const int nc = min(kScatterChannels, C - c0);
  const int m = min_idx[(size_t)b * N + n];
  const bool ok = m >= 0 && m < M;
  const float* pr = pooled + ((size_t)b * C + c0) * M + (ok ? m : 0);
  float* o = scattered + ((size_t)b * C + c0) * N + n;
#pragma unroll 4
  for (int c = 0; c < nc; ++c) o[(size_t)c * N] = ok ? pr[(size_t)c * M] : __int_as_float(0x7fc00000);
}

template <int KK>
__global__ void __launch_bounds__(kKnnThreads)
    knn_search_kernel(const float* __restrict__ query, const float* __restrict__ database, int M, int N, int K,
                      int32_t* __restrict__ knn_idx) {
  extern __shared__ __align__(16) float s_db[];              // [3][N]
  const int b = blockIdx.y, tid = threadIdx.x;
  const float* db = database + (size_t)b * 3 * N;
  for (int i = tid; i < 3 * N; i += kKnnThreads) s_db[i] = db[i];
  __syncthreads();
  const int m = blockIdx.x * kKnnThreads + tid;
  if (m >= M) return;
  const float* q = query + (size_t)b * 3 * M;
  const float x = q[m], y = q[(size_t)M + m], z = q[2 * (size_t)M + m];
  int bi[KK];
  if (!nearest_k<KK, false>(x, y, z, s_db, N, bi)) nearest_k<KK, true>(x, y, z, s_db, N, bi);
  int32_t* o = knn_idx + ((size_t)b * M + m) * K;
#pragma unroll
  for (int j = 0; j < KK; ++j)
    if (j < K) o[j] = bi[j];
}

// knn_idx [B][M][K] of knn_group_forward_f32 (also the indices knn_fusion.cu groups by); the caller checks the shape
int knn_search_launch(const float* query, const float* database, int B, int M, int N, int K, int32_t* knn_idx,
                      cudaStream_t stream) {
  const size_t smem = (size_t)3 * N * sizeof(float);            // <= 24 KB
  dim3 grid((M + kKnnThreads - 1) / kKnnThreads, B);
#define DIB_KS_LAUNCH(KK) \
  knn_search_kernel<KK><<<grid, kKnnThreads, smem, stream>>>(query, database, M, N, K, knn_idx)
  if (K <= 1) DIB_KS_LAUNCH(1);
  else if (K <= 2) DIB_KS_LAUNCH(2);
  else if (K <= 4) DIB_KS_LAUNCH(4);
  else if (K <= 8) DIB_KS_LAUNCH(8);
  else if (K <= 16) DIB_KS_LAUNCH(16);
  else DIB_KS_LAUNCH(32);
#undef DIB_KS_LAUNCH
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

// grid (ceil(M * K / 256), ceil((3 + C) / 16), B)
__global__ void __launch_bounds__(kGroupThreads)
    knn_group_kernel(const float* __restrict__ query, const float* __restrict__ database,
                     const float* __restrict__ features, const int32_t* __restrict__ knn_idx, int C, int M, int N,
                     int K, float* __restrict__ grouped) {
  const int e = blockIdx.x * kGroupThreads + threadIdx.x, b = blockIdx.z;
  const size_t MK = (size_t)M * K;
  if ((size_t)e >= MK) return;
  const int n = knn_idx[b * MK + e], m = e / K;
  const int r0 = blockIdx.y * kGroupRows, r1 = min(3 + C, r0 + kGroupRows);
  float* o = grouped + (size_t)b * (3 + C) * MK + e;
#pragma unroll 4
  for (int r = r0; r < r1; ++r) {
    const float v = r < 3 ? __fsub_rn(database[((size_t)b * 3 + r) * N + n], query[((size_t)b * 3 + r) * M + m])
                          : features[((size_t)b * C + (r - 3)) * N + n];
    o[(size_t)r * MK] = v;
  }
}

// grid (slices * ranges, ceil(C / 32), B), 32 threads.  g element (b, c, l) at b * g_batch_stride + c * L + l; seg
// [B][L] int32, a value outside [0, S) joins no segment.  Partials [B][slices][C][S] f64.  The next tile's g and seg
// are loaded into registers while the current one is accumulated.
__global__ void __launch_bounds__(kSegChannels)
    segment_sum_kernel(const float* __restrict__ g, int64_t g_batch_stride, const int32_t* __restrict__ seg, int C,
                       int L, int S, int slices, int slice_len, double* __restrict__ partial) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int ranges = (S + kSegRange - 1) / kSegRange;
  const int s = blockIdx.x / ranges, r = blockIdx.x % ranges;
  const int m0 = r * kSegRange, mr = min(kSegRange, S - m0);
  const int stride = mr | 1;                                  // odd: the lanes' doubles fall in distinct bank pairs
  double* acc = reinterpret_cast<double*>(smem_raw);          // [32][stride]
  float* s_g = reinterpret_cast<float*>(acc + kSegChannels * stride);   // [32][kSegTile + 1]
  int32_t* s_i = reinterpret_cast<int32_t*>(s_g + kSegChannels * (kSegTile + 1));   // [kSegTile]
  const int b = blockIdx.z, c0 = blockIdx.y * kSegChannels, lane = threadIdx.x;
  const int nc = min(kSegChannels, C - c0);
  for (int i = lane; i < kSegChannels * stride; i += 32) acc[i] = 0.0;
  const int l_begin = s * slice_len, l_end = min(L, l_begin + slice_len);
  const float* gb = g + (size_t)b * g_batch_stride + (size_t)c0 * L;
  const int32_t* sb = seg + (size_t)b * L;
  double* my = acc + lane * stride;
  float pg[kSegChannels];
  int32_t pi = -1;
  auto fetch = [&](int t0) {                                  // lane = element of the tile
    const int tn = min(kSegTile, l_end - t0);
#pragma unroll
    for (int c = 0; c < kSegChannels; ++c) pg[c] = (c < nc && lane < tn) ? gb[(size_t)c * L + t0 + lane] : 0.f;
    pi = lane < tn ? sb[t0 + lane] : -1;
  };
  if (l_begin < l_end) fetch(l_begin);
  for (int t0 = l_begin; t0 < l_end; t0 += kSegTile) {
    const int tn = min(kSegTile, l_end - t0);
    __syncwarp();
#pragma unroll
    for (int c = 0; c < kSegChannels; ++c) s_g[c * (kSegTile + 1) + lane] = pg[c];
    s_i[lane] = pi;
    __syncwarp();
    if (t0 + kSegTile < l_end) fetch(t0 + kSegTile);
    if (lane < nc) {
      const float* gr = s_g + lane * (kSegTile + 1);
      for (int t = 0; t < tn; ++t) {
        const int v = s_i[t];                                 // the same in every lane: no divergence
        if (v >= m0 && v < m0 + mr) my[v - m0] += (double)gr[t];
      }
    }
  }
  __syncwarp();
  double* pb = partial + (((size_t)b * slices + s) * C + c0) * S + m0;
  for (int c = 0; c < nc; ++c)
    for (int m = lane; m < mr; m += 32) pb[(size_t)c * S + m] = acc[c * stride + m];
}

// one warp per (b, c); gP [B][C][M] (may be NULL), partial [B][slices][C][M] (NULL: no scattered gradient).
__global__ void pool_finish_kernel(const float* __restrict__ gP, const double* __restrict__ partial, int slices,
                                   const int32_t* __restrict__ sel, const float* __restrict__ mask, int B, int C,
                                   int N, int M, float* __restrict__ gF) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= (long long)B * C) return;                           // warp-uniform
  const int b = (int)(w / C), c = (int)(w % C);
  const size_t row = (size_t)w * M;
  const size_t cm = (size_t)C * M;
  float* out = gF + (size_t)w * N;
  double z = 0.0;
  bool any0 = false;
  for (int mb = 0; mb < M; mb += 32) {
    const int m = mb + lane;
    double t = 0.0;
    int n = -1;
    if (m < M) {
      double sum = 0.0;
      if (partial) {
        const double* p = partial + (size_t)b * slices * cm + (size_t)c * M + m;
        sum = p[0];
        for (int s = 1; s < slices; ++s) sum += p[(size_t)s * cm];
        if (gP) sum = (double)gP[row + m] + sum;
      } else {
        sum = (double)gP[row + m];
      }
      t = sum * (double)mask[(size_t)b * M + m];
      n = sel[row + m];
      if (n != 0) out[n] = (float)t;                           // one segment per point: no other writer
    }
    unsigned zm = __ballot_sync(0xffffffffu, m < M && n == 0);
    while (zm) {                                               // ascending m
      const int l = __ffs(zm) - 1;
      const double v = __shfl_sync(0xffffffffu, t, l);
      z = any0 ? z + v : v;
      any0 = true;
      zm &= zm - 1;
    }
  }
  if (lane == 0 && any0) out[0] = (float)z;
}

// one thread per (b, c, n)
__global__ void knn_reduce_kernel(const double* __restrict__ partial, int C, int N, int slices, size_t total,
                                  float* __restrict__ gF) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const size_t cn = (size_t)C * N, b = i / cn, r = i % cn;
  const double* p = partial + b * slices * cn + r;
  double sum = p[0];
  for (int s = 1; s < slices; ++s) sum += p[(size_t)s * cn];
  gF[i] = (float)sum;
}

// Slices of the segment sum: a function of the shape alone, so a given shape always sums in the same order.
inline void seg_slices(int B, int C, int L, int S, int* slices, int* slice_len) {
  const long long base = (long long)B * ((C + kSegChannels - 1) / kSegChannels) * ((S + kSegRange - 1) / kSegRange);
  const int tiles = (L + kSegTile - 1) / kSegTile;
  long long s = (kSegTargetCtas + base - 1) / base;
  const long long cap = (tiles + kSegMinTiles - 1) / kSegMinTiles;
  if (s > cap) s = cap;
  if (s < 1) s = 1;
  const int tiles_per = (tiles + (int)s - 1) / (int)s;
  *slice_len = tiles_per * kSegTile;
  *slices = (L + *slice_len - 1) / *slice_len;
  if (*slices < 1) *slices = 1;
}

inline size_t seg_smem(int S) {
  const int mr = S < kSegRange ? S : kSegRange;
  return (size_t)kSegChannels * (mr | 1) * sizeof(double) + kSegChannels * (kSegTile + 1) * sizeof(float) +
         kSegTile * sizeof(int32_t);
}

inline size_t seg_workspace_bytes(int B, int C, int L, int S) {
  if (B <= 0 || C <= 0 || L <= 0 || S <= 0) return 0;
  int slices, slice_len;
  seg_slices(B, C, L, S, &slices, &slice_len);
  return (size_t)B * slices * (size_t)C * S * sizeof(double);
}

// partial [B][slices][C][S] from g (element (b, c, l) at b * g_batch_stride + c * L + l) and seg [B][L]
inline int launch_segment_sum(const float* g, int64_t g_batch_stride, const int32_t* seg, int B, int C, int L, int S,
                              double* partial, int* slices, cudaStream_t stream) {
  int slice_len;
  seg_slices(B, C, L, S, slices, &slice_len);
  const int ranges = (S + kSegRange - 1) / kSegRange;
  dim3 grid(*slices * ranges, (C + kSegChannels - 1) / kSegChannels, B);
  segment_sum_kernel<<<grid, kSegChannels, seg_smem(S), stream>>>(g, g_batch_stride, seg, C, L, S, *slices, slice_len,
                                                                  partial);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

}  // namespace dib

extern "C" {

int cluster_pool_forward_f32(const float* features, const int32_t* min_idx, int B, int C, int N, int M, int32_t* sel,
                             float* mask, float* pooled, float* scattered, dib_stream_t stream_) {
  using namespace dib;
  cudaStream_t stream = (cudaStream_t)stream_;
  DIB_REQUIRE(B >= 0 && C >= 0 && B <= 65535, "cluster_pool: need 0 <= B <= 65535, C >= 0");
  DIB_REQUIRE(N >= 1 && M >= 1, "cluster_pool: need N >= 1 and M >= 1");
  if (B == 0) return DIB_OK;
  DIB_REQUIRE(min_idx && mask, "cluster_pool: NULL argument");
  DIB_CHECK_CUDA(cudaMemsetAsync(mask, 0, (size_t)B * M * sizeof(float), stream));
  pool_mask_kernel<<<dim3((N + 255) / 256, B), 256, 0, stream>>>(min_idx, N, M, mask);
  DIB_CHECK_CUDA(cudaGetLastError());
  if (C == 0) return DIB_OK;
  DIB_REQUIRE(features && sel && pooled, "cluster_pool: NULL argument");
  DIB_REQUIRE((C + kScatterChannels - 1) / kScatterChannels <= 65535, "cluster_pool: too many channels");
  const int rc = index_max_forward(features, min_idx, sel, B, C, N, M, stream_);
  if (rc != DIB_OK) return rc;
  const size_t total = (size_t)B * C * M;
  pool_gather_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(features, sel, mask, C, N, M, total, pooled);
  DIB_CHECK_CUDA(cudaGetLastError());
  if (scattered) {
    dim3 grid((N + kScatterThreads - 1) / kScatterThreads, (C + kScatterChannels - 1) / kScatterChannels, B);
    pool_scatter_kernel<<<grid, kScatterThreads, 0, stream>>>(pooled, min_idx, C, N, M, scattered);
    DIB_CHECK_CUDA(cudaGetLastError());
  }
  return DIB_OK;
}

size_t cluster_pool_backward_workspace_bytes(int B, int C, int N, int M) {
  return dib::seg_workspace_bytes(B, C, N, M);
}

int cluster_pool_backward_f32(const float* grad_pooled, const float* grad_scattered, int64_t grad_scattered_batch_stride,
                              const int32_t* min_idx, const int32_t* sel, const float* mask, int B, int C, int N, int M,
                              float* grad_features, void* workspace, size_t workspace_bytes, dib_stream_t stream_) {
  using namespace dib;
  cudaStream_t stream = (cudaStream_t)stream_;
  DIB_REQUIRE(B >= 0 && C >= 0 && B <= 65535, "cluster_pool_backward: need 0 <= B <= 65535, C >= 0");
  DIB_REQUIRE(N >= 1 && M >= 1, "cluster_pool_backward: need N >= 1 and M >= 1");
  if (B == 0 || C == 0) return DIB_OK;
  DIB_REQUIRE(grad_features && sel && mask, "cluster_pool_backward: NULL argument");
  DIB_CHECK_CUDA(cudaMemsetAsync(grad_features, 0, (size_t)B * C * N * sizeof(float), stream));
  if (!grad_pooled && !grad_scattered) return DIB_OK;
  double* partial = nullptr;
  int slices = 0;
  if (grad_scattered) {
    DIB_REQUIRE(min_idx, "cluster_pool_backward: NULL argument");
    DIB_REQUIRE(grad_scattered_batch_stride >= 0, "cluster_pool_backward: grad_scattered_batch_stride < 0");
    DIB_REQUIRE((C + kSegChannels - 1) / kSegChannels <= 65535, "cluster_pool_backward: too many channels");
    const size_t need = cluster_pool_backward_workspace_bytes(B, C, N, M);
    DIB_REQUIRE(workspace && workspace_bytes >= need && ((uintptr_t)workspace & 7) == 0,
                "cluster_pool_backward: workspace too small or misaligned");
    partial = (double*)workspace;
    const int rc = launch_segment_sum(grad_scattered, grad_scattered_batch_stride, min_idx, B, C, N, M, partial,
                                      &slices, stream);
    if (rc != DIB_OK) return rc;
  }
  const long long warps = (long long)B * C;
  pool_finish_kernel<<<(unsigned)((warps + 3) / 4), 128, 0, stream>>>(grad_pooled, partial, slices, sel, mask, B, C,
                                                                      N, M, grad_features);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

int knn_group_forward_f32(const float* query, const float* database, const float* features, int B, int C, int M,
                          int N, int K, int32_t* knn_idx, float* grouped, dib_stream_t stream_) {
  using namespace dib;
  cudaStream_t stream = (cudaStream_t)stream_;
  DIB_REQUIRE(B >= 0 && C >= 0 && M >= 0 && B <= 65535, "knn_group: need 0 <= B <= 65535, C, M >= 0");
  DIB_REQUIRE(N >= 1 && N <= kKnnMaxNodes, "knn_group: need 1 <= N <= 2048");
  DIB_REQUIRE(K >= 1 && K <= kKnnMaxK && K <= N, "knn_group: need 1 <= K <= min(32, N)");
  if (B == 0 || M == 0) return DIB_OK;
  DIB_REQUIRE(query && database && knn_idx && grouped && (C == 0 || features), "knn_group: NULL argument");
  DIB_REQUIRE((3 + C + kGroupRows - 1) / kGroupRows <= 65535, "knn_group: too many channels");
  DIB_REQUIRE((long long)M * K <= 0x7fffffffLL, "knn_group: M * K must fit in int32");
  const int rc = knn_search_launch(query, database, B, M, N, K, knn_idx, stream);
  if (rc != DIB_OK) return rc;
  const long long MK = (long long)M * K;
  dim3 ggrid((unsigned)((MK + kGroupThreads - 1) / kGroupThreads), (3 + C + kGroupRows - 1) / kGroupRows, B);
  knn_group_kernel<<<ggrid, kGroupThreads, 0, stream>>>(query, database, features, knn_idx, C, M, N, K, grouped);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

size_t knn_group_backward_workspace_bytes(int B, int C, int M, int N, int K) {
  if ((long long)M * K > 0x7fffffffLL) return 0;
  return dib::seg_workspace_bytes(B, C, M * K, N);
}

int knn_group_backward_f32(const float* grad_grouped, int64_t grad_batch_stride, const int32_t* knn_idx, int B, int C,
                           int M, int N, int K, float* grad_features, void* workspace, size_t workspace_bytes,
                           dib_stream_t stream_) {
  using namespace dib;
  cudaStream_t stream = (cudaStream_t)stream_;
  DIB_REQUIRE(B >= 0 && C >= 0 && M >= 0 && B <= 65535, "knn_group_backward: need 0 <= B <= 65535, C, M >= 0");
  DIB_REQUIRE(N >= 1 && N <= kKnnMaxNodes, "knn_group_backward: need 1 <= N <= 2048");
  DIB_REQUIRE(K >= 1 && K <= kKnnMaxK && K <= N, "knn_group_backward: need 1 <= K <= min(32, N)");
  DIB_REQUIRE((long long)M * K <= 0x7fffffffLL, "knn_group_backward: M * K must fit in int32");
  if (B == 0 || C == 0) return DIB_OK;
  DIB_REQUIRE(grad_features, "knn_group_backward: NULL argument");
  if (M == 0) {
    DIB_CHECK_CUDA(cudaMemsetAsync(grad_features, 0, (size_t)B * C * N * sizeof(float), stream));
    return DIB_OK;
  }
  DIB_REQUIRE(grad_grouped && knn_idx, "knn_group_backward: NULL argument");
  DIB_REQUIRE(grad_batch_stride >= 0, "knn_group_backward: grad_batch_stride < 0");
  DIB_REQUIRE((C + kSegChannels - 1) / kSegChannels <= 65535, "knn_group_backward: too many channels");
  const size_t need = knn_group_backward_workspace_bytes(B, C, M, N, K);
  DIB_REQUIRE(workspace && workspace_bytes >= need && ((uintptr_t)workspace & 7) == 0,
              "knn_group_backward: workspace too small or misaligned");
  const int L = M * K;
  double* partial = (double*)workspace;
  int slices;
  const int rc = launch_segment_sum(grad_grouped + (size_t)3 * L, grad_batch_stride, knn_idx, B, C, L, N, partial,
                                    &slices, stream);
  if (rc != DIB_OK) return rc;
  const size_t total = (size_t)B * C * N;
  knn_reduce_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(partial, C, N, slices, total, grad_features);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

}  // extern "C"
