// Point -> node clustering front-end of the point-cloud encoder (SURVEY.md 8f row N4, first half):
// models/networks_pc.py:60-85 without the B x N x Ma intermediates.  The reference materialises
// pc_B3NMa - node_a_B3NMa, its norm, a B x N x Ma mask (byte and float) and a B x 3 x N x Ma masked copy
// of the cloud (8 x 3 x 20480 x 128 floats = 252 MB each at the shipped configuration) to obtain
//
//   min_k_idx [B,N,k]  the k nearest nodes of every point, nearest first        (:63-64, torch.topk)
//   min_idx   [B,N]    = min_k_idx[..., 0], the `index` argument of index_max    (:65, :88-90)
//   count     [B,Ma]   points per node; mask_row_max = count > 0                 (:66-72)
//   cluster_mean [B,3,Ma] = sum of the node's points / (count + 1e-5)            (:74-76)
//   pc_centers [B,3,N] = cluster_mean gathered by min_idx;  pc_decentered = pc - pc_centers  (:78-82)
//
// Here: kernel 1 keeps the nodes of one batch item in shared memory, one thread per point scans them,
// keeps the k best in registers and adds the point to its node's count and coordinate sums; kernel 2
// turns sums into means; kernel 3 gathers and subtracts.  HBM traffic = the cloud twice + the outputs.
//
// Arithmetic contract (oracle: oracle.cluster_assign):
//   * ordering key d2 = ((dx*dx + dy*dy) + dz*dz), float32, no fma, d = point - node; ties -> lower
//     node index (torch.topk leaves tie order unspecified; sqrt is monotone so the order on d2 is a
//     valid order on the reference's norm).  +inf orders after every finite d2 and NaN after +inf, so
//     the k slots always hold k distinct nodes.
//   * coordinate sums are fixed point: each coordinate is rounded to the 2^-24 grid (rint(x * 2^24),
//     an error of at most 2^-25 per point, none for |x| >= 0.5 or any multiple of 2^-24) and the
//     integers are added exactly in a two-word accumulator (64-bit low word, 32-bit high word) --
//     associative, so the result does not depend on the order the atomics land in (the reference's
//     float tree-sum has no defined order).  A point with a coordinate of magnitude >= 2^39 (where x * 2^24 leaves int64) or a
//     non-finite one is left out of its node's count and sums.  mean = round_f32(sum * 2^-24) /
//     (float(count) + 1e-5f), the first rounding done once from the two-word sum.
#include <cfloat>

#include "common.cuh"
#include "nearest_k.cuh"

namespace dib {

constexpr int kCaThreads = 256;
constexpr int kCaPointsPerThread = 1;
constexpr int kCaMaxK = 8;
constexpr int kCaMaxNodes = 2048;
constexpr double kCaFixedScale = 16777216.0;        // 2^24
constexpr float kCaFixedLimit = 549755813888.0f;    // 2^39: |x| * 2^24 < 2^63

// hi:lo += v (two's complement): the returned old low word tells whether this addition carried, so the high word
// receives exactly the carries and sign extensions, whatever order the additions land in.
__device__ __forceinline__ void add_wide_shared(unsigned long long* lo, int* hi, long long v) {
  const unsigned long long u = (unsigned long long)v;
  const unsigned long long old = atomicAdd(lo, u);
  const int h = (int)(old + u < old) - (int)(v < 0);
  if (h) atomicAdd(hi, h);
}

template <int K>
__global__ void __launch_bounds__(kCaThreads)
    cluster_assign_kernel(const float* __restrict__ pc, const float* __restrict__ node, int N, int M,
                          int32_t* __restrict__ topk, int32_t* __restrict__ min_idx, int32_t* __restrict__ count,
                          unsigned long long* __restrict__ sum_lo, unsigned* __restrict__ sum_hi) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  unsigned long long* s_lo = reinterpret_cast<unsigned long long*>(smem_raw);      // [3][M]
  float* s_node = reinterpret_cast<float*>(s_lo + 3 * (size_t)M);                  // [3][M]
  int* s_hi = reinterpret_cast<int*>(s_node + 3 * (size_t)M);                      // [3][M]: at most 256 adds per CTA
  int* s_cnt = s_hi + 3 * (size_t)M;                                               // [M]
  const int b = blockIdx.y, tid = threadIdx.x;
  const float* nb = node + (size_t)b * 3 * M;
  for (int i = tid; i < 3 * M; i += kCaThreads) { s_node[i] = nb[i]; s_lo[i] = 0ull; s_hi[i] = 0; }
  for (int i = tid; i < M; i += kCaThreads) s_cnt[i] = 0;
  __syncthreads();

  const float* px = pc + (size_t)b * 3 * N;
  const int base = blockIdx.x * (kCaThreads * kCaPointsPerThread);
#pragma unroll 1
  for (int q = 0; q < kCaPointsPerThread; ++q) {
    const int n = base + q * kCaThreads + tid;
    if (n >= N) break;
    const float x = px[n], y = px[(size_t)N + n], z = px[2 * (size_t)N + n];
    int bi[K];
    if (!nearest_k<K, false>(x, y, z, s_node, M, bi)) nearest_k<K, true>(x, y, z, s_node, M, bi);
    int32_t* o = topk + ((size_t)b * N + n) * K;
#pragma unroll
    for (int j = 0; j < K; ++j) o[j] = bi[j];
    const int m0 = bi[0];
    min_idx[(size_t)b * N + n] = m0;
    // a point with a coordinate that has no int64 fixed-point image (|x| >= 2^39, inf, NaN) is left out of its node's
    // count and sums; it keeps its min_k_idx / min_idx
    if (fabsf(x) < kCaFixedLimit && fabsf(y) < kCaFixedLimit && fabsf(z) < kCaFixedLimit) {
      atomicAdd(&s_cnt[m0], 1);
      add_wide_shared(&s_lo[m0], &s_hi[m0], __double2ll_rn((double)x * kCaFixedScale));
      add_wide_shared(&s_lo[M + m0], &s_hi[M + m0], __double2ll_rn((double)y * kCaFixedScale));
      add_wide_shared(&s_lo[2 * M + m0], &s_hi[2 * M + m0], __double2ll_rn((double)z * kCaFixedScale));
    }
  }
  __syncthreads();
  for (int i = tid; i < M; i += kCaThreads) {
    const int c = s_cnt[i];
    if (c) {
      atomicAdd(&count[(size_t)b * M + i], c);
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        const size_t g = ((size_t)b * 3 + a) * M + i;
        const unsigned long long u = s_lo[a * M + i];
        const unsigned long long old = atomicAdd(&sum_lo[g], u);
        const int h = s_hi[a * M + i] + (int)(old + u < old);
        if (h) atomicAdd(&sum_hi[g], (unsigned)h);                 // modulo 2^32: only the final value must fit
      }
    }
  }
}

// round_f32(hi * 2^64 + lo), correctly rounded: the magnitude is cut to its top 64 bits with a sticky bit for the rest
// (|value| < 2^94: fewer than 2^31 points of |x * 2^24| < 2^63)
__device__ __forceinline__ float wide_to_float(long long hi, unsigned long long lo) {
  const bool neg = hi < 0;
  if (neg) { lo = ~lo + 1ull; hi = ~hi + (lo == 0ull ? 1 : 0); }
  float f;
  if (hi == 0) {
    f = __ull2float_rn(lo);
  } else {
    const int s = 64 - __clzll(hi);                  // 1..31: shift the 96-bit magnitude right by s
    const unsigned long long m = ((unsigned long long)hi << (64 - s)) | (lo >> s) | ((lo << (64 - s)) != 0ull ? 1ull : 0ull);
    f = __fmul_rn(__ull2float_rn(m), __int_as_float((127 + s) << 23));      // exact: a power of two
  }
  return neg ? -f : f;
}

// one thread per sum: the sums' low and high words and the counts start at zero, in one launch
__global__ void cluster_zero_kernel(unsigned long long* __restrict__ sum_lo, unsigned* __restrict__ sum_hi,
                                    int32_t* __restrict__ count, int sums, int counts) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < sums) { sum_lo[i] = 0ull; sum_hi[i] = 0u; }
  if (i < counts) count[i] = 0;
}

// one thread per (b, axis, node); hi_then_mean holds the high words on entry and the means (as float bits) on exit
__global__ void cluster_mean_kernel(const unsigned long long* __restrict__ sum_lo, const int32_t* __restrict__ count,
                                    int M, int total, int32_t* __restrict__ hi_then_mean) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int m = i % M, b = i / (3 * M);
  const float num = __fmul_rn(wide_to_float(hi_then_mean[i], sum_lo[i]), 0x1p-24f);     // exact: a power of two
  hi_then_mean[i] = __float_as_int(__fdiv_rn(num, __fadd_rn((float)count[(size_t)b * M + m], 1e-5f)));
}

// one thread per (b, n)
__global__ void cluster_decenter_kernel(const float* __restrict__ pc, const int32_t* __restrict__ min_idx,
                                        const float* __restrict__ mean, int N, int M, float* __restrict__ centers,
                                        float* __restrict__ decentered) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (n >= N) return;
  const int m = min_idx[(size_t)b * N + n];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const size_t i = ((size_t)b * 3 + a) * N + n;
    const float c = mean[((size_t)b * 3 + a) * M + m];
    if (centers) centers[i] = c;
    if (decentered) decentered[i] = __fsub_rn(pc[i], c);
  }
}

}  // namespace dib

extern "C" {

size_t cluster_assign_workspace_bytes(int B, int M) {
  if (B <= 0 || M <= 0) return 0;
  return (size_t)B * 3 * (size_t)M * sizeof(unsigned long long);          // the low words of the sums
}

// pc [B][3][N] f32, node [B][3][M] f32 [dev]; outputs [dev]: min_k_idx [B][N][k] i32, min_idx [B][N] i32,
// count [B][M] i32, cluster_mean [B][3][M] f32, pc_centers / pc_decentered [B][3][N] f32 (either may be
// NULL).  1 <= k <= min(8, M), M <= 2048.
int cluster_assign_forward(const float* pc, const float* node, int B, int N, int M, int k, int32_t* min_k_idx,
                           int32_t* min_idx, int32_t* count, float* cluster_mean, float* pc_centers,
                           float* pc_decentered, void* workspace, size_t workspace_bytes, dib_stream_t stream_) {
  using namespace dib;
  cudaStream_t stream = (cudaStream_t)stream_;
  DIB_REQUIRE(B >= 0 && N >= 0 && M >= 1 && M <= kCaMaxNodes, "cluster_assign: need 1 <= M <= 2048");
  DIB_REQUIRE(k >= 1 && k <= kCaMaxK && k <= M, "cluster_assign: need 1 <= k <= min(8, M)");
  if (B == 0) return DIB_OK;
  DIB_REQUIRE(node && count && cluster_mean && (N == 0 || (pc && min_k_idx && min_idx)), "cluster_assign: NULL argument");
  DIB_REQUIRE(B <= 65535, "cluster_assign: B <= 65535");
  const size_t need = cluster_assign_workspace_bytes(B, M);
  DIB_REQUIRE(workspace && workspace_bytes >= need && ((uintptr_t)workspace & 7) == 0,
              "cluster_assign: workspace too small or misaligned");
  // The high words of the sums are 32-bit: |sum| < 2^31 points x 2^63 < 2^94, so the final high word is below 2^30 in
  // magnitude, and additions modulo 2^32 reach it exactly.  They live in cluster_mean, which has one 4-byte element
  // per sum, until cluster_mean_kernel replaces each with its mean.
  unsigned long long* sum_lo = (unsigned long long*)workspace;
  unsigned* sum_hi = reinterpret_cast<unsigned*>(cluster_mean);
  const int total = B * 3 * M;
  cluster_zero_kernel<<<(total + 255) / 256, 256, 0, stream>>>(sum_lo, sum_hi, count, total, B * M);
  DIB_CHECK_CUDA(cudaGetLastError());
  constexpr size_t kSmemPerNode = 3 * sizeof(unsigned long long) + 3 * sizeof(float) + 3 * sizeof(int) + sizeof(int);
  if (N > 0) {
    const size_t smem = (size_t)M * kSmemPerNode;
    const int per_cta = kCaThreads * kCaPointsPerThread;
    dim3 grid((N + per_cta - 1) / per_cta, B);
#define DIB_CA_LAUNCH(KK)                                                                                         \
  case KK:                                                                                                        \
    if (smem > 48 * 1024)                                                                                         \
      DIB_CHECK_CUDA(cudaFuncSetAttribute(cluster_assign_kernel<KK>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                          (int)(kCaMaxNodes * kSmemPerNode)));                                    \
    cluster_assign_kernel<KK><<<grid, kCaThreads, smem, stream>>>(pc, node, N, M, min_k_idx, min_idx, count, sum_lo, \
                                                                  sum_hi);                                        \
    break;
    switch (k) {
      DIB_CA_LAUNCH(1) DIB_CA_LAUNCH(2) DIB_CA_LAUNCH(3) DIB_CA_LAUNCH(4)
      DIB_CA_LAUNCH(5) DIB_CA_LAUNCH(6) DIB_CA_LAUNCH(7) DIB_CA_LAUNCH(8)
    }
#undef DIB_CA_LAUNCH
    DIB_CHECK_CUDA(cudaGetLastError());
  }
  cluster_mean_kernel<<<(total + 255) / 256, 256, 0, stream>>>(sum_lo, count, M, total,
                                                               reinterpret_cast<int32_t*>(cluster_mean));
  DIB_CHECK_CUDA(cudaGetLastError());
  if (N > 0 && (pc_centers || pc_decentered)) {
    dim3 grid((N + 255) / 256, B);
    cluster_decenter_kernel<<<grid, 256, 0, stream>>>(pc, min_idx, cluster_mean, N, M, pc_centers, pc_decentered);
    DIB_CHECK_CUDA(cudaGetLastError());
  }
  return DIB_OK;
}

}  // extern "C"
