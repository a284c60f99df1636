// The K nearest nodes of one point by cluster_assign's key, shared by cluster_assign.cu (K <= 8) and encoder_ops.cu
// (the node kNN grouping, K <= 32).
//
//   key d2 = ((dx*dx + dy*dy) + dz*dz), float32 without fma, d = point - node; ties -> lower node index; +inf after
//   every finite key and NaN after +inf, so the K slots always hold K distinct nodes (K <= M).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

namespace dib {

constexpr unsigned kCaNanKey = 0x7f800001u;         // every NaN d2 maps here: after +inf (0x7f800000)

// The K nearest nodes of (x, y, z) by (key, node index), nearest first.  kAll = false keys on the float d2 and keeps
// finite ones only: one compare per node, and enough unless fewer than K distances are finite, which the return value
// reports.  kAll = true keys on the bits of d2 (never negative, so the bit order is the value order) with every NaN
// clamped to kCaNanKey, just above +inf; the empty slots' key is above every node's, so every node has a place.
// s_node holds the nodes as [3][M].
template <int K, bool kAll>
__device__ __forceinline__ bool nearest_k(float x, float y, float z, const float* s_node, int M, int (&bi)[K]) {
  using Key = typename std::conditional<kAll, unsigned, float>::type;
  Key bd[K];
#pragma unroll
  for (int j = 0; j < K; ++j) {
    if constexpr (kAll) bd[j] = 0xffffffffu; else bd[j] = __int_as_float(0x7f800000);
    bi[j] = j;
  }
#pragma unroll 4
  for (int m = 0; m < M; ++m) {
    const float dx = __fsub_rn(x, s_node[m]), dy = __fsub_rn(y, s_node[M + m]), dz = __fsub_rn(z, s_node[2 * M + m]);
    const float f = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
    Key d2;
    if constexpr (kAll) d2 = min(__float_as_uint(f), kCaNanKey); else d2 = f;
    if (!(d2 < bd[K - 1])) continue;                  // strict: on a tie the earlier (lower) node stays
    // sorted insert from the back; all indices are compile-time, so bd / bi stay in registers
#pragma unroll
    for (int j = K - 1; j >= 1; --j) {
      const bool shift = d2 < bd[j - 1];
      const bool here = !shift && d2 < bd[j];
      bd[j] = shift ? bd[j - 1] : (here ? d2 : bd[j]);
      bi[j] = shift ? bi[j - 1] : (here ? m : bi[j]);
    }
    if (d2 < bd[0]) { bd[0] = d2; bi[0] = m; }
  }
  if constexpr (kAll) return true; else return bd[K - 1] < __int_as_float(0x7f800000);
}

// knn_idx [B][M][K] int32: nearest_k of every query [B][3][M] among the database [B][3][N], K <= min(32, N) <= 2048
// (encoder_ops.cu's knn_search_kernel, launched on `stream`).  knn_group and knn_fusion group by these indices.
int knn_search_launch(const float* query, const float* database, int B, int M, int N, int K, int32_t* knn_idx,
                      cudaStream_t stream);

}  // namespace dib
