// nuScenes dataset list (data/nuscenes/make_datasets.py: search_nearby_cameras) for E kept LIDAR_TOP sweeps at once.
// DESIGN.md 4.28 states the contract.
//
//   count: one thread per (entry, camera, direction) walk follows the camera's next / prev chain from its first
//          neighbour, tests each later record against the radius and counts the records it appends;
//   scan:  an exclusive scan of the counts into int64 offsets (block sums, one block scanning them, block rescans);
//   fill:  the same walks again, writing the appended records' sample_data indices at their offsets.
//
// Each step evaluates t_lc = rows 0-2 of inv(P_l) (t_c, 1) and its norm in fp64 together with a bound on how far any
// summation order, with or without FMA, can move the norm (walk_step).  A step whose norm is within the bound of
// max_translation is not decided here: the walk stops with status DIB_NSW_DEFERRED and the host resumes it with numpy.
// No atomics; the decisions depend on the inputs alone, so two runs give the same bits.
#include <math.h>

#include "common.cuh"

namespace dib {
namespace {

constexpr int kWalkThreads = 128;
constexpr int kScanThreads = 1024;
constexpr int kCameras = 6;

// gamma_4 = 4u / (1 - 4u), u = 2^-53, rounded up: the relative error bound of a sum of four rounded products in any
// order (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., 3.1 and 4.2).
constexpr double kGamma4 = 4.440892098500632e-16;

enum Step { kAppend = 0, kStop = 1, kDefer = 2 };

// One candidate: t_i = ((a_i0 + a_i1) + a_i2) + a_i3 with a_ij = inv_ij p_j, p = (t_c, 1); N = sqrt((t0 t0 + t1 t1) +
// t2 t2).  numpy's dgemm / ddot may sum in another order and contract products into FMAs; DESIGN.md 4.28 shows
// |N_numpy - N| <= 4 gamma_4 (sum_ij |a_ij| + N), so outside that distance of max_translation both decide alike.  A
// non-finite N or bound is deferred as well.
__device__ __forceinline__ Step walk_step(const double (&inv)[12], const float* __restrict__ trans, int32_t cand,
                                          double max_translation) {
  const double p0 = trans[3 * (int64_t)cand], p1 = trans[3 * (int64_t)cand + 1], p2 = trans[3 * (int64_t)cand + 2];
  double t[3], s = 0.0;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const double a0 = inv[4 * i] * p0, a1 = inv[4 * i + 1] * p1, a2 = inv[4 * i + 2] * p2, a3 = inv[4 * i + 3];
    t[i] = ((a0 + a1) + a2) + a3;
    s += ((fabs(a0) + fabs(a1)) + fabs(a2)) + fabs(a3);
  }
  const double n = sqrt((t[0] * t[0] + t[1] * t[1]) + t[2] * t[2]);
  const double bound = 4.0 * kGamma4 * (s + n);
  if (!(fabs(n - max_translation) > bound)) return kDefer;   // also NaN and infinite norms or bounds
  return n < max_translation ? kAppend : kStop;
}

// Lane w = 2 (e C + c) + d.  The own record is never tested; the first neighbour is walked over but never tested or
// appended; each later record is appended while walk_step says so.
template <bool kFill>
__global__ void __launch_bounds__(kWalkThreads) walk_kernel(const int32_t* __restrict__ next,
                                                            const int32_t* __restrict__ prev,
                                                            const float* __restrict__ trans, int32_t n_sd,
                                                            const int32_t* __restrict__ own,
                                                            const double* __restrict__ inv_rows, int W,
                                                            double max_translation, int32_t* __restrict__ counts,
                                                            int32_t* __restrict__ status,
                                                            const int64_t* __restrict__ offsets,
                                                            int32_t* __restrict__ tokens) {
  const int w = blockIdx.x * kWalkThreads + threadIdx.x;
  if (w >= W) return;
  const int32_t* __restrict__ link = (w & 1) ? prev : next;
  const int64_t ec = w >> 1, e = ec / kCameras;
  double inv[12];
#pragma unroll
  for (int k = 0; k < 12; ++k) inv[k] = inv_rows[12 * e + k];
  int32_t* out = kFill ? tokens + offsets[w] : nullptr;
  int32_t cur = own[ec], count = 0, st = DIB_NSW_DONE;
  if (cur < 0 || cur >= n_sd) {
    st = DIB_NSW_BAD_LINK;
  } else {
    cur = link[cur];                                   // the first neighbour
    if (cur < -1 || cur >= n_sd) st = DIB_NSW_BAD_LINK;
    for (int32_t steps = 0; st == DIB_NSW_DONE && cur >= 0;) {
      const int32_t cand = link[cur];
      if (cand == -1) break;
      if (cand < -1 || cand >= n_sd) {
        st = DIB_NSW_BAD_LINK;
        break;
      }
      if (++steps > n_sd) {                            // a cycle in the chain
        st = DIB_NSW_CYCLE;
        break;
      }
      const Step r = walk_step(inv, trans, cand, max_translation);
      if (r == kDefer) st = DIB_NSW_DEFERRED;
      if (r != kAppend) break;
      if (kFill) out[count] = cand;
      ++count;
      cur = cand;
    }
  }
  if (!kFill) {
    counts[w] = count;
    status[w] = st;
  }
}

// Inclusive scan of one value per thread over the block (blockDim.x == kScanThreads); returns it and leaves the block
// total in *total.
__device__ int64_t block_inclusive_scan(int64_t v, int64_t* s_warp, int64_t* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int64_t u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += u;
  }
  if (lane == 31) s_warp[wid] = v;
  __syncthreads();
  if (wid == 0) {
    int64_t x = s_warp[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t u = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += u;
    }
    s_warp[lane] = x;
  }
  __syncthreads();
  const int64_t r = v + (wid ? s_warp[wid - 1] : 0);
  *total = s_warp[31];
  __syncthreads();
  return r;
}

__global__ void __launch_bounds__(kScanThreads) block_sum_kernel(const int32_t* __restrict__ counts, int W,
                                                                 int64_t* __restrict__ partial) {
  __shared__ int64_t s_warp[32];
  const int i = blockIdx.x * kScanThreads + threadIdx.x;
  int64_t total;
  block_inclusive_scan(i < W ? counts[i] : 0, s_warp, &total);
  if (threadIdx.x == 0) partial[blockIdx.x] = total;
}

// One block: partial[b] becomes the exclusive prefix of the block sums; offsets[W] the grand total.
__global__ void __launch_bounds__(kScanThreads) partial_scan_kernel(int64_t* __restrict__ partial, int nb, int W,
                                                                    int64_t* __restrict__ offsets) {
  __shared__ int64_t s_warp[32];
  int64_t carry = 0;
  for (int base = 0; base < nb; base += kScanThreads) {
    const int i = base + threadIdx.x;
    const int64_t v = i < nb ? partial[i] : 0;
    int64_t total;
    const int64_t inc = block_inclusive_scan(v, s_warp, &total);
    if (i < nb) partial[i] = carry + inc - v;
    carry += total;
  }
  if (threadIdx.x == 0) offsets[W] = carry;
}

__global__ void __launch_bounds__(kScanThreads) offsets_kernel(const int32_t* __restrict__ counts, int W,
                                                               const int64_t* __restrict__ partial,
                                                               int64_t* __restrict__ offsets) {
  __shared__ int64_t s_warp[32];
  const int i = blockIdx.x * kScanThreads + threadIdx.x;
  const int64_t v = i < W ? counts[i] : 0;
  int64_t total;
  const int64_t inc = block_inclusive_scan(v, s_warp, &total);
  if (i < W) offsets[i] = partial[blockIdx.x] + inc - v;
}

int check_walk_args(const int32_t* next, const int32_t* prev, const float* trans, int64_t n_sd, const int32_t* own,
                    const double* inv_rows, int E, double max_translation) {
  DIB_REQUIRE(E >= 0 && (int64_t)E * kCameras * 2 < INT32_MAX, "E must be in [0, (2^31 - 1) / 12) (got %d)", E);
  DIB_REQUIRE(n_sd >= 0 && n_sd < INT32_MAX, "n_sd must be in [0, 2^31 - 1) (got %lld)", (long long)n_sd);
  DIB_REQUIRE(isfinite(max_translation) && max_translation >= 0, "max_translation must be finite and >= 0");
  DIB_REQUIRE(E == 0 || (next && prev && trans && own && inv_rows), "a required pointer is null");
  return 0;
}

}  // namespace
}  // namespace dib

using namespace dib;

extern "C" {

int nuscenes_walk_count(const int32_t* next, const int32_t* prev, const float* trans, int64_t n_sd,
                        const int32_t* own, const double* inv_rows, int E, double max_translation, int32_t* counts,
                        int32_t* status, dib_stream_t stream) {
  const int rc = check_walk_args(next, prev, trans, n_sd, own, inv_rows, E, max_translation);
  if (rc) return rc;
  if (E == 0) return 0;
  DIB_REQUIRE(counts && status, "a required pointer is null");
  const int W = E * kCameras * 2;
  walk_kernel<false><<<(W + kWalkThreads - 1) / kWalkThreads, kWalkThreads, 0, (cudaStream_t)stream>>>(
      next, prev, trans, (int32_t)n_sd, own, inv_rows, W, max_translation, counts, status, nullptr, nullptr);
  DIB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

size_t nuscenes_walk_scan_workspace_bytes(int W) {
  if (W < 0) return 0;
  return (size_t)((W + kScanThreads - 1) / kScanThreads) * sizeof(int64_t);
}

int nuscenes_walk_scan(const int32_t* counts, int W, int64_t* offsets, void* workspace, size_t workspace_bytes,
                       dib_stream_t stream) {
  DIB_REQUIRE(W >= 0, "W must be >= 0 (got %d)", W);
  DIB_REQUIRE(offsets && (W == 0 || (counts && workspace)), "a required pointer is null");
  const size_t need = nuscenes_walk_scan_workspace_bytes(W);
  if (workspace_bytes < need) {
    set_error("nuscenes_walk_scan: workspace is %zu bytes, %zu needed", workspace_bytes, need);
    return DIB_ENOMEM;
  }
  cudaStream_t cs = (cudaStream_t)stream;
  if (W == 0) {
    DIB_CHECK_CUDA(cudaMemsetAsync(offsets, 0, sizeof(int64_t), cs));
    return 0;
  }
  const int nb = (W + kScanThreads - 1) / kScanThreads;
  int64_t* partial = (int64_t*)workspace;
  block_sum_kernel<<<nb, kScanThreads, 0, cs>>>(counts, W, partial);
  DIB_CHECK_CUDA(cudaGetLastError());
  partial_scan_kernel<<<1, kScanThreads, 0, cs>>>(partial, nb, W, offsets);
  DIB_CHECK_CUDA(cudaGetLastError());
  offsets_kernel<<<nb, kScanThreads, 0, cs>>>(counts, W, partial, offsets);
  DIB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int nuscenes_walk_fill(const int32_t* next, const int32_t* prev, const float* trans, int64_t n_sd,
                       const int32_t* own, const double* inv_rows, int E, double max_translation,
                       const int64_t* offsets, int32_t* tokens, dib_stream_t stream) {
  const int rc = check_walk_args(next, prev, trans, n_sd, own, inv_rows, E, max_translation);
  if (rc) return rc;
  if (E == 0) return 0;
  DIB_REQUIRE(offsets && tokens, "a required pointer is null");
  const int W = E * kCameras * 2;
  walk_kernel<true><<<(W + kWalkThreads - 1) / kWalkThreads, kWalkThreads, 0, (cudaStream_t)stream>>>(
      next, prev, trans, (int32_t)n_sd, own, inv_rows, W, max_translation, nullptr, nullptr, offsets, tokens);
  DIB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
