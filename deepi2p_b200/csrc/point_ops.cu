// index_max (segmented arg-max) and ball_query (first-K-within-radius) for sm_90a.
//
// index_max replaces models/index_max_ext/index_max_cuda.cu:30-62 (one thread per (b,c) scanning
// N floats with stride C*N between neighbouring threads).  Here a CTA owns (b, a group of
// channels): the cluster-id row index[b,:] is loaded once per group, data rows are streamed with
// coalesced 128-bit loads, and the per-segment winner is kept in shared memory as a 64-bit key
// (order-preserving float bits << 32 | ~n) under atomicMax -- max over a total order is
// independent of arrival order, so the result is deterministic and equals the reference's
// "strict > in ascending n" scan: largest value, lowest n on ties, values <= -1000 and NaN never
// win, untouched segments stay 0.
//
// ball_query replaces models/ball_query_ext/ball_query_cuda.cu:11-50 (one thread per (b,m) row).
// Here a warp owns a row: coalesced loads, ballot + popc ordered compaction, early exit once K
// hits are found, then the reference's padding rule (none -> 0, fewer -> cyclic repeat).
#include "common.cuh"
#include "feature_type.cuh"

namespace dib {

constexpr int kImThreads = 128;     // 4096 (b, channel-group) CTAs' worth of work stays co-resident: no wave tail

__device__ __forceinline__ uint32_t ordered_bits(float v) {
  const uint32_t b = __float_as_uint(v + 0.0f);   // -0 -> +0 so that -0 == +0 as in float compare
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// Common path: one shared-memory load and one float compare.  bestf is only a FILTER: it is updated
// with plain (racy) stores, so it may lag behind the true running maximum, which merely lets a few
// extra candidates through; the winner is decided by the 64-bit atomicMax on bestk alone.
// `>=` lets equal values through (a tie must still be able to win with a lower n); NaN fails it.
template <int CPB>
__device__ __forceinline__ void im_consider(float* bestf, unsigned long long* bestk, int K, int c, int k,
                                            float v, uint32_t n) {
  float* pf = bestf + c * K + k;
  if (v >= *pf) {
    if (!(v > -1000.0f)) return;                  // the floor itself never wins (strict > in the reference)
    *pf = v;
    atomicMax(bestk + c * K + k,
              ((unsigned long long)ordered_bits(v) << 32) | (unsigned long long)(0xFFFFFFFFu - n));
  }
}

// Four consecutive elements of a row as floats: one 128-bit load of float, one 64-bit load of bf16 (widened exactly).
__device__ __forceinline__ float4 ldg4(const float* row, int i) { return __ldg(reinterpret_cast<const float4*>(row) + i); }
__device__ __forceinline__ float4 ldcs4(const float* row, int i) {
  return __ldcs(reinterpret_cast<const float4*>(row) + i);
}
__device__ __forceinline__ float4 widen4(uint2 u) {
  return make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xFFFF0000u), __uint_as_float(u.y << 16),
                     __uint_as_float(u.y & 0xFFFF0000u));
}
__device__ __forceinline__ float4 ldg4(const bf16* row, int i) {
  return widen4(__ldg(reinterpret_cast<const uint2*>(row) + i));
}
__device__ __forceinline__ float4 ldcs4(const bf16* row, int i) {
  return widen4(__ldcs(reinterpret_cast<const uint2*>(row) + i));
}

// grid = (ceil(C / CPB), B); dynamic smem = CPB * K * 12 bytes.  T = float or bf16: the values are compared as floats.
template <int CPB, bool VEC, typename T>
__global__ void __launch_bounds__(kImThreads) index_max_kernel(const T* __restrict__ data,
                                                               const int32_t* __restrict__ index,
                                                               int32_t* __restrict__ out, int B, int C, int N, int K) {
  extern __shared__ __align__(16) unsigned char im_smem[];
  unsigned long long* bestk = reinterpret_cast<unsigned long long*>(im_smem);
  float* bestv = reinterpret_cast<float*>(bestk + (size_t)CPB * K);
  const int b = blockIdx.y;
  const int c0 = blockIdx.x * CPB;
  const int nc = min(CPB, C - c0);
  for (int i = threadIdx.x; i < CPB * K; i += kImThreads) { bestk[i] = 0ull; bestv[i] = -1000.0f; }
  __syncthreads();
  const int32_t* idx = index + (size_t)b * N;
  const T* rows = data + ((size_t)b * C + c0) * N;

  if (VEC) {
    const int n4 = N >> 2;
    // Pre-pass over the first 1/16 of the row: seed the filter thresholds with plain (racy) stores.
    // All threads scan "in parallel", so without it the thresholds lag and ~13 % of the elements
    // (instead of ~1 %) would take the divergent slow path (measured: 24 instructions / element).
    // Every threshold is the value of a real element of its segment, so it can never exceed the
    // segment maximum, and the main pass below re-scans these elements with the full logic.
    {
      const int npre = n4 >> 4;
      for (int i = threadIdx.x; i < npre; i += kImThreads) {
        const int4 kk = __ldg(reinterpret_cast<const int4*>(idx) + i);
        const int k4[4] = {kk.x, kk.y, kk.z, kk.w};
#pragma unroll
        for (int c = 0; c < CPB; ++c) {
          if (c < nc) {
            const float4 v = ldg4(rows + (size_t)c * N, i);
            const float v4[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              if ((unsigned)k4[j] < (unsigned)K) {
                float* pf = bestv + c * K + k4[j];
                if (v4[j] > *pf) *pf = v4[j];
              }
            }
          }
        }
      }
      __syncthreads();
    }
    // software pipeline: the loads of iteration i + 1 are in flight while iteration i is scanned
    int i = threadIdx.x;
    int4 kk = make_int4(0, 0, 0, 0);
    float4 vv[CPB];
    if (i < n4) {
      kk = __ldg(reinterpret_cast<const int4*>(idx) + i);
#pragma unroll
      for (int c = 0; c < CPB; ++c)
        if (c < nc) vv[c] = ldcs4(rows + (size_t)c * N, i);
    }
    while (i < n4) {
      const int inext = i + kImThreads;
      int4 kn = make_int4(0, 0, 0, 0);
      float4 vn[CPB];
      if (inext < n4) {
        kn = __ldg(reinterpret_cast<const int4*>(idx) + inext);
#pragma unroll
        for (int c = 0; c < CPB; ++c)
          if (c < nc) vn[c] = ldcs4(rows + (size_t)c * N, inext);
      }
      const uint32_t n = (uint32_t)i << 2;
#pragma unroll
      for (int c = 0; c < CPB; ++c) {
        if (c < nc) {
          if ((unsigned)kk.x < (unsigned)K) im_consider<CPB>(bestv, bestk, K, c, kk.x, vv[c].x, n);
          if ((unsigned)kk.y < (unsigned)K) im_consider<CPB>(bestv, bestk, K, c, kk.y, vv[c].y, n + 1);
          if ((unsigned)kk.z < (unsigned)K) im_consider<CPB>(bestv, bestk, K, c, kk.z, vv[c].z, n + 2);
          if ((unsigned)kk.w < (unsigned)K) im_consider<CPB>(bestv, bestk, K, c, kk.w, vv[c].w, n + 3);
        }
      }
      kk = kn;
#pragma unroll
      for (int c = 0; c < CPB; ++c) vv[c] = vn[c];
      i = inext;
    }
  } else {
    for (int i = threadIdx.x; i < N; i += kImThreads) {
      const int k = __ldg(idx + i);
      if ((unsigned)k >= (unsigned)K) continue;
#pragma unroll
      for (int c = 0; c < CPB; ++c)
        if (c < nc) im_consider<CPB>(bestv, bestk, K, c, k, load_f32(__ldcs(rows + (size_t)c * N + i)), (uint32_t)i);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nc * K; i += kImThreads) {
    const unsigned long long key = bestk[i];
    out[((size_t)b * C + c0) * K + i] = key ? (int32_t)(0xFFFFFFFFu - (uint32_t)(key & 0xFFFFFFFFull)) : 0;
  }
}

constexpr int kBqWarps = 8;
constexpr int kBqUnroll = 32;       // 4 KB per warp in flight

// One warp per (b,m) row.  Two register buffers of kBqHalf loads per lane: the next 512 elements are
// in flight while the current 512 are compacted.
constexpr int kBqHalf = kBqUnroll / 2;

__device__ __forceinline__ void bq_load(const float* d, int base, int N, int lane, float v[kBqHalf]) {
#pragma unroll
  for (int j = 0; j < kBqHalf; ++j) {
    const int n = base + j * 32 + lane;
    v[j] = (n < N) ? __ldcs(d + n) : __int_as_float(0x7fc00000);   // NaN never hits
  }
}

__device__ __forceinline__ void bq_scan(const float v[kBqHalf], float radius, int base, int lane, int K, int32_t* o,
                                        int& cnt) {
#pragma unroll
  for (int j = 0; j < kBqHalf; ++j) {
    const bool hit = v[j] <= radius;
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    if (m) {                                       // warp-uniform; hits are rare
      if (hit) {
        const int pos = cnt + __popc(m & ((1u << lane) - 1u));
        if (pos < K) o[pos] = base + j * 32 + lane;
      }
      cnt += __popc(m);
    }
  }
}

__global__ void __launch_bounds__(kBqWarps * 32) ball_query_kernel(const float* __restrict__ dist, float radius,
                                                                   int32_t* __restrict__ out, long long rows, int N,
                                                                   int K) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * kBqWarps + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* d = dist + (size_t)row * N;
  int32_t* o = out + (size_t)row * K;
  constexpr int kStep = 32 * kBqHalf;
  int cnt = 0;
  float va[kBqHalf], vb[kBqHalf];
  bq_load(d, 0, N, lane, va);
  for (int base = 0; base < N && cnt < K; base += 2 * kStep) {
    if (base + kStep < N) bq_load(d, base + kStep, N, lane, vb);
    bq_scan(va, radius, base, lane, K, o, cnt);
    if (cnt >= K || base + kStep >= N) break;
    if (base + 2 * kStep < N) bq_load(d, base + 2 * kStep, N, lane, va);
    bq_scan(vb, radius, base + kStep, lane, K, o, cnt);
  }
  __syncwarp();
  if (cnt == 0) {
    for (int i = lane; i < K; i += 32) o[i] = 0;
  } else if (cnt < K) {
    for (int i = lane; i < K - cnt; i += 32) o[cnt + i] = o[i % cnt];   // sources are all < cnt: never overwritten
  }
}

// 128-bit variant of bq_load / bq_scan for 16-byte aligned rows: kBqVec float4 per lane = 512 elements per warp and
// half, lane l holding elements 4l .. 4l+3 of each 128-element block.  Hits are rare (K of N), so the common block
// costs four compares, four ballots and one warp-uniform branch; only a block with a hit computes positions: the
// hits of lower lanes (all four components) come first, then this lane's own lower components -- index order.
constexpr int kBqVec = kBqHalf / 4;

__device__ __forceinline__ void bq_load4(const float4* d4, int lane, float4 v[kBqVec]) {
#pragma unroll
  for (int j = 0; j < kBqVec; ++j) v[j] = __ldcs(d4 + j * 32 + lane);
}

__device__ __forceinline__ void bq_scan4(const float4 v[kBqVec], float radius, int base, int lane, int K, int32_t* o,
                                         int& cnt) {
#pragma unroll
  for (int j = 0; j < kBqVec; ++j) {
    const bool h0 = v[j].x <= radius, h1 = v[j].y <= radius, h2 = v[j].z <= radius, h3 = v[j].w <= radius;
    const unsigned m0 = __ballot_sync(0xffffffffu, h0), m1 = __ballot_sync(0xffffffffu, h1);
    const unsigned m2 = __ballot_sync(0xffffffffu, h2), m3 = __ballot_sync(0xffffffffu, h3);
    if (m0 | m1 | m2 | m3) {                       // warp-uniform
      const unsigned lt = (1u << lane) - 1u;
      int pos = cnt + __popc(m0 & lt) + __popc(m1 & lt) + __popc(m2 & lt) + __popc(m3 & lt);
      const int e = base + j * 128 + lane * 4;
      if (h0) { if (pos < K) o[pos] = e; ++pos; }
      if (h1) { if (pos < K) o[pos] = e + 1; ++pos; }
      if (h2) { if (pos < K) o[pos] = e + 2; ++pos; }
      if (h3) { if (pos < K) o[pos] = e + 3; }
      cnt += __popc(m0) + __popc(m1) + __popc(m2) + __popc(m3);
    }
  }
}

// Row split over the 4 warps of a CTA (one CTA per row): each warp compacts its quarter of the row
// into its own shared-memory list (at most K hits), then the lists are concatenated in order.  Four
// times as many independent load streams as the warp-per-row kernel; used when 4 K ints fit in
// shared memory.  A later quarter cannot know that earlier quarters already hold K hits, so rows
// whose K-th hit comes early read more than they strictly need.
constexpr int kBqSplit = 4;

template <bool VEC>
__global__ void __launch_bounds__(kBqSplit * 32) ball_query_split_kernel(const float* __restrict__ dist, float radius,
                                                                         int32_t* __restrict__ out, int N, int K) {
  extern __shared__ int32_t bq_hits[];          // [kBqSplit][K]
  __shared__ int bq_cnt[kBqSplit];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const float* d = dist + (size_t)blockIdx.x * N;
  int32_t* o = out + (size_t)blockIdx.x * K;
  // quarter boundaries on multiples of 32 elements
  const int per = (((N + kBqSplit - 1) / kBqSplit) + 31) & ~31;
  const int lo = min(w * per, N), hi = min(lo + per, N);
  int32_t* mine = bq_hits + w * K;
  constexpr int kStep = 32 * kBqHalf;
  int cnt = 0;
  if (VEC) {
    // quarters are whole multiples of kStep elements and 16-byte aligned (checked by the host)
    float4 va[kBqVec], vb[kBqVec];
    if (lo < hi) {
      const float4* d4 = reinterpret_cast<const float4*>(d);
      bq_load4(d4 + (lo >> 2), lane, va);
      for (int base = lo; base < hi && cnt < K; base += 2 * kStep) {
        if (base + kStep < hi) bq_load4(d4 + ((base + kStep) >> 2), lane, vb);
        bq_scan4(va, radius, base, lane, K, mine, cnt);
        if (cnt >= K || base + kStep >= hi) break;
        if (base + 2 * kStep < hi) bq_load4(d4 + ((base + 2 * kStep) >> 2), lane, va);
        bq_scan4(vb, radius, base + kStep, lane, K, mine, cnt);
      }
    }
  } else {
    float va[kBqHalf], vb[kBqHalf];
    if (lo < hi) {
      bq_load(d, lo, hi, lane, va);
      for (int base = lo; base < hi && cnt < K; base += 2 * kStep) {
        if (base + kStep < hi) bq_load(d, base + kStep, hi, lane, vb);
        bq_scan(va, radius, base, lane, K, mine, cnt);
        if (cnt >= K || base + kStep >= hi) break;
        if (base + 2 * kStep < hi) bq_load(d, base + 2 * kStep, hi, lane, va);
        bq_scan(vb, radius, base + kStep, lane, K, mine, cnt);
      }
    }
  }
  if (lane == 0) bq_cnt[w] = min(cnt, K);
  __syncthreads();
  int start = 0, total = 0;
#pragma unroll
  for (int q = 0; q < kBqSplit; ++q) { if (q < w) start += bq_cnt[q]; total += bq_cnt[q]; }
  const int have = min(total, K);
  for (int i = lane; i < bq_cnt[w]; i += 32)
    if (start + i < K) o[start + i] = mine[i];
  __syncthreads();                              // the first `have` outputs are in place (block-visible)
  if (have == 0) {
    for (int i = threadIdx.x; i < K; i += kBqSplit * 32) o[i] = 0;
  } else if (have < K) {
    for (int i = threadIdx.x; i < K - have; i += kBqSplit * 32) o[have + i] = o[i % have];
  }
}

// index_max_forward's launch for float or bf16 data (cluster_pool_forward_* launch it too)
template <typename T>
int index_max_launch(const T* data, const int32_t* index, int32_t* out, int B, int C, int N, int K,
                     dib_stream_t stream) {
  DIB_REQUIRE(data && index && out, "NULL argument");
  DIB_REQUIRE(B >= 0 && C >= 0 && N >= 0 && K >= 1, "bad shape B=%d C=%d N=%d K=%d", B, C, N, K);
  DIB_REQUIRE(B <= 65535, "B too large for grid.y");
  if (B == 0 || C == 0) return DIB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const bool vec = (N % 4 == 0) && ((uintptr_t)data % (4 * sizeof(T)) == 0) && ((uintptr_t)index % 16 == 0);
  const size_t per_c = (size_t)K * 12;
  const size_t limit = 227 * 1024;
  int cpb = 4;
  while (cpb > 1 && per_c * cpb > limit) cpb >>= 1;
  DIB_REQUIRE(per_c * cpb <= limit, "K=%d too large for the shared-memory segment table", K);
  const size_t smem = per_c * cpb;
  dim3 grid((C + cpb - 1) / cpb, B);
#define DIB_IM_LAUNCH(CPB, VEC)                                                                              \
  do {                                                                                                       \
    auto kern = index_max_kernel<CPB, VEC, T>;                                                               \
    DIB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));      \
    kern<<<grid, kImThreads, smem, st>>>(data, index, out, B, C, N, K);                                      \
  } while (0)
  if (cpb == 4) { if (vec) DIB_IM_LAUNCH(4, true); else DIB_IM_LAUNCH(4, false); }
  else if (cpb == 2) { if (vec) DIB_IM_LAUNCH(2, true); else DIB_IM_LAUNCH(2, false); }
  else { if (vec) DIB_IM_LAUNCH(1, true); else DIB_IM_LAUNCH(1, false); }
#undef DIB_IM_LAUNCH
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}
template int index_max_launch<float>(const float*, const int32_t*, int32_t*, int, int, int, int, dib_stream_t);
template int index_max_launch<bf16>(const bf16*, const int32_t*, int32_t*, int, int, int, int, dib_stream_t);

}  // namespace dib

extern "C" {

int index_max_forward(const float* data, const int32_t* index, int32_t* out, int B, int C, int N, int K,
                      dib_stream_t stream) {
  return dib::index_max_launch(data, index, out, B, C, N, K, stream);
}

int ball_query_forward(const float* dist, float radius, int32_t* out, int B, int M, int N, int K,
                       dib_stream_t stream) {
  using namespace dib;
  DIB_REQUIRE(dist && out, "NULL argument");
  DIB_REQUIRE(B >= 0 && M >= 0 && N >= 0 && K >= 1, "bad shape B=%d M=%d N=%d K=%d", B, M, N, K);
  const long long rows = (long long)B * M;
  if (rows == 0) return DIB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t split_smem = (size_t)kBqSplit * K * sizeof(int32_t);
  if (split_smem <= 32 * 1024 && N >= 4096 && rows < (1ll << 31)) {
    // 128-bit loads when every quarter of every row is a 16-byte aligned whole number of 512-element steps
    const bool vec = (N % (kBqSplit * 32 * kBqHalf) == 0) && ((uintptr_t)dist % 16 == 0);
    if (vec) ball_query_split_kernel<true><<<(unsigned)rows, kBqSplit * 32, split_smem, st>>>(dist, radius, out, N, K);
    else ball_query_split_kernel<false><<<(unsigned)rows, kBqSplit * 32, split_smem, st>>>(dist, radius, out, N, K);
  } else {
    const long long blocks = (rows + kBqWarps - 1) / kBqWarps;
    DIB_REQUIRE(blocks < (1ll << 31), "too many rows");
    ball_query_kernel<<<(unsigned)blocks, kBqWarps * 32, 0, st>>>(dist, radius, out, rows, N, K);
  }
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

}  // extern "C"
