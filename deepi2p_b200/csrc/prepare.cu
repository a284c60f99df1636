// On-device front end of the multi-start driver: get_initial_guess (evaluation/registration_lsq.py:196-220)
// and the random perturbed inits (registration_lsq.py:163-164), so that a batch goes from
// (cloud, predicted labels) to solver inputs without a host round-trip.
//
// Per sample (one CTA): mean of the predicted-inside points -> init_y_angle =
// wrap_pi(atan2(mean_z, mean_x) - pi/2); zmin = min over predicted-inside points of the rotated z;
// keep points with rotated z > zmin - 10, order-preserving compaction into the solver's
// device record (xyz f32 SoA + int8 label, tail padded with ignored points); inits
// ry_i = init_y_angle + N(0, sigma), t_i = (0, 0, U(-amp, amp)) from a counter-based Philox4x32-10
// keyed by (seed; sample, init) so that a CPU restatement can reproduce them.
// The reference draws from Python's unseeded `random`, so only the distribution can be matched.
#include <cfloat>
#include <cmath>

#include "common.cuh"

namespace dib {

constexpr int kPrepThreads = 1024;
constexpr int kPrepWarps = kPrepThreads / 32;
constexpr int kSortMax = 32768;          // points sortable in shared memory (32-bit composite keys)
constexpr double kPi = 3.14159265358979323846;

template <typename T, typename Op>
__device__ T block_reduce(T v, T* scratch, Op op) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) scratch[threadIdx.x >> 5] = v;
  __syncthreads();
  T t = scratch[0];
  for (int w = 1; w < kPrepWarps; ++w) t = op(t, scratch[w]);   // fixed order
  return t;
}

__device__ __forceinline__ uint32_t spread6(uint32_t v) {   // 6 bits -> every other bit
  v &= 0x3f;
  v = (v | (v << 4)) & 0x30f;
  v = (v | (v << 2)) & 0x333;
  v = (v | (v << 1)) & 0x555;
  return v;
}

// One stable counting-sort pass over 7 bits of the 16-bit keys (all kPrepThreads threads call).  `in` = current order
// of the point indices (NULL = identity), `out` = the order after this digit.  Warp w owns a contiguous range of the
// input and walks it 32 elements at a time, so equal digits keep their input order (match_any gives the rank among the
// lanes of a tile, the per-(warp, digit) cursor the rank among earlier tiles, the scan the rank among earlier warps).
__device__ void radix_pass(const uint16_t* k16, const uint16_t* in, uint16_t* out, int n, int shift, uint32_t* hist,
                           uint32_t* tot) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < kPrepWarps * 128; i += kPrepThreads) hist[i] = 0u;
  __syncthreads();
  const int R = ((((n + kPrepWarps - 1) / kPrepWarps) + 31) / 32) * 32;
  const int lo = min(warp * R, n), hi = min(lo + R, n);
  for (int j = lo + lane; j < hi; j += 32) {
    const int src = in ? (int)in[j] : j;
    atomicAdd(&hist[warp * 128 + ((k16[src] >> shift) & 127)], 1u);
  }
  __syncthreads();
  if (tid < 128) {                                 // per digit: exclusive prefix over the warps, and the digit's total
    uint32_t sum = 0;
    for (int w = 0; w < kPrepWarps; ++w) { const uint32_t v = hist[w * 128 + tid]; hist[w * 128 + tid] = sum; sum += v; }
    tot[tid] = sum;
  }
  __syncthreads();
  if (tid < 32) {                                  // exclusive scan of the 128 totals (one warp, 4 digits per lane)
    uint32_t v[4], run = 0;
#pragma unroll
    for (int q = 0; q < 4; ++q) { v[q] = tot[4 * tid + q]; run += v[q]; }
    uint32_t inc = run;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
    uint32_t base = inc - run;
#pragma unroll
    for (int q = 0; q < 4; ++q) { tot[4 * tid + q] = base; base += v[q]; }
  }
  __syncthreads();
  if (tid < 128) {
    const uint32_t base = tot[tid];
    for (int w = 0; w < kPrepWarps; ++w) hist[w * 128 + tid] += base;
  }
  __syncthreads();
  const unsigned lt = (1u << lane) - 1u;
  for (int j0 = lo; j0 < hi; j0 += 32) {
    const int j = j0 + lane;
    const bool valid = j < hi;
    const int src = valid ? (in ? (int)in[j] : j) : 0;
    const unsigned d = valid ? ((k16[src] >> shift) & 127u) : (128u + (unsigned)lane);     // invalid lanes match nobody
    const unsigned m = __match_any_sync(0xffffffffu, d);
    const int rank = __popc(m & lt);
    uint32_t base = 0;
    if (valid) base = hist[warp * 128 + d];
    __syncwarp();
    if (valid) {
      out[base + rank] = (uint16_t)src;
      if (rank == 0) hist[warp * 128 + d] = base + (uint32_t)__popc(m);
    }
    __syncwarp();
  }
  __syncthreads();
}

// grid = S.  xyz_in [S][3][n_in_stride] f32, pred [S][n_in_stride] int8, n_in points valid.
// do_sort: order the kept points by (label class, 12-bit Morton cell of (x, z), original index) with an
// in-shared-memory stable radix sort (needs n_in <= kSortMax and radix_smem_bytes(n2) of dynamic shared memory,
// n2 = n_in rounded up to 8); otherwise the original order is kept.
__global__ void __launch_bounds__(kPrepThreads)
    frustum_prepare_kernel(const float* __restrict__ xyz_in, const int8_t* __restrict__ pred, int n_in,
                           int n_in_stride, int n_out_stride, int I, unsigned long long seed, double ry_sigma,
                           double t_amp, int do_sort, int keep_all, int n2, float* __restrict__ xyz_out,
                           int8_t* __restrict__ label_out, int32_t* __restrict__ n_pts, double* __restrict__ init,
                           double* __restrict__ init_y_angle, int32_t* __restrict__ degenerate) {
  extern __shared__ __align__(16) unsigned char prep_smem[];
  // sort scratch (do_sort only): per-warp digit histograms, bucket totals, 16-bit keys and two index arrays
  uint32_t* hist = reinterpret_cast<uint32_t*>(prep_smem);                 // [kPrepWarps][128]
  uint32_t* tot = hist + kPrepWarps * 128;                                 // [128]
  uint16_t* k16 = reinterpret_cast<uint16_t*>(tot + 128);                  // [n2]
  uint16_t* ord1 = k16 + n2;                                               // [n2]
  uint16_t* ord2 = ord1 + n2;                                              // [n2]
  __shared__ double scratch[kPrepWarps];
  __shared__ float fscratch[kPrepWarps];
  __shared__ int iscratch[kPrepWarps];
  __shared__ int warp_cnt[kPrepWarps];
  __shared__ int s_base;
  const int s = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* px = xyz_in + (size_t)s * 3 * n_in_stride;
  const float* py = px + n_in_stride;
  const float* pz = py + n_in_stride;
  const int8_t* lab = pred + (size_t)s * n_in_stride;
  auto dsum = [](double a, double b) { return a + b; };
  auto dmin = [](double a, double b) { return fmin(a, b); };

  // pass 1: mean of predicted-inside points (fixed reduction order)
  double sx = 0, sz = 0, cnt = 0;
  for (int i = tid; i < n_in; i += kPrepThreads)
    if (lab[i] == 1) { sx += (double)px[i]; sz += (double)pz[i]; cnt += 1.0; }
  sx = block_reduce(sx, scratch, dsum); sz = block_reduce(sz, scratch, dsum); cnt = block_reduce(cnt, scratch, dsum);
  // keep_all (frustum_sort_batch_f32): no front filter -- the caller's cloud is only reordered
  const bool degen = !(cnt > 0.0) || keep_all != 0;
  double ang = 0.0;
  if (!degen) {
    double a = atan2(sz / cnt, sx / cnt) - 0.5 * kPi;    // registration_lsq.py:203-207
    a = fmod(a + kPi, 2.0 * kPi);                          // wrap_in_pi, :189-193
    if (a < 0) a += 2.0 * kPi;
    ang = a - kPi;
  }
  double sn, cs;
  sincos(ang, &sn, &cs);

  // pass 2: min rotated z over predicted-inside points (:209-212)
  double zmin = DBL_MAX;
  for (int i = tid; i < n_in; i += kPrepThreads)
    if (lab[i] == 1) zmin = fmin(zmin, -sn * (double)px[i] + cs * (double)pz[i]);
  zmin = block_reduce(zmin, scratch, dmin);
  const double thresh = zmin - 10.0;

  float* ox = xyz_out + (size_t)s * 3 * n_out_stride;
  float* oy = ox + n_out_stride;
  float* oz = oy + n_out_stride;
  int8_t* ol = label_out + (size_t)s * n_out_stride;
  int n_front;

  if (do_sort) {
    // pass 3a: extent of the kept points in (x, z) for the Morton quantisation
    float xlo = 3e38f, xhi = -3e38f, zlo = 3e38f, zhi = -3e38f;
    int kept = 0;
    for (int i = tid; i < n_in; i += kPrepThreads) {
      const float x = px[i], z = pz[i];
      if (degen || (-sn * (double)x + cs * (double)z) > thresh) {
        ++kept;
        xlo = fminf(xlo, x); xhi = fmaxf(xhi, x); zlo = fminf(zlo, z); zhi = fmaxf(zhi, z);
      }
    }
    auto fmn = [](float a, float b) { return fminf(a, b); };
    auto fmx = [](float a, float b) { return fmaxf(a, b); };
    auto isum = [](int a, int b) { return a + b; };
    xlo = block_reduce(xlo, fscratch, fmn); xhi = block_reduce(xhi, fscratch, fmx);
    zlo = block_reduce(zlo, fscratch, fmn); zhi = block_reduce(zhi, fscratch, fmx);
    n_front = block_reduce(kept, iscratch, isum);
    const float xs = (xhi > xlo) ? 64.0f / (xhi - xlo) : 0.0f, zs = (zhi > zlo) ? 64.0f / (zhi - zlo) : 0.0f;
    // pass 3b: 14-bit sort keys  [class:2 | morton:12]  (dropped points: all ones, they sort last)
    for (int i = tid; i < n_in; i += kPrepThreads) {
      uint32_t key = 0x3FFFu;
      const float x = px[i], z = pz[i];
      if (degen || (-sn * (double)x + cs * (double)z) > thresh) {
        const int l = lab[i];
        const uint32_t cls = (l == 0) ? 0u : (l == 1 ? 1u : 2u);
        const uint32_t qx = (uint32_t)fminf(fmaxf((x - xlo) * xs, 0.0f), 63.0f);
        const uint32_t qz = (uint32_t)fminf(fmaxf((z - zlo) * zs, 0.0f), 63.0f);
        key = (cls << 12) | (spread6(qx) << 1) | spread6(qz);
      }
      k16[i] = (uint16_t)key;
    }
    __syncthreads();
    // pass 3c: STABLE least-significant-digit radix sort of the point indices by that key, two 7-bit digits.  Stable +
    // ascending input order = ties broken by the original index, i.e. exactly the order of the unique composite key
    // [class | morton | index]; O(n) per digit instead of the O(n log^2 n) bitonic network this replaces.
    radix_pass(k16, nullptr, ord1, n_in, 0, hist, tot);
    radix_pass(k16, ord1, ord2, n_in, 7, hist, tot);
    // pass 3d: gather in sorted order
    if (n_front > n_out_stride) n_front = n_out_stride;
    for (int i = tid; i < n_front; i += kPrepThreads) {
      const int src = (int)ord2[i];
      const int8_t l = lab[src];
      ox[i] = px[src]; oy[i] = py[src]; oz[i] = pz[src];
      ol[i] = (l == 0 || l == 1) ? l : (int8_t)-1;
    }
  } else {
    // pass 3: order-preserving compaction of the front points (:213-215)
    if (tid == 0) s_base = 0;
    __syncthreads();
    for (int start = 0; start < n_in; start += kPrepThreads) {
      const int i = start + tid;
      bool keep = false;
      float x = 0, y = 0, z = 0;
      int8_t l = -1;
      if (i < n_in) {
        x = px[i]; y = py[i]; z = pz[i]; l = lab[i];
        keep = degen ? true : ((-sn * (double)x + cs * (double)z) > thresh);
      }
      const unsigned m = __ballot_sync(0xffffffffu, keep);
      if (lane == 0) warp_cnt[warp] = __popc(m);
      __syncthreads();
      int off = s_base;
      for (int w = 0; w < warp; ++w) off += warp_cnt[w];
      if (keep) {
        const int o = off + __popc(m & ((1u << lane) - 1u));
        if (o < n_out_stride) { ox[o] = x; oy[o] = y; oz[o] = z; ol[o] = (l == 0 || l == 1) ? l : (int8_t)-1; }
      }
      __syncthreads();
      if (tid == 0) { int t = 0; for (int w = 0; w < kPrepWarps; ++w) t += warp_cnt[w]; s_base += t; }
      __syncthreads();
    }
    n_front = min(s_base, n_out_stride);
  }
  for (int i = n_front + tid; i < n_out_stride; i += kPrepThreads) { ox[i] = 0.f; oy[i] = 0.f; oz[i] = 0.f; ol[i] = -1; }
  if (tid == 0) {
    n_pts[s] = n_front;
    if (init_y_angle) init_y_angle[s] = ang;
    if (degenerate) degenerate[s] = degen ? 1 : 0;
  }
  // inits (:163-164)
  for (int i = tid; i < I; i += kPrepThreads) {
    uint32_t c[4] = {(uint32_t)i, (uint32_t)s, 0u, 0u};
    philox4x32_10(c, (uint32_t)(seed & 0xffffffffull), (uint32_t)(seed >> 32));
    const double u1 = 1.0 - ((double)(c[0] >> 5) * 67108864.0 + (double)(c[1] >> 6)) * (1.0 / 9007199254740992.0);
    const double u2 = ((double)c[2] + 0.5) * (1.0 / 4294967296.0);
    const double u3 = ((double)c[3] + 0.5) * (1.0 / 4294967296.0);
    const double gauss = sqrt(-2.0 * log(u1)) * cos(2.0 * kPi * u2);
    double* o = init + ((size_t)s * I + i) * 4;
    o[0] = ang + ry_sigma * gauss;
    o[1] = 0.0;
    o[2] = 0.0;
    o[3] = (2.0 * u3 - 1.0) * t_amp;
  }
}

}  // namespace dib

extern "C" {

size_t frustum_prepare_workspace_bytes(int S, int I) {
  (void)S; (void)I;
  return 0;
}

// xyz_in [S][3][n_in_stride] f32 [dev], pred [S][n_in_stride] int8 [dev] (1 = predicted inside);
// outputs: xyz_out [S][3][n_out_stride], label_out [S][n_out_stride], n_pts [S], init [S][I][4],
// init_y_angle [S], degenerate [S] (1 = no predicted-inside point; registration_lsq.py:329-332).
// n_out_stride = round_up(n_in, 16).  sort != 0 reorders the kept points by (label, Morton cell) -- the
// solver's sums are order-independent up to rounding and its box culling is far more effective on it.
int frustum_prepare_batch_f32(const float* xyz_in, const int8_t* pred, int n_in, int n_in_stride, int S, int I,
                              uint64_t seed, double ry_sigma, double t_amp, int sort, float* xyz_out, int8_t* label_out,
                              int32_t* n_pts, double* init, double* init_y_angle, int32_t* degenerate,
                              void* workspace, size_t workspace_bytes, dib_stream_t stream) {
  using namespace dib;
  (void)workspace; (void)workspace_bytes;
  DIB_REQUIRE(xyz_in && pred && xyz_out && label_out && n_pts && init && init_y_angle && degenerate, "NULL argument");
  DIB_REQUIRE(S >= 0 && I >= 1 && n_in >= 0 && n_in <= n_in_stride, "bad sizes");
  const int n_out_stride = (n_in + 15) & ~15;
  if (S == 0) return DIB_OK;
  const int do_sort = (sort != 0 && n_in <= kSortMax && n_in > 1) ? 1 : 0;
  const int n2 = (n_in + 7) & ~7;                  // array stride of the three 16-bit sort arrays
  const size_t smem = do_sort ? (size_t)(kPrepWarps * 128 + 128) * sizeof(uint32_t) + (size_t)3 * n2 * sizeof(uint16_t) : 0;
  if (smem > 48 * 1024)
    DIB_CHECK_CUDA(cudaFuncSetAttribute(frustum_prepare_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  frustum_prepare_kernel<<<S, kPrepThreads, smem, (cudaStream_t)stream>>>(
      xyz_in, pred, n_in, n_in_stride, n_out_stride, I, seed, ry_sigma, t_amp, do_sort, 0, n2, xyz_out, label_out, n_pts,
      init, init_y_angle, degenerate);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

// Reorder clouds by (label, Morton cell of (x, z)) WITHOUT filtering: every point is kept, labels other than 0 / 1
// become -1 (ignored) and sort last.  For callers that hand the solver an already filtered cloud (the drop-in
// solvePGivenK, registration.cpp:190-206): the solver's sums do not depend on the order beyond rounding, its box cull
// does.  xyz_in [S][3][n_in_stride], label [S][n_in_stride]; xyz_out [S][3][round_up(n_in,16)], label_out, n_pts [S].
// Clouds of more than 32768 points keep their order.
int frustum_sort_batch_f32(const float* xyz_in, const int8_t* label, int n_in, int n_in_stride, int S, float* xyz_out,
                           int8_t* label_out, int32_t* n_pts, dib_stream_t stream) {
  using namespace dib;
  DIB_REQUIRE(xyz_in && label && xyz_out && label_out && n_pts, "NULL argument");
  DIB_REQUIRE(S >= 0 && n_in >= 0 && n_in <= n_in_stride, "bad sizes");
  const int n_out_stride = (n_in + 15) & ~15;
  if (S == 0) return DIB_OK;
  const int do_sort = (n_in <= kSortMax && n_in > 1) ? 1 : 0;
  const int n2 = (n_in + 7) & ~7;
  const size_t smem = do_sort ? (size_t)(kPrepWarps * 128 + 128) * sizeof(uint32_t) + (size_t)3 * n2 * sizeof(uint16_t) : 0;
  if (smem > 48 * 1024)
    DIB_CHECK_CUDA(cudaFuncSetAttribute(frustum_prepare_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  frustum_prepare_kernel<<<S, kPrepThreads, smem, (cudaStream_t)stream>>>(
      xyz_in, label, n_in, n_in_stride, n_out_stride, /*I=*/0, 0ull, 0.0, 0.0, do_sort, /*keep_all=*/1, n2, xyz_out,
      label_out, n_pts, nullptr, nullptr, nullptr);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

}  // extern "C"
