// Inverse-distance feature interpolation of the classifier's decoder (SURVEY.md 8f row N9):
// KeypointDetector.upsample_by_interpolation (models/networks_united.py:76-103) without its B x C x Nq x k
// intermediates, with a deterministic backward with respect to the features.
//
//   interp_weights_kernel   one thread per query point: d_j = sqrt((dx*dx + dy*dy) + dz*dz), S = sum_j d_j in
//                           ascending j, w_j = 1 - d_j / S; writes w [B][Nq][k] f32 and the indices as int32.
//                           A point with any index outside [0, M) gets w = NaN and idx = -1 in all k slots.
//   interp_forward_kernel   CTA per (n-tile, channel chunk, b): the chunk's features [cc][M] sit in shared memory,
//                           one query point per thread, out[b][c][n] = ((w_0 F_0 + w_1 F_1) + ...) written along n.
//   interp_backward_kernel  CTA (one warp) per (N-slice x node range, 32-channel chunk, b): the g tile [32][T] is
//                           staged coalesced and read transposed; lane c owns the fp64 accumulators of channel c over
//                           the node range in padded shared memory and adds the exact fp32 products w * g in ascending
//                           (n, j).  Each accumulator has one owner and a fixed order: no atomics.  When a point's
//                           k indices are distinct its k updates are issued together.
//   interp_reduce_kernel    gF[b][c][m] = float(((p_0 + p_1) + ...) + p_{S-1}) over the slice partials, in slice order.
//
// All arithmetic is IEEE single precision without contraction (this file is compiled with --fmad=false; the
// intrinsics below make the rounding explicit anyway).  oracle_interp restates it.  The forward and backward are
// templated on the feature type (float, or bf16 for the *_bf16 entry points, feature_type.cuh): the features (staged
// in shared memory as they are), the output and the gradients convert at load and store; the weights stay f32.
#include <math.h>

#include "common.cuh"
#include "feature_type.cuh"

namespace dib {

constexpr int kInterpMaxK = 8;
constexpr int kInterpMaxNodes = 2048;
constexpr int kFwdThreads = 256;               // query points per forward CTA
constexpr int kFwdSmemFloats = 16384;          // features staged per forward CTA (64 KB)
constexpr int kFwdMaxChunk = 64;               // channels per forward CTA
constexpr int kBwdChannels = 32;               // channels per backward CTA = its one warp
constexpr int kBwdTile = 32;                   // query points staged per step
constexpr int kBwdNodeRange = 128;             // nodes per backward CTA (accumulators per lane)
constexpr int kBwdTargetCtas = 2048;           // slices are added until the grid has about this many CTAs

__host__ __device__ inline int fwd_chunk(int M) {
  const int c = kFwdSmemFloats / M;
  return c < kFwdMaxChunk ? c : kFwdMaxChunk;
}

template <typename IdxT, int K>
__global__ void __launch_bounds__(256)
    interp_weights_kernel(const IdxT* __restrict__ topk, const float* __restrict__ query,
                          const float* __restrict__ node, int Nq, int M, float* __restrict__ w_out,
                          int32_t* __restrict__ idx_out) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (n >= Nq) return;
  const size_t row = ((size_t)b * Nq + n) * K;
  int32_t id[K];
  bool ok = true;
#pragma unroll
  for (int j = 0; j < K; ++j) {
    const long long v = (long long)topk[row + j];
    ok = ok && v >= 0 && v < M;
    id[j] = (int32_t)v;
  }
  if (!ok) {                                            // nothing is read through an index that is out of range
#pragma unroll
    for (int j = 0; j < K; ++j) { w_out[row + j] = __int_as_float(0x7fc00000); idx_out[row + j] = -1; }
    return;
  }
  const float* qb = query + (size_t)b * 3 * Nq;
  const float* nb = node + (size_t)b * 3 * M;
  const float x = qb[n], y = qb[(size_t)Nq + n], z = qb[2 * (size_t)Nq + n];
  float d[K];
  float S = 0.f;
#pragma unroll
  for (int j = 0; j < K; ++j) {
    const int m = id[j];
    const float dx = __fsub_rn(x, nb[m]), dy = __fsub_rn(y, nb[M + m]), dz = __fsub_rn(z, nb[2 * M + m]);
    d[j] = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
    S = j == 0 ? d[0] : __fadd_rn(S, d[j]);
  }
#pragma unroll
  for (int j = 0; j < K; ++j) {
    w_out[row + j] = __fsub_rn(1.f, __fdiv_rn(d[j], S));
    idx_out[row + j] = id[j];
  }
}

template <int K, typename T>
__global__ void __launch_bounds__(kFwdThreads)
    interp_forward_kernel(const T* __restrict__ features, const float* __restrict__ w,
                          const int32_t* __restrict__ idx, int C, int Nq, int M, int cc, T* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char s_raw[];
  T* s_f = reinterpret_cast<T*>(s_raw);                     // [cc][M]
  const int b = blockIdx.z, c0 = blockIdx.y * cc, tid = threadIdx.x;
  const int nc = min(cc, C - c0);
  const T* fb = features + ((size_t)b * C + c0) * M;        // the chunk's rows are contiguous
  for (int i = tid; i < nc * M; i += kFwdThreads) s_f[i] = fb[i];
  __syncthreads();
  const int n = blockIdx.x * kFwdThreads + tid;
  if (n >= Nq) return;
  const size_t row = ((size_t)b * Nq + n) * K;
  float wj[K];
  int ij[K];
#pragma unroll
  for (int j = 0; j < K; ++j) { wj[j] = w[row + j]; ij[j] = idx[row + j]; }
  T* ob = out + ((size_t)b * C + c0) * Nq + n;
  if (ij[0] < 0) {                                           // an index was out of range: the whole column is NaN
    for (int c = 0; c < nc; ++c) ob[(size_t)c * Nq] = store_as<T>(__int_as_float(0x7fc00000));
    return;
  }
#pragma unroll 4
  for (int c = 0; c < nc; ++c) {
    const T* f = s_f + c * M;
    float acc = __fmul_rn(wj[0], load_f32(f[ij[0]]));
#pragma unroll
    for (int j = 1; j < K; ++j) acc = __fadd_rn(acc, __fmul_rn(wj[j], load_f32(f[ij[j]])));
    ob[(size_t)c * Nq] = store_as<T>(acc);
  }
}

// grid (slices * ranges, ceil(C / 32), B), 32 threads.  Partials [B][slices][C][M] f64.  The next tile's g, w and
// idx are loaded into registers while the current one is accumulated.
template <int K, typename T>
__global__ void __launch_bounds__(kBwdChannels)
    interp_backward_kernel(const T* __restrict__ g, int64_t g_batch_stride, const float* __restrict__ w,
                           const int32_t* __restrict__ idx, int C, int Nq, int M, int slices, int slice_len,
                           double* __restrict__ partial) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int ranges = (M + kBwdNodeRange - 1) / kBwdNodeRange;
  const int s = blockIdx.x / ranges, r = blockIdx.x % ranges;
  const int m0 = r * kBwdNodeRange, mr = min(kBwdNodeRange, M - m0);
  const int stride = mr | 1;                                  // odd: the lanes' doubles fall in distinct bank pairs
  double* acc = reinterpret_cast<double*>(smem_raw);          // [32][stride]
  float* s_g = reinterpret_cast<float*>(acc + kBwdChannels * stride);   // [32][kBwdTile + 1]
  float* s_w = s_g + kBwdChannels * (kBwdTile + 1);           // [kBwdTile * K]
  int32_t* s_i = reinterpret_cast<int32_t*>(s_w + kBwdTile * kInterpMaxK);
  const int b = blockIdx.z, c0 = blockIdx.y * kBwdChannels, lane = threadIdx.x;
  const int nc = min(kBwdChannels, C - c0);
  for (int i = lane; i < kBwdChannels * stride; i += 32) acc[i] = 0.0;
  const int n_begin = s * slice_len, n_end = min(Nq, n_begin + slice_len);
  const T* gb = g + (size_t)b * g_batch_stride + (size_t)c0 * Nq;
  const size_t wb = (size_t)b * Nq * K;
  double* my = acc + lane * stride;
  float pg[kBwdChannels], pw[K];
  int32_t pi[K];
  auto fetch = [&](int t0) {                                  // lane = point of the tile for g, flat (point, j) for w
    const int tn = min(kBwdTile, n_end - t0);
#pragma unroll
    for (int c = 0; c < kBwdChannels; ++c) pg[c] = (c < nc && lane < tn) ? load_f32(gb[(size_t)c * Nq + t0 + lane]) : 0.f;
#pragma unroll
    for (int q = 0; q < K; ++q) {
      const int i = q * 32 + lane;
      pw[q] = i < tn * K ? w[wb + (size_t)t0 * K + i] : 0.f;
      pi[q] = i < tn * K ? idx[wb + (size_t)t0 * K + i] : -1;
    }
  };
  if (n_begin < n_end) fetch(n_begin);
  for (int t0 = n_begin; t0 < n_end; t0 += kBwdTile) {
    const int tn = min(kBwdTile, n_end - t0);
    __syncwarp();
#pragma unroll
    for (int c = 0; c < kBwdChannels; ++c) s_g[c * (kBwdTile + 1) + lane] = pg[c];
#pragma unroll
    for (int q = 0; q < K; ++q) { s_w[q * 32 + lane] = pw[q]; s_i[q * 32 + lane] = pi[q]; }
    __syncwarp();
    if (t0 + kBwdTile < n_end) fetch(t0 + kBwdTile);
    if (lane < nc) {
      const float* gr = s_g + lane * (kBwdTile + 1);
      for (int t = 0; t < tn; ++t) {
        const double gv = (double)gr[t];
        int mj[K];
        double pj[K];
        bool distinct = true;
#pragma unroll
        for (int j = 0; j < K; ++j) {
          mj[j] = s_i[t * K + j] - m0;                        // -1 - m0 (bad point) and other ranges fail the test
          pj[j] = (double)s_w[t * K + j] * gv;                // exact: 24 x 24 bits
#pragma unroll
          for (int a = 0; a < j; ++a) distinct = distinct && mj[a] != mj[j];
        }
        // the indices are the same in every lane, so this branch is warp-uniform.  Either way each accumulator
        // receives at most one addition per j, in ascending j: the sums are the same bit for bit.
        if (distinct) {
          double v[K];
#pragma unroll
          for (int j = 0; j < K; ++j) v[j] = (unsigned)mj[j] < (unsigned)mr ? my[mj[j]] : 0.0;
#pragma unroll
          for (int j = 0; j < K; ++j)
            if ((unsigned)mj[j] < (unsigned)mr) my[mj[j]] = v[j] + pj[j];
        } else {
#pragma unroll
          for (int j = 0; j < K; ++j)
            if ((unsigned)mj[j] < (unsigned)mr) my[mj[j]] += pj[j];
        }
      }
    }
  }
  __syncwarp();
  double* pb = partial + (((size_t)b * slices + s) * C + c0) * M + m0;
  for (int c = 0; c < nc; ++c)
    for (int m = lane; m < mr; m += 32) pb[(size_t)c * M + m] = acc[c * stride + m];
}

// one thread per (b, c, m)
template <typename T>
__global__ void interp_reduce_kernel(const double* __restrict__ partial, int C, int M, int slices, size_t total,
                                     T* __restrict__ gF) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const size_t cm = (size_t)C * M, b = i / cm, r = i % cm;
  const double* p = partial + b * slices * cm + r;
  double sum = p[0];
  for (int s = 1; s < slices; ++s) sum += p[(size_t)s * cm];
  gF[i] = store_as<T>((float)sum);
}

// Slices of the backward: a function of the shape alone, so a given shape always sums in the same order.
inline void bwd_slices(int B, int C, int Nq, int M, int* slices, int* slice_len) {
  const long long base = (long long)B * ((C + kBwdChannels - 1) / kBwdChannels) *
                         ((M + kBwdNodeRange - 1) / kBwdNodeRange);
  const int tiles = (Nq + kBwdTile - 1) / kBwdTile;
  long long s = (kBwdTargetCtas + base - 1) / base;
  if (s > tiles) s = tiles;
  if (s < 1) s = 1;
  const int tiles_per = (tiles + (int)s - 1) / (int)s;
  *slice_len = tiles_per * kBwdTile;
  *slices = (Nq + *slice_len - 1) / *slice_len;
  if (*slices < 1) *slices = 1;
}

inline size_t bwd_smem(int M) {
  const int mr = M < kBwdNodeRange ? M : kBwdNodeRange;
  return (size_t)kBwdChannels * (mr | 1) * sizeof(double) + kBwdChannels * (kBwdTile + 1) * sizeof(float) +
         kBwdTile * kInterpMaxK * (sizeof(float) + sizeof(int32_t));
}

}  // namespace dib

extern "C" {

int interp_weights_f32(const void* topk_idx, int idx_bytes, const float* query, const float* node, int B, int Nq,
                       int M, int k, float* w_out, int32_t* idx_out, dib_stream_t stream_) {
  using namespace dib;
  cudaStream_t stream = (cudaStream_t)stream_;
  DIB_REQUIRE(idx_bytes == 4 || idx_bytes == 8, "interp_weights: idx_bytes must be 4 or 8");
  DIB_REQUIRE(B >= 0 && Nq >= 0 && B <= 65535, "interp_weights: need 0 <= B <= 65535, Nq >= 0");
  DIB_REQUIRE(M >= 1 && M <= kInterpMaxNodes, "interp_weights: need 1 <= M <= 2048");
  DIB_REQUIRE(k >= 1 && k <= kInterpMaxK, "interp_weights: need 1 <= k <= 8");
  if (B == 0 || Nq == 0) return DIB_OK;
  DIB_REQUIRE(topk_idx && query && node && w_out && idx_out, "interp_weights: NULL argument");
  dim3 grid((Nq + 255) / 256, B);
#define DIB_IW_LAUNCH(KK)                                                                                         \
  case KK:                                                                                                        \
    if (idx_bytes == 8)                                                                                           \
      interp_weights_kernel<long long, KK><<<grid, 256, 0, stream>>>((const long long*)topk_idx, query, node, Nq, M, \
                                                                     w_out, idx_out);                             \
    else                                                                                                          \
      interp_weights_kernel<int32_t, KK><<<grid, 256, 0, stream>>>((const int32_t*)topk_idx, query, node, Nq, M,  \
                                                                   w_out, idx_out);                               \
    break;
  switch (k) {
    DIB_IW_LAUNCH(1) DIB_IW_LAUNCH(2) DIB_IW_LAUNCH(3) DIB_IW_LAUNCH(4)
    DIB_IW_LAUNCH(5) DIB_IW_LAUNCH(6) DIB_IW_LAUNCH(7) DIB_IW_LAUNCH(8)
  }
#undef DIB_IW_LAUNCH
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

}  // extern "C"

namespace dib {

template <typename T>
int interp_forward(const T* features, const float* w, const int32_t* idx, int B, int C, int Nq, int M, int k, T* out,
                   dib_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  DIB_REQUIRE(B >= 0 && C >= 0 && Nq >= 0 && B <= 65535, "interp_forward: need 0 <= B <= 65535, C, Nq >= 0");
  DIB_REQUIRE(M >= 1 && M <= kInterpMaxNodes, "interp_forward: need 1 <= M <= 2048");
  DIB_REQUIRE(k >= 1 && k <= kInterpMaxK, "interp_forward: need 1 <= k <= 8");
  if (B == 0 || C == 0 || Nq == 0) return DIB_OK;
  DIB_REQUIRE(features && w && idx && out, "interp_forward: NULL argument");
  const int cc = fwd_chunk(M);
  DIB_REQUIRE((C + cc - 1) / cc <= 65535, "interp_forward: too many channels");
  const size_t smem = (size_t)cc * M * sizeof(T);
  dim3 grid((Nq + kFwdThreads - 1) / kFwdThreads, (C + cc - 1) / cc, B);
#define DIB_IF_LAUNCH(KK)                                                                                      \
  case KK:                                                                                                     \
    if (smem > 48 * 1024)                                                                                      \
      DIB_CHECK_CUDA(cudaFuncSetAttribute(interp_forward_kernel<KK, T>,                                        \
                                          cudaFuncAttributeMaxDynamicSharedMemorySize,                         \
                                          kFwdSmemFloats * (int)sizeof(T)));                                   \
    interp_forward_kernel<KK, T><<<grid, kFwdThreads, smem, stream>>>(features, w, idx, C, Nq, M, cc, out);    \
    break;
  switch (k) {
    DIB_IF_LAUNCH(1) DIB_IF_LAUNCH(2) DIB_IF_LAUNCH(3) DIB_IF_LAUNCH(4)
    DIB_IF_LAUNCH(5) DIB_IF_LAUNCH(6) DIB_IF_LAUNCH(7) DIB_IF_LAUNCH(8)
  }
#undef DIB_IF_LAUNCH
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

inline size_t bwd_workspace_bytes(int B, int C, int Nq, int M) {
  if (B <= 0 || C <= 0 || Nq <= 0 || M <= 0) return 0;
  int slices, slice_len;
  bwd_slices(B, C, Nq, M, &slices, &slice_len);
  return (size_t)B * slices * (size_t)C * M * sizeof(double);
}

template <typename T>
int interp_backward(const T* grad_out, int64_t grad_batch_stride, const float* w, const int32_t* idx, int B, int C,
                    int Nq, int M, int k, T* grad_features, void* workspace, size_t workspace_bytes,
                    dib_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  DIB_REQUIRE(B >= 0 && C >= 0 && Nq >= 0 && B <= 65535, "interp_backward: need 0 <= B <= 65535, C, Nq >= 0");
  DIB_REQUIRE(M >= 1 && M <= kInterpMaxNodes, "interp_backward: need 1 <= M <= 2048");
  DIB_REQUIRE(k >= 1 && k <= kInterpMaxK, "interp_backward: need 1 <= k <= 8");
  if (B == 0 || C == 0) return DIB_OK;
  DIB_REQUIRE(grad_features, "interp_backward: NULL argument");
  if (Nq == 0) {
    DIB_CHECK_CUDA(cudaMemsetAsync(grad_features, 0, (size_t)B * C * M * sizeof(T), stream));
    return DIB_OK;
  }
  DIB_REQUIRE(grad_out && w && idx, "interp_backward: NULL argument");
  DIB_REQUIRE(grad_batch_stride >= 0, "interp_backward: grad_batch_stride < 0");
  DIB_REQUIRE((C + kBwdChannels - 1) / kBwdChannels <= 65535, "interp_backward: too many channels");
  const size_t need = bwd_workspace_bytes(B, C, Nq, M);
  DIB_REQUIRE(workspace && workspace_bytes >= need && ((uintptr_t)workspace & 7) == 0,
              "interp_backward: workspace too small or misaligned");
  int slices, slice_len;
  bwd_slices(B, C, Nq, M, &slices, &slice_len);
  const int ranges = (M + kBwdNodeRange - 1) / kBwdNodeRange;
  const size_t smem = bwd_smem(M);                            // <= 39 KB: no opt-in needed
  dim3 grid(slices * ranges, (C + kBwdChannels - 1) / kBwdChannels, B);
  double* partial = (double*)workspace;
#define DIB_IB_LAUNCH(KK)                                                                                    \
  case KK:                                                                                                   \
    interp_backward_kernel<KK, T><<<grid, kBwdChannels, smem, stream>>>(grad_out, grad_batch_stride, w, idx, C, Nq,  \
                                                                        M, slices, slice_len, partial);          \
    break;
  switch (k) {
    DIB_IB_LAUNCH(1) DIB_IB_LAUNCH(2) DIB_IB_LAUNCH(3) DIB_IB_LAUNCH(4)
    DIB_IB_LAUNCH(5) DIB_IB_LAUNCH(6) DIB_IB_LAUNCH(7) DIB_IB_LAUNCH(8)
  }
#undef DIB_IB_LAUNCH
  DIB_CHECK_CUDA(cudaGetLastError());
  const size_t total = (size_t)B * C * M;
  interp_reduce_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(partial, C, M, slices, total,
                                                                             grad_features);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

}  // namespace dib

extern "C" {

int interp_forward_f32(const float* features, const float* w, const int32_t* idx, int B, int C, int Nq, int M, int k,
                       float* out, dib_stream_t stream) {
  return dib::interp_forward(features, w, idx, B, C, Nq, M, k, out, stream);
}

int interp_forward_bf16(const uint16_t* features, const float* w, const int32_t* idx, int B, int C, int Nq, int M,
                        int k, uint16_t* out, dib_stream_t stream) {
  return dib::interp_forward(dib::as_bf16(features), w, idx, B, C, Nq, M, k, dib::as_bf16(out), stream);
}

size_t interp_backward_workspace_bytes(int B, int C, int Nq, int M) { return dib::bwd_workspace_bytes(B, C, Nq, M); }

int interp_backward_f32(const float* grad_out, int64_t grad_batch_stride, const float* w, const int32_t* idx, int B,
                        int C, int Nq, int M, int k, float* grad_features, void* workspace, size_t workspace_bytes,
                        dib_stream_t stream) {
  return dib::interp_backward(grad_out, grad_batch_stride, w, idx, B, C, Nq, M, k, grad_features, workspace,
                              workspace_bytes, stream);
}

int interp_backward_bf16(const uint16_t* grad_out, int64_t grad_batch_stride, const float* w, const int32_t* idx,
                         int B, int C, int Nq, int M, int k, uint16_t* grad_features, void* workspace,
                         size_t workspace_bytes, dib_stream_t stream) {
  return dib::interp_backward(dib::as_bf16(grad_out), grad_batch_stride, w, idx, B, C, Nq, M, k,
                              dib::as_bf16(grad_features), workspace, workspace_bytes, stream);
}

}  // extern "C"
