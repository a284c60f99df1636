// Fused inference of the classifier's ResNet-34 image encoder (SURVEY.md 8f row N25, DESIGN.md 4.30): every
// convolution with its eval-mode BatchNorm folded into the weights on the host, as an implicit GEMM on the TF32 tensor
// cores over NHWC float32 activations, with bias, residual and ReLU in the epilogue.
//
//   rn_conv_kernel   CTA = 128 output pixels x 64 output channels, 4 warps of 64 x 32, K in tiles of 32 staged by
//                    cp.async into a 3-stage shared ring.  GEMM M = B * H_out * W_out, N = C_out, K = kh * kw * C_in
//                    (+ C_in of the shortcut: a block's 1x1 stride-2 downsample runs as extra K tiles of its second
//                    convolution, out = W2 y + Wd x_strided + (b2 + bd)).  Two gathers: NHWC with C_in % 32 == 0 (a K
//                    tile lies inside one tap, 16-byte copies), and NCHW with any C_in (the 7x7 stem reads the [B,3,H,W]
//                    image directly, 4-byte copies).  The epilogue adds the bias and an optional NHWC residual, applies
//                    ReLU, and stores NHWC and/or channel-major [B][C_out][H_out * W_out].
//   rn_maxpool_kernel  3x3 stride-2 pad-1 max-pool over NHWC, one thread per output element; a NaN in the window wins.
//   rn_mean_kernel   one warp per (sample, channel): the mean over P of a channel-major map as a float64 sum in a fixed
//                    order (lane-strided, then a fixed shuffle tree), divided by P and rounded once.
//
// Operand rounding is the project's (tf32_mma.cuh): weights once when packed, activations when read from shared memory
// into fragments; accumulation, bias, residual and ReLU (NaN stays NaN) are f32.  No atomics: every output has one
// writer and every sum a fixed order.
#include <math.h>

#include "common.cuh"
#include "tf32_mma.cuh"

namespace dib {

constexpr int kRnBM = 128;            // output pixels per CTA
constexpr int kRnBN = 64;             // output channels per CTA
constexpr int kRnBK = 32;             // K per stage
constexpr int kRnStride = 36;         // floats per shared row: (36 g + t) % 32 = 4 g + t keeps fragment loads conflict-free
constexpr int kRnStages = 3;
constexpr int kRnThreads = 128;
constexpr size_t kRnSmem = (size_t)kRnStages * (kRnBM + kRnBN) * kRnStride * sizeof(float) + kRnBM * sizeof(int4);

struct RnSeg {                        // one gathered operand: the main input or the shortcut
  const float* x; int H, W, C, kh, kw, stride, pad, nchw, kt;   // kt: K tiles of this segment
};
struct RnParams {
  RnSeg seg[2];
  int n_seg, Kpad;                    // Kpad = 32 * (seg[0].kt + seg[1].kt), the packed weights' row length
  int B, Ho, Wo, M, C_out, relu;
  const float* w;                     // [C_out][Kpad], TF32-rounded, zero-padded
  const float* bias;                  // [C_out]
  const float* residual;              // NHWC [M][C_out] or NULL
  float* out_nhwc;                    // [M][C_out] or NULL
  float* out_cm;                      // [B][C_out][Ho * Wo] or NULL
};

__device__ __forceinline__ void cp_async16(float* dst, const float* src, bool ok) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(ok ? 16 : 0)
               : "memory");
}
__device__ __forceinline__ void cp_async4(float* dst, const float* src, bool ok) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(ok ? 4 : 0)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_stages() {
  asm volatile("cp.async.wait_group %0;" ::"n"(kRnStages - 2) : "memory");
}

// Stage K tile `kt` (global, over both segments) into As / Bs.  rows[r] = (sample or -1, oh, ow) of the CTA's pixels.
__device__ __forceinline__ void rn_load_tile(const RnParams& p, const int4* rows, float* As, float* Bs, int kt,
                                             int n0, int tid) {
  const RnSeg& s = (p.n_seg > 1 && kt >= p.seg[0].kt) ? p.seg[1] : p.seg[0];
  const int kseg = (kt >= p.seg[0].kt ? kt - p.seg[0].kt : kt) * kRnBK;     // K offset inside the segment
  if (!s.nchw) {
    // a tile lies inside one tap (C % 32 == 0): 8 float4 per row
    const int tap = kseg / s.C, c0 = kseg - tap * s.C, r = tap / s.kw, q = tap - r * s.kw;
    const int c4 = (tid & 7) * 4;
#pragma unroll
    for (int j = 0; j < kRnBM / 16; ++j) {
      const int row = (tid >> 3) + 16 * j;
      const int4 ri = rows[row];
      const int ih = ri.y * s.stride - s.pad + r, iw = ri.z * s.stride - s.pad + q;
      const bool ok = ri.x >= 0 && ih >= 0 && ih < s.H && iw >= 0 && iw < s.W;
      const float* src = ok ? s.x + (((size_t)ri.x * s.H + ih) * s.W + iw) * s.C + c0 + c4 : s.x;
      cp_async16(As + row * kRnStride + c4, src, ok);
    }
  } else {
    // one K column per thread: k -> (tap, channel) of the [C_out][kh][kw][C] packing, read from NCHW
    const int col = tid & 31, k = kseg + col, K = s.kh * s.kw * s.C;
    const int tap = k / s.C, c = k - tap * s.C, r = tap / s.kw, q = tap - r * s.kw;
#pragma unroll 4
    for (int j = 0; j < kRnBM / 4; ++j) {
      const int row = (tid >> 5) + 4 * j;
      const int4 ri = rows[row];
      const int ih = ri.y * s.stride - s.pad + r, iw = ri.z * s.stride - s.pad + q;
      const bool ok = k < K && ri.x >= 0 && ih >= 0 && ih < s.H && iw >= 0 && iw < s.W;
      const float* src = ok ? s.x + (((size_t)ri.x * s.C + c) * s.H + ih) * s.W + iw : s.x;
      cp_async4(As + row * kRnStride + col, src, ok);
    }
  }
  const int c4 = (tid & 7) * 4;
#pragma unroll
  for (int j = 0; j < kRnBN / 16; ++j) {
    const int n = (tid >> 3) + 16 * j;
    const bool ok = n0 + n < p.C_out;
    const float* src = ok ? p.w + (size_t)(n0 + n) * p.Kpad + kt * kRnBK + c4 : p.w;
    cp_async16(Bs + n * kRnStride + c4, src, ok);
  }
}

__global__ void __launch_bounds__(kRnThreads) rn_conv_kernel(const __grid_constant__ RnParams p) {
  extern __shared__ __align__(16) float rn_smem[];
  float* As = rn_smem;                                         // [stages][BM][stride]
  float* Bs = rn_smem + kRnStages * kRnBM * kRnStride;         // [stages][BN][stride]
  int4* rows = reinterpret_cast<int4*>(Bs + kRnStages * kRnBN * kRnStride);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3, wm = warp >> 1, wn = warp & 1;
  // the N tiles of one M tile are consecutive blocks, so an activation tile is read from HBM about once
  const int n_tiles = (p.C_out + kRnBN - 1) / kRnBN;
  const int n0 = (int)(blockIdx.x % n_tiles) * kRnBN, m0 = (int)(blockIdx.x / n_tiles) * kRnBM;
  const int P = p.Ho * p.Wo;
  {
    const int m = m0 + tid;                                    // kRnThreads == kRnBM
    int4 ri = make_int4(-1, 0, 0, 0);
    if (m < p.M) {
      const int b = m / P, pix = m - b * P, oh = pix / p.Wo;
      ri = make_int4(b, oh, pix - oh * p.Wo, 0);
    }
    rows[tid] = ri;
  }
  __syncthreads();

  const int KT = p.seg[0].kt + (p.n_seg > 1 ? p.seg[1].kt : 0);
#pragma unroll
  for (int st = 0; st < kRnStages - 1; ++st) {
    if (st < KT) rn_load_tile(p, rows, As + st * kRnBM * kRnStride, Bs + st * kRnBN * kRnStride, st, n0, tid);
    cp_async_commit();
  }
  float acc[4][4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;

  for (int kt = 0; kt < KT; ++kt) {
    cp_async_wait_stages();
    __syncthreads();
    {
      const int nk = kt + kRnStages - 1, st = nk % kRnStages;
      if (nk < KT) rn_load_tile(p, rows, As + st * kRnBM * kRnStride, Bs + st * kRnBN * kRnStride, nk, n0, tid);
      cp_async_commit();
    }
    const float* A = As + (kt % kRnStages) * kRnBM * kRnStride + (wm * 64) * kRnStride;
    const float* Bt = Bs + (kt % kRnStages) * kRnBN * kRnStride + (wn * 32) * kRnStride;
#pragma unroll
    for (int k8 = 0; k8 < kRnBK; k8 += 8) {
      float4 a[4];
      uint32_t b0[4], b1[4];
#pragma unroll
      for (int mt = 0; mt < 4; ++mt) {
        const float* r0 = A + (mt * 16 + g) * kRnStride + k8 + t;
        const float* r8 = r0 + 8 * kRnStride;
        a[mt] = make_float4(tf32_rna(r0[0]), tf32_rna(r8[0]), tf32_rna(r0[4]), tf32_rna(r8[4]));
      }
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        const float* c = Bt + (nt * 8 + g) * kRnStride + k8 + t;
        b0[nt] = __float_as_uint(c[0]);
        b1[nt] = __float_as_uint(c[4]);
      }
#pragma unroll
      for (int mt = 0; mt < 4; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) mma_tf32(acc[mt][nt], a[mt], b0[nt], b1[nt]);
    }
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");

  // epilogue: (acc + bias) + residual, ReLU; row g / g + 8 of each 16-row tile, columns 2t, 2t + 1 of each 8
#pragma unroll
  for (int mt = 0; mt < 4; ++mt) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = wm * 64 + mt * 16 + g + 8 * h;
      const int4 ri = rows[row];
      if (ri.x < 0) continue;
      const size_t m = (size_t)(m0 + row);
      const size_t pix = (size_t)ri.y * p.Wo + ri.z;
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        const int n = n0 + wn * 32 + nt * 8 + 2 * t;
        if (n >= p.C_out) continue;                            // C_out % 8 == 0: n < C_out implies n + 1 < C_out
        float v0 = acc[mt][nt][2 * h] + __ldg(p.bias + n), v1 = acc[mt][nt][2 * h + 1] + __ldg(p.bias + n + 1);
        if (p.residual) {
          const float2 r = __ldg(reinterpret_cast<const float2*>(p.residual + m * p.C_out + n));
          v0 += r.x;
          v1 += r.y;
        }
        if (p.relu) {                                          // NaN < 0 is false: NaN stays NaN
          v0 = v0 < 0.f ? 0.f : v0;
          v1 = v1 < 0.f ? 0.f : v1;
        }
        if (p.out_nhwc) *reinterpret_cast<float2*>(p.out_nhwc + m * p.C_out + n) = make_float2(v0, v1);
        if (p.out_cm) {
          float* o = p.out_cm + ((size_t)ri.x * p.C_out + n) * P + pix;
          o[0] = v0;
          o[P] = v1;
        }
      }
    }
  }
}

__global__ void rn_maxpool_kernel(const float* __restrict__ x, int B, int H, int W, int C, int Ho, int Wo,
                                  float* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, total = (size_t)B * Ho * Wo * C;
  if (i >= total) return;
  const int c = (int)(i % C);
  size_t r = i / C;
  const int ow = (int)(r % Wo);
  r /= Wo;
  const int oh = (int)(r % Ho), b = (int)(r / Ho);
  float m = -INFINITY;
  for (int dh = 0; dh < 3; ++dh) {
    const int ih = oh * 2 - 1 + dh;
    if (ih < 0 || ih >= H) continue;
    for (int dw = 0; dw < 3; ++dw) {
      const int iw = ow * 2 - 1 + dw;
      if (iw < 0 || iw >= W) continue;
      const float v = __ldg(x + (((size_t)b * H + ih) * W + iw) * C + c);
      if (v > m || v != v) m = v;                              // once m is NaN nothing replaces it
    }
  }
  out[i] = m;
}

__global__ void rn_mean_kernel(const float* __restrict__ x, int rows, int P, float* __restrict__ out) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* s = x + (size_t)row * P;
  double acc = 0.0;
  for (int i = lane; i < P; i += 32) acc += (double)__ldg(s + i);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) out[row] = (float)(acc / (double)P);
}

__global__ void rn_pack_kernel(const float* __restrict__ w, int C_out, int K, int Kpad, float* __restrict__ packed) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)C_out * Kpad) return;
  const int k = (int)(i % Kpad);
  const size_t n = i / Kpad;
  packed[i] = k < K ? __uint_as_float(tf32_rna_bits(__float_as_uint(w[n * K + k]))) : 0.f;
}

}  // namespace dib

extern "C" {

size_t resnet_conv_packed_bytes(int C_out, int K) {
  if (C_out < 1 || K < 1) return 0;
  return (size_t)C_out * ((K + dib::kRnBK - 1) / dib::kRnBK * dib::kRnBK) * sizeof(float);
}

int resnet_conv_pack_f32(const float* w, int C_out, int K, void* packed, size_t packed_bytes, dib_stream_t stream) {
  using namespace dib;
  DIB_REQUIRE(C_out >= 1 && K >= 1, "resnet_conv_pack: need C_out >= 1 and K >= 1");
  DIB_REQUIRE(w != nullptr, "resnet_conv_pack: w is NULL");
  DIB_REQUIRE(packed && ((uintptr_t)packed & 15) == 0, "resnet_conv_pack: packed is NULL or not 16-byte aligned");
  if (packed_bytes < resnet_conv_packed_bytes(C_out, K)) {
    set_error("resnet_conv_pack: packed buffer too small");
    return DIB_ENOMEM;
  }
  const int Kpad = (K + kRnBK - 1) / kRnBK * kRnBK;
  const size_t n = (size_t)C_out * Kpad;
  rn_pack_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(w, C_out, K, Kpad, (float*)packed);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

int resnet_conv_f32(const float* x, int nchw, int B, int H, int W, int C_in, int kernel, int stride, int pad,
                    const float* shortcut, int H2, int W2, int C2, int stride2, const void* packed,
                    size_t packed_bytes, const float* bias, const float* residual, int relu, int C_out,
                    float* out_nhwc, float* out_cm, dib_stream_t stream) {
  using namespace dib;
  DIB_REQUIRE(B >= 1 && B <= 65535 && H >= 1 && W >= 1 && C_in >= 1,
              "resnet_conv: need 1 <= B <= 65535, H >= 1, W >= 1 and C_in >= 1");
  DIB_REQUIRE(kernel >= 1 && kernel <= 7 && stride >= 1 && stride <= 2 && pad >= 0 && pad < kernel,
              "resnet_conv: need 1 <= kernel <= 7, stride 1 or 2 and 0 <= pad < kernel");
  DIB_REQUIRE(C_out >= 8 && C_out % 8 == 0, "resnet_conv: C_out must be a positive multiple of 8");
  DIB_REQUIRE(nchw || C_in % 32 == 0, "resnet_conv: an NHWC input needs C_in %% 32 == 0");
  DIB_REQUIRE(x != nullptr && bias != nullptr, "resnet_conv: x or bias is NULL");
  DIB_REQUIRE(nchw || ((uintptr_t)x & 15) == 0, "resnet_conv: an NHWC input must be 16-byte aligned");
  DIB_REQUIRE(out_nhwc != nullptr || out_cm != nullptr, "resnet_conv: both outputs are NULL");
  DIB_REQUIRE((!out_nhwc || ((uintptr_t)out_nhwc & 7) == 0) && (!residual || ((uintptr_t)residual & 7) == 0),
              "resnet_conv: out_nhwc and residual must be 8-byte aligned");
  const int Ho = (H + 2 * pad - kernel) / stride + 1, Wo = (W + 2 * pad - kernel) / stride + 1;
  DIB_REQUIRE(H + 2 * pad >= kernel && W + 2 * pad >= kernel, "resnet_conv: the input is smaller than the kernel");
  const long long M = (long long)B * Ho * Wo;
  DIB_REQUIRE(M <= (1LL << 31) - 1 - 8 * kRnBM, "resnet_conv: too many output pixels");
  const int K1 = kernel * kernel * C_in;
  RnParams p = {};
  p.seg[0] = RnSeg{x, H, W, C_in, kernel, kernel, stride, pad, nchw ? 1 : 0, (K1 + kRnBK - 1) / kRnBK};
  p.n_seg = 1;
  if (shortcut) {
    DIB_REQUIRE(!nchw && C2 >= 32 && C2 % 32 == 0 && ((uintptr_t)shortcut & 15) == 0 && stride2 >= 1 && H2 >= 1 &&
                    W2 >= 1,
                "resnet_conv: the shortcut must be NHWC, 16-byte aligned, with C2 a positive multiple of 32");
    DIB_REQUIRE(K1 % kRnBK == 0, "resnet_conv: a shortcut needs kernel^2 * C_in %% 32 == 0");
    DIB_REQUIRE((H2 - 1) / stride2 + 1 == Ho && (W2 - 1) / stride2 + 1 == Wo,
                "resnet_conv: the shortcut's strided size differs from the output's");
    p.seg[1] = RnSeg{shortcut, H2, W2, C2, 1, 1, stride2, 0, 0, C2 / kRnBK};
    p.n_seg = 2;
  }
  p.Kpad = (p.seg[0].kt + (shortcut ? p.seg[1].kt : 0)) * kRnBK;
  DIB_REQUIRE(packed && ((uintptr_t)packed & 15) == 0 && packed_bytes >= (size_t)C_out * p.Kpad * sizeof(float),
              "resnet_conv: packed is NULL, misaligned or smaller than C_out x the padded K");
  p.B = B, p.Ho = Ho, p.Wo = Wo, p.M = (int)M, p.C_out = C_out, p.relu = relu ? 1 : 0;
  p.w = (const float*)packed, p.bias = bias, p.residual = residual, p.out_nhwc = out_nhwc, p.out_cm = out_cm;
  DIB_CHECK_CUDA(cudaFuncSetAttribute(rn_conv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kRnSmem));
  const long long blocks = (M + kRnBM - 1) / kRnBM * ((C_out + kRnBN - 1) / kRnBN);
  DIB_REQUIRE(blocks < (1LL << 31), "resnet_conv: too many output pixels x channels");
  rn_conv_kernel<<<(unsigned)blocks, kRnThreads, kRnSmem, (cudaStream_t)stream>>>(p);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

int resnet_maxpool_f32(const float* x, int B, int H, int W, int C, float* out, dib_stream_t stream) {
  using namespace dib;
  DIB_REQUIRE(B >= 1 && H >= 1 && W >= 1 && C >= 1, "resnet_maxpool: need B, H, W and C >= 1");
  DIB_REQUIRE(x != nullptr && out != nullptr, "resnet_maxpool: x or out is NULL");
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  const size_t n = (size_t)B * Ho * Wo * C;
  rn_maxpool_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, B, H, W, C, Ho, Wo, out);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

int resnet_mean_f32(const float* x, int rows, int P, float* out, dib_stream_t stream) {
  using namespace dib;
  DIB_REQUIRE(rows >= 1 && P >= 1, "resnet_mean: need rows >= 1 and P >= 1");
  DIB_REQUIRE(x != nullptr && out != nullptr, "resnet_mean: x or out is NULL");
  rn_mean_kernel<<<(rows + 7) / 8, 256, 0, (cudaStream_t)stream>>>(x, rows, P, out);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

}  // extern "C"
