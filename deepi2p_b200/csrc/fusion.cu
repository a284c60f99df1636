// The classifier's attention-weighted image-feature fusion (SURVEY.md 8f row N13): the two
// torch.mean(img_map.unsqueeze(3) * attention.unsqueeze(1), dim=2) lines of KeypointDetector.forward
// (models/networks_united.py:149-150, 172-174) without their B x C x P x M product tensor.
//
//   forward   out [b][c][m] = float(S / P), S = sum over p ascending of F[b][c][p] * A[b][p][m]
//   backward  gF  [b][c][p] = float((sum over m ascending of gO[b][c][m] * A[b][p][m]) / P)
//             gA  [b][p][m] = float((sum over c ascending of F[b][c][p] * gO[b][c][m]) / P)
//
// fusion_tile_kernel<BM, BN, XK, YK> computes all three as out[b][i][j] = float((sum over k ascending of X[b][i][k] *
// Y[b][k][j]) / P) for operands with any strides; XK (YK) says whether X (Y) has unit stride along k, which decides the
// direction of the coalesced loads.  Each CTA owns a BM x BN output tile.  k advances in chunks of 16: a chunk of both
// operands is read coalesced into registers while the previous one is used, then converted to fp64 once and stored in
// shared memory (two buffers).  Each thread owns a 4 x 4 block of outputs, rows ty + (BM / 4) r and columns
// tx + (BN / 4) s, so a warp's shared-memory reads of X are broadcasts and its reads of Y are consecutive doubles.
//
// Every output has one fp64 accumulator that starts at +0.0 and takes one fma per k in ascending k.  A product of two
// floats is exact in fp64, so the fma equals a multiply and an add: the result is the plain ascending sum, which a numpy
// loop reproduces bit for bit whatever the tile size.  k past the end is zero in both operands, and fma(0, 0, s) == s
// for every s the sum can hold (never -0.0: it starts at +0.0 and an exact cancellation rounds to +0.0).  No atomics
// and no workspace: bit-identical across runs, streams and batch compositions.
//
// The kernel is templated on the operand type T (float, or bf16 for the *_bf16 entry points, feature_type.cuh): the
// operands are widened at load, the result rounded float -> T at store; the fp64 accumulation is the same.
#include "common.cuh"
#include "feature_type.cuh"

namespace dib {

constexpr int kFusionBK = 16;                  // k per shared-memory chunk
constexpr int kFusionMaxRowTiles = 65535;      // grid y: row tiles of the 32-row kernel
constexpr long long kFusionBigTiles = 264;     // 64 x 64 tiles from two per SM of a 132-SM H100 up, else 32 x 32

template <int BM, int BN, bool XK, bool YK, typename T>
__global__ void __launch_bounds__((BM / 4) * (BN / 4))
    fusion_tile_kernel(const T* __restrict__ x, int64_t xb, int64_t xi, int64_t xk, const T* __restrict__ y,
                       int64_t yb, int64_t yk, int64_t yj, int I, int J, int K, double div, T* __restrict__ out) {
  constexpr int TX = BN / 4, TY = BM / 4, NT = TX * TY, BK = kFusionBK;
  constexpr int XL = BK * BM / NT, YL = BK * BN / NT;         // elements each thread stages per chunk
  // rows padded by one double: the k-fastest stores of a k-contiguous operand fall in distinct banks
  __shared__ double sx[2][BK][BM + 1];
  __shared__ double sy[2][BK][BN + 1];
  const int tid = threadIdx.x, tx = tid % TX, ty = tid / TX;
  const int b = blockIdx.z, i0 = blockIdx.y * BM, j0 = blockIdx.x * BN;
  x += (int64_t)b * xb;
  y += (int64_t)b * yb;
  float rx[XL], ry[YL];
  auto fetch = [&](int k0) {
#pragma unroll
    for (int e = 0; e < XL; ++e) {
      const int t = tid + e * NT;
      const int kk = XK ? t % BK : t / BM, ii = XK ? t / BK : t % BM;
      const int i = i0 + ii, k = k0 + kk;
      rx[e] = (i < I && k < K) ? load_f32(x[i * xi + k * xk]) : 0.f;
    }
#pragma unroll
    for (int e = 0; e < YL; ++e) {
      const int t = tid + e * NT;
      const int kk = YK ? t % BK : t / BN, jj = YK ? t / BK : t % BN;
      const int j = j0 + jj, k = k0 + kk;
      ry[e] = (j < J && k < K) ? load_f32(y[k * yk + j * yj]) : 0.f;
    }
  };
  auto stage = [&](int buf) {
#pragma unroll
    for (int e = 0; e < XL; ++e) {
      const int t = tid + e * NT;
      sx[buf][XK ? t % BK : t / BM][XK ? t / BK : t % BM] = (double)rx[e];
    }
#pragma unroll
    for (int e = 0; e < YL; ++e) {
      const int t = tid + e * NT;
      sy[buf][YK ? t % BK : t / BN][YK ? t / BK : t % BN] = (double)ry[e];
    }
  };
  double acc[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int s = 0; s < 4; ++s) acc[r][s] = 0.0;
  const int chunks = (K + BK - 1) / BK;
  fetch(0);
  stage(0);
  __syncthreads();
  for (int t = 0; t < chunks; ++t) {
    const int buf = t & 1;
    if (t + 1 < chunks) fetch((t + 1) * BK);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      double a[4], c[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) a[r] = sx[buf][kk][ty + TY * r];
#pragma unroll
      for (int s = 0; s < 4; ++s) c[s] = sy[buf][kk][tx + TX * s];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int s = 0; s < 4; ++s) acc[r][s] = __fma_rn(a[r], c[s], acc[r][s]);
    }
    // the other buffer was last read in chunk t - 1, which every thread finished before the barrier below it
    if (t + 1 < chunks) stage(buf ^ 1);
    __syncthreads();
  }
  T* ob = out + (int64_t)b * I * J;
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int i = i0 + ty + TY * r;
    if (i >= I) continue;
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      const int j = j0 + tx + TX * s;
      if (j < J) ob[(int64_t)i * J + j] = store_as<T>(__double2float_rn(__ddiv_rn(acc[r][s], div)));
    }
  }
}

// out [B][I][J] contiguous; X element (b, i, k) at x + b xb + i xi + k xk, Y element (b, k, j) at y + b yb + k yk + j yj.
// The tile size follows from the shape and never changes a result.
template <bool XK, bool YK, typename T>
int launch_fusion(const T* x, int64_t xb, int64_t xi, int64_t xk, const T* y, int64_t yb, int64_t yk, int64_t yj,
                  int B, int I, int J, int K, int P, T* out, cudaStream_t stream) {
  const long long tiles64 = (long long)B * ((I + 63) / 64) * ((J + 63) / 64);
  if (tiles64 >= kFusionBigTiles) {
    dim3 grid((J + 63) / 64, (I + 63) / 64, B);
    fusion_tile_kernel<64, 64, XK, YK, T><<<grid, 256, 0, stream>>>(x, xb, xi, xk, y, yb, yk, yj, I, J, K, (double)P, out);
  } else {
    dim3 grid((J + 31) / 32, (I + 31) / 32, B);
    fusion_tile_kernel<32, 32, XK, YK, T><<<grid, 64, 0, stream>>>(x, xb, xi, xk, y, yb, yk, yj, I, J, K, (double)P, out);
  }
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

static int check_fusion_shape(int B, int C, int P, int M, const char* what) {
  DIB_REQUIRE(B >= 1 && B <= 65535, "%s: need 1 <= B <= 65535, got %d", what, B);
  DIB_REQUIRE(C >= 1 && P >= 1 && M >= 1, "%s: need C, P, M >= 1, got %d, %d, %d", what, C, P, M);
  DIB_REQUIRE((C + 31) / 32 <= kFusionMaxRowTiles && (P + 31) / 32 <= kFusionMaxRowTiles,
              "%s: need C, P <= %d, got %d, %d", what, 32 * kFusionMaxRowTiles, C, P);
  return DIB_OK;
}

template <typename T>
int attn_fusion_forward(const T* img_features, const T* attention, int B, int C, int P, int M, T* out,
                        dib_stream_t stream_) {
  const int rc = check_fusion_shape(B, C, P, M, "attn_fusion_forward");
  if (rc != DIB_OK) return rc;
  DIB_REQUIRE(img_features && attention && out, "attn_fusion_forward: NULL argument");
  // X = F [C][P] (k = p contiguous), Y = A [P][M] (j = m contiguous)
  return launch_fusion<true, false>(img_features, (int64_t)C * P, P, 1, attention, (int64_t)P * M, M, 1, B, C, M, P, P,
                                    out, (cudaStream_t)stream_);
}

template <typename T>
int attn_fusion_backward(const T* grad_out, int64_t grad_batch_stride, const T* img_features, const T* attention,
                         int B, int C, int P, int M, T* grad_img_features, T* grad_attention, dib_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  int rc = check_fusion_shape(B, C, P, M, "attn_fusion_backward");
  if (rc != DIB_OK) return rc;
  DIB_REQUIRE(grad_batch_stride >= 0, "attn_fusion_backward: grad_batch_stride < 0");
  if (!grad_img_features && !grad_attention) return DIB_OK;
  DIB_REQUIRE(grad_out, "attn_fusion_backward: NULL argument");
  if (grad_img_features) {
    DIB_REQUIRE(attention, "attn_fusion_backward: NULL argument");
    // gF [C][P]: X = gO [C][M] (k = m contiguous), Y = A^T [M][P] (k = m contiguous)
    rc = launch_fusion<true, true>(grad_out, grad_batch_stride, M, 1, attention, (int64_t)P * M, 1, M, B, C, P, M, P,
                                   grad_img_features, stream);
    if (rc != DIB_OK) return rc;
  }
  if (grad_attention) {
    DIB_REQUIRE(img_features, "attn_fusion_backward: NULL argument");
    // gA [P][M]: X = F^T [P][C] (i = p contiguous), Y = gO [C][M] (j = m contiguous)
    rc = launch_fusion<false, false>(img_features, (int64_t)C * P, 1, P, grad_out, grad_batch_stride, M, 1, B, P, M, C,
                                     P, grad_attention, stream);
    if (rc != DIB_OK) return rc;
  }
  return DIB_OK;
}

}  // namespace dib

extern "C" {

int attn_fusion_forward_f32(const float* img_features, const float* attention, int B, int C, int P, int M, float* out,
                            dib_stream_t stream) {
  return dib::attn_fusion_forward(img_features, attention, B, C, P, M, out, stream);
}

int attn_fusion_forward_bf16(const uint16_t* img_features, const uint16_t* attention, int B, int C, int P, int M,
                             uint16_t* out, dib_stream_t stream) {
  using dib::as_bf16;
  return dib::attn_fusion_forward(as_bf16(img_features), as_bf16(attention), B, C, P, M, as_bf16(out), stream);
}

int attn_fusion_backward_f32(const float* grad_out, int64_t grad_batch_stride, const float* img_features,
                             const float* attention, int B, int C, int P, int M, float* grad_img_features,
                             float* grad_attention, dib_stream_t stream) {
  return dib::attn_fusion_backward(grad_out, grad_batch_stride, img_features, attention, B, C, P, M,
                                   grad_img_features, grad_attention, stream);
}

int attn_fusion_backward_bf16(const uint16_t* grad_out, int64_t grad_batch_stride, const uint16_t* img_features,
                              const uint16_t* attention, int B, int C, int P, int M, uint16_t* grad_img_features,
                              uint16_t* grad_attention, dib_stream_t stream) {
  using dib::as_bf16;
  return dib::attn_fusion_backward(as_bf16(grad_out), grad_batch_stride, as_bf16(img_features), as_bf16(attention), B,
                                   C, P, M, as_bf16(grad_img_features), as_bf16(grad_attention), stream);
}

}  // extern "C"
