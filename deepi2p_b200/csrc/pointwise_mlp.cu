// Fused inference path of the classifier's per-point layers (SURVEY.md 8f row N16, DESIGN.md 4.21): a chain of one to
// three 1x1 convolutions over the points of a batch, BatchNorm folded into the weights on the host, with the layer-1
// input the virtual concatenation of dense sources and interpolated node features, and the arg-max of network.predict
// as an output mode.  Nothing wider than the sources and the predictions touches global memory.
//
//   mlp_pack_kernel   W [C_out][ld] f32 -> the m16n8k8 A-fragment order [m tile][k tile][lane][4], each weight rounded
//                     to TF32 once (tf32_rna), zero in the padding.  A lane's fragment is one 16-byte load.
//   mlp_kernel        CTA = 64 points of one sample, 8 warps as 4 (output channels, 64 each) x 2 (points, 32 each).
//                     Layer 1:  z = W1[:, dense rows] x  (tensor cores; the dense rows staged 64 at a time, rounded to
//                     TF32)  +  sum over interpolated sources s, neighbours j of w_sj P_s[idx_sj]  (f32 fma chain in
//                     that order, gathered by one warp per point from the projected node features P_s = W1[:, rows of
//                     s] F_s, [B][M][C1] so that a node is one contiguous row)  +  b1.  Interpolation is linear, so
//                     this equals the layer over the interpolated rows; it takes them out of the per-point product.
//                     Layers 2, 3 read the previous activations from shared memory (rounded to TF32 when stored).
//                     The last layer's scores stay f32 in shared memory and leave as [B][C][N] activations, as the
//                     arg-max over [0, c_split) and [c_split, C) by torch.max's rule, or (the projection launches)
//                     transposed as [B][N][C_pad].
//
// Operand rounding is defined, not left to the instruction: tf32_rna (tf32_mma.cuh) is round-to-nearest, ties away
// from zero, onto 10 mantissa bits, with overflow (-> inf) and NaN (unchanged) defined too.  Products accumulate in
// f32 in the tensor core; bias, ReLU (NaN stays NaN) and the arg-max are f32.  oracle_pointwise restates this
// formulation.
#include <math.h>

#include "common.cuh"
#include "tf32_mma.cuh"

namespace dib {

constexpr int kMlpTile = 64;          // points per CTA
constexpr int kMlpStride = 72;        // floats per shared row: 72 % 32 == 8 makes the B-fragment loads conflict-free
constexpr int kMlpThreads = 256;
constexpr int kMlpChunk = 64;         // dense input rows staged per step
constexpr int kMlpMaxWidth = 256;     // 4 warp rows x 4 m tiles x 16
constexpr int kMlpMaxIn = 1024;
constexpr int kMlpMaxSources = 4;
constexpr int kMlpMaxLayers = 3;
constexpr int kMlpMaxK = 8;
constexpr int kMlpMaxNodes = 2048;

enum { kOutActivations = 0, kOutTransposed = 1, kOutArgmax = 2 };

struct MlpDense { const float* p; long long bstride; int C; int row0; };
struct MlpInterp { const float* P; const float* w; const int32_t* idx; int M; int k; };
struct MlpLayer { const float* W; const float* bias; int C; int Cpad; int relu; };
struct MlpParams {
  MlpDense dense[kMlpMaxSources];
  MlpInterp interp[kMlpMaxSources];
  MlpLayer layer[kMlpMaxLayers];
  int n_dense, n_interp, n_layers, Kd, N, xs_floats, buf_floats, out_mode, c_split;
  float* out;
  int8_t* pred_a;
  int32_t* pred_b;
};

// torch.max's order: NaN beats everything, otherwise the larger value; equal values (or two NaN) -> the lower index
__device__ __forceinline__ bool mlp_better(float v, int i, float bv, int bi) {
  if (i < 0) return false;
  if (bi < 0) return true;
  const bool vn = v != v, bn = bv != bv;
  if (vn != bn) return vn;
  if (!vn && v != bv) return v > bv;
  return i < bi;
}

__global__ void __launch_bounds__(kMlpThreads, 2) mlp_kernel(const __grid_constant__ MlpParams p) {
  extern __shared__ __align__(16) float mlp_smem[];
  float* xs = mlp_smem;                       // [<= kMlpChunk][kMlpStride] staged dense rows
  float* bufA = xs + p.xs_floats;             // activations [Cpad][kMlpStride], ping
  float* bufB = bufA + p.buf_floats;          // pong; before layer 1 the gathered interpolation [64][C1pad + 4]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3, wm = warp >> 1, n_base = (warp & 1) * 32;
  const int b = blockIdx.y, n0 = blockIdx.x * kMlpTile, N = p.N;
  const int C1pad = p.layer[0].Cpad, IS = C1pad + 4;

  if (p.n_interp > 0) {
    // lane l holds the weight and index of (source l / 8, neighbour l % 8) of the warp's current point
    const int ls = lane >> 3, lj = lane & 7;
    const bool mine = ls < p.n_interp && lj < p.interp[ls].k;
    for (int pt = warp; pt < kMlpTile; pt += kMlpThreads / 32) {
      const int n = n0 + pt;
      float wv = 0.f;
      int iv = 0;
      if (mine && n < N) {
        const size_t e = ((size_t)b * N + n) * p.interp[ls].k + lj;
        wv = p.interp[ls].w[e];
        iv = p.interp[ls].idx[e];
        if (iv < 0 || iv >= p.interp[ls].M) iv = -1;
      }
      const bool bad = __any_sync(0xffffffffu, iv < 0);        // interp_forward's rule: the whole column is NaN
      for (int c0 = 0; c0 < C1pad; c0 += 128) {              // uniform trip count: the shuffles below need every lane
        const int c4 = c0 + lane * 4;
        const bool active = c4 < C1pad;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int s = 0; s < p.n_interp; ++s) {
          const float* Ps = p.interp[s].P + (size_t)b * p.interp[s].M * C1pad + c4;
          for (int j = 0; j < p.interp[s].k; ++j) {
            const float w = __shfl_sync(0xffffffffu, wv, s * 8 + j);
            const int id = __shfl_sync(0xffffffffu, iv, s * 8 + j);
            if (active && !bad && n < N) {
              const float4 v = __ldg(reinterpret_cast<const float4*>(Ps + (size_t)id * C1pad));
              acc.x = fmaf(w, v.x, acc.x); acc.y = fmaf(w, v.y, acc.y);
              acc.z = fmaf(w, v.z, acc.z); acc.w = fmaf(w, v.w, acc.w);
            }
          }
        }
        if (bad) acc.x = acc.y = acc.z = acc.w = __int_as_float(0x7fc00000);
        if (active) *reinterpret_cast<float4*>(bufB + pt * IS + c4) = acc;
      }
    }
  }

  float* in = xs;
  for (int l = 0; l < p.n_layers; ++l) {
    const MlpLayer L = p.layer[l];
    const int MT = L.Cpad >> 4;
    float acc[4][4][4];
#pragma unroll
    for (int mt = 0; mt < 4; ++mt)
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[mt][nt][i] = 0.f;
    const float4* Wp = reinterpret_cast<const float4*>(L.W);
    if (l == 0) {
      const int KT = (p.Kd + 7) >> 3;
      for (int k0 = 0; k0 < p.Kd; k0 += kMlpChunk) {
        const int kc8 = (min(kMlpChunk, p.Kd - k0) + 7) & ~7;
        __syncthreads();                                       // the previous chunk has been consumed
        for (int r = tid >> 6; r < kc8; r += kMlpThreads / kMlpTile) {
          const int n = tid & 63, row = k0 + r;
          float v = 0.f;
          if (row < p.Kd && n0 + n < N) {
            int s = 0;
#pragma unroll
            for (int q = 1; q < kMlpMaxSources; ++q)
              if (q < p.n_dense && row >= p.dense[q].row0) s = q;
            v = tf32_rna(p.dense[s].p[(size_t)b * p.dense[s].bstride + (size_t)(row - p.dense[s].row0) * N + n0 + n]);
          }
          xs[r * kMlpStride + n] = v;
        }
        __syncthreads();
        mma_block_64x32<kMlpStride>(acc, xs, Wp, KT, MT, k0 >> 3, kc8 >> 3, wm, n_base, lane);
      }
    } else {
      const int KT = p.layer[l - 1].Cpad >> 3;
      mma_block_64x32<kMlpStride>(acc, in, Wp, KT, MT, 0, KT, wm, n_base, lane);
    }
    if (l == 0 && p.n_interp > 0) __syncthreads();             // the gathered tile is complete (and visible)
    float* out = (l & 1) ? bufB : bufA;
    const bool last = l == p.n_layers - 1;
#pragma unroll
    for (int mt = 0; mt < 4; ++mt) {
      if (wm * 4 + mt < MT) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int m = (wm * 4 + mt) * 16 + g + (i >> 1) * 8;
          const float bias = L.bias != nullptr ? L.bias[m] : 0.f;
#pragma unroll
          for (int nt = 0; nt < 4; ++nt) {
            const int n = n_base + nt * 8 + 2 * t + (i & 1);
            float v = acc[mt][nt][i];
            if (l == 0 && p.n_interp > 0) v += bufB[n * IS + m];
            v += bias;
            if (L.relu) v = v < 0.f ? 0.f : v;                 // NaN < 0 is false: NaN stays, as torch.relu
            if (m >= L.C) v = 0.f;                             // padding rows feed zero weights: keep them finite
            out[m * kMlpStride + n] = last ? v : tf32_rna(v);
          }
        }
      }
    }
    __syncthreads();
    in = out;
  }

  const MlpLayer L = p.layer[p.n_layers - 1];
  const float* S = in;
  if (p.out != nullptr) {
    if (p.out_mode == kOutTransposed) {
      for (int i = tid; i < kMlpTile * L.Cpad; i += kMlpThreads) {
        const int n = i / L.Cpad, c = i - n * L.Cpad;
        if (n0 + n < N) p.out[((size_t)b * N + n0 + n) * L.Cpad + c] = S[c * kMlpStride + n];
      }
    } else {
      for (int i = tid; i < kMlpTile * L.C; i += kMlpThreads) {
        const int c = i >> 6, n = i & 63;
        if (n0 + n < N) p.out[((size_t)b * L.C + c) * N + n0 + n] = S[c * kMlpStride + n];
      }
    }
  }
  if (p.out_mode == kOutArgmax) {
    // 4 lanes per point, lane q scans channels lo + q, lo + q + 4, ... (conflict-free), then a butterfly merge
    const int n = tid >> 2, q = tid & 3;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int lo = r == 0 ? 0 : p.c_split, hi = r == 0 ? p.c_split : L.C;
      if (lo >= hi) continue;                                  // uniform: a coarse-only head has no second range
      float bv = 0.f;
      int bi = -1;
      for (int c = lo + q; c < hi; c += 4) {
        const float v = S[c * kMlpStride + n];
        if (mlp_better(v, c, bv, bi)) { bv = v; bi = c; }
      }
#pragma unroll
      for (int d = 1; d < 4; d <<= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, d);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, d);
        if (mlp_better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
      }
      if (q == 0 && n0 + n < N) {
        if (r == 0) p.pred_a[(size_t)b * N + n0 + n] = (int8_t)bi;
        else p.pred_b[(size_t)b * N + n0 + n] = bi - lo;
      }
    }
  }
}

// One thread per packed float.  Packed column c of the matrix is column seg_orig[s] + (c - seg_start[s]) of W for the
// segment s holding c (the dense sources of layer 1 are up to four column ranges of W1).
struct MlpPackSeg { int start[kMlpMaxSources + 1]; int orig[kMlpMaxSources]; int n; };

__global__ void mlp_pack_kernel(const float* __restrict__ W, int ld, int C_out, int K, int KT, int total,
                                MlpPackSeg seg, float* __restrict__ out) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  int row, col;
  a_frag_row_col(e, KT, row, col);
  float v = 0.f;
  if (row < C_out && col < K) {
    int s = 0;
    for (int q = 1; q < seg.n; ++q)
      if (col >= seg.start[q]) s = q;
    v = tf32_rna(W[(size_t)row * ld + seg.orig[s] + col - seg.start[s]]);
  }
  out[e] = v;
}

__global__ void mlp_bias_kernel(const float* __restrict__ b, int C, int Cpad, float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < Cpad) out[c] = c < C && b != nullptr ? b[c] : 0.f;
}

// Where everything lives in the packed buffer (floats) and the workspace (bytes); a function of the widths alone.
struct MlpPlan {
  int n_src, n_layers, n_dense, n_interp, Kd, c_in;
  int src_C[kMlpMaxSources], src_M[kMlpMaxSources], src_k[kMlpMaxSources], src_col[kMlpMaxSources];
  int C[kMlpMaxLayers], Cpad[kMlpMaxLayers], relu[kMlpMaxLayers];
  size_t proj_off[kMlpMaxSources], w_off[kMlpMaxLayers], b_off[kMlpMaxLayers], packed_floats;
};

static inline int pad_to(int x, int m) { return (x + m - 1) / m * m; }

static int mlp_plan(const int64_t* sources, int n_sources, const int64_t* layers, int n_layers, MlpPlan* pl) {
  DIB_REQUIRE(sources && layers, "pointwise_mlp: NULL descriptor table");
  DIB_REQUIRE(n_sources >= 1 && n_sources <= kMlpMaxSources, "pointwise_mlp: need 1 <= n_sources <= 4");
  DIB_REQUIRE(n_layers >= 1 && n_layers <= kMlpMaxLayers, "pointwise_mlp: need 1 <= n_layers <= 3");
  pl->n_src = n_sources; pl->n_layers = n_layers; pl->n_dense = pl->n_interp = pl->Kd = pl->c_in = 0;
  for (int s = 0; s < n_sources; ++s) {
    const int64_t* d = sources + (size_t)s * DIB_MLP_SRC;
    DIB_REQUIRE(d[DIB_MLP_SRC_CHANNELS] >= 1 && d[DIB_MLP_SRC_CHANNELS] <= kMlpMaxIn,
                "pointwise_mlp: a source needs 1 <= channels <= 1024");
    DIB_REQUIRE(d[DIB_MLP_SRC_NODES] >= 0 && d[DIB_MLP_SRC_NODES] <= kMlpMaxNodes,
                "pointwise_mlp: an interpolated source needs 1 <= M <= 2048 (0 marks a dense source)");
    pl->src_C[s] = (int)d[DIB_MLP_SRC_CHANNELS];
    pl->src_M[s] = (int)d[DIB_MLP_SRC_NODES];
    pl->src_k[s] = (int)d[DIB_MLP_SRC_K];
    pl->src_col[s] = pl->c_in;
    pl->c_in += pl->src_C[s];
    if (pl->src_M[s] > 0) {
      DIB_REQUIRE(d[DIB_MLP_SRC_K] >= 1 && d[DIB_MLP_SRC_K] <= kMlpMaxK, "pointwise_mlp: need 1 <= k <= 8");
      pl->n_interp++;
    } else {
      pl->n_dense++;
      pl->Kd += pl->src_C[s];
    }
  }
  DIB_REQUIRE(pl->c_in <= kMlpMaxIn, "pointwise_mlp: the concatenated input has more than 1024 rows");
  for (int l = 0; l < n_layers; ++l) {
    const int64_t* d = layers + (size_t)l * DIB_MLP_LAYER;
    DIB_REQUIRE(d[DIB_MLP_LAYER_COUT] >= 1 && d[DIB_MLP_LAYER_COUT] <= kMlpMaxWidth,
                "pointwise_mlp: a layer needs 1 <= C_out <= 256");
    DIB_REQUIRE(d[DIB_MLP_LAYER_RELU] == 0 || d[DIB_MLP_LAYER_RELU] == 1, "pointwise_mlp: relu must be 0 or 1");
    pl->C[l] = (int)d[DIB_MLP_LAYER_COUT];
    pl->Cpad[l] = pad_to(pl->C[l], 16);
    pl->relu[l] = (int)d[DIB_MLP_LAYER_RELU];
  }
  size_t off = 0;
  for (int s = 0; s < n_sources; ++s) {
    pl->proj_off[s] = off;
    if (pl->src_M[s] > 0) off += (size_t)pl->Cpad[0] * pad_to(pl->src_C[s], 8);
  }
  for (int l = 0; l < n_layers; ++l) {
    pl->w_off[l] = off;
    off += (size_t)pl->Cpad[l] * (l == 0 ? pad_to(pl->Kd, 8) : pl->Cpad[l - 1]);
    pl->b_off[l] = off;
    off += pl->Cpad[l];
  }
  pl->packed_floats = off;
  return DIB_OK;
}

static size_t mlp_smem_bytes(const MlpParams& p) {
  return ((size_t)p.xs_floats + 2 * (size_t)p.buf_floats) * sizeof(float);
}

static int mlp_launch(MlpParams& p, int B, cudaStream_t stream) {
  int cmax = 0;
  for (int l = 0; l < p.n_layers; ++l) cmax = p.layer[l].Cpad > cmax ? p.layer[l].Cpad : cmax;
  p.xs_floats = (p.Kd < kMlpChunk ? pad_to(p.Kd, 8) : kMlpChunk) * kMlpStride;
  p.buf_floats = cmax * kMlpStride;
  if (p.n_interp > 0 && kMlpTile * (p.layer[0].Cpad + 4) > p.buf_floats)
    p.buf_floats = kMlpTile * (p.layer[0].Cpad + 4);
  const size_t smem = mlp_smem_bytes(p);
  if (smem > 48 * 1024)
    DIB_CHECK_CUDA(cudaFuncSetAttribute(mlp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  dim3 grid((p.N + kMlpTile - 1) / kMlpTile, B);
  mlp_kernel<<<grid, kMlpThreads, smem, stream>>>(p);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

}  // namespace dib

extern "C" {

size_t pointwise_mlp_packed_bytes(const int64_t* sources, int n_sources, const int64_t* layers, int n_layers) {
  dib::MlpPlan pl;
  if (dib::mlp_plan(sources, n_sources, layers, n_layers, &pl) != DIB_OK) return 0;
  return pl.packed_floats * sizeof(float);
}

int pointwise_mlp_pack_f32(const int64_t* sources, int n_sources, const int64_t* layers, int n_layers, void* packed,
                           size_t packed_bytes, dib_stream_t stream_) {
  using namespace dib;
  cudaStream_t stream = (cudaStream_t)stream_;
  MlpPlan pl;
  const int rc = mlp_plan(sources, n_sources, layers, n_layers, &pl);
  if (rc != DIB_OK) return rc;
  DIB_REQUIRE(packed && ((uintptr_t)packed & 15) == 0, "pointwise_mlp_pack: packed is NULL or not 16-byte aligned");
  if (packed_bytes < pl.packed_floats * sizeof(float)) {
    set_error("pointwise_mlp_pack: packed buffer too small");
    return DIB_ENOMEM;
  }
  float* out = (float*)packed;
  // K columns of W packed into KT >= ceil(K / 8) k tiles (the kernel's count for this matrix)
  auto pack = [&](const float* W, int ld, int C_out, int K, int KT, const MlpPackSeg& seg, float* dst) -> int {
    const int total = pad_to(C_out, 16) * KT * 8;
    if (total == 0) return DIB_OK;
    mlp_pack_kernel<<<(total + 255) / 256, 256, 0, stream>>>(W, ld, C_out, K, KT, total, seg, dst);
    DIB_CHECK_CUDA(cudaGetLastError());
    return DIB_OK;
  };
  for (int l = 0; l < n_layers; ++l) {
    const int64_t* d = layers + (size_t)l * DIB_MLP_LAYER;
    const float* W = (const float*)(uintptr_t)d[DIB_MLP_LAYER_W];
    const float* bias = (const float*)(uintptr_t)d[DIB_MLP_LAYER_B];
    DIB_REQUIRE(W != nullptr, "pointwise_mlp_pack: a layer's W is NULL");
    MlpPackSeg seg = {};
    if (l == 0) {
      for (int s = 0; s < n_sources; ++s) {
        if (pl.src_M[s] > 0) {
          MlpPackSeg one = {};
          one.n = 1; one.orig[0] = pl.src_col[s];
          const int r = pack(W, pl.c_in, pl.C[0], pl.src_C[s], pad_to(pl.src_C[s], 8) / 8, one, out + pl.proj_off[s]);
          if (r != DIB_OK) return r;
        } else {                               // the dense segments start at the running sums of the dense widths
          seg.orig[seg.n] = pl.src_col[s];
          seg.start[seg.n + 1] = seg.start[seg.n] + pl.src_C[s];
          seg.n++;
        }
      }
      const int r = pack(W, pl.c_in, pl.C[0], pl.Kd, pad_to(pl.Kd, 8) / 8, seg, out + pl.w_off[0]);
      if (r != DIB_OK) return r;
    } else {
      // rows [C, Cpad) of the previous layer are zero activations; their weight columns are zero padding
      seg.n = 1;
      const int r = pack(W, pl.C[l - 1], pl.C[l], pl.C[l - 1], pl.Cpad[l - 1] / 8, seg, out + pl.w_off[l]);
      if (r != DIB_OK) return r;
    }
    mlp_bias_kernel<<<(pl.Cpad[l] + 255) / 256, 256, 0, stream>>>(bias, pl.C[l], pl.Cpad[l], out + pl.b_off[l]);
    DIB_CHECK_CUDA(cudaGetLastError());
  }
  return DIB_OK;
}

size_t pointwise_mlp_workspace_bytes(const int64_t* sources, int n_sources, const int64_t* layers, int n_layers,
                                     int B) {
  dib::MlpPlan pl;
  if (B <= 0 || dib::mlp_plan(sources, n_sources, layers, n_layers, &pl) != DIB_OK) return 0;
  size_t bytes = 0;
  for (int s = 0; s < n_sources; ++s) bytes += (size_t)B * pl.src_M[s] * pl.Cpad[0] * sizeof(float);
  return bytes;
}

int pointwise_mlp_f32(const int64_t* sources, int n_sources, const int64_t* layers, int n_layers, const void* packed,
                      size_t packed_bytes, int B, int N, int c_split, float* out, int8_t* pred_a, int32_t* pred_b,
                      void* workspace, size_t workspace_bytes, dib_stream_t stream_) {
  using namespace dib;
  cudaStream_t stream = (cudaStream_t)stream_;
  MlpPlan pl;
  const int rc = mlp_plan(sources, n_sources, layers, n_layers, &pl);
  if (rc != DIB_OK) return rc;
  DIB_REQUIRE(B >= 0 && B <= 65535 && N >= 0, "pointwise_mlp: need 0 <= B <= 65535 and N >= 0");
  const int C_last = pl.C[n_layers - 1];
  DIB_REQUIRE(c_split >= 0 && c_split <= C_last && c_split <= 128,
              "pointwise_mlp: need 0 <= c_split <= min(C_out, 128) (0 selects the activations)");
  if (B == 0 || N == 0) return DIB_OK;
  DIB_REQUIRE(packed && ((uintptr_t)packed & 15) == 0 && packed_bytes >= pl.packed_floats * sizeof(float),
              "pointwise_mlp: packed is NULL, misaligned or smaller than pointwise_mlp_packed_bytes");
  if (c_split == 0) DIB_REQUIRE(out != nullptr, "pointwise_mlp: out is NULL");
  else DIB_REQUIRE(pred_a != nullptr && (c_split == C_last || pred_b != nullptr), "pointwise_mlp: a prediction output is NULL");
  const size_t need = pointwise_mlp_workspace_bytes(sources, n_sources, layers, n_layers, B);
  if (need > 0) {
    DIB_REQUIRE(workspace && ((uintptr_t)workspace & 15) == 0, "pointwise_mlp: workspace is NULL or misaligned");
    if (workspace_bytes < need) {
      set_error("pointwise_mlp: workspace too small");
      return DIB_ENOMEM;
    }
  }
  const float* pk = (const float*)packed;
  MlpParams p = {};
  p.N = N;
  char* ws = (char*)workspace;
  for (int s = 0; s < n_sources; ++s) {
    const int64_t* d = sources + (size_t)s * DIB_MLP_SRC;
    const float* data = (const float*)(uintptr_t)d[DIB_MLP_SRC_DATA];
    DIB_REQUIRE(data != nullptr, "pointwise_mlp: a source's data is NULL");
    if (pl.src_M[s] > 0) {
      const float* w = (const float*)(uintptr_t)d[DIB_MLP_SRC_W];
      const int32_t* idx = (const int32_t*)(uintptr_t)d[DIB_MLP_SRC_IDX];
      DIB_REQUIRE(w && idx, "pointwise_mlp: an interpolated source's w or idx is NULL");
      DIB_REQUIRE(d[DIB_MLP_SRC_BSTRIDE] >= (int64_t)pl.src_C[s] * pl.src_M[s],
                  "pointwise_mlp: a source's batch stride is smaller than channels x M");
      // P_s = W1[:, rows of s] . F_s for every node, [B][M][C1pad]: the same kernel with the nodes as its points
      MlpParams q = {};
      q.N = pl.src_M[s];
      q.n_dense = 1; q.Kd = pl.src_C[s]; q.n_layers = 1;
      q.dense[0] = MlpDense{data, (long long)d[DIB_MLP_SRC_BSTRIDE], pl.src_C[s], 0};
      q.layer[0] = MlpLayer{pk + pl.proj_off[s], nullptr, pl.C[0], pl.Cpad[0], 0};
      q.out_mode = kOutTransposed;
      q.out = (float*)ws;
      const int r = mlp_launch(q, B, stream);
      if (r != DIB_OK) return r;
      p.interp[p.n_interp++] = MlpInterp{(const float*)ws, w, idx, pl.src_M[s], pl.src_k[s]};
      ws += (size_t)B * pl.src_M[s] * pl.Cpad[0] * sizeof(float);
    } else {
      DIB_REQUIRE(d[DIB_MLP_SRC_BSTRIDE] >= (int64_t)pl.src_C[s] * N,
                  "pointwise_mlp: a source's batch stride is smaller than channels x N");
      p.dense[p.n_dense] = MlpDense{data, (long long)d[DIB_MLP_SRC_BSTRIDE], pl.src_C[s], p.Kd};
      p.n_dense++;
      p.Kd += pl.src_C[s];
    }
  }
  p.n_layers = n_layers;
  for (int l = 0; l < n_layers; ++l)
    p.layer[l] = MlpLayer{pk + pl.w_off[l], pk + pl.b_off[l], pl.C[l], pl.Cpad[l], pl.relu[l]};
  p.out_mode = c_split == 0 ? kOutActivations : kOutArgmax;
  p.c_split = c_split;
  p.out = out;
  p.pred_a = pred_a;
  p.pred_b = pred_b;
  return mlp_launch(p, B, stream);
}

}  // extern "C"
