// Fused inference of the point encoder's node kNN module and of its global feature (SURVEY.md 8f row N21, DESIGN.md
// 4.26): GeneralKNNFusionModule.forward (models/layers_pc.py:793-818) and final_pointnet + torch.max over the nodes
// (models/networks_pc.py:107-115), BatchNorm folded into the weights on the host.  No [B, C, M, K] or [B, C, M]
// activation touches global memory.
//
//   kf_kernel, kNN mode   CTA = one tile of 32 columns = G = min(32 / K, 8) query nodes x their K neighbours, 8 warps
//                         of 64 output rows x 32 columns (widths up to 512).  Columns are staged from
//                         knn_search_launch's indices as knn_group_kernel computes them (rows 0-2 database[idx] -
//                         query by __fsub_rn, rows 3.. features[idx]), rounded to TF32.  The "before" layers run on
//                         the tensor cores with the activations in shared memory; the max over each node's K columns
//                         of the last one (stored rounded, so the max is exact) is projected once per node by the
//                         pooled half of the first "after" layer's weights (f32 fma chain in ascending input row) and
//                         added to that layer's columns like a bias: W [max; x] = W_p max + W_x x.  The "after" layers
//                         follow and the max over each node's K columns of the last one (f32, not rounded) is written
//                         to out [B][C_out][M].
//   kf_kernel, dense mode CTA = 32 columns of up to four dense sources, one to three layers, the max over the tile's
//                         columns of the last one to partial [B][C_out][tiles];
//   kf_max_kernel         out [B][C_out] = the max over the tiles in ascending order (pointwise_mlp_max_f32).
//
// Operand rounding is pointwise_mlp's (tf32_mma.cuh): weights once when packed, staged values and the activations fed
// to the next layer when stored; bias, ReLU (NaN stays NaN) and the maxes are f32, a NaN anywhere in a group gives NaN
// (torch.max(dim)'s rule).  No atomics: every output has one writer and every sum a fixed order.
#include <math.h>

#include "common.cuh"
#include "nearest_k.cuh"
#include "tf32_mma.cuh"

namespace dib {

constexpr int kKfTile = 32;           // columns per CTA
constexpr int kKfStride = 40;         // floats per shared row: 40 % 32 == 8 keeps the B-fragment loads conflict-free
constexpr int kKfThreads = 256;       // 8 warps x 64 rows
constexpr int kKfMaxWidth = 512;
constexpr int kKfMaxSide = 3;         // layers before and after the per-node max
constexpr int kKfMaxLayers = 2 * kKfMaxSide;
constexpr int kKfMaxGroups = 8;       // nodes per tile
constexpr int kKfMaxSources = 4;
constexpr int kKfMaxK = 32;
constexpr int kKfMaxNodes = 2048;

struct KfLayer { const float* W; const float* bias; int C; int Cpad; int KT; int relu; };
struct KfParams {
  const float* query; const float* database; const float* features; const int32_t* idx;
  const float* src[kKfMaxSources]; long long bstride[kKfMaxSources]; int src_row0[kKfMaxSources + 1];
  int n_src, dense, c_in, c_in_pad, M, N, K, G, Kg, n_layers, n_before;
  KfLayer layer[kKfMaxLayers];
  const float* projT;                 // [C_before][Cpad of the first after layer], rounded
  int x_floats, y_floats;
  float* out;
  int out_cols;                       // out [B][C_out][out_cols]
};

__device__ __forceinline__ float kf_max(float a, float v) { return (v != v || v > a) ? v : a; }   // NaN sticks

__global__ void __launch_bounds__(kKfThreads, 1) kf_kernel(const __grid_constant__ KfParams p) {
  extern __shared__ __align__(16) float kf_smem[];
  float* bufX = kf_smem;                                   // [rows][kKfStride]: the staged input, then odd layers
  float* bufY = bufX + p.x_floats;                         // even layers
  float* pooled = bufY + p.y_floats;                       // [C_before][G]
  const int tid = threadIdx.x, lane = tid & 31, wm = tid >> 5;
  const int g4 = lane >> 2, t4 = lane & 3;
  const int b = blockIdx.y, tile = blockIdx.x, G = p.G, Kg = p.Kg;

  // stage the input columns, rounded to TF32; padding rows and columns are zero
  for (int i = tid; i < p.c_in_pad * kKfTile; i += kKfThreads) {
    const int r = i >> 5, n = i & 31;
    float v = 0.f;
    if (r < p.c_in) {
      if (p.dense) {
        const int col = tile * kKfTile + n;
        if (col < p.N) {
          int s = 0;
#pragma unroll
          for (int q = 1; q < kKfMaxSources; ++q)
            if (q < p.n_src && r >= p.src_row0[q]) s = q;
          v = p.src[s][(size_t)b * p.bstride[s] + (size_t)(r - p.src_row0[s]) * p.N + col];
        }
      } else {
        const int g = n / Kg, m = tile * G + g;
        if (g < G && m < p.M) {
          const int id = p.idx[((size_t)b * p.M + m) * Kg + (n - g * Kg)];
          v = r < 3 ? __fsub_rn(p.database[((size_t)b * 3 + r) * p.N + id], p.query[((size_t)b * 3 + r) * p.M + m])
                    : p.features[((size_t)b * (p.c_in - 3) + (r - 3)) * p.N + id];
        }
      }
    }
    bufX[r * kKfStride + n] = tf32_rna(v);
  }
  __syncthreads();

  float* in = bufX;
  float* proj = nullptr;                                   // [Cpad of the first after layer][G]
  for (int l = 0; l < p.n_layers; ++l) {
    const KfLayer L = p.layer[l];
    const bool split = !p.dense && l == p.n_before;
    if (split) {
      // the per-node max of the last "before" layer (stored rounded), then its projection by W_p, once per node
      const int Cb = p.layer[l - 1].C;
      for (int i = tid; i < Cb * G; i += kKfThreads) {
        const int c = i / G, g = i - c * G;
        const float* row = in + c * kKfStride + g * Kg;
        float v = row[0];
        for (int j = 1; j < Kg; ++j) v = kf_max(v, row[j]);
        pooled[i] = v;
      }
      proj = pooled + Cb * G;
      __syncthreads();
      for (int m = tid; m < L.Cpad; m += kKfThreads) {
        float acc[kKfMaxGroups];
#pragma unroll
        for (int g = 0; g < kKfMaxGroups; ++g) acc[g] = 0.f;
        for (int c = 0; c < Cb; ++c) {
          const float w = __ldg(p.projT + (size_t)c * L.Cpad + m);
#pragma unroll
          for (int g = 0; g < kKfMaxGroups; ++g)
            if (g < G) acc[g] = fmaf(w, pooled[c * G + g], acc[g]);
        }
#pragma unroll
        for (int g = 0; g < kKfMaxGroups; ++g)
          if (g < G) proj[m * G + g] = acc[g];
      }
      __syncthreads();
    }
    float acc[4][4][4];
#pragma unroll
    for (int mt = 0; mt < 4; ++mt)
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[mt][nt][i] = 0.f;
    mma_block_64x32<kKfStride>(acc, in, reinterpret_cast<const float4*>(L.W), L.KT, L.Cpad >> 4, 0, L.KT, wm, 0,
                               lane);
    float* out = (l & 1) ? bufX : bufY;
    const bool last = l == p.n_layers - 1;
#pragma unroll
    for (int mt = 0; mt < 4; ++mt) {
      if ((wm * 4 + mt) * 16 < L.Cpad) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int m = (wm * 4 + mt) * 16 + g4 + (i >> 1) * 8;
          const float bias = L.bias[m];
#pragma unroll
          for (int nt = 0; nt < 4; ++nt) {
            const int n = nt * 8 + 2 * t4 + (i & 1);
            float v = acc[mt][nt][i];
            if (split) {
              const int g = n / Kg;
              if (g < G) v += proj[m * G + g];
            }
            v += bias;
            if (L.relu) v = v < 0.f ? 0.f : v;             // NaN < 0 is false: NaN stays, as torch.relu
            if (m >= L.C) v = 0.f;                         // padding rows feed zero weights: keep them finite
            out[m * kKfStride + n] = last ? v : tf32_rna(v);
          }
        }
      }
    }
    __syncthreads();
    in = out;
  }

  // the max over each group's columns of the last layer (f32)
  const int C = p.layer[p.n_layers - 1].C;
  for (int i = tid; i < C * G; i += kKfThreads) {
    const int c = i / G, g = i - c * G;
    int cols, o;
    if (p.dense) {
      cols = min(kKfTile, p.N - tile * kKfTile);
      o = tile;
    } else {
      o = tile * G + g;
      if (o >= p.M) continue;
      cols = Kg;
    }
    const float* row = in + c * kKfStride + g * Kg;
    float v = row[0];
    for (int j = 1; j < cols; ++j) v = kf_max(v, row[j]);
    p.out[((size_t)b * C + c) * p.out_cols + o] = v;
  }
}

// one thread per (b, c): the max over the tiles in ascending order
__global__ void kf_max_kernel(const float* __restrict__ partial, int tiles, int total, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const float* row = partial + (size_t)i * tiles;
  float v = row[0];
  for (int t = 1; t < tiles; ++t) v = kf_max(v, row[t]);
  out[i] = v;
}

// W [C_out][ld] columns [col0, col0 + K) -> the A-fragment order with KT k tiles, rounded to TF32, zero padding
__global__ void kf_pack_kernel(const float* __restrict__ W, int ld, int col0, int C_out, int K, int KT, int total,
                               float* __restrict__ out) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  int row, col;
  a_frag_row_col(e, KT, row, col);
  out[e] = row < C_out && col < K ? tf32_rna(W[(size_t)row * ld + col0 + col]) : 0.f;
}

// W [C_out][ld] columns [0, K) -> transposed [K][Cpad], rounded to TF32, zero padding; and the bias padded to Cpad
__global__ void kf_pack_t_kernel(const float* __restrict__ W, int ld, int C_out, int K, int Cpad,
                                 float* __restrict__ out) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= K * Cpad) return;
  const int c = e / Cpad, m = e - c * Cpad;
  out[e] = m < C_out ? tf32_rna(W[(size_t)m * ld + c]) : 0.f;
}

__global__ void kf_bias_kernel(const float* __restrict__ b, int C, int Cpad, float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < Cpad) out[c] = c < C && b != nullptr ? b[c] : 0.f;
}

// Where every layer lives in the packed buffer (floats); a function of the widths alone.
struct KfPlan {
  int c_in, c_in_pad, n_layers, n_before;
  int C[kKfMaxLayers], Cpad[kKfMaxLayers], KT[kKfMaxLayers], relu[kKfMaxLayers];
  size_t w_off[kKfMaxLayers], b_off[kKfMaxLayers], projT_off, packed_floats;
};

static inline int kf_pad(int x, int m) { return (x + m - 1) / m * m; }

// n_after = 0: a plain chain of n_before layers (pointwise_mlp_max)
static int kf_plan(const char* who, int c_in, const int64_t* layers, int n_before, int n_after, KfPlan* pl) {
  DIB_REQUIRE(layers != nullptr, "%s: NULL layer table", who);
  DIB_REQUIRE(n_before >= 1 && n_before <= kKfMaxSide && n_after >= 0 && n_after <= kKfMaxSide,
              "%s: need 1 to 3 layers on each side of the max", who);
  DIB_REQUIRE(c_in >= 1 && c_in <= kKfMaxWidth, "%s: need 1 <= input rows <= 512", who);
  pl->c_in = c_in;
  pl->c_in_pad = kf_pad(c_in, 8);
  pl->n_layers = n_before + n_after;
  pl->n_before = n_before;
  size_t off = 0;
  for (int l = 0; l < pl->n_layers; ++l) {
    const int64_t* d = layers + (size_t)l * DIB_MLP_LAYER;
    DIB_REQUIRE(d[DIB_MLP_LAYER_COUT] >= 1 && d[DIB_MLP_LAYER_COUT] <= kKfMaxWidth,
                "%s: a layer needs 1 <= C_out <= 512", who);
    DIB_REQUIRE(d[DIB_MLP_LAYER_RELU] == 0 || d[DIB_MLP_LAYER_RELU] == 1, "%s: relu must be 0 or 1", who);
    pl->C[l] = (int)d[DIB_MLP_LAYER_COUT];
    pl->Cpad[l] = kf_pad(pl->C[l], 16);
    pl->relu[l] = (int)d[DIB_MLP_LAYER_RELU];
    pl->KT[l] = (l == 0 ? pl->c_in_pad : pl->Cpad[l - 1]) / 8;
    pl->w_off[l] = off;
    off += (size_t)pl->Cpad[l] * pl->KT[l] * 8;
    pl->b_off[l] = off;
    off += pl->Cpad[l];
  }
  pl->projT_off = off;
  if (n_after > 0) off += (size_t)pl->C[n_before - 1] * pl->Cpad[n_before];
  pl->packed_floats = off;
  return DIB_OK;
}

static int kf_pack(const char* who, const KfPlan& pl, const int64_t* layers, float* out, cudaStream_t stream) {
  for (int l = 0; l < pl.n_layers; ++l) {
    const int64_t* d = layers + (size_t)l * DIB_MLP_LAYER;
    const float* W = (const float*)(uintptr_t)d[DIB_MLP_LAYER_W];
    const float* bias = (const float*)(uintptr_t)d[DIB_MLP_LAYER_B];
    DIB_REQUIRE(W != nullptr, "%s: a layer's W is NULL", who);
    const int K = l == 0 ? pl.c_in : pl.C[l - 1];
    const bool split = l == pl.n_before;                   // W = [W_p | W_x], [C_out][2 C_before]
    const int ld = split ? 2 * K : K;
    const int total = pl.Cpad[l] * pl.KT[l] * 8;
    kf_pack_kernel<<<(total + 255) / 256, 256, 0, stream>>>(W, ld, split ? K : 0, pl.C[l], K, pl.KT[l], total,
                                                            out + pl.w_off[l]);
    DIB_CHECK_CUDA(cudaGetLastError());
    if (split) {
      const int tt = K * pl.Cpad[l];
      kf_pack_t_kernel<<<(tt + 255) / 256, 256, 0, stream>>>(W, ld, pl.C[l], K, pl.Cpad[l], out + pl.projT_off);
      DIB_CHECK_CUDA(cudaGetLastError());
    }
    kf_bias_kernel<<<(pl.Cpad[l] + 255) / 256, 256, 0, stream>>>(bias, pl.C[l], pl.Cpad[l], out + pl.b_off[l]);
    DIB_CHECK_CUDA(cudaGetLastError());
  }
  return DIB_OK;
}

static void kf_fill_layers(const KfPlan& pl, const float* pk, KfParams& p) {
  p.c_in = pl.c_in;
  p.c_in_pad = pl.c_in_pad;
  p.n_layers = pl.n_layers;
  p.n_before = pl.n_before;
  int x_rows = pl.c_in_pad, y_rows = 0;
  for (int l = 0; l < pl.n_layers; ++l) {
    p.layer[l] = KfLayer{pk + pl.w_off[l], pk + pl.b_off[l], pl.C[l], pl.Cpad[l], pl.KT[l], pl.relu[l]};
    int& rows = (l & 1) ? x_rows : y_rows;
    rows = pl.Cpad[l] > rows ? pl.Cpad[l] : rows;
  }
  p.projT = pk + pl.projT_off;
  p.x_floats = x_rows * kKfStride;
  p.y_floats = y_rows * kKfStride;
}

static int kf_launch(const KfPlan& pl, KfParams& p, int B, int tiles, cudaStream_t stream) {
  size_t floats = (size_t)p.x_floats + p.y_floats;
  if (!p.dense && pl.n_layers > pl.n_before)
    floats += (size_t)p.G * (pl.C[pl.n_before - 1] + pl.Cpad[pl.n_before]);
  const size_t smem = floats * sizeof(float);              // <= 2 x 512 x 40 + 2 x 512 x 8 floats = 192 KB
  if (smem > 48 * 1024)
    DIB_CHECK_CUDA(cudaFuncSetAttribute(kf_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  kf_kernel<<<dim3(tiles, B), kKfThreads, smem, stream>>>(p);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

}  // namespace dib

extern "C" {

size_t knn_fusion_packed_bytes(int C_in, const int64_t* layers, int n_before, int n_after) {
  dib::KfPlan pl;
  if (n_after < 1) {
    dib::set_error("knn_fusion: need 1 to 3 layers on each side of the max");
    return 0;
  }
  if (dib::kf_plan("knn_fusion", C_in, layers, n_before, n_after, &pl) != DIB_OK) return 0;
  return pl.packed_floats * sizeof(float);
}

int knn_fusion_pack_f32(int C_in, const int64_t* layers, int n_before, int n_after, void* packed, size_t packed_bytes,
                        dib_stream_t stream) {
  using namespace dib;
  DIB_REQUIRE(n_after >= 1, "knn_fusion: need 1 to 3 layers on each side of the max");
  KfPlan pl;
  const int rc = kf_plan("knn_fusion", C_in, layers, n_before, n_after, &pl);
  if (rc != DIB_OK) return rc;
  DIB_REQUIRE(packed && ((uintptr_t)packed & 15) == 0, "knn_fusion_pack: packed is NULL or not 16-byte aligned");
  if (packed_bytes < pl.packed_floats * sizeof(float)) {
    set_error("knn_fusion_pack: packed buffer too small");
    return DIB_ENOMEM;
  }
  return kf_pack("knn_fusion_pack", pl, layers, (float*)packed, (cudaStream_t)stream);
}

int knn_fusion_f32(const float* query, const float* database, const float* features, int B, int C, int M, int N,
                   int K, const int64_t* layers, int n_before, int n_after, const void* packed, size_t packed_bytes,
                   int32_t* knn_idx, float* out, dib_stream_t stream_) {
  using namespace dib;
  cudaStream_t stream = (cudaStream_t)stream_;
  DIB_REQUIRE(n_after >= 1, "knn_fusion: need 1 to 3 layers on each side of the max");
  DIB_REQUIRE(C >= 1 && C <= kKfMaxWidth - 3, "knn_fusion: need 1 <= C <= 509 (3 + C input rows)");
  KfPlan pl;
  const int rc = kf_plan("knn_fusion", 3 + C, layers, n_before, n_after, &pl);
  if (rc != DIB_OK) return rc;
  DIB_REQUIRE(B >= 0 && B <= 65535 && M >= 0, "knn_fusion: need 0 <= B <= 65535 and M >= 0");
  DIB_REQUIRE(N >= 1 && N <= kKfMaxNodes, "knn_fusion: need 1 <= N <= 2048");
  DIB_REQUIRE(K >= 1 && K <= kKfMaxK && K <= N, "knn_fusion: need 1 <= K <= min(32, N)");
  if (B == 0 || M == 0) return DIB_OK;
  DIB_REQUIRE(query && database && features && knn_idx && out, "knn_fusion: NULL argument");
  DIB_REQUIRE(packed && ((uintptr_t)packed & 15) == 0 && packed_bytes >= pl.packed_floats * sizeof(float),
              "knn_fusion: packed is NULL, misaligned or smaller than knn_fusion_packed_bytes");
  DIB_REQUIRE((long long)M * K <= 0x7fffffffLL, "knn_fusion: M * K must fit in int32");
  const int r = knn_search_launch(query, database, B, M, N, K, knn_idx, stream);
  if (r != DIB_OK) return r;
  KfParams p = {};
  p.query = query; p.database = database; p.features = features; p.idx = knn_idx;
  p.M = M; p.N = N; p.K = K;
  p.G = kKfTile / K < kKfMaxGroups ? kKfTile / K : kKfMaxGroups;
  p.Kg = K;
  kf_fill_layers(pl, (const float*)packed, p);
  p.out = out;
  p.out_cols = M;
  return kf_launch(pl, p, B, (M + p.G - 1) / p.G, stream);
}

size_t pointwise_mlp_max_packed_bytes(int C_in, const int64_t* layers, int n_layers) {
  dib::KfPlan pl;
  if (dib::kf_plan("pointwise_mlp_max", C_in, layers, n_layers, 0, &pl) != DIB_OK) return 0;
  return pl.packed_floats * sizeof(float);
}

int pointwise_mlp_max_pack_f32(int C_in, const int64_t* layers, int n_layers, void* packed, size_t packed_bytes,
                               dib_stream_t stream) {
  using namespace dib;
  KfPlan pl;
  const int rc = kf_plan("pointwise_mlp_max", C_in, layers, n_layers, 0, &pl);
  if (rc != DIB_OK) return rc;
  DIB_REQUIRE(packed && ((uintptr_t)packed & 15) == 0, "pointwise_mlp_max_pack: packed is NULL or not 16-byte aligned");
  if (packed_bytes < pl.packed_floats * sizeof(float)) {
    set_error("pointwise_mlp_max_pack: packed buffer too small");
    return DIB_ENOMEM;
  }
  return kf_pack("pointwise_mlp_max_pack", pl, layers, (float*)packed, (cudaStream_t)stream);
}

size_t pointwise_mlp_max_workspace_bytes(int C_out, int B, int N) {
  if (C_out < 1 || B < 1 || N < 1) return 0;
  return (size_t)B * C_out * ((N + dib::kKfTile - 1) / dib::kKfTile) * sizeof(float);
}

int pointwise_mlp_max_f32(const int64_t* sources, int n_sources, const int64_t* layers, int n_layers,
                          const void* packed, size_t packed_bytes, int B, int N, float* out, void* workspace,
                          size_t workspace_bytes, dib_stream_t stream_) {
  using namespace dib;
  cudaStream_t stream = (cudaStream_t)stream_;
  DIB_REQUIRE(sources != nullptr, "pointwise_mlp_max: NULL source table");
  DIB_REQUIRE(n_sources >= 1 && n_sources <= kKfMaxSources, "pointwise_mlp_max: need 1 <= n_sources <= 4");
  KfParams p = {};
  p.dense = 1;
  p.n_src = n_sources;
  int c_in = 0;
  for (int s = 0; s < n_sources; ++s) {
    const int64_t* d = sources + (size_t)s * DIB_MLP_SRC;
    DIB_REQUIRE(d[DIB_MLP_SRC_NODES] == 0, "pointwise_mlp_max: every source must be dense (NODES = 0)");
    DIB_REQUIRE(d[DIB_MLP_SRC_CHANNELS] >= 1 && d[DIB_MLP_SRC_CHANNELS] <= kKfMaxWidth,
                "pointwise_mlp_max: a source needs 1 <= channels <= 512");
    p.src[s] = (const float*)(uintptr_t)d[DIB_MLP_SRC_DATA];
    p.bstride[s] = (long long)d[DIB_MLP_SRC_BSTRIDE];
    p.src_row0[s] = c_in;
    c_in += (int)d[DIB_MLP_SRC_CHANNELS];
    DIB_REQUIRE(c_in <= kKfMaxWidth, "pointwise_mlp_max: the concatenated input has more than 512 rows");
  }
  p.src_row0[n_sources] = c_in;
  KfPlan pl;
  const int rc = kf_plan("pointwise_mlp_max", c_in, layers, n_layers, 0, &pl);
  if (rc != DIB_OK) return rc;
  DIB_REQUIRE(B >= 0 && B <= 65535 && N >= 0, "pointwise_mlp_max: need 0 <= B <= 65535 and N >= 0");
  if (B == 0) return DIB_OK;
  DIB_REQUIRE(N >= 1, "pointwise_mlp_max: the max over no columns is undefined (N = 0)");
  for (int s = 0; s < n_sources; ++s) {
    DIB_REQUIRE(p.src[s] != nullptr, "pointwise_mlp_max: a source's data is NULL");
    DIB_REQUIRE(p.bstride[s] >= (long long)(p.src_row0[s + 1] - p.src_row0[s]) * N,
                "pointwise_mlp_max: a source's batch stride is smaller than channels x N");
  }
  DIB_REQUIRE(out != nullptr, "pointwise_mlp_max: out is NULL");
  DIB_REQUIRE(packed && ((uintptr_t)packed & 15) == 0 && packed_bytes >= pl.packed_floats * sizeof(float),
              "pointwise_mlp_max: packed is NULL, misaligned or smaller than pointwise_mlp_max_packed_bytes");
  const int C_out = pl.C[n_layers - 1];
  const size_t need = pointwise_mlp_max_workspace_bytes(C_out, B, N);
  DIB_REQUIRE(workspace && ((uintptr_t)workspace & 15) == 0, "pointwise_mlp_max: workspace is NULL or misaligned");
  if (workspace_bytes < need) {
    set_error("pointwise_mlp_max: workspace too small");
    return DIB_ENOMEM;
  }
  const int tiles = (N + kKfTile - 1) / kKfTile;
  p.N = N;
  p.G = 1;
  p.Kg = kKfTile;
  kf_fill_layers(pl, (const float*)packed, p);
  p.out = (float*)workspace;
  p.out_cols = tiles;
  const int r = kf_launch(pl, p, B, tiles, stream);
  if (r != DIB_OK) return r;
  const int total = B * C_out;
  kf_max_kernel<<<(total + 255) / 256, 256, 0, stream>>>((const float*)workspace, tiles, total, out);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

}  // extern "C"
