// Fused inference of the decoder's node-level PointNets (SURVEY.md 8f row N22, DESIGN.md 4.27): node_b_attention_pn,
// node_b_pn, node_a_attention_pn and node_a_pn of KeypointDetector.forward (models/networks_united.py:147-189), BatchNorm
// folded into the weights on the host.  The input concatenation is never built, and a source that is the same for every
// node of a sample is projected once per sample instead of once per column.
//
//   nm_proj_kernel   one thread per (output row of layer 1, group of kNmProjB samples): proj[b][m] = the broadcast
//                    rows' block of W1 times the sample's broadcast values, as an f32 fma chain in ascending input row
//                    (one launch per broadcast source, each continuing the previous one's sums).
//   nm_kernel        CTA = 32 columns of up to four dense sources, 8 warps, one to three layers of up to 1024 rows.  The
//                    activations live in one shared buffer [rows][kNmStride] that every layer overwrites in place: a
//                    warp computes 64 rows per pass and keeps kPasses (1 or 2) passes of accumulators in registers, so
//                    1024 rows are held until every warp has read the layer's input.  Layer 1 adds proj[b][m] before
//                    the bias; the last layer (f32, not rounded) is written to out [B][C_out][M].
//
// Operand rounding is pointwise_mlp's (tf32_mma.cuh): weights once when packed, staged values (dense and broadcast) and
// the activations fed to the next layer when stored; the broadcast products are exact in f32 (two TF32 operands), bias
// and ReLU (NaN stays NaN) are f32.  No atomics: every output has one writer and every sum a fixed order.
#include <math.h>

#include "common.cuh"
#include "tf32_mma.cuh"
#include "tf32_pack.cuh"

namespace dib {

constexpr int kNmTile = 32;           // columns per CTA
constexpr int kNmStride = 40;         // floats per shared row: 40 % 32 == 8 keeps the B-fragment loads conflict-free
constexpr int kNmThreads = 256;       // 8 warps x 64 rows per pass
constexpr int kNmPassRows = 512;
constexpr int kNmMaxWidth = 1024;     // dense input rows and every layer
constexpr int kNmMaxBcast = 65536;    // per-sample input rows
constexpr int kNmMaxLayers = 3;
constexpr int kNmMaxDense = 4;
constexpr int kNmProjB = 8;           // samples per thread of nm_proj_kernel: each weight is read once per 8 samples
static_assert(kNmMaxDense <= kPackMaxSegs, "the dense sources are column segments of W1");

struct NmLayer { const float* W; const float* bias; int C; int Cpad; int KT; int relu; };
struct NmParams {
  const float* src[kNmMaxDense]; long long bstride[kNmMaxDense]; int src_row0[kNmMaxDense + 1];
  int n_src, c_in, c_in_pad, M, n_layers;
  NmLayer layer[kNmMaxLayers];
  const float* proj;                  // [B][Cpad of layer 1], or NULL without broadcast rows
  float* out;                         // [B][C_out][M]
};

template <int kPasses>
__global__ void __launch_bounds__(kNmThreads, 1) nm_kernel(const __grid_constant__ NmParams p) {
  extern __shared__ __align__(16) float nm_smem[];
  float* buf = nm_smem;
  const int tid = threadIdx.x, lane = tid & 31, wm = tid >> 5;
  const int g4 = lane >> 2, t4 = lane & 3;
  const int b = blockIdx.y, col0 = blockIdx.x * kNmTile;

  // stage the dense rows, rounded to TF32; padding rows and columns are zero
  for (int i = tid; i < p.c_in_pad * kNmTile; i += kNmThreads) {
    const int r = i >> 5, n = i & 31, col = col0 + n;
    float v = 0.f;
    if (r < p.c_in && col < p.M) {
      int s = 0;
#pragma unroll
      for (int q = 1; q < kNmMaxDense; ++q)
        if (q < p.n_src && r >= p.src_row0[q]) s = q;
      v = p.src[s][(size_t)b * p.bstride[s] + (size_t)(r - p.src_row0[s]) * p.M + col];
    }
    buf[r * kNmStride + n] = tf32_rna(v);
  }
  __syncthreads();

  for (int l = 0; l < p.n_layers; ++l) {
    const NmLayer L = p.layer[l];
    const bool last = l == p.n_layers - 1;
    const float* proj = l == 0 && p.proj != nullptr ? p.proj + (size_t)b * L.Cpad : nullptr;
    float acc[kPasses][4][4][4];
#pragma unroll
    for (int h = 0; h < kPasses; ++h) {
#pragma unroll
      for (int mt = 0; mt < 4; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
          for (int i = 0; i < 4; ++i) acc[h][mt][nt][i] = 0.f;
      if (h * kNmPassRows < L.Cpad)
        mma_block_64x32<kNmStride>(acc[h], buf, reinterpret_cast<const float4*>(L.W), L.KT, L.Cpad >> 4, 0, L.KT,
                                   h * (kNmPassRows / 64) + wm, 0, lane);
    }
    __syncthreads();                                       // every warp has read the layer's input: overwrite it
#pragma unroll
    for (int h = 0; h < kPasses; ++h) {
#pragma unroll
      for (int mt = 0; mt < 4; ++mt) {
        const int m0 = h * kNmPassRows + (wm * 4 + mt) * 16;
        if (m0 < L.Cpad) {
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int m = m0 + g4 + (i >> 1) * 8;
            const float add = proj != nullptr ? proj[m] : 0.f;
            const float bias = L.bias[m];
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
              const int n = nt * 8 + 2 * t4 + (i & 1);
              buf[m * kNmStride + n] = layer_value(acc[h][mt][nt][i], proj != nullptr, [&] { return add; }, bias,
                                                   L.relu, m >= L.C, last);
            }
          }
        }
      }
    }
    __syncthreads();
  }

  const int C = p.layer[p.n_layers - 1].C;
  const int cols = min(kNmTile, p.M - col0);
  for (int i = tid; i < C * kNmTile; i += kNmThreads) {
    const int c = i >> 5, n = i & 31;
    if (n < cols) p.out[((size_t)b * C + c) * p.M + col0 + n] = buf[c * kNmStride + n];
  }
}

// proj[b][m] (+)= sum over the source's C rows c, ascending, of WbT[c][m] * tf32(v[b][c]) as an f32 fma chain; first = 1
// starts the sums at zero, later sources continue them.  Grid ((Cpad + 255) / 256, ceil(B / kNmProjB)).
__global__ void nm_proj_kernel(const float* __restrict__ v, long long bstride, int C, const float* __restrict__ WbT,
                               int Cpad, int B, int first, float* __restrict__ proj) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  const int b0 = blockIdx.y * kNmProjB;
  if (m >= Cpad) return;
  float acc[kNmProjB];
#pragma unroll
  for (int j = 0; j < kNmProjB; ++j) acc[j] = first || b0 + j >= B ? 0.f : proj[(size_t)(b0 + j) * Cpad + m];
  for (int c = 0; c < C; ++c) {
    const float w = __ldg(WbT + (size_t)c * Cpad + m);
#pragma unroll
    for (int j = 0; j < kNmProjB; ++j)
      if (b0 + j < B) acc[j] = fmaf(w, tf32_rna(__ldg(v + (size_t)(b0 + j) * bstride + c)), acc[j]);
  }
#pragma unroll
  for (int j = 0; j < kNmProjB; ++j)
    if (b0 + j < B) proj[(size_t)(b0 + j) * Cpad + m] = acc[j];
}

// Where every layer lives in the packed buffer (floats) and which sources are dense; a function of the source
// widths, their kinds and the layer widths alone.
struct NmPlan {
  int n_dense, c_dense, c_dense_pad, c_bcast, c_in, n_layers;
  PackSegs dense;                     // dense input row r is W1's column dense.col[s] + r - dense.start[s]
  PackedLayer layer[kNmMaxLayers];
  size_t wbt_off, packed_floats;
};

static int nm_plan(const char* who, const int64_t* sources, int n_sources, const int64_t* layers, int n_layers,
                   NmPlan* pl) {
  DIB_REQUIRE(sources != nullptr && layers != nullptr, "%s: NULL source or layer table", who);
  DIB_REQUIRE(n_sources >= 1, "%s: need at least one source", who);
  DIB_REQUIRE(n_layers >= 1 && n_layers <= kNmMaxLayers, "%s: need 1 to 3 layers", who);
  pl->n_dense = pl->c_dense = pl->c_bcast = 0;
  int c_in = 0;
  for (int s = 0; s < n_sources; ++s) {
    const int64_t* d = sources + (size_t)s * DIB_MLP_SRC;
    DIB_REQUIRE(d[DIB_MLP_SRC_NODES] == 0, "%s: a source cannot be interpolated (NODES must be 0)", who);
    DIB_REQUIRE(d[DIB_MLP_SRC_BCAST] == 0 || d[DIB_MLP_SRC_BCAST] == 1, "%s: BCAST must be 0 or 1", who);
    DIB_REQUIRE(d[DIB_MLP_SRC_CHANNELS] >= 1 && d[DIB_MLP_SRC_CHANNELS] <= kNmMaxBcast,
                "%s: a source needs 1 <= channels <= 65536", who);
    const int C = (int)d[DIB_MLP_SRC_CHANNELS];
    if (d[DIB_MLP_SRC_BCAST]) {
      DIB_REQUIRE(pl->c_bcast + C <= kNmMaxBcast, "%s: more than 65536 per-sample rows", who);
      pl->c_bcast += C;
    } else {
      DIB_REQUIRE(pl->c_dense + C <= kNmMaxWidth, "%s: the dense sources have more than 1024 rows", who);
      DIB_REQUIRE(pl->n_dense < kNmMaxDense, "%s: at most 4 dense sources", who);
      pl->dense.start[pl->n_dense] = pl->c_dense;
      pl->dense.col[pl->n_dense] = c_in;
      ++pl->n_dense;
      pl->c_dense += C;
    }
    c_in += C;
  }
  pl->dense.n = pl->n_dense;
  pl->dense.start[pl->n_dense] = pl->c_dense;
  pl->c_in = c_in;
  pl->c_dense_pad = pad_to(pl->c_dense, 8);
  pl->n_layers = n_layers;
  size_t off = 0;
  const int rc = plan_packed_layers(who, kNmMaxWidth, layers, n_layers, pl->c_dense_pad, &off, pl->layer);
  if (rc != DIB_OK) return rc;
  pl->wbt_off = off;
  off += (size_t)pl->c_bcast * pl->layer[0].Cpad;
  pl->packed_floats = off;
  return DIB_OK;
}

static int nm_pack(const NmPlan& pl, const int64_t* sources, int n_sources, const int64_t* layers, float* out,
                   cudaStream_t stream) {
  for (int l = 0; l < pl.n_layers; ++l) {
    const PackedLayer& L = pl.layer[l];
    const int64_t* d = layers + (size_t)l * DIB_MLP_LAYER;
    const float* W = (const float*)(uintptr_t)d[DIB_MLP_LAYER_W];
    DIB_REQUIRE(W != nullptr, "node_mlp_pack: a layer's W is NULL");
    const int ld = l == 0 ? pl.c_in : pl.layer[l - 1].C;
    int r = pack_tf32_a(W, ld, L.C, L.KT, l == 0 ? pl.dense : pack_cols(0, ld), out + L.w_off, stream);
    if (r != DIB_OK) return r;
    if (l == 0) {                                          // the broadcast columns, transposed, in input order
      for (int s = 0, col = 0, row = 0; s < n_sources; ++s) {
        const int64_t* d = sources + (size_t)s * DIB_MLP_SRC;
        const int C = (int)d[DIB_MLP_SRC_CHANNELS];
        if (d[DIB_MLP_SRC_BCAST]) {
          r = pack_tf32_t(W, ld, col, L.C, C, L.Cpad, out + pl.wbt_off + (size_t)row * L.Cpad, stream);
          if (r != DIB_OK) return r;
          row += C;
        }
        col += C;
      }
    }
    r = pack_bias((const float*)(uintptr_t)d[DIB_MLP_LAYER_B], L.C, L.Cpad, out + L.b_off, stream);
    if (r != DIB_OK) return r;
  }
  return DIB_OK;
}

template <int kPasses>
static int nm_launch(const NmParams& p, int B, int tiles, size_t smem, cudaStream_t stream) {
  if (smem > 48 * 1024)
    DIB_CHECK_CUDA(cudaFuncSetAttribute(nm_kernel<kPasses>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  nm_kernel<kPasses><<<dim3(tiles, B), kNmThreads, smem, stream>>>(p);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

}  // namespace dib

extern "C" {

size_t node_mlp_packed_bytes(const int64_t* sources, int n_sources, const int64_t* layers, int n_layers) {
  dib::NmPlan pl;
  if (dib::nm_plan("node_mlp", sources, n_sources, layers, n_layers, &pl) != DIB_OK) return 0;
  return pl.packed_floats * sizeof(float);
}

int node_mlp_pack_f32(const int64_t* sources, int n_sources, const int64_t* layers, int n_layers, void* packed,
                      size_t packed_bytes, dib_stream_t stream) {
  using namespace dib;
  NmPlan pl;
  const int rc = nm_plan("node_mlp", sources, n_sources, layers, n_layers, &pl);
  if (rc != DIB_OK) return rc;
  DIB_REQUIRE(packed && ((uintptr_t)packed & 15) == 0, "node_mlp_pack: packed is NULL or not 16-byte aligned");
  if (packed_bytes < pl.packed_floats * sizeof(float)) {
    set_error("node_mlp_pack: packed buffer too small");
    return DIB_ENOMEM;
  }
  return nm_pack(pl, sources, n_sources, layers, (float*)packed, (cudaStream_t)stream);
}

size_t node_mlp_workspace_bytes(const int64_t* sources, int n_sources, const int64_t* layers, int n_layers, int B) {
  dib::NmPlan pl;
  if (B < 1 || dib::nm_plan("node_mlp", sources, n_sources, layers, n_layers, &pl) != DIB_OK) return 0;
  return pl.c_bcast > 0 ? (size_t)B * pl.layer[0].Cpad * sizeof(float) : 0;
}

int node_mlp_f32(const int64_t* sources, int n_sources, const int64_t* layers, int n_layers, const void* packed,
                 size_t packed_bytes, int B, int M, float* out, void* workspace, size_t workspace_bytes,
                 dib_stream_t stream_) {
  using namespace dib;
  cudaStream_t stream = (cudaStream_t)stream_;
  NmPlan pl;
  const int rc = nm_plan("node_mlp", sources, n_sources, layers, n_layers, &pl);
  if (rc != DIB_OK) return rc;
  DIB_REQUIRE(B >= 0 && B <= 65535 && M >= 0, "node_mlp: need 0 <= B <= 65535 and M >= 0");
  if (B == 0 || M == 0) return DIB_OK;
  NmParams p = {};
  for (int s = 0; s < n_sources; ++s) {
    const int64_t* d = sources + (size_t)s * DIB_MLP_SRC;
    DIB_REQUIRE(d[DIB_MLP_SRC_DATA] != 0, "node_mlp: a source's data is NULL");
    const long long need = d[DIB_MLP_SRC_CHANNELS] * (d[DIB_MLP_SRC_BCAST] ? 1LL : (long long)M);
    DIB_REQUIRE(B == 1 || (long long)d[DIB_MLP_SRC_BSTRIDE] >= need,
                "node_mlp: a source's batch stride is smaller than channels (x M for a dense source)");
  }
  DIB_REQUIRE(out != nullptr, "node_mlp: out is NULL");
  DIB_REQUIRE(packed && ((uintptr_t)packed & 15) == 0 && packed_bytes >= pl.packed_floats * sizeof(float),
              "node_mlp: packed is NULL, misaligned or smaller than node_mlp_packed_bytes");
  const float* pk = (const float*)packed;
  const int Cpad0 = pl.layer[0].Cpad;
  float* proj = nullptr;
  if (pl.c_bcast > 0) {
    DIB_REQUIRE(workspace && ((uintptr_t)workspace & 15) == 0, "node_mlp: workspace is NULL or misaligned");
    if (workspace_bytes < (size_t)B * Cpad0 * sizeof(float)) {
      set_error("node_mlp: workspace too small");
      return DIB_ENOMEM;
    }
    proj = (float*)workspace;
    for (int s = 0, row = 0; s < n_sources; ++s) {
      const int64_t* d = sources + (size_t)s * DIB_MLP_SRC;
      if (!d[DIB_MLP_SRC_BCAST]) continue;
      const int C = (int)d[DIB_MLP_SRC_CHANNELS];
      const dim3 grid((Cpad0 + 255) / 256, (B + kNmProjB - 1) / kNmProjB);
      nm_proj_kernel<<<grid, 256, 0, stream>>>((const float*)(uintptr_t)d[DIB_MLP_SRC_DATA],
                                               (long long)d[DIB_MLP_SRC_BSTRIDE], C,
                                               pk + pl.wbt_off + (size_t)row * Cpad0, Cpad0, B, row == 0, proj);
      DIB_CHECK_CUDA(cudaGetLastError());
      row += C;
    }
  }
  p.n_src = pl.n_dense;
  for (int s = 0, k = 0; s < n_sources; ++s) {
    const int64_t* d = sources + (size_t)s * DIB_MLP_SRC;
    if (d[DIB_MLP_SRC_BCAST]) continue;
    p.src[k] = (const float*)(uintptr_t)d[DIB_MLP_SRC_DATA];
    p.bstride[k] = (long long)d[DIB_MLP_SRC_BSTRIDE];
    p.src_row0[k] = pl.dense.start[k];
    ++k;
  }
  p.src_row0[pl.n_dense] = pl.c_dense;
  p.c_in = pl.c_dense;
  p.c_in_pad = pl.c_dense_pad;
  p.M = M;
  p.n_layers = pl.n_layers;
  int rows = pl.c_dense_pad, widest = 0;
  for (int l = 0; l < pl.n_layers; ++l) {
    const PackedLayer& L = pl.layer[l];
    p.layer[l] = NmLayer{pk + L.w_off, pk + L.b_off, L.C, L.Cpad, L.KT, L.relu};
    rows = L.Cpad > rows ? L.Cpad : rows;
    widest = L.Cpad > widest ? L.Cpad : widest;
  }
  p.proj = proj;
  p.out = out;
  const size_t smem = (size_t)rows * kNmStride * sizeof(float);   // <= 1024 x 40 floats = 160 KB
  const int tiles = (M + kNmTile - 1) / kNmTile;
  return widest > kNmPassRows ? nm_launch<2>(p, B, tiles, smem, stream) : nm_launch<1>(p, B, tiles, smem, stream);
}

}  // extern "C"
