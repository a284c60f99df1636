// Training path of the classifier's per-point layers (SURVEY.md 8f row N29, DESIGN.md 4.34): one 1x1 layer of a
// chain per call, in train mode, with batch-statistics BatchNorm, ReLU and dropout applied where the next layer loads
// its operand, and the backward.  The host (point_ops.point_chain) strings the calls together.
//
//   chain_gemm_kernel   CTA = 64 points of one sample, 8 warps as 4 (output rows, 64 each) x 2 (points, 32 each), the
//                       product of pointwise_mlp (mma_block_64x32 over weights packed by pointwise_mlp_pack_f32, the
//                       operand staged 64 rows at a time and rounded to TF32).  The operand is read through a
//                       transform: plain rows (up to four dense sources, in row order), act (BN scale/shift, ReLU,
//                       dropout of a previous layer's pre-norm Y) or bn_grad (dY = k1 dZ + k2 Y + k3).  Without weights
//                       the kernel is elementwise: the value is the transformed operand itself.  The epilogue adds
//                       bias and an additive [B][C][N] term, writes [B][C][N] and, when asked, per-CTA fp64 channel
//                       sums (sum v and sum v^2; or, for the backward, dZ = v masked by the recomputed dropout and
//                       ReLU of a BN layer, sum dZ and sum dZ x^).
//   chain_bn_kernel     one CTA per channel: the per-CTA partials in a fixed order (strided per thread, then a fixed
//                       tree), then mean / biased variance / scale / shift and the running statistics (forward) or
//                       dgamma, dbeta and the dY coefficients (backward).
//   chain_dw_kernel     dW = dY . X^T over the B N columns: CTA = 64 x 64 of dW over one contiguous range of 32-point
//                       chunks (a split), 4 warps of 32 x 32; both operands through the same transforms; db from the
//                       unrounded dY rows.  chain_dw_reduce_kernel sums the splits in order in fp64.
//
// Everything is deterministic: no atomics, every sum in a fixed order.  Dropout keeps (layer, b, c, n) when word 0 of
// Philox4x32-10 at counter (n, c | layer << 24, b, offset) with key (seed lo, seed hi ^ offset hi) is >= p 2^32; the
// seed and offset are read from a device int64 pair, so a captured graph that advances the offset draws new masks on
// every replay.
#include <math.h>

#include "common.cuh"
#include "tf32_mma.cuh"

namespace dib {

constexpr int kPcTile = 64;
constexpr int kPcStride = 72;
constexpr int kPcThreads = 256;
constexpr int kPcChunk = 64;
constexpr int kPcMaxWidth = 256;      // output rows per CTA: a wider layer runs as row blocks (grid z)
constexpr int kPcMaxRows = 1024;      // rows of a wide layer (point_chain_gemm_group_f32, point_chain_bn_f32)
constexpr int kPcMaxSources = 4;
constexpr int kDwTile = 64;
constexpr int kDwPts = 32;
constexpr int kDwStride = 36;   // % 32 == 4: the fragment loads of both operands are conflict-free
constexpr int kDwThreads = 128;
constexpr int kDwTargetCtas = 1056;

enum { kOpPlain = 0, kOpAct = 1, kOpBnGrad = 2, kOpMaxGrad = DIB_PC_MODE_MAX_GRAD };
enum { kEpWrite = 0, kEpStats = 1, kEpActGrad = 2 };

// BN + ReLU + dropout of one layer, recomputed from its pre-norm Y: z = scale y + shift, a = relu(z), kept a / (1 - p)
struct ChainAct {
  const float* scale; const float* shift; const float* mean; const float* invstd;
  const int64_t* drop_state; uint32_t drop_thresh; float drop_scale; int layer;
};

struct ChainOperand {
  const float* p[kPcMaxSources]; long long bstride[kPcMaxSources]; int row0[kPcMaxSources];
  int n_src, K, mode;
  ChainAct act;                                   // kOpAct
  const float* y; const float* k1; const float* k2; const float* k3;   // kOpBnGrad: rows of Y [B][K][N]
  const int* idx; int group;                      // kOpMaxGrad: p[0] and idx are [B][K][N / group]
};

struct ChainGemm {
  ChainOperand x;
  const float* W; const float* bias; const float* add;   // W packed [Cpad][pad8(K)] or NULL (elementwise, C == K)
  int C, Cpad, N, ntiles, epilogue, add_group;           // add [B][C][N / add_group]
  float* out; double* part;
  ChainAct eg; const float* ey;                           // kEpActGrad: the layer whose output's gradient v is
};

__device__ __forceinline__ bool chain_keep(const int64_t* st, int layer, int b, int c, int n, uint32_t thresh) {
  const uint64_t seed = (uint64_t)st[0], off = (uint64_t)st[1];
  uint32_t ctr[4] = {(uint32_t)n, (uint32_t)c | ((uint32_t)layer << 24), (uint32_t)b, (uint32_t)off};
  philox4x32_10(ctr, (uint32_t)seed, (uint32_t)(seed >> 32) ^ (uint32_t)(off >> 32));
  return ctr[0] >= thresh;
}

__device__ __forceinline__ float chain_act(const ChainAct& a, float y, int b, int c, int n) {
  float v = fmaf(a.scale[c], y, a.shift[c]);
  v = v > 0.f ? v : 0.f;
  if (a.drop_state != nullptr) v = chain_keep(a.drop_state, a.layer, b, c, n, a.drop_thresh) ? v * a.drop_scale : 0.f;
  return v;
}

// Row `row` of the operand at point n of sample b (row < K, n < N).
__device__ __forceinline__ float chain_load(const ChainOperand& x, int b, int row, int n, int N) {
  if (x.mode == kOpMaxGrad) {                     // the group max's gradient, at the index the forward kept
    const int j = n / x.group;
    const size_t e = (size_t)b * x.bstride[0] + (size_t)row * (N / x.group) + j;
    return x.idx[e] == n - j * x.group ? x.p[0][e] : 0.f;
  }
  int s = 0;
#pragma unroll
  for (int q = 1; q < kPcMaxSources; ++q)
    if (q < x.n_src && row >= x.row0[q]) s = q;
  const size_t e = (size_t)(row - x.row0[s]) * N + n;
  const float v = x.p[s][(size_t)b * x.bstride[s] + e];
  if (x.mode == kOpAct) return chain_act(x.act, v, b, row, n);
  if (x.mode == kOpBnGrad) {
    const float y = x.y[(size_t)b * x.K * N + e];
    return fmaf(x.k1[row], v, fmaf(x.k2[row], y, x.k3[row]));
  }
  return v;
}

__global__ void __launch_bounds__(kPcThreads) chain_gemm_kernel(const __grid_constant__ ChainGemm p) {
  extern __shared__ __align__(16) float pc_smem[];
  float* xs = pc_smem;                               // [kPcChunk][kPcStride]
  float* ta = xs + kPcChunk * kPcStride;             // [block rows][kPcStride]: the values (dZ for kEpActGrad)
  float* tb = ta + min(p.Cpad, kPcMaxWidth) * kPcStride;   // kEpActGrad: dZ x^
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3, wm = warp >> 1, n_base = (warp & 1) * 32;
  const int b = blockIdx.y, n0 = blockIdx.x * kPcTile, N = p.N;
  // row block blockIdx.z: output rows c0 .. c0 + Cb of the layer's C
  const int c0 = blockIdx.z * kPcMaxWidth, Cb = min(kPcMaxWidth, p.C - c0);
  const int MT = min(kPcMaxWidth, p.Cpad - c0) >> 4;

  if (p.W != nullptr) {
    float acc[4][4][4];
#pragma unroll
    for (int mt = 0; mt < 4; ++mt)
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[mt][nt][i] = 0.f;
    const int K = p.x.K, KT = (K + 7) >> 3;
    const float4* Wp = reinterpret_cast<const float4*>(p.W) + (size_t)(c0 >> 4) * KT * 32;
    for (int k0 = 0; k0 < K; k0 += kPcChunk) {
      const int kc8 = (min(kPcChunk, K - k0) + 7) & ~7;
      __syncthreads();
      for (int r = tid >> 6; r < kc8; r += kPcThreads / kPcTile) {
        const int n = tid & 63, row = k0 + r;
        const float v = row < K && n0 + n < N ? chain_load(p.x, b, row, n0 + n, N) : 0.f;
        xs[r * kPcStride + n] = tf32_rna(v);
      }
      __syncthreads();
      mma_block_64x32<kPcStride>(acc, xs, Wp, KT, MT, k0 >> 3, kc8 >> 3, wm, n_base, lane);
    }
#pragma unroll
    for (int mt = 0; mt < 4; ++mt) {
      if (wm * 4 + mt < MT) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int m = (wm * 4 + mt) * 16 + g + (i >> 1) * 8;
#pragma unroll
          for (int nt = 0; nt < 4; ++nt) ta[m * kPcStride + n_base + nt * 8 + 2 * t + (i & 1)] = acc[mt][nt][i];
        }
      }
    }
  }
  __syncthreads();

  // epilogue, one (channel, point) per thread step: bias, the additive term, the backward's masks; invalid -> 0
  for (int i = tid; i < Cb * kPcTile; i += kPcThreads) {
    const int c = i >> 6, n = i & 63, gn = n0 + n, gc = c0 + c;
    float v = 0.f, w = 0.f;
    if (gn < N) {
      const size_t e = ((size_t)b * p.C + gc) * N + gn;
      v = p.W != nullptr ? ta[c * kPcStride + n] : chain_load(p.x, b, gc, gn, N);
      if (p.bias != nullptr) v += p.bias[gc];
      if (p.add != nullptr)
        v += p.add_group == 1 ? p.add[e] : p.add[((size_t)b * p.C + gc) * (N / p.add_group) + gn / p.add_group];
      if (p.epilogue == kEpActGrad) {
        const float y = p.ey[e];
        const float z = fmaf(p.eg.scale[gc], y, p.eg.shift[gc]);
        bool keep = z > 0.f;
        if (keep && p.eg.drop_state != nullptr) keep = chain_keep(p.eg.drop_state, p.eg.layer, b, gc, gn, p.eg.drop_thresh);
        v = keep ? (p.eg.drop_state != nullptr ? v * p.eg.drop_scale : v) : 0.f;
        w = v * ((y - p.eg.mean[gc]) * p.eg.invstd[gc]);
      }
      p.out[e] = v;
    }
    ta[c * kPcStride + n] = v;
    if (p.epilogue == kEpActGrad) tb[c * kPcStride + n] = w;
  }
  if (p.epilogue == kEpWrite) return;
  __syncthreads();
  // fixed order per channel: points 0..63 of the tile, in fp64
  double* part = p.part + (size_t)(b * p.ntiles + blockIdx.x) * 2 * p.C;
  for (int c = tid; c < Cb; c += kPcThreads) {
    double s = 0.0, q = 0.0;
    for (int n = 0; n < kPcTile; ++n) {
      const double v = ta[c * kPcStride + n];
      s += v;
      q += p.epilogue == kEpStats ? v * v : (double)tb[c * kPcStride + n];
    }
    part[c0 + c] = s;
    part[p.C + c0 + c] = q;
  }
}

// One thread per (b, c, group of G columns): the operand's values over the group in column order (written to act when
// act is not NULL) and their max by torch.max's rule: the first maximal value, a NaN (the first) over any number.
__global__ void chain_group_max_kernel(const __grid_constant__ ChainOperand x, int B, int N, int G, float* act,
                                       float* __restrict__ mx, int* __restrict__ idx) {
  const int NG = N / G, C = x.K;
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)B * C * NG) return;
  const int j = (int)(e % NG), c = (int)((e / NG) % C), b = (int)(e / ((long long)NG * C));
  float best = 0.f;
  int bi = 0;
  for (int k = 0; k < G; ++k) {
    const int n = j * G + k;
    const float v = chain_load(x, b, c, n, N);
    if (act != nullptr) act[((size_t)b * C + c) * N + n] = v;
    if (k == 0 || v > best || (v != v && best == best)) { best = v; bi = k; }
  }
  mx[e] = best;
  idx[e] = bi;
}

// out [B][C][N / G] = the operand's sum over each group of G columns, in column order in fp64, rounded once.
__global__ void chain_group_sum_kernel(const __grid_constant__ ChainOperand x, int B, int N, int G,
                                       float* __restrict__ out) {
  const int NG = N / G, C = x.K;
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)B * C * NG) return;
  const int j = (int)(e % NG), c = (int)((e / NG) % C), b = (int)(e / ((long long)NG * C));
  double s = 0.0;
  for (int k = 0; k < G; ++k) s += chain_load(x, b, c, j * G + k, N);
  out[e] = (float)s;
}

// Forward (grad == 0): stats [4][C] = mean, invstd, scale, shift; running statistics; num_batches_tracked.
// Backward (grad == 1): stats as the forward wrote them; dgamma, dbeta; coef [3][C] = k1, k2, k3 of dY = k1 dZ + k2 Y
// + k3.  M = B N.
__global__ void __launch_bounds__(256) chain_bn_kernel(const double* __restrict__ part, int G, int C, double M,
                                                       int grad, const float* __restrict__ gamma,
                                                       const float* __restrict__ beta, float eps, float momentum,
                                                       float* stats, float* running_mean, float* running_var,
                                                       int64_t* nbt, float* dgamma, float* dbeta, float* coef) {
  __shared__ double rs[256], rq[256];
  const int c = blockIdx.x, tid = threadIdx.x;
  double s = 0.0, q = 0.0;
  for (int i = tid; i < G; i += 256) {
    s += part[(size_t)i * 2 * C + c];
    q += part[(size_t)i * 2 * C + C + c];
  }
  rs[tid] = s; rq[tid] = q;
  __syncthreads();
  for (int h = 128; h > 0; h >>= 1) {
    if (tid < h) { rs[tid] += rs[tid + h]; rq[tid] += rq[tid + h]; }
    __syncthreads();
  }
  if (tid != 0) return;
  s = rs[0]; q = rq[0];
  const double gm = gamma[c];
  if (!grad) {
    const double mean = s / M;
    double var = q / M - mean * mean;
    var = var > 0.0 ? var : 0.0;
    const double invstd = 1.0 / sqrt(var + (double)eps);
    const double scale = gm * invstd;
    stats[c] = (float)mean;
    stats[C + c] = (float)invstd;
    stats[2 * C + c] = (float)scale;
    stats[3 * C + c] = (float)((double)beta[c] - mean * scale);
    const double unbiased = M > 1.0 ? var * M / (M - 1.0) : var;
    running_mean[c] = (float)((1.0 - momentum) * running_mean[c] + momentum * mean);
    running_var[c] = (float)((1.0 - momentum) * running_var[c] + momentum * unbiased);
    if (c == 0 && nbt != nullptr) nbt[0] += 1;
  } else {
    const double mean = stats[c], invstd = stats[C + c];
    dbeta[c] = (float)s;
    dgamma[c] = (float)q;
    const double k1 = gm * invstd, k2 = -k1 * invstd * q / M;
    coef[c] = (float)k1;
    coef[C + c] = (float)k2;
    coef[2 * C + c] = (float)(-k1 * s / M - k2 * mean);
  }
}

__device__ __forceinline__ float4 dw_frag(const float* s, int r, int k, int g, int t) {
  return make_float4(tf32_rna(s[(r + g) * kDwStride + k + t]), tf32_rna(s[(r + g + 8) * kDwStride + k + t]),
                     tf32_rna(s[(r + g) * kDwStride + k + t + 4]), tf32_rna(s[(r + g + 8) * kDwStride + k + t + 4]));
}

// part [splits][C][K] f32, dbp [splits][C] f64 (written by the CTAs of column tile 0)
__global__ void __launch_bounds__(kDwThreads) chain_dw_kernel(const __grid_constant__ ChainOperand dy,
                                                              const __grid_constant__ ChainOperand x, int B, int N,
                                                              int splits, float* __restrict__ part,
                                                              double* __restrict__ dbp) {
  __shared__ __align__(16) float As[kDwTile * kDwStride], Xs[kDwTile * kDwStride];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
  const int wm = warp >> 1, wn = warp & 1;
  const int C = dy.K, K = x.K;
  const int m0 = blockIdx.x * kDwTile, k0 = blockIdx.y * kDwTile, s = blockIdx.z;
  const int per_b = (N + kDwPts - 1) / kDwPts;
  const long long Q = (long long)B * per_b, q0 = Q * s / splits, q1 = Q * (s + 1) / splits;
  float acc[2][4][4];
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[a][nt][i] = 0.f;
  double db = 0.0;
  const bool do_db = blockIdx.y == 0 && tid < kDwTile;
  for (long long q = q0; q < q1; ++q) {
    const int b = (int)(q / per_b), n0 = (int)(q % per_b) * kDwPts, n = n0 + lane;
    __syncthreads();
    for (int r = warp; r < kDwTile; r += kDwThreads / 32) {
      const bool ok = n < N;
      As[r * kDwStride + lane] = ok && m0 + r < C ? chain_load(dy, b, m0 + r, n, N) : 0.f;
      Xs[r * kDwStride + lane] = ok && k0 + r < K ? chain_load(x, b, k0 + r, n, N) : 0.f;
    }
    __syncthreads();
    if (do_db)
      for (int j = 0; j < kDwPts; ++j) db += As[tid * kDwStride + j];
#pragma unroll
    for (int kk = 0; kk < kDwPts; kk += 8) {
      float4 a[2];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) a[mt] = dw_frag(As, wm * 32 + mt * 16, kk, g, t);
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        const int col = wn * 32 + nt * 8 + g;
        const uint32_t b0 = __float_as_uint(tf32_rna(Xs[col * kDwStride + kk + t]));
        const uint32_t b1 = __float_as_uint(tf32_rna(Xs[col * kDwStride + kk + t + 4]));
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) mma_tf32(acc[mt][nt], a[mt], b0, b1);
      }
    }
  }
  float* out = part + (size_t)s * C * K;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int m = m0 + wm * 32 + mt * 16 + g + (i >> 1) * 8, k = k0 + wn * 32 + nt * 8 + 2 * t + (i & 1);
        if (m < C && k < K) out[(size_t)m * K + k] = acc[mt][nt][i];
      }
  if (do_db && m0 + tid < C) dbp[(size_t)s * C + m0 + tid] = db;
}

__global__ void chain_dw_reduce_kernel(const float* __restrict__ part, const double* __restrict__ dbp, int splits,
                                       int C, int K, float* __restrict__ dW, float* __restrict__ db) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e < C * K) {
    double v = 0.0;
    for (int s = 0; s < splits; ++s) v += part[(size_t)s * C * K + e];
    dW[e] = (float)v;
  }
  if (e < C && db != nullptr) {
    double v = 0.0;
    for (int s = 0; s < splits; ++s) v += dbp[(size_t)s * C + e];
    db[e] = (float)v;
  }
}

__global__ void chain_mask_kernel(const int64_t* st, int layer, int B, int C, int N, uint32_t thresh,
                                  uint8_t* __restrict__ out) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)B * C * N) return;
  const int n = (int)(e % N), c = (int)((e / N) % C), b = (int)(e / ((long long)N * C));
  out[e] = chain_keep(st, layer, b, c, n, thresh) ? 1 : 0;
}

static uint32_t drop_threshold(double p) {
  const double t = p * 4294967296.0;
  return t >= 4294967295.0 ? 4294967295u : (uint32_t)llrint(t);
}

static int read_act(const int64_t* d, ChainAct* a) {
  a->scale = (const float*)(uintptr_t)d[DIB_PC_ACT_STATS];
  DIB_REQUIRE(a->scale != nullptr, "point_chain: a BN layer's statistics are NULL");
  const int C = (int)d[DIB_PC_ACT_C];
  const float* st = a->scale;
  a->mean = st; a->invstd = st + C; a->scale = st + 2 * C; a->shift = st + 3 * C;
  a->drop_state = (const int64_t*)(uintptr_t)d[DIB_PC_ACT_DROP_STATE];
  const double pd = (double)d[DIB_PC_ACT_DROP_PPM] / 1e6;
  DIB_REQUIRE(pd >= 0.0 && pd < 1.0, "point_chain: need 0 <= dropout p < 1");
  if (pd == 0.0) a->drop_state = nullptr;
  a->drop_thresh = drop_threshold(pd);
  a->drop_scale = (float)(1.0 / (1.0 - pd));
  a->layer = (int)d[DIB_PC_ACT_LAYER];
  return DIB_OK;
}

static int read_operand(const int64_t* d, int n_src, int N, ChainOperand* x) {
  DIB_REQUIRE(d != nullptr && n_src >= 1 && n_src <= kPcMaxSources, "point_chain: need 1 to 4 operand sources");
  *x = ChainOperand{};
  x->n_src = n_src;
  const int64_t* h = d + (size_t)n_src * DIB_PC_SRC;                    // the transform row after the sources
  x->mode = (int)h[DIB_PC_OP_MODE];
  DIB_REQUIRE(x->mode >= kOpPlain && x->mode <= kOpMaxGrad, "point_chain: unknown operand transform");
  int cols = N;                                                         // a source row's columns
  if (x->mode == kOpMaxGrad) {
    x->group = (int)h[DIB_PC_OP_LAYER];
    x->idx = (const int*)(uintptr_t)h[DIB_PC_OP_Y];
    DIB_REQUIRE(x->group >= 1 && N % x->group == 0 && x->idx != nullptr,
                "point_chain: max_grad needs a group that divides N and the max's indices");
    cols = N / x->group;
  }
  for (int s = 0; s < n_src; ++s) {
    const int64_t* r = d + (size_t)s * DIB_PC_SRC;
    x->p[s] = (const float*)(uintptr_t)r[DIB_PC_SRC_DATA];
    x->bstride[s] = r[DIB_PC_SRC_BSTRIDE];
    x->row0[s] = x->K;
    DIB_REQUIRE(x->p[s] != nullptr && r[DIB_PC_SRC_CHANNELS] >= 1 &&
                r[DIB_PC_SRC_BSTRIDE] >= r[DIB_PC_SRC_CHANNELS] * cols,
                "point_chain: a source is NULL, has no channel or a batch stride below channels x N");
    x->K += (int)r[DIB_PC_SRC_CHANNELS];
  }
  DIB_REQUIRE(x->mode == kOpPlain || n_src == 1, "point_chain: a transformed operand has one source");
  if (x->mode == kOpAct) {
    const int64_t a[DIB_PC_ACT] = {h[DIB_PC_OP_STATS], x->K, h[DIB_PC_OP_DROP_STATE], h[DIB_PC_OP_DROP_PPM],
                                   h[DIB_PC_OP_LAYER]};
    const int r = read_act(a, &x->act);
    if (r != DIB_OK) return r;
  } else if (x->mode == kOpBnGrad) {
    x->y = (const float*)(uintptr_t)h[DIB_PC_OP_Y];
    const float* k = (const float*)(uintptr_t)h[DIB_PC_OP_STATS];
    DIB_REQUIRE(x->y != nullptr && k != nullptr, "point_chain: bn_grad needs Y and its coefficients");
    x->k1 = k; x->k2 = k + x->K; x->k3 = k + 2 * x->K;
  }
  return DIB_OK;
}

}  // namespace dib

extern "C" {

size_t point_chain_partial_bytes(int B, int N, int C) {
  if (B <= 0 || N <= 0 || C <= 0) return 0;
  return (size_t)B * ((N + dib::kPcTile - 1) / dib::kPcTile) * 2 * C * sizeof(double);
}

static int chain_gemm(const int64_t* operand, int n_src, const void* packed, const float* bias, const float* add,
                      int add_group, int C, int B, int N, int epilogue, const int64_t* act, const float* act_y,
                      float* out, void* partials, size_t partial_bytes, cudaStream_t stream) {
  using namespace dib;
  DIB_REQUIRE(B >= 1 && B <= 65535 && N >= 1, "point_chain: need 1 <= B <= 65535 and N >= 1");
  DIB_REQUIRE(epilogue >= kEpWrite && epilogue <= kEpActGrad, "point_chain: unknown epilogue");
  DIB_REQUIRE(out != nullptr, "point_chain: out is NULL");
  ChainGemm p = {};
  int rc = read_operand(operand, n_src, N, &p.x);
  if (rc != DIB_OK) return rc;
  DIB_REQUIRE(p.x.K <= 1024, "point_chain: the operand has more than 1024 rows");
  DIB_REQUIRE(packed != nullptr || p.x.K == C, "point_chain: an elementwise call needs C == the operand's rows");
  DIB_REQUIRE(packed == nullptr || ((uintptr_t)packed & 15) == 0, "point_chain: packed is not 16-byte aligned");
  DIB_REQUIRE(add_group >= 1 && N % add_group == 0, "point_chain: add_group must divide N");
  p.W = (const float*)packed; p.bias = bias; p.add = add; p.add_group = add_group;
  p.C = C; p.Cpad = (C + 15) / 16 * 16; p.N = N; p.ntiles = (N + kPcTile - 1) / kPcTile; p.epilogue = epilogue;
  p.out = out;
  if (epilogue != kEpWrite) {
    DIB_REQUIRE(partials != nullptr && partial_bytes >= point_chain_partial_bytes(B, N, C),
                "point_chain: the partials buffer is NULL or smaller than point_chain_partial_bytes");
    p.part = (double*)partials;
  }
  if (epilogue == kEpActGrad) {
    DIB_REQUIRE(act != nullptr && act_y != nullptr, "point_chain: act_grad needs the layer's act row and Y");
    const int64_t a[DIB_PC_ACT] = {act[DIB_PC_ACT_STATS], C, act[DIB_PC_ACT_DROP_STATE], act[DIB_PC_ACT_DROP_PPM],
                                   act[DIB_PC_ACT_LAYER]};
    rc = read_act(a, &p.eg);
    if (rc != DIB_OK) return rc;
    p.ey = act_y;
  }
  const size_t rows = (size_t)(p.Cpad < kPcMaxWidth ? p.Cpad : kPcMaxWidth);
  const size_t smem = ((size_t)kPcChunk * kPcStride + (size_t)(epilogue == kEpActGrad ? 2 : 1) * rows * kPcStride) *
                      sizeof(float);
  DIB_CHECK_CUDA(cudaFuncSetAttribute(chain_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  chain_gemm_kernel<<<dim3(p.ntiles, B, (C + kPcMaxWidth - 1) / kPcMaxWidth), kPcThreads, smem, stream>>>(p);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

int point_chain_gemm_f32(const int64_t* operand, int n_src, const void* packed, const float* bias, const float* add,
                         int C, int B, int N, int epilogue, const int64_t* act, const float* act_y, float* out,
                         void* partials, size_t partial_bytes, dib_stream_t stream) {
  DIB_REQUIRE(C >= 1 && C <= dib::kPcMaxWidth, "point_chain: need 1 <= C_out <= 256");
  return chain_gemm(operand, n_src, packed, bias, add, 1, C, B, N, epilogue, act, act_y, out, partials, partial_bytes,
                    (cudaStream_t)stream);
}

int point_chain_gemm_group_f32(const int64_t* operand, int n_src, const void* packed, const float* bias,
                               const float* add, int add_group, int C, int B, int N, int epilogue, const int64_t* act,
                               const float* act_y, float* out, void* partials, size_t partial_bytes,
                               dib_stream_t stream) {
  DIB_REQUIRE(C >= 1 && C <= dib::kPcMaxRows, "point_chain: need 1 <= C_out <= 1024");
  return chain_gemm(operand, n_src, packed, bias, add, add_group, C, B, N, epilogue, act, act_y, out, partials,
                    partial_bytes, (cudaStream_t)stream);
}

int point_chain_group_max_f32(const int64_t* operand, int B, int N, int group, float* act, float* max, int* idx,
                              dib_stream_t stream) {
  using namespace dib;
  DIB_REQUIRE(B >= 1 && B <= 65535 && N >= 1 && group >= 1 && N % group == 0 && max != nullptr && idx != nullptr,
              "point_chain_group_max: need 1 <= B <= 65535, a group that divides N >= 1, and max and idx");
  ChainOperand x;
  const int rc = read_operand(operand, 1, N, &x);
  if (rc != DIB_OK) return rc;
  DIB_REQUIRE(x.mode != kOpMaxGrad, "point_chain_group_max: the operand is a max's gradient");
  const long long total = (long long)B * x.K * (N / group);
  chain_group_max_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, B, N, group, act, max,
                                                                                           idx);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

int point_chain_group_sum_f32(const int64_t* operand, int B, int N, int group, float* out, dib_stream_t stream) {
  using namespace dib;
  DIB_REQUIRE(B >= 1 && B <= 65535 && N >= 1 && group >= 1 && N % group == 0 && out != nullptr,
              "point_chain_group_sum: need 1 <= B <= 65535, a group that divides N >= 1, and out");
  ChainOperand x;
  const int rc = read_operand(operand, 1, N, &x);
  if (rc != DIB_OK) return rc;
  const long long total = (long long)B * x.K * (N / group);
  chain_group_sum_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, B, N, group, out);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

int point_chain_bn_f32(const void* partials, int B, int N, int C, int grad, const float* gamma, const float* beta,
                       float eps, float momentum, float* stats, float* running_mean, float* running_var,
                       int64_t* num_batches_tracked, float* dgamma, float* dbeta, float* coef, dib_stream_t stream_) {
  using namespace dib;
  DIB_REQUIRE(B >= 1 && N >= 1 && C >= 1 && C <= kPcMaxRows, "point_chain_bn: need B, N >= 1 and 1 <= C <= 1024");
  DIB_REQUIRE(partials && gamma && beta && stats, "point_chain_bn: a pointer is NULL");
  if (grad) DIB_REQUIRE(dgamma && dbeta && coef, "point_chain_bn: a gradient output is NULL");
  else DIB_REQUIRE(running_mean && running_var, "point_chain_bn: the running statistics are NULL");
  const int G = B * ((N + kPcTile - 1) / kPcTile);
  chain_bn_kernel<<<C, 256, 0, (cudaStream_t)stream_>>>((const double*)partials, G, C, (double)B * N, grad, gamma,
                                                          beta, eps, momentum, stats, running_mean, running_var,
                                                          num_batches_tracked, dgamma, dbeta, coef);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

static int dw_splits(int B, int N, int C, int K) {
  const long long tiles = (long long)((C + 63) / 64) * ((K + 63) / 64);
  const long long Q = (long long)B * ((N + 31) / 32);
  // about 1056 CTAs in all, eight per SM of a 132-SM H100.  A constant rather than the device's SM count: the split,
  // and so the summation order of dW, is then the same on every device, and the results are bit-identical across them.
  long long s = (dib::kDwTargetCtas + tiles - 1) / tiles;
  if (s > 256) s = 256;
  if (s > Q) s = Q;
  return (int)(s < 1 ? 1 : s);
}

size_t point_chain_dw_workspace_bytes(int B, int N, int C, int K) {
  if (B <= 0 || N <= 0 || C <= 0 || K <= 0) return 0;
  const size_t s = dw_splits(B, N, C, K);
  return s * C * K * sizeof(float) + s * C * sizeof(double) + 16;
}

int point_chain_dw_f32(const int64_t* dy, const int64_t* x, int n_src, int B, int N, float* dW, float* db,
                       void* workspace, size_t workspace_bytes, dib_stream_t stream_) {
  using namespace dib;
  cudaStream_t stream = (cudaStream_t)stream_;
  DIB_REQUIRE(B >= 1 && N >= 1 && dW != nullptr, "point_chain_dw: need B, N >= 1 and dW");
  ChainOperand a, o;
  int rc = read_operand(dy, 1, N, &a);
  if (rc != DIB_OK) return rc;
  rc = read_operand(x, n_src, N, &o);
  if (rc != DIB_OK) return rc;
  DIB_REQUIRE(a.K <= 1024 && o.K <= 1024, "point_chain_dw: more than 1024 rows");
  const int C = a.K, K = o.K, S = dw_splits(B, N, C, K);
  DIB_REQUIRE(workspace && ((uintptr_t)workspace & 15) == 0 && workspace_bytes >= point_chain_dw_workspace_bytes(B, N, C, K),
              "point_chain_dw: the workspace is NULL, misaligned or too small");
  double* dbp = (double*)workspace;
  float* part = (float*)(dbp + (size_t)S * C);
  chain_dw_kernel<<<dim3((C + 63) / 64, (K + 63) / 64, S), kDwThreads, 0, stream>>>(a, o, B, N, S, part, dbp);
  DIB_CHECK_CUDA(cudaGetLastError());
  const int total = C * K > C ? C * K : C;
  chain_dw_reduce_kernel<<<(total + 255) / 256, 256, 0, stream>>>(part, dbp, S, C, K, dW, db);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

int point_chain_dropout_mask(const int64_t* drop_state, int layer, float p, int B, int C, int N, uint8_t* out,
                             dib_stream_t stream_) {
  using namespace dib;
  DIB_REQUIRE(drop_state && out && B >= 1 && C >= 1 && N >= 1, "point_chain_dropout_mask: bad argument");
  DIB_REQUIRE(p >= 0.f && p < 1.f, "point_chain_dropout_mask: need 0 <= p < 1");
  const long long total = (long long)B * C * N;
  chain_mask_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream_>>>(drop_state, layer, B, C, N,
                                                                                       drop_threshold((double)p), out);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

}  // extern "C"
