// Weight packing of the fused TF32 chains (pointwise_mlp.cu, knn_fusion.cu, node_mlp.cu; DESIGN.md 4.21): every
// weight rounded to TF32 once (tf32_rna), in the m16n8k8 A-fragment order of tf32_mma.cuh with rows padded to 16 and
// k tiles to 8 columns, zero in the padding; biases padded to the layer's padded width.  tf32_pack.cu holds the kernels.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace dib {

constexpr int kPackMaxSegs = 4;

inline int pad_to(int x, int m) { return (x + m - 1) / m * m; }

// Column segments of W: packed column c of segment s (start[s] <= c < start[s + 1]) is column col[s] + c - start[s] of
// W.  Packed columns from start[n] on are zero padding.
struct PackSegs { int n; int start[kPackMaxSegs + 1]; int col[kPackMaxSegs]; };

// One segment: packed columns [0, K) are W's columns [col0, col0 + K).
inline PackSegs pack_cols(int col0, int K) {
  PackSegs s = {};
  s.n = 1;
  s.start[1] = K;
  s.col[0] = col0;
  return s;
}

// One layer of a packed chain: C_out, padded to Cpad = 16 rows; KT k tiles of input; ReLU; where its weights and its
// bias start in the packed buffer (floats).
struct PackedLayer { int C, Cpad, KT, relu; size_t w_off, b_off; };

// Plans layers [0, n_layers) of a DIB_MLP_LAYER table: every C_out in [1, max_width] and relu 0 or 1 (who names the op
// in the errors); layer 0 takes k0_pad input rows (a multiple of 8), each later layer its predecessor's Cpad.  Each
// layer's weights and then its bias go at the running offset *off, which ends past the last bias.
int plan_packed_layers(const char* who, int max_width, const int64_t* layers, int n_layers, int k0_pad, size_t* off,
                       PackedLayer* out);

// W [C_out][ld] -> out [pad16(C_out) x KT x 8] in the A-fragment order, the columns mapped by segs.  One launch, none
// when KT is 0.
int pack_tf32_a(const float* W, int ld, int C_out, int KT, const PackSegs& segs, float* out, cudaStream_t stream);

// W [C_out][ld] columns [col0, col0 + K) -> transposed out [K][Cpad], rounded to TF32, zero padding.  One launch.
int pack_tf32_t(const float* W, int ld, int col0, int C_out, int K, int Cpad, float* out, cudaStream_t stream);

// bias [C] (or NULL: zeros) -> out [Cpad], zero padding.  One launch.
int pack_bias(const float* bias, int C, int Cpad, float* out, cudaStream_t stream);

}  // namespace dib
