// TF32 tensor-core helpers shared by the fused per-point chains (pointwise_mlp.cu, knn_fusion.cu, node_mlp.cu,
// point_chain.cu; DESIGN.md 4.21): the operand rounding rule, the m16n8k8 instruction, the A-fragment order weights
// are packed in (by tf32_pack.cu), the warp's 64-row x 32-column product over activations kept in shared memory, and
// the value a layer stores between layers.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace dib {

// Round-to-nearest, ties away from zero, onto 10 mantissa bits (cvt.rna.tf32.f32's rule for every finite value that
// stays finite), written with integer operations so that overflow (-> inf) and NaN (unchanged) are defined too.
__host__ __device__ __forceinline__ uint32_t tf32_rna_bits(uint32_t u) {
  if ((u & 0x7fffffffu) > 0x7f800000u) return u;                 // NaN
  return (u + 0x1000u) & 0xffffe000u;
}
__device__ __forceinline__ float tf32_rna(float x) { return __uint_as_float(tf32_rna_bits(__float_as_uint(x))); }

__device__ __forceinline__ void mma_tf32(float (&d)[4], const float4& a, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(__float_as_uint(a.x)), "r"(__float_as_uint(a.y)), "r"(__float_as_uint(a.z)), "r"(__float_as_uint(a.w)),
        "r"(b0), "r"(b1));
}

// Packed float e of a matrix in the m16n8k8 A-fragment order [m tile][k tile][lane][4] with KT k tiles: its (row,
// col) in the unpacked matrix.  A lane's fragment is then one 16-byte load.
__device__ __forceinline__ void a_frag_row_col(int e, int KT, int& row, int& col) {
  const int i = e & 3, lane = (e >> 2) & 31, tile = e >> 7, kt = tile % KT, mt = tile / KT;
  row = mt * 16 + (lane >> 2) + (i & 1) * 8;
  col = kt * 8 + (lane & 3) + (i >> 1) * 4;
}

// acc += W[warp's 64 rows][k tiles kt0 .. kt0 + nkt) . xin[nkt * 8][Stride] over the warp's 32 columns from n_base.
// Stride % 32 == 8 makes the B-fragment loads conflict-free.  The next step's A fragments are loaded while the current
// step's products are issued.
template <int Stride>
__device__ __forceinline__ void mma_block_64x32(float (&acc)[4][4][4], const float* __restrict__ xin,
                                                const float4* __restrict__ Wp, int KT, int MT, int kt0, int nkt,
                                                int wm, int n_base, int lane) {
  static_assert(Stride % 32 == 8, "the B-fragment loads need Stride % 32 == 8");
  const int g = lane >> 2, t = lane & 3;
  float4 a[4], an[4];
#pragma unroll
  for (int mt = 0; mt < 4; ++mt) {
    const int m = wm * 4 + mt;
    a[mt] = m < MT && nkt > 0 ? __ldg(Wp + ((size_t)m * KT + kt0) * 32 + lane) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  for (int kt = 0; kt < nkt; ++kt) {
#pragma unroll
    for (int mt = 0; mt < 4; ++mt) {
      const int m = wm * 4 + mt;
      an[mt] = m < MT && kt + 1 < nkt ? __ldg(Wp + ((size_t)m * KT + kt0 + kt + 1) * 32 + lane)
                                      : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    const float* x0 = xin + (kt * 8 + t) * Stride + n_base + g;
    uint32_t b0[4], b1[4];
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      b0[nt] = __float_as_uint(x0[nt * 8]);
      b1[nt] = __float_as_uint(x0[4 * Stride + nt * 8]);
    }
#pragma unroll
    for (int mt = 0; mt < 4; ++mt) {
      if (wm * 4 + mt < MT) {
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) mma_tf32(acc[mt][nt], a[mt], b0[nt], b1[nt]);
      }
    }
#pragma unroll
    for (int mt = 0; mt < 4; ++mt) a[mt] = an[mt];
  }
}

// The value a fused layer stores for one output row and column: the product v, plus add() when has_add (read only
// then), plus the bias; ReLU keeps NaN (NaN < 0 is false), as torch.relu; a padding row (m >= C) is zero, since it
// feeds zero weights and must stay finite; rounded to TF32 unless it is the chain's last layer.
template <class Add>
__device__ __forceinline__ float layer_value(float v, bool has_add, Add add, float bias, bool relu, bool padding,
                                             bool last) {
  if (has_add) v += add();
  v += bias;
  if (relu) v = v < 0.f ? 0.f : v;
  if (padding) v = 0.f;
  return last ? v : tf32_rna(v);
}

}  // namespace dib
