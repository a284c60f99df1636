// The packing kernels and layer plan of tf32_pack.cuh, in one translation unit so that each kernel is defined once.
#include "common.cuh"
#include "tf32_mma.cuh"
#include "tf32_pack.cuh"

namespace dib {

// one thread per packed float
__global__ void pack_tf32_a_kernel(const float* __restrict__ W, int ld, int C_out, int KT, int total, PackSegs segs,
                                   float* __restrict__ out) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  int row, col;
  a_frag_row_col(e, KT, row, col);
  float v = 0.f;
  if (row < C_out && col < segs.start[segs.n]) {
    int s = 0;
    for (int q = 1; q < segs.n; ++q)
      if (col >= segs.start[q]) s = q;
    v = tf32_rna(W[(size_t)row * ld + segs.col[s] + col - segs.start[s]]);
  }
  out[e] = v;
}

__global__ void pack_tf32_t_kernel(const float* __restrict__ W, int ld, int col0, int C_out, int K, int Cpad,
                                   float* __restrict__ out) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= K * Cpad) return;
  const int c = e / Cpad, m = e - c * Cpad;
  out[e] = m < C_out ? tf32_rna(W[(size_t)m * ld + col0 + c]) : 0.f;
}

__global__ void pack_bias_kernel(const float* __restrict__ b, int C, int Cpad, float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < Cpad) out[c] = c < C && b != nullptr ? b[c] : 0.f;
}

int plan_packed_layers(const char* who, int max_width, const int64_t* layers, int n_layers, int k0_pad, size_t* off,
                       PackedLayer* out) {
  for (int l = 0; l < n_layers; ++l) {
    const int64_t* d = layers + (size_t)l * DIB_MLP_LAYER;
    DIB_REQUIRE(d[DIB_MLP_LAYER_COUT] >= 1 && d[DIB_MLP_LAYER_COUT] <= max_width,
                "%s: a layer needs 1 <= C_out <= %d", who, max_width);
    DIB_REQUIRE(d[DIB_MLP_LAYER_RELU] == 0 || d[DIB_MLP_LAYER_RELU] == 1, "%s: relu must be 0 or 1", who);
    PackedLayer& L = out[l];
    L.C = (int)d[DIB_MLP_LAYER_COUT];
    L.Cpad = pad_to(L.C, 16);
    L.KT = (l == 0 ? k0_pad : out[l - 1].Cpad) / 8;
    L.relu = (int)d[DIB_MLP_LAYER_RELU];
    L.w_off = *off;
    *off += (size_t)L.Cpad * L.KT * 8;
    L.b_off = *off;
    *off += L.Cpad;
  }
  return DIB_OK;
}

int pack_tf32_a(const float* W, int ld, int C_out, int KT, const PackSegs& segs, float* out, cudaStream_t stream) {
  const int total = pad_to(C_out, 16) * KT * 8;
  if (total == 0) return DIB_OK;
  pack_tf32_a_kernel<<<(total + 255) / 256, 256, 0, stream>>>(W, ld, C_out, KT, total, segs, out);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

int pack_tf32_t(const float* W, int ld, int col0, int C_out, int K, int Cpad, float* out, cudaStream_t stream) {
  pack_tf32_t_kernel<<<(K * Cpad + 255) / 256, 256, 0, stream>>>(W, ld, col0, C_out, K, Cpad, out);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

int pack_bias(const float* bias, int C, int Cpad, float* out, cudaStream_t stream) {
  pack_bias_kernel<<<(Cpad + 255) / 256, 256, 0, stream>>>(bias, C, Cpad, out);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

}  // namespace dib
