// Training targets, losses, accuracies and predictions of the classifier (SURVEY.md 8f row N11):
// MMClassifer.foraward_pass (models/multimodal_classifier.py:135-191, the coarse-only variant :482-508) without a host
// synchronisation.  DESIGN.md 4.15 states the contract.
//
//   cls_forward_kernel   one thread per point, grid (ceil(N / 256), B): the label rule of project.cuh, kornia's focal
//                        term over the two coarse logits, an online max / sum-exp / argmax over the L fine logits (the
//                        loads at stride N are coalesced across the warp), the per-point log-sum-exp for the backward
//                        (as the row max and the log of the shifted sum), and per-CTA partials: fp64 sums of the
//                        focal and cross-entropy terms, integer counts of inside points and correct predictions.
//   cls_reduce_kernel    one CTA: each sample's partials summed in CTA order, then a fixed tree over the samples;
//                        writes the per-sample counts, the three losses, the accuracies and the inside total.
//   cls_backward_kernel  one thread per point: both gradients in one pass, the fine softmax recomputed from the logits
//                        and the saved log-sum-exp, the scale factors read from device memory.
// No atomics: every sum has an order fixed by the shape.  Per-point arithmetic is fp32, sums over points fp64.  The
// file is compiled with --fmad=false (build.py NOFMA_SOURCES) so that the coarse label is inside_mask_kernel's
// decision bit for bit.
#include <math.h>

#include "common.cuh"
#include "project.cuh"

namespace dib {

constexpr int kClsThreads = 256;
constexpr int kClsWarps = kClsThreads / 32;
constexpr int kClsChunk = 8;                 // fine logits loaded per thread before they are consumed

struct Focal2 {
  float loss;    // sum_c (onehot_c + eps) f_c
  float dz0;     // d loss / d z_0 (d loss / d z_1 = -dz0)
};

// kornia's focal loss on two logits as the reference calls it: p = softmax(z) + eps,
// f_c = -alpha (1 - p_c)^gamma log p_c, loss = sum_c (onehot_c + eps) f_c.  With two classes 1 - p_c = s_o - eps
// (s_o the other class's softmax) and log p_c = log1p(eps - s_o), which keep the digits that 1 - p_c and log p_c
// lose when p_c is near 1.
__device__ __forceinline__ Focal2 focal2(float z0, float z1, int label, float alpha, int gamma, float eps) {
  const float m = z0 > z1 ? z0 : z1;
  const float e0 = expf(z0 - m), e1 = expf(z1 - m);
  const float S = e0 + e1;
  const float s[2] = {e0 / S, e1 / S};
  float loss = 0.f, a[2];
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    const float sc = s[c], so = s[1 - c];
    const float p = sc + eps;
    const float q = so - eps;                               // 1 - p
    const float lg = sc > 0.5f ? log1pf(eps - so) : logf(p);
    float qg1 = 1.f;                                        // q^(gamma - 1) for gamma >= 1
    for (int k = 1; k < gamma; ++k) qg1 *= q;
    const float qg = gamma == 0 ? 1.f : qg1 * q;            // q^gamma
    const float w = (c == label ? 1.f : 0.f) + eps;
    loss += w * (-alpha * qg * lg);
    // d f_c / d p_c = alpha (gamma q^(gamma-1) log p - q^gamma / p)
    const float df = gamma == 0 ? -alpha / p : alpha * ((float)gamma * qg1 * lg - qg / p);
    a[c] = w * df;
  }
  // d / d z_0 of sum_c a_c s_c: s_0 (a_0 - (a_0 s_0 + a_1 s_1)) = s_0 s_1 (a_0 - a_1)
  return {loss, s[0] * s[1] * (a[0] - a[1])};
}

struct FineState {
  float m = -INFINITY, sum = 0.f, best = 0.f, zl = 0.f;
  int arg = -1;
  // online log-sum-exp, torch.max's argmax (first maximal index, NaN maximal) and the label's logit
  __device__ __forceinline__ void step(float z, int l, int label) {
    if (arg < 0 || (best == best && (z != z || z > best))) { best = z; arg = l; }
    if (z > m) {
      sum = sum * expf(m - z) + 1.f;
      m = z;
    } else {
      sum += expf(z == -INFINITY ? -INFINITY : z - m);    // -inf adds nothing, also when m = -inf
    }
    if (l == label) zl = z;
  }
};

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return v;
}

// Partials [2][B][nblk] f64 (focal sum, cross-entropy sum over inside points) and [3][B][nblk] int32 (inside points,
// correct coarse predictions, correct fine predictions of inside points).
__global__ void __launch_bounds__(kClsThreads)
    cls_forward_kernel(const float* __restrict__ coarse, long long cbs, const float* __restrict__ fine, long long fbs,
                       int L, const float* __restrict__ pc, const double* __restrict__ P12,
                       const double* __restrict__ K9, int B, int N, double H, double W, double s, int Wf, float alpha,
                       int gamma, float eps, int8_t* __restrict__ coarse_lab, int32_t* __restrict__ fine_lab,
                       int8_t* __restrict__ coarse_pred, int32_t* __restrict__ fine_pred, float* __restrict__ lse,
                       double* __restrict__ part_d, int32_t* __restrict__ part_i) {
  __shared__ double sh_d[2][kClsWarps];
  __shared__ int sh_i[3][kClsWarps];
  const int b = blockIdx.y, n = blockIdx.x * kClsThreads + threadIdx.x;
  double focal = 0.0, ce = 0.0;
  int inside = 0, c_ok = 0, f_ok = 0;
  if (n < N) {
    const float* p = pc + (size_t)b * 3 * N + n;
    double u, v;
    const bool in = project_inside(P12 + (size_t)b * 12, K9 + (size_t)b * 9, p[0], p[N], p[2 * (size_t)N], H, W, &u, &v);
    const size_t bn = (size_t)b * N + n;
    const float* zc = coarse + (size_t)b * cbs + n;
    const float z0 = zc[0], z1 = zc[N];
    const Focal2 f = focal2(z0, z1, in ? 1 : 0, alpha, gamma, eps);
    const int cp = (z0 == z0 && (z1 != z1 || z1 > z0)) ? 1 : 0;   // torch.max over two values
    coarse_lab[bn] = in ? 1 : 0;
    coarse_pred[bn] = (int8_t)cp;
    focal = (double)f.loss;
    inside = in ? 1 : 0;
    c_ok = cp == inside ? 1 : 0;
    if (fine) {
      const int label = in ? (int)floor(u / s) + (int)floor(v / s) * Wf : -1;
      const float* row = fine + (size_t)b * fbs + n;
      FineState st;
      int l = 0;
      for (; l + kClsChunk <= L; l += kClsChunk) {
        float z[kClsChunk];
#pragma unroll
        for (int j = 0; j < kClsChunk; ++j) z[j] = row[(size_t)(l + j) * N];
#pragma unroll
        for (int j = 0; j < kClsChunk; ++j) st.step(z[j], l + j, label);
      }
      for (; l < L; ++l) st.step(row[(size_t)l * N], l, label);
      // the log-sum-exp kept in two parts, max and log of the shifted sum: z - m is exact near the top of the row, so
      // softmax = exp((z - m) - log_sum) keeps its digits when the logits are large
      const float ls = logf(st.sum);
      fine_lab[bn] = label;
      fine_pred[bn] = st.arg;
      lse[bn] = st.m;
      lse[(size_t)B * N + bn] = ls;
      if (in) {
        ce = (double)((st.m - st.zl) + ls);
        f_ok = st.arg == label ? 1 : 0;
      }
    }
  }
  focal = warp_sum(focal);
  ce = warp_sum(ce);
  inside = warp_sum(inside);
  c_ok = warp_sum(c_ok);
  f_ok = warp_sum(f_ok);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
    sh_d[0][warp] = focal; sh_d[1][warp] = ce;
    sh_i[0][warp] = inside; sh_i[1][warp] = c_ok; sh_i[2][warp] = f_ok;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double d0 = 0.0, d1 = 0.0;
    int i0 = 0, i1 = 0, i2 = 0;
    for (int w = 0; w < kClsWarps; ++w) {
      d0 += sh_d[0][w]; d1 += sh_d[1][w];
      i0 += sh_i[0][w]; i1 += sh_i[1][w]; i2 += sh_i[2][w];
    }
    const size_t nblk = gridDim.x, slot = (size_t)b * nblk + blockIdx.x, plane = (size_t)B * nblk;
    part_d[slot] = d0; part_d[plane + slot] = d1;
    part_i[slot] = i0; part_i[plane + slot] = i1; part_i[2 * plane + slot] = i2;
  }
}

// One CTA of kClsThreads.  Thread t sums samples t, t + 256, ... in that order; the threads' sums meet in a fixed tree.
__global__ void __launch_bounds__(kClsThreads)
    cls_reduce_kernel(const double* __restrict__ part_d, const int32_t* __restrict__ part_i, int B, int N, int nblk,
                      int has_fine, double coarse_alpha, float* __restrict__ loss, float* __restrict__ coarse_loss,
                      float* __restrict__ fine_loss, float* __restrict__ accuracy, int32_t* __restrict__ n_inside,
                      int32_t* __restrict__ coarse_correct, int32_t* __restrict__ fine_correct,
                      int32_t* __restrict__ n_inside_total) {
  __shared__ double sh_d[2][kClsThreads];
  __shared__ long long sh_i[3][kClsThreads];
  const size_t plane = (size_t)B * nblk;
  double d0 = 0.0, d1 = 0.0;
  long long i0 = 0, i1 = 0, i2 = 0;
  for (int b = threadIdx.x; b < B; b += kClsThreads) {
    double e0 = 0.0, e1 = 0.0;
    int j0 = 0, j1 = 0, j2 = 0;
    for (int k = 0; k < nblk; ++k) {
      const size_t slot = (size_t)b * nblk + k;
      e0 += part_d[slot]; e1 += part_d[plane + slot];
      j0 += part_i[slot]; j1 += part_i[plane + slot]; j2 += part_i[2 * plane + slot];
    }
    n_inside[b] = j0;
    coarse_correct[b] = j1;
    if (fine_correct) fine_correct[b] = j2;
    d0 += e0; d1 += e1;
    i0 += j0; i1 += j1; i2 += j2;
  }
  const int t = threadIdx.x;
  sh_d[0][t] = d0; sh_d[1][t] = d1;
  sh_i[0][t] = i0; sh_i[1][t] = i1; sh_i[2][t] = i2;
  __syncthreads();
  for (int h = kClsThreads / 2; h > 0; h >>= 1) {
    if (t < h) {
      sh_d[0][t] += sh_d[0][t + h]; sh_d[1][t] += sh_d[1][t + h];
      sh_i[0][t] += sh_i[0][t + h]; sh_i[1][t] += sh_i[1][t + h]; sh_i[2][t] += sh_i[2][t + h];
    }
    __syncthreads();
  }
  if (t == 0) {
    const double points = (double)B * (double)N;
    const long long n_in = sh_i[0][0];
    const float c = (float)(coarse_alpha * (sh_d[0][0] / points));
    const float f = (has_fine && n_in > 0) ? (float)(sh_d[1][0] / (double)n_in) : 0.f;
    *coarse_loss = c;
    *fine_loss = f;
    *loss = c + f;
    accuracy[0] = (float)((double)sh_i[1][0] / points);
    accuracy[1] = has_fine ? (float)((double)sh_i[2][0] / (double)n_in) : 0.f;   // 0 / 0 = NaN: no inside point
    *n_inside_total = (int32_t)n_in;
  }
}

__global__ void __launch_bounds__(kClsThreads)
    cls_backward_kernel(const float* __restrict__ coarse, long long cbs, const float* __restrict__ fine, long long fbs,
                        int L, int N, const int8_t* __restrict__ coarse_lab, const int32_t* __restrict__ fine_lab,
                        const float* __restrict__ lse, const int32_t* __restrict__ n_inside_total,
                        const float* __restrict__ g_loss, const float* __restrict__ g_coarse,
                        const float* __restrict__ g_fine, double coarse_scale, float alpha, int gamma, float eps,
                        float* __restrict__ grad_coarse, float* __restrict__ grad_fine) {
  const int b = blockIdx.y, n = blockIdx.x * kClsThreads + threadIdx.x;
  if (n >= N) return;
  const size_t bn = (size_t)b * N + n;
  const float gl = *g_loss;
  if (grad_coarse) {
    const float sc = (float)(((double)gl + (double)*g_coarse) * coarse_scale);
    const float* zc = coarse + (size_t)b * cbs + n;
    const Focal2 f = focal2(zc[0], zc[N], coarse_lab[bn], alpha, gamma, eps);
    const float d = f.dz0 * sc;
    float* gc = grad_coarse + (size_t)b * 2 * N + n;
    gc[0] = d;
    gc[N] = -d;
  }
  if (grad_fine) {
    float* gr = grad_fine + (size_t)b * L * N + n;
    const int label = fine_lab[bn];
    if (label < 0) {
      for (int l = 0; l < L; ++l) gr[(size_t)l * N] = 0.f;
      return;
    }
    const float sf = (float)(((double)gl + (double)*g_fine) / (double)*n_inside_total);
    const float m = lse[bn], ls = lse[(size_t)gridDim.y * N + bn];
    const float* row = fine + (size_t)b * fbs + n;
    int l = 0;
    for (; l + kClsChunk <= L; l += kClsChunk) {
      float z[kClsChunk];
#pragma unroll
      for (int j = 0; j < kClsChunk; ++j) z[j] = row[(size_t)(l + j) * N];
#pragma unroll
      for (int j = 0; j < kClsChunk; ++j)
        gr[(size_t)(l + j) * N] = (expf((z[j] - m) - ls) - (l + j == label ? 1.f : 0.f)) * sf;
    }
    for (; l < L; ++l) gr[(size_t)l * N] = (expf((row[(size_t)l * N] - m) - ls) - (l == label ? 1.f : 0.f)) * sf;
  }
}

inline int cls_blocks(int N) { return (N + kClsThreads - 1) / kClsThreads; }

}  // namespace dib

extern "C" {

size_t classifier_loss_workspace_bytes(int B, int N) {
  if (B <= 0 || N <= 0) return 0;
  const size_t slots = (size_t)B * dib::cls_blocks(N);
  return slots * (2 * sizeof(double) + 3 * sizeof(int32_t));
}

// Shared host checks of both entry points.
static int cls_check(const float* coarse, long long cbs, const float* fine, long long fbs, int L, int B, int N,
                     int gamma, const char* what) {
  DIB_REQUIRE(B >= 1 && B <= 65535 && N >= 1, "%s: need 1 <= B <= 65535 and N >= 1", what);
  DIB_REQUIRE((long long)B * N < (1LL << 31), "%s: B * N must be below 2^31", what);
  DIB_REQUIRE(coarse && cbs >= 0, "%s: NULL coarse scores or negative batch stride", what);
  DIB_REQUIRE(!fine || (L >= 1 && fbs >= 0), "%s: need L >= 1 and a non-negative fine batch stride", what);
  DIB_REQUIRE(gamma >= 0, "%s: focal_gamma must be a non-negative integer", what);
  return DIB_OK;
}

int classifier_loss_forward_f32(const float* coarse, int64_t coarse_batch_stride, const float* fine,
                                int64_t fine_batch_stride, int L, const float* pc, const double* P12, const double* K9,
                                int B, int N, double H, double W, double fine_scale, int H_f, int W_f,
                                double coarse_loss_alpha, double focal_alpha, int focal_gamma, double eps,
                                int8_t* coarse_labels, int32_t* fine_labels, int8_t* coarse_pred, int32_t* fine_pred,
                                float* lse, float* loss, float* coarse_loss, float* fine_loss, float* accuracy,
                                int32_t* n_inside, int32_t* coarse_correct, int32_t* fine_correct,
                                int32_t* n_inside_total, void* workspace, size_t workspace_bytes, dib_stream_t stream_) {
  using namespace dib;
  cudaStream_t stream = (cudaStream_t)stream_;
  const int rc = cls_check(coarse, coarse_batch_stride, fine, fine_batch_stride, L, B, N, focal_gamma,
                           "classifier_loss_forward");
  if (rc != DIB_OK) return rc;
  DIB_REQUIRE(pc && P12 && K9 && coarse_labels && coarse_pred && loss && coarse_loss && fine_loss && accuracy &&
                  n_inside && coarse_correct && n_inside_total,
              "classifier_loss_forward: NULL argument");
  DIB_REQUIRE(H >= 1.0 && W >= 1.0 && fine_scale > 0.0, "classifier_loss_forward: need H, W >= 1 and fine_scale > 0");
  if (fine) {
    DIB_REQUIRE(fine_labels && fine_pred && lse && fine_correct, "classifier_loss_forward: NULL fine output");
    DIB_REQUIRE(H_f >= 1 && W_f >= 1 && (long long)H_f * W_f == L,
                "classifier_loss_forward: L = %d is not H_f * W_f = %d * %d", L, H_f, W_f);
    // with these every fine label of an inside point lies in [0, L)
    DIB_REQUIRE(floor((W - 1.0) / fine_scale) < W_f && floor((H - 1.0) / fine_scale) < H_f,
                "classifier_loss_forward: the last pixel row / column falls outside the %d x %d cell grid", H_f, W_f);
  }
  const size_t need = classifier_loss_workspace_bytes(B, N);
  DIB_REQUIRE(workspace && workspace_bytes >= need && ((uintptr_t)workspace & 7) == 0,
              "classifier_loss_forward: workspace too small or misaligned");
  const int nblk = cls_blocks(N);
  double* part_d = (double*)workspace;
  int32_t* part_i = (int32_t*)(part_d + 2 * (size_t)B * nblk);
  cls_forward_kernel<<<dim3(nblk, B), kClsThreads, 0, stream>>>(
      coarse, coarse_batch_stride, fine, fine_batch_stride, L, pc, P12, K9, B, N, H, W, fine_scale, W_f,
      (float)focal_alpha, focal_gamma, (float)eps, coarse_labels, fine_labels, coarse_pred, fine_pred, lse, part_d,
      part_i);
  DIB_CHECK_CUDA(cudaGetLastError());
  cls_reduce_kernel<<<1, kClsThreads, 0, stream>>>(part_d, part_i, B, N, nblk, fine ? 1 : 0, coarse_loss_alpha, loss,
                                                   coarse_loss, fine_loss, accuracy, n_inside, coarse_correct,
                                                   fine ? fine_correct : nullptr, n_inside_total);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

int classifier_loss_backward_f32(const float* coarse, int64_t coarse_batch_stride, const float* fine,
                                 int64_t fine_batch_stride, int L, int B, int N, const int8_t* coarse_labels,
                                 const int32_t* fine_labels, const float* lse, const int32_t* n_inside_total,
                                 const float* grad_loss, const float* grad_coarse_loss, const float* grad_fine_loss,
                                 double coarse_loss_alpha, double focal_alpha, int focal_gamma, double eps,
                                 float* grad_coarse, float* grad_fine, dib_stream_t stream_) {
  using namespace dib;
  cudaStream_t stream = (cudaStream_t)stream_;
  const int rc = cls_check(coarse, coarse_batch_stride, fine, fine_batch_stride, L, B, N, focal_gamma,
                           "classifier_loss_backward");
  if (rc != DIB_OK) return rc;
  DIB_REQUIRE(grad_loss && coarse_labels, "classifier_loss_backward: NULL argument");
  DIB_REQUIRE(!grad_coarse || grad_coarse_loss, "classifier_loss_backward: NULL coarse upstream gradient");
  DIB_REQUIRE(!grad_fine || (fine && fine_labels && lse && n_inside_total && grad_fine_loss),
              "classifier_loss_backward: NULL fine argument");
  if (!grad_coarse && !grad_fine) return DIB_OK;
  const double coarse_scale = coarse_loss_alpha / ((double)B * (double)N);
  cls_backward_kernel<<<dim3(cls_blocks(N), B), kClsThreads, 0, stream>>>(
      coarse, coarse_batch_stride, fine, fine_batch_stride, L, N, coarse_labels, fine_labels, lse, n_inside_total,
      grad_loss, grad_coarse_loss, grad_fine_loss, coarse_scale, (float)focal_alpha, focal_gamma, (float)eps,
      grad_coarse, grad_fine);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

}  // extern "C"
