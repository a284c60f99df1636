// Monodepth depth clouds for the ICP baseline (evaluation/icp/save_depth_map.py; SURVEY.md 8f row N26, DESIGN.md
// 4.31): the network's input side and its output side on the device, so a batch goes from decoded frames to the
// target clouds of icp_register_batch_f32 without a host round trip.
//
//   md_resample_kernel  one separable pass of Pillow's 8-bit Lanczos resize (Resample.c) over uint8 HWC frames, one
//                       thread per output pixel (3 channels): int32 accumulator starting at 2^21, the host's
//                       fixed-point coefficients (2^-22 units), >> 22 and a clip to 0..255.  The pass writes a uint8
//                       intermediate, or, as the last pass, the encoder's input ((v / 255 - sub) * mul, NCHW f32).
//   md_cloud_kernel     one thread per output pixel: torch's CUDA upsample_bilinear2d (align_corners=False) of the
//                       disparity, its reciprocal, and the back-projection K^-1 (d x, d y, d) in fp64; writes the
//                       unscaled fp64 cloud, or, in the second pass, float32(p * scale[s]); each CTA also leaves the
//                       fp64 sum of its z values for the scale (a fixed shared-memory tree).
//   md_scale_kernel     one CTA per frame: the fp64 z sum of the LiDAR points inside the image under P_gt
//                       (project.cuh) and of the CTA partials, both in a fixed order, and scale = mean / mean.
//
// Compiled without FMA contraction (build.py NOFMA_SOURCES): the contractions of torch's bilinear kernel are written
// out with __fmaf_rn, and the back-projection and the inside test are plain products and sums.  No atomics.
#include <math.h>

#include "common.cuh"
#include "project.cuh"

namespace dib {

constexpr int kMdThreads = 256;

__global__ void __launch_bounds__(kMdThreads)
md_resample_kernel(const uint8_t* __restrict__ in, const int64_t* __restrict__ off, int h_in, int w_in, int h_out,
                   int w_out, int axis, const int32_t* __restrict__ tab, int ksize, uint8_t* __restrict__ out_u8,
                   float* __restrict__ out_f32, float sub, float mul) {
  const long long P = (long long)h_out * w_out;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int s = blockIdx.y;
  if (i >= P) return;
  const int y = (int)(i / w_out), x = (int)(i - (long long)y * w_out);
  const uint8_t* src = in + (off ? off[s] : (long long)s * h_in * w_in * 3);
  int v0, v1, v2;
  if (tab == nullptr) {
    const uint8_t* p = src + ((size_t)y * w_in + x) * 3;
    v0 = p[0], v1 = p[1], v2 = p[2];
  } else {
    const int32_t* t = tab + (size_t)(axis == 0 ? x : y) * (2 + ksize);
    const int lo = t[0], n = t[1];
    const size_t step = axis == 0 ? 3 : (size_t)w_in * 3;
    const uint8_t* p = axis == 0 ? src + ((size_t)y * w_in + lo) * 3 : src + ((size_t)lo * w_in + x) * 3;
    int a0 = 1 << 21, a1 = 1 << 21, a2 = 1 << 21;
    for (int j = 0; j < n; ++j, p += step) {
      const int k = t[2 + j];
      a0 += p[0] * k, a1 += p[1] * k, a2 += p[2] * k;
    }
    v0 = min(max(a0 >> 22, 0), 255), v1 = min(max(a1 >> 22, 0), 255), v2 = min(max(a2 >> 22, 0), 255);
  }
  if (out_u8) {
    uint8_t* q = out_u8 + ((size_t)s * P + i) * 3;
    q[0] = (uint8_t)v0, q[1] = (uint8_t)v1, q[2] = (uint8_t)v2;
  }
  if (out_f32) {
    float* q = out_f32 + (size_t)s * 3 * P + i;
    q[0] = (__fdiv_rn((float)v0, 255.0f) - sub) * mul;
    q[P] = (__fdiv_rn((float)v1, 255.0f) - sub) * mul;
    q[2 * P] = (__fdiv_rn((float)v2, 255.0f) - sub) * mul;
  }
}

// torch.reciprocal(F.interpolate(disp, (H, W), mode="bilinear", align_corners=False)) at (oy, ox): torch's
// upsample_bilinear2d_out_frame with its float32 accumulation, rh = h / H and rw = w / W.
__device__ __forceinline__ float md_depth(const float* __restrict__ d, int h, int w, int H, int W, float rh, float rw,
                                          int oy, int ox) {
  if (h == H && w == W) return __frcp_rn(d[(size_t)oy * w + ox]);
  float h1r = __fmaf_rn(rh, (float)oy + 0.5f, -0.5f);
  h1r = h1r < 0.0f ? 0.0f : h1r;
  const int h1 = (int)h1r;
  const int h1p = h1 < h - 1 ? 1 : 0;
  const float h1l = h1r - (float)h1, h0l = 1.0f - h1l;
  float w1r = __fmaf_rn(rw, (float)ox + 0.5f, -0.5f);
  w1r = w1r < 0.0f ? 0.0f : w1r;
  const int w1 = (int)w1r;
  const int w1p = w1 < w - 1 ? 1 : 0;
  const float w1l = w1r - (float)w1, w0l = 1.0f - w1l;
  const float* r0 = d + (size_t)h1 * w + w1;
  const float* r1 = r0 + (size_t)h1p * w;
  const float top = __fmaf_rn(w0l, r0[0], __fmul_rn(w1l, r0[w1p]));
  const float bot = __fmaf_rn(w0l, r1[0], __fmul_rn(w1l, r1[w1p]));
  return __frcp_rn(__fmaf_rn(h0l, top, __fmul_rn(h1l, bot)));
}

struct MdCloud {
  const float* disp;                  // [S][h][w]
  int h, w, H, W;
  float rh, rw;
  const double* K_inv;                // [S][9]
  float* depth;                       // [S][H*W] or NULL
  double* out64;                      // [S][3][H*W] or NULL
  float* out32;                       // [S][3][H*W] or NULL (then scale is read)
  const double* scale;                // [S]
  double* partial;                    // [S][gridDim.x] or NULL
};

__global__ void __launch_bounds__(kMdThreads) md_cloud_kernel(MdCloud p) {
  __shared__ double red[kMdThreads];
  const int s = blockIdx.y;
  const long long P = (long long)p.H * p.W;
  const long long i = (long long)blockIdx.x * kMdThreads + threadIdx.x;
  double z = 0.0;
  if (i < P) {
    const int oy = (int)(i / p.W), ox = (int)(i - (long long)oy * p.W);
    const float dep = md_depth(p.disp + (size_t)s * p.h * p.w, p.h, p.w, p.H, p.W, p.rh, p.rw, oy, ox);
    if (p.depth) p.depth[(size_t)s * P + i] = dep;
    // depth_np * meshgrid_np: exact products of a float32 depth and integers below 2^24
    const double D = (double)dep, X = D * (double)ox, Y = D * (double)oy;
    const double* k = p.K_inv + 9 * (size_t)s;
    const double px = k[0] * X + k[1] * Y + k[2] * D;
    const double py = k[3] * X + k[4] * Y + k[5] * D;
    const double pz = k[6] * X + k[7] * Y + k[8] * D;
    z = pz;
    if (p.out64) {
      double* q = p.out64 + (size_t)s * 3 * P + i;
      q[0] = px, q[P] = py, q[2 * P] = pz;
    }
    if (p.out32) {
      const double c = p.scale[s];
      float* q = p.out32 + (size_t)s * 3 * P + i;
      q[0] = (float)(px * c), q[P] = (float)(py * c), q[2 * P] = (float)(pz * c);
    }
  }
  if (p.partial == nullptr) return;
  red[threadIdx.x] = z;
  __syncthreads();
  for (int h = kMdThreads / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) p.partial[(size_t)s * gridDim.x + blockIdx.x] = red[0];
}

__global__ void __launch_bounds__(kMdThreads)
md_scale_kernel(const float* __restrict__ src, const int32_t* __restrict__ n_pts, int Ns,
                const double* __restrict__ P16, const double* __restrict__ K9, double H, double W,
                const double* __restrict__ partial, int n_part, long long n_pix, double* __restrict__ scale) {
  __shared__ double red[2][kMdThreads];
  const int s = blockIdx.x;
  const int n = n_pts ? n_pts[s] : Ns;
  const float* b = src + (size_t)s * 3 * Ns;
  const double* P = P16 + 16 * (size_t)s;
  const double* K = K9 + 9 * (size_t)s;
  double lz = 0.0, cnt = 0.0, dz = 0.0;
  for (int i = threadIdx.x; i < n; i += kMdThreads) {
    const double x = b[i], y = b[(size_t)Ns + i], zz = b[2 * (size_t)Ns + i];
    double u, v;
    if (project_inside(P, K, x, y, zz, H, W, &u, &v)) {
      lz += P[8] * x + P[9] * y + P[10] * zz + P[11];
      cnt += 1.0;
    }
  }
  for (int i = threadIdx.x; i < n_part; i += kMdThreads) dz += partial[(size_t)s * n_part + i];
  red[0][threadIdx.x] = lz;
  red[1][threadIdx.x] = dz;
  __shared__ double rc[kMdThreads];
  rc[threadIdx.x] = cnt;
  __syncthreads();
  for (int h = kMdThreads / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) {
      red[0][threadIdx.x] += red[0][threadIdx.x + h];
      red[1][threadIdx.x] += red[1][threadIdx.x + h];
      rc[threadIdx.x] += rc[threadIdx.x + h];
    }
    __syncthreads();
  }
  // np.mean(z[mask]) / np.mean(depth_pc[2]); no inside point gives NaN, as numpy's mean of an empty array does
  if (threadIdx.x == 0) scale[s] = (red[0][0] / rc[0]) / (red[1][0] / (double)n_pix);
}

}  // namespace dib

extern "C" {

int monodepth_resize_f32(const uint8_t* data, const int64_t* offsets, int S, int h, int w, int out_h, int out_w,
                         const int32_t* tab_x, int kx, const int32_t* tab_y, int ky, float sub, float mul,
                         uint8_t* tmp, size_t tmp_bytes, float* out, dib_stream_t stream) {
  using namespace dib;
  DIB_REQUIRE(S >= 1 && S <= 65535 && h >= 1 && w >= 1 && out_h >= 1 && out_w >= 1,
              "monodepth_resize: need 1 <= S <= 65535 and positive sizes");
  DIB_REQUIRE(data != nullptr && out != nullptr, "monodepth_resize: data or out is NULL");
  DIB_REQUIRE((w == out_w) == (tab_x == nullptr) && (h == out_h) == (tab_y == nullptr),
              "monodepth_resize: a table is given exactly for each axis that changes size");
  DIB_REQUIRE((!tab_x || kx >= 1) && (!tab_y || ky >= 1), "monodepth_resize: tables need ksize >= 1");
  const long long mid = (long long)h * out_w;
  DIB_REQUIRE((long long)out_h * out_w < (1LL << 31) && mid < (1LL << 31), "monodepth_resize: frames too large");
  cudaStream_t st = (cudaStream_t)stream;
  if (tab_x && tab_y) {
    DIB_REQUIRE(tmp != nullptr && tmp_bytes >= (size_t)S * mid * 3, "monodepth_resize: tmp is NULL or too small");
    md_resample_kernel<<<dim3((unsigned)((mid + kMdThreads - 1) / kMdThreads), S), kMdThreads, 0, st>>>(
        data, offsets, h, w, h, out_w, 0, tab_x, kx, tmp, nullptr, 0.f, 0.f);
    DIB_CHECK_CUDA(cudaGetLastError());
    data = tmp, offsets = nullptr, w = out_w;
  }
  const long long P = (long long)out_h * out_w;
  const int axis = tab_y ? 1 : 0;
  md_resample_kernel<<<dim3((unsigned)((P + kMdThreads - 1) / kMdThreads), S), kMdThreads, 0, st>>>(
      data, offsets, h, w, out_h, out_w, axis, tab_y ? tab_y : tab_x, tab_y ? ky : kx, nullptr, out, sub, mul);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

size_t monodepth_cloud_workspace_bytes(int S, int H, int W) {
  if (S < 1 || H < 1 || W < 1) return 0;
  const long long P = (long long)H * W;
  return (size_t)S * (size_t)((P + dib::kMdThreads - 1) / dib::kMdThreads) * sizeof(double);
}

int monodepth_cloud_f32(const float* disp, int S, int h, int w, int H, int W, const double* K_inv, float* depth,
                        double* out64, const float* src, const int32_t* n_pts, int Ns, const double* P_gt,
                        const double* K, double* scale, float* out32, void* workspace, size_t workspace_bytes,
                        dib_stream_t stream) {
  using namespace dib;
  DIB_REQUIRE(S >= 1 && S <= 65535 && h >= 1 && w >= 1 && H >= 1 && W >= 1,
              "monodepth_cloud: need 1 <= S <= 65535 and positive sizes");
  DIB_REQUIRE((long long)H * W < (1LL << 31) - kMdThreads, "monodepth_cloud: output frames too large");
  DIB_REQUIRE(disp != nullptr && K_inv != nullptr, "monodepth_cloud: disp or K_inv is NULL");
  DIB_REQUIRE(depth || out64 || scale, "monodepth_cloud: no output requested");
  const bool calib = scale != nullptr;
  DIB_REQUIRE(!calib || (src && P_gt && K && Ns >= 0), "monodepth_cloud: the scale needs src, P_gt and K");
  DIB_REQUIRE(!out32 || calib, "monodepth_cloud: the scaled float32 cloud needs the scale");
  const long long P = (long long)H * W;
  const int nblk = (int)((P + kMdThreads - 1) / kMdThreads);
  MdCloud p = {};
  p.disp = disp, p.h = h, p.w = w, p.H = H, p.W = W;
  // torch's area_pixel_compute_scale: (float)input_size / output_size
  p.rh = (float)h / (float)H, p.rw = (float)w / (float)W;
  p.K_inv = K_inv, p.depth = depth, p.out64 = out64;
  if (calib) {
    DIB_REQUIRE(workspace && workspace_bytes >= monodepth_cloud_workspace_bytes(S, H, W),
                "monodepth_cloud: workspace is NULL or too small");
    p.partial = (double*)workspace;
  }
  cudaStream_t st = (cudaStream_t)stream;
  md_cloud_kernel<<<dim3(nblk, S), kMdThreads, 0, st>>>(p);
  DIB_CHECK_CUDA(cudaGetLastError());
  if (!calib) return DIB_OK;
  md_scale_kernel<<<S, kMdThreads, 0, st>>>(src, n_pts, Ns, P_gt, K, (double)H, (double)W, p.partial, nblk, P, scale);
  DIB_CHECK_CUDA(cudaGetLastError());
  if (!out32) return DIB_OK;
  MdCloud q = {};
  q.disp = disp, q.h = h, q.w = w, q.H = H, q.W = W, q.rh = p.rh, q.rw = p.rw, q.K_inv = K_inv;
  q.out32 = out32, q.scale = scale;
  md_cloud_kernel<<<dim3(nblk, S), kMdThreads, 0, st>>>(q);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

}  // extern "C"
