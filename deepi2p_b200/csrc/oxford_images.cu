// Oxford RobotCar stereo-centre frames: GBRG Bayer demosaicing and LUT undistortion fused, bit for bit with the
// RobotCar SDK's load_image(path, CameraModel) (colour_demosaicing's bilinear demosaic in float64, scipy's
// map_coordinates(order=1) per channel, then a uint8 cast).  DESIGN.md 4.25 states the contract;
// oracle_oxford_images/ restates it on the CPU and deepi2p_b200/oxford_images.py is the host side.
//
// oxford_debayer_kernel  thread per output pixel, all three channels: reads the pixel's LUT coordinate (x, y), then
//                        for each of the four interpolation taps the demosaiced values, computed on the fly from the
//                        raw mosaic's 3 x 3 neighbourhood with reflected borders.  The float64 RGB image is never
//                        materialised.
//
// Compiled with --fmad=false (build.py NOFMA_SOURCES): the interpolation's products and sums are rounded one by one
// in scipy's order.  The demosaiced values are integer tap sums times 0.25, exact in fp64.
#include <vector>

#include "common.cuh"

namespace dib {
namespace oxford_images {

constexpr int kMaxS = 65535;
constexpr int kThreads = 256;
enum { kIn = 0, kOut, kH, kW, kLut };   // descriptor slots, DIB_OXIMG_DESC of them per image
static_assert(kLut < DIB_OXIMG_DESC, "descriptor slots");

// GBRG: (even row, even column) G, (even, odd) B, (odd, even) R, (odd, odd) G.  Channel 0 R, 1 G, 2 B.
__device__ __forceinline__ int bayer_channel(int r, int c) {
  return (r & 1) ? ((c & 1) ? 1 : 0) : ((c & 1) ? 2 : 1);
}

// 4 x the demosaiced value of channel ch at (r, c): the masked 3 x 3 tap sum with the integer kernels
// H_G = [[0,1,0],[1,4,1],[0,1,0]] and H_RB = [[1,2,1],[2,4,2],[1,2,1]] and scipy's 'reflect' borders (-1 -> 0,
// n -> n - 1), the mask read at the reflected pixel.
__device__ __forceinline__ void demosaic4(const uint8_t* __restrict__ img, int H, int W, int r, int c, int out[3]) {
  out[0] = out[1] = out[2] = 0;
#pragma unroll
  for (int dy = -1; dy <= 1; ++dy) {
    int rr = r + dy;
    rr = rr < 0 ? 0 : rr >= H ? H - 1 : rr;
#pragma unroll
    for (int dx = -1; dx <= 1; ++dx) {
      int cc = c + dx;
      cc = cc < 0 ? 0 : cc >= W ? W - 1 : cc;
      const int v = img[(size_t)rr * W + cc];
      const int ch = bayer_channel(rr, cc);
      const int wrb = (dy == 0 ? 2 : 1) * (dx == 0 ? 2 : 1);
      const int wg = (dy == 0 && dx == 0) ? 4 : (dy == 0 || dx == 0) ? 1 : 0;
      out[0] += ch == 0 ? v * wrb : 0;                              // selects, so out[] stays in registers
      out[1] += ch == 1 ? v * wg : 0;
      out[2] += ch == 2 ? v * wrb : 0;
    }
  }
}

__global__ void __launch_bounds__(kThreads) oxford_debayer_kernel(const uint8_t* __restrict__ grey,
                                                                  const double2* __restrict__ lut,
                                                                  const int64_t* __restrict__ desc,
                                                                  uint8_t* __restrict__ out) {
  const int64_t* q = desc + (size_t)blockIdx.y * DIB_OXIMG_DESC;
  const int H = (int)q[kH], W = (int)q[kW];
  const int64_t p = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (p >= (int64_t)H * W) return;
  const uint8_t* img = grey + q[kIn];
  const double2 xy = lut[q[kLut] + p];
  const double x = xy.x, y = xy.y;
  uint8_t* o = out + q[kOut] + 3 * p;
  // map_coordinates' 'constant' mode: a coordinate below 0 or above n - 1 on either axis gives cval 0.
  if (!(y >= 0.0 && y <= (double)(H - 1) && x >= 0.0 && x <= (double)(W - 1))) {
    o[0] = o[1] = o[2] = 0;
    return;
  }
  const double fy = floor(y), fx = floor(x);
  const double ty = __dsub_rn(y, fy), tx = __dsub_rn(x, fx);
  const double wy0 = __dsub_rn(1.0, ty), wx0 = __dsub_rn(1.0, tx);
  const double wy1 = __dsub_rn(1.0, wy0), wx1 = __dsub_rn(1.0, wx0);
  const int r0 = (int)fy, c0 = (int)fx;
  const int r1 = min(r0 + 1, H - 1), c1 = min(c0 + 1, W - 1);   // a tap past the edge has weight 0
  int v00[3], v01[3], v10[3], v11[3];
  demosaic4(img, H, W, r0, c0, v00);
  demosaic4(img, H, W, r0, c1, v01);
  demosaic4(img, H, W, r1, c0, v10);
  demosaic4(img, H, W, r1, c1, v11);
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    double acc = 0.0;
    acc = __dadd_rn(acc, __dmul_rn(__dmul_rn((double)v00[ch] * 0.25, wy0), wx0));
    acc = __dadd_rn(acc, __dmul_rn(__dmul_rn((double)v01[ch] * 0.25, wy0), wx1));
    acc = __dadd_rn(acc, __dmul_rn(__dmul_rn((double)v10[ch] * 0.25, wy1), wx0));
    acc = __dadd_rn(acc, __dmul_rn(__dmul_rn((double)v11[ch] * 0.25, wy1), wx1));
    // numpy's float64 -> uint8 cast on x86-64: truncate to a 32-bit integer, keep the low byte.  Values above 255
    // occur at the mosaic's borders, where the reflected taps count a pixel twice.
    o[ch] = (uint8_t)(uint32_t)(int32_t)acc;
  }
}

int run(const uint8_t* grey, size_t grey_bytes, const double* lut, int64_t lut_pairs, const int64_t* desc, int S,
        uint8_t* out, size_t out_bytes, void* workspace, size_t workspace_bytes, cudaStream_t cs) {
  DIB_REQUIRE(S >= 0 && S <= kMaxS, "S must be in [0, %d] (got %d)", kMaxS, S);
  if (S == 0) return 0;
  DIB_REQUIRE(grey && lut && desc && out && workspace, "a required pointer is null");
  DIB_REQUIRE(((uintptr_t)lut & 15) == 0, "lut must be 16-byte aligned");
  int64_t max_px = 0;
  for (int s = 0; s < S; ++s) {
    const int64_t* q = desc + (size_t)s * DIB_OXIMG_DESC;
    const int64_t n = q[kH] * q[kW];
    DIB_REQUIRE(q[kH] >= 2 && q[kW] >= 2 && q[kH] <= (1 << 16) && q[kW] <= (1 << 16),
                "image %d: size %lld x %lld (each side must be in 2..65536)", s, (long long)q[kH], (long long)q[kW]);
    DIB_REQUIRE(q[kIn] >= 0 && (size_t)(q[kIn] + n) <= grey_bytes, "image %d: mosaic outside the input", s);
    DIB_REQUIRE(q[kOut] >= 0 && (size_t)(q[kOut] + 3 * n) <= out_bytes, "image %d: output outside the buffer", s);
    DIB_REQUIRE(q[kLut] >= 0 && q[kLut] + n <= lut_pairs, "image %d: LUT range outside the %lld LUT entries", s,
                (long long)lut_pairs);
    max_px = n > max_px ? n : max_px;
  }
  const size_t need = (size_t)S * DIB_OXIMG_DESC * sizeof(int64_t);
  if (workspace_bytes < need) {
    set_error("oxford_debayer: workspace is %zu bytes, %zu needed", workspace_bytes, need);
    return DIB_ENOMEM;
  }
  DIB_CHECK_CUDA(cudaMemcpyAsync(workspace, desc, need, cudaMemcpyHostToDevice, cs));
  const dim3 grid((unsigned)((max_px + kThreads - 1) / kThreads), (unsigned)S);
  oxford_debayer_kernel<<<grid, kThreads, 0, cs>>>(grey, (const double2*)lut, (const int64_t*)workspace, out);
  DIB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace oxford_images
}  // namespace dib

extern "C" {

size_t oxford_debayer_workspace_bytes(int S) {
  return S < 0 ? 0 : (size_t)(S > 0 ? S : 1) * DIB_OXIMG_DESC * sizeof(int64_t);
}

int oxford_debayer_undistort_u8(const uint8_t* grey, size_t grey_bytes, const double* lut, int64_t lut_pairs,
                                const int64_t* desc, int S, uint8_t* out, size_t out_bytes, void* workspace,
                                size_t workspace_bytes, dib_stream_t stream) {
  return dib::oxford_images::run(grey, grey_bytes, lut, lut_pairs, desc, S, out, out_bytes, workspace,
                                 workspace_bytes, (cudaStream_t)stream);
}

}  // extern "C"
