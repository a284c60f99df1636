// The image side of the classifier's input batches: the part of the KITTI / Oxford / nuScenes loaders' __getitem__
// that turns a raw camera frame into `img` (data/kitti_pc_img_pose_loader.py:326-349,360-362,439-440,
// data/oxford_pc_img_pose_loader.py:238-259,300-301,368).  DESIGN.md 4.13 states the contract; oracle_image/ is its
// numpy restatement, bit for bit against cv2 and Pillow.
//
// Per sample: a row cut of a ragged HWC uint8 frame (a view), cv2.resize(INTER_LINEAR) to (dh, dw) by OpenCV's
// fixed-point path, the H x W window at (dy, dx) -- only the window is computed --, torchvision's ColorJitter steps
// on a PIL image in the sample's order, a column flip, and the CHW write.
//
// image_luma_partials_kernel  CTA per (32 x 32 output tile, sample) of the jittered samples: the chain up to the
//                             contrast step, then the exact integer sum of the tile's L into partial[s][tile]
// image_assemble_kernel       CTA per (tile, sample): warp 0 adds the sample's partials in tile order (an exact
//                             integer sum, so the run is bit-identical without float atomics) into the contrast
//                             grey level; every thread recomputes the chain from the raw pixels for 4 pixels of one
//                             output column and writes them
//
// The flip commutes with every colour step (they are per pixel, and the contrast mean does not depend on the pixel
// order), so it is an index map: output column xo reads crop column W-1-xo.
// The file is compiled with --fmad=false (build.py NOFMA_SOURCES); the intrinsics make each rounding explicit anyway.
#include <cmath>
#include <vector>

#include "common.cuh"

namespace dib {
namespace img {

constexpr int kMaxS = 65535;
constexpr int kMaxSide = 16384;
constexpr int kTileW = 32, kTileRows = 8, kRowsPerThread = 4;
constexpr int kTileH = kTileRows * kRowsPerThread;
enum { kBrightness = 0, kContrast = 1, kSaturation = 2, kHue = 3 };

__host__ __device__ inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }
inline int tiles_of(int H, int W) { return ((W + kTileW - 1) / kTileW) * ((H + kTileH - 1) / kTileH); }

struct Layout {
  size_t params, offsets, factors, partial, head, total;
};

inline Layout layout(int S, int H, int W) {
  Layout L;
  L.params = 0;
  L.offsets = align256((size_t)S * DIB_IMAGE_PARAMS * sizeof(int32_t));
  L.factors = L.offsets + align256((size_t)S * sizeof(int64_t));
  L.head = L.factors + align256((size_t)S * 3 * sizeof(float));
  L.partial = L.head;
  L.total = L.partial + align256((size_t)S * tiles_of(H, W) * sizeof(uint32_t));
  return L;
}

struct Rgb {
  int r, g, b;
};

// ImagingBlend(deg, x, a) with a float32 factor: t = (float)deg + a * (float)(x - deg); 0 <= a <= 1 truncates,
// any other a clips to [0, 255] first.
__device__ __forceinline__ int blend1(int deg, int x, float a, bool in01) {
  const float t = __fadd_rn((float)deg, __fmul_rn(a, (float)(x - deg)));
  if (in01) return (int)t;
  return t <= 0.f ? 0 : (t >= 255.f ? 255 : (int)t);
}

__device__ __forceinline__ Rgb blend3(Rgb d, Rgb x, float a) {
  const bool in01 = a >= 0.f && a <= 1.f;
  return Rgb{blend1(d.r, x.r, a, in01), blend1(d.g, x.g, a, in01), blend1(d.b, x.b, a, in01)};
}

__device__ __forceinline__ int luma(Rgb p) { return (19595 * p.r + 38470 * p.g + 7471 * p.b + 0x8000) >> 16; }

__device__ __forceinline__ int clip8(int v) { return v < 0 ? 0 : (v > 255 ? 255 : v); }

// Pillow Convert.c: rgb2hsv (float cr, s, rc, gc, bc; the 2.0 / 4.0 / 6.0 / 1.0 / 255.0 steps in double), the hue
// byte shifted modulo 256, hsv2rgb (double i, f stored as float, float fs, round() half away from zero).
__device__ Rgb hue_shift(Rgb p, int shift) {
  const int mx = max(p.r, max(p.g, p.b)), mn = min(p.r, min(p.g, p.b));
  int h = 0, s = 0;
  const int v = mx;
  if (mx != mn) {
    const float cr = (float)(mx - mn);
    const float sf = __fdiv_rn(cr, (float)mx);
    const float rc = __fdiv_rn((float)(mx - p.r), cr);
    const float gc = __fdiv_rn((float)(mx - p.g), cr);
    const float bc = __fdiv_rn((float)(mx - p.b), cr);
    float hf;
    if (p.r == mx) hf = __fsub_rn(bc, gc);
    else if (p.g == mx) hf = __double2float_rn(__dsub_rn(__dadd_rn(2.0, (double)rc), (double)bc));
    else hf = __double2float_rn(__dsub_rn(__dadd_rn(4.0, (double)gc), (double)rc));
    hf = __double2float_rn(fmod(__dadd_rn(__ddiv_rn((double)hf, 6.0), 1.0), 1.0));
    h = clip8((int)__dmul_rn((double)hf, 255.0));
    s = clip8((int)__dmul_rn((double)sf, 255.0));
  }
  h = (h + shift) & 255;
  if (s == 0) return Rgb{v, v, v};
  const double hd = __ddiv_rn(__dmul_rn((double)h, 6.0), 255.0);
  const int i = (int)floor(hd);
  const float f = __double2float_rn(__dsub_rn(hd, (double)i));
  const float fs = __double2float_rn(__ddiv_rn((double)s, 255.0));
  const double vd = (double)v;
  const int pp = clip8((int)round(__dmul_rn(vd, __dsub_rn(1.0, (double)fs))));
  const int q = clip8((int)round(__dmul_rn(vd, __dsub_rn(1.0, (double)__fmul_rn(fs, f)))));
  const int t = clip8((int)round(__dmul_rn(vd, __dsub_rn(1.0, __dmul_rn((double)fs, __dsub_rn(1.0, (double)f))))));
  switch (i % 6) {
    case 0: return Rgb{v, t, pp};
    case 1: return Rgb{q, v, pp};
    case 2: return Rgb{pp, v, t};
    case 3: return Rgb{pp, q, v};
    case 4: return Rgb{t, pp, v};
    default: return Rgb{v, pp, q};
  }
}

struct Sample {
  const uint8_t* view;   // first row of the row-cut view
  int w, rows, dh, dw, dy, dx, flip, jitter, shift;
  int order[4];
  float fb, fc, fs;
};

__device__ __forceinline__ Sample load_sample(const uint8_t* src, const int64_t* offsets, const int32_t* params,
                                              const float* factors, int s) {
  const int32_t* p = params + (size_t)s * DIB_IMAGE_PARAMS;
  Sample a;
  a.w = p[DIB_IMG_W];
  a.view = src + offsets[s] + (size_t)p[DIB_IMG_ROW0] * a.w * 3;
  a.rows = p[DIB_IMG_ROWS];
  a.dh = p[DIB_IMG_DH];
  a.dw = p[DIB_IMG_DW];
  a.dy = p[DIB_IMG_DY];
  a.dx = p[DIB_IMG_DX];
  a.flip = p[DIB_IMG_FLIP];
  a.jitter = p[DIB_IMG_JITTER];
  a.shift = p[DIB_IMG_SHIFT];
#pragma unroll
  for (int o = 0; o < 4; ++o) a.order[o] = p[DIB_IMG_ORDER + o];
  a.fb = factors[3 * s];
  a.fc = factors[3 * s + 1];
  a.fs = factors[3 * s + 2];
  return a;
}

// cv2's linear source index and 11-bit weights for destination index d along an axis of n source pixels:
// f = (float)((d + 0.5) scale - 0.5), s = floor(f), f -= s, both borders clamp with f = 0, a = rint_even(w 2048).
__device__ __forceinline__ void axis_coeff(int d, int n, double scale, int& s0, int& s1, int& a0, int& a1) {
  float f = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)d, 0.5), scale), 0.5));
  int sx = (int)floorf(f);
  f = __fsub_rn(f, (float)sx);
  if (sx < 0) { sx = 0; f = 0.f; }
  if (sx >= n - 1) { sx = n - 1; f = 0.f; }
  a0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, f), 2048.f));
  a1 = __float2int_rn(__fmul_rn(f, 2048.f));
  s0 = sx;
  s1 = min(sx + 1, n - 1);
}

// One resized pixel: horizontal int rows S[sx] a0 + S[sx+1] a1, then OpenCV's SIMD vertical step
// sat_u8((((r0 >> 4) b0) >> 16) + (((r1 >> 4) b1) >> 16) + 2) >> 2).
__device__ __forceinline__ Rgb resize_px(const uint8_t* row0, const uint8_t* row1, int x0, int x1, int a0, int a1,
                                         int b0, int b1) {
  int o[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int h0 = (int)row0[x0 + c] * a0 + (int)row0[x1 + c] * a1;
    const int h1 = (int)row1[x0 + c] * a0 + (int)row1[x1 + c] * a1;
    o[c] = clip8(((((h0 >> 4) * b0) >> 16) + (((h1 >> 4) * b1) >> 16) + 2) >> 2);
  }
  return Rgb{o[0], o[1], o[2]};
}

// The sample's colour steps in order; with kUpToContrast, stop before the contrast step (its input is what pass 1
// sums).  contrast_grey is int(mean(L) + 0.5) of the contrast step's input.
template <bool kUpToContrast>
__device__ __forceinline__ Rgb jitter_chain(Rgb c, const Sample& a, int contrast_grey) {
#pragma unroll
  for (int o = 0; o < 4; ++o) {
    const int op = a.order[o];
    if (op == kContrast) {
      if (kUpToContrast) break;
      c = blend3(Rgb{contrast_grey, contrast_grey, contrast_grey}, c, a.fc);
    } else if (op == kBrightness) {
      c = blend3(Rgb{0, 0, 0}, c, a.fb);
    } else if (op == kSaturation) {
      const int l = luma(c);
      c = blend3(Rgb{l, l, l}, c, a.fs);
    } else {
      c = hue_shift(c, a.shift);
    }
  }
  return c;
}

template <typename OutT>
__device__ __forceinline__ OutT to_out(int v);
template <>
__device__ __forceinline__ float to_out<float>(int v) { return (float)v; }
template <>
__device__ __forceinline__ uint8_t to_out<uint8_t>(int v) { return (uint8_t)v; }

// grid (ceil(W / 32), ceil(H / 32), S), block (32, 8); each thread takes output column xo and rows y + 8 k.
template <bool kWrite, typename OutT>
__device__ __forceinline__ void image_tile(const uint8_t* __restrict__ src, const int64_t* __restrict__ offsets,
                                           const int32_t* __restrict__ params, const float* __restrict__ factors,
                                           int H, int W, uint32_t* __restrict__ partial, OutT* __restrict__ out) {
  const int s = blockIdx.z;
  const Sample a = load_sample(src, offsets, params, factors, s);
  if (!kWrite && !a.jitter) return;
  const int tiles = gridDim.x * gridDim.y, tile = blockIdx.y * gridDim.x + blockIdx.x;
  const int lane = threadIdx.x, wy = threadIdx.y;
  __shared__ unsigned long long s_red[kTileRows];
  int grey = 0;
  if (kWrite && a.jitter) {
    if (wy == 0) {
      unsigned long long t = 0;
      for (int i = lane; i < tiles; i += 32) t += partial[(size_t)s * tiles + i];
#pragma unroll
      for (int off = 16; off; off >>= 1) t += __shfl_xor_sync(0xffffffffu, t, off);
      if (lane == 0) s_red[0] = t;
    }
    __syncthreads();
    grey = (int)__dadd_rn(__ddiv_rn((double)s_red[0], (double)H * (double)W), 0.5);
  }
  const int xo = blockIdx.x * kTileW + lane;
  uint32_t lsum = 0;
  if (xo < W) {
    const int x = a.flip ? W - 1 - xo : xo;
    int sx0, sx1, a0, a1;
    axis_coeff(a.dx + x, a.w, __ddiv_rn(1.0, __ddiv_rn((double)a.dw, (double)a.w)), sx0, sx1, a0, a1);
    sx0 *= 3;
    sx1 *= 3;
    const double yscale = __ddiv_rn(1.0, __ddiv_rn((double)a.dh, (double)a.rows));
    const size_t w3 = (size_t)a.w * 3, plane = (size_t)H * W;
#pragma unroll
    for (int k = 0; k < kRowsPerThread; ++k) {
      const int y = blockIdx.y * kTileH + wy + kTileRows * k;
      if (y >= H) break;
      int sy0, sy1, b0, b1;
      axis_coeff(a.dy + y, a.rows, yscale, sy0, sy1, b0, b1);
      Rgb c = resize_px(a.view + sy0 * w3, a.view + sy1 * w3, sx0, sx1, a0, a1, b0, b1);
      if (kWrite) {
        if (a.jitter) c = jitter_chain<false>(c, a, grey);
        OutT* o = out + (size_t)s * 3 * plane + (size_t)y * W + xo;
        o[0] = to_out<OutT>(c.r);
        o[plane] = to_out<OutT>(c.g);
        o[2 * plane] = to_out<OutT>(c.b);
      } else {
        lsum += (uint32_t)luma(jitter_chain<true>(c, a, 0));
      }
    }
  }
  if (!kWrite) {
#pragma unroll
    for (int off = 16; off; off >>= 1) lsum += __shfl_xor_sync(0xffffffffu, lsum, off);
    if (lane == 0) s_red[wy] = lsum;
    __syncthreads();
    if (wy == 0 && lane == 0) {
      uint32_t t = 0;
      for (int i = 0; i < kTileRows; ++i) t += (uint32_t)s_red[i];
      partial[(size_t)s * tiles + tile] = t;
    }
  }
}

__global__ void __launch_bounds__(kTileW * kTileRows)
    image_luma_partials_kernel(const uint8_t* __restrict__ src, const int64_t* __restrict__ offsets,
                               const int32_t* __restrict__ params, const float* __restrict__ factors, int H, int W,
                               uint32_t* __restrict__ partial) {
  image_tile<false, float>(src, offsets, params, factors, H, W, partial, nullptr);
}

template <typename OutT>
__global__ void __launch_bounds__(kTileW * kTileRows)
    image_assemble_kernel(const uint8_t* __restrict__ src, const int64_t* __restrict__ offsets,
                          const int32_t* __restrict__ params, const float* __restrict__ factors, int H, int W,
                          const uint32_t* __restrict__ partial, OutT* __restrict__ out) {
  image_tile<true, OutT>(src, offsets, params, factors, H, W, const_cast<uint32_t*>(partial), out);
}

template <typename OutT>
int assemble(const uint8_t* src, size_t src_bytes, const int64_t* offsets, const int32_t* params,
             const float* factors, int S, int H, int W, OutT* out, void* workspace, size_t workspace_bytes,
             cudaStream_t stream) {
  DIB_REQUIRE(S >= 0 && S <= kMaxS, "S must be in [0, %d] (got %d)", kMaxS, S);
  DIB_REQUIRE(H >= 1 && W >= 1 && H <= kMaxSide && W <= kMaxSide, "img_H, img_W must be in [1, %d] (got %d, %d)",
              kMaxSide, H, W);
  if (S == 0) return 0;
  DIB_REQUIRE(src && offsets && params && factors && out && workspace, "a required pointer is null");
  const Layout L = layout(S, H, W);
  if (workspace_bytes < L.total) {
    set_error("image_assemble: workspace is %zu bytes, %zu needed", workspace_bytes, L.total);
    return DIB_ENOMEM;
  }
  bool any_jitter = false;
  for (int s = 0; s < S; ++s) {
    const int32_t* p = params + (size_t)s * DIB_IMAGE_PARAMS;
    const int h = p[DIB_IMG_H], w = p[DIB_IMG_W], row0 = p[DIB_IMG_ROW0], rows = p[DIB_IMG_ROWS];
    const int dh = p[DIB_IMG_DH], dw = p[DIB_IMG_DW], dy = p[DIB_IMG_DY], dx = p[DIB_IMG_DX];
    DIB_REQUIRE(h >= 1 && w >= 1 && h <= kMaxSide && w <= kMaxSide, "sample %d: frame %d x %d is not in [1, %d]^2",
                s, h, w, kMaxSide);
    DIB_REQUIRE(offsets[s] >= 0 && (size_t)offsets[s] + (size_t)h * w * 3 <= src_bytes,
                "sample %d: frame bytes [%lld, +%zu) are outside the %zu-byte buffer", s, (long long)offsets[s],
                (size_t)h * w * 3, src_bytes);
    DIB_REQUIRE(row0 >= 0 && rows >= 1 && row0 + rows <= h, "sample %d: rows [%d, %d) are not inside the %d-row frame",
                s, row0, row0 + rows, h);
    DIB_REQUIRE(dh >= 1 && dh <= rows && dw >= 1 && dw <= w,
                "sample %d: resize %d x %d -> %d x %d is not a downscale", s, rows, w, dh, dw);
    DIB_REQUIRE(dh >= H && dw >= W, "sample %d: the resized %d x %d image is smaller than the %d x %d output", s, dh,
                dw, H, W);
    DIB_REQUIRE(dy >= 0 && dy <= dh - H && dx >= 0 && dx <= dw - W,
                "sample %d: crop offset (%d, %d) is outside [0, %d] x [0, %d]", s, dy, dx, dh - H, dw - W);
    DIB_REQUIRE((p[DIB_IMG_FLIP] == 0 || p[DIB_IMG_FLIP] == 1) && (p[DIB_IMG_JITTER] == 0 || p[DIB_IMG_JITTER] == 1),
                "sample %d: flip and jitter must be 0 or 1", s);
    if (p[DIB_IMG_JITTER]) {
      int seen = 0;
      for (int o = 0; o < 4; ++o) {
        const int op = p[DIB_IMG_ORDER + o];
        DIB_REQUIRE(op >= 0 && op < 4 && !(seen >> op & 1), "sample %d: order must be a permutation of 0..3", s);
        seen |= 1 << op;
      }
      DIB_REQUIRE(p[DIB_IMG_SHIFT] >= 0 && p[DIB_IMG_SHIFT] <= 255, "sample %d: hue shift must be in [0, 255]", s);
      for (int j = 0; j < 3; ++j)
        DIB_REQUIRE(std::isfinite(factors[3 * s + j]), "sample %d: colour factors must be finite", s);
      any_jitter = true;
    }
  }
  // One upload of the per-sample parameters (pageable memory is staged before cudaMemcpyAsync returns).
  std::vector<unsigned char> head(L.head, 0);
  memcpy(head.data() + L.params, params, (size_t)S * DIB_IMAGE_PARAMS * sizeof(int32_t));
  memcpy(head.data() + L.offsets, offsets, (size_t)S * sizeof(int64_t));
  memcpy(head.data() + L.factors, factors, (size_t)S * 3 * sizeof(float));
  unsigned char* ws = (unsigned char*)workspace;
  DIB_CHECK_CUDA(cudaMemcpyAsync(ws, head.data(), L.head, cudaMemcpyHostToDevice, stream));
  const int32_t* d_params = (const int32_t*)(ws + L.params);
  const int64_t* d_off = (const int64_t*)(ws + L.offsets);
  const float* d_fac = (const float*)(ws + L.factors);
  uint32_t* d_part = (uint32_t*)(ws + L.partial);
  const dim3 grid((W + kTileW - 1) / kTileW, (H + kTileH - 1) / kTileH, S), block(kTileW, kTileRows);
  if (any_jitter) {
    image_luma_partials_kernel<<<grid, block, 0, stream>>>(src, d_off, d_params, d_fac, H, W, d_part);
    DIB_CHECK_CUDA(cudaGetLastError());
  }
  image_assemble_kernel<OutT><<<grid, block, 0, stream>>>(src, d_off, d_params, d_fac, H, W, d_part, out);
  DIB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace img
}  // namespace dib

extern "C" {

size_t image_assemble_workspace_bytes(int S, int img_H, int img_W) {
  if (S < 0 || S > dib::img::kMaxS || img_H < 1 || img_W < 1 || img_H > dib::img::kMaxSide ||
      img_W > dib::img::kMaxSide)
    return 0;
  return dib::img::layout(S, img_H, img_W).total;
}

int image_assemble_f32(const uint8_t* src, size_t src_bytes, const int64_t* offsets, const int32_t* params,
                       const float* factors, int S, int img_H, int img_W, float* img_out, void* workspace,
                       size_t workspace_bytes, dib_stream_t stream) {
  return dib::img::assemble<float>(src, src_bytes, offsets, params, factors, S, img_H, img_W, img_out, workspace,
                                   workspace_bytes, (cudaStream_t)stream);
}

int image_assemble_u8(const uint8_t* src, size_t src_bytes, const int64_t* offsets, const int32_t* params,
                      const float* factors, int S, int img_H, int img_W, uint8_t* img_out, void* workspace,
                      size_t workspace_bytes, dib_stream_t stream) {
  return dib::img::assemble<uint8_t>(src, src_bytes, offsets, params, factors, S, img_H, img_W, img_out, workspace,
                                     workspace_bytes, (cudaStream_t)stream);
}

}  // extern "C"
