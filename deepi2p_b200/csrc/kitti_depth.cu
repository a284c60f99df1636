// KITTI camera-frame scan records and LiDAR depth maps (data/kitti/kitti_pc_bin_to_npy_in_img_frame.py, the body of
// its per-scan, per-camera loop) for T (scan, camera) pairs at once, all of one image size.  DESIGN.md 4.33 states
// the contract.
//
//   project_min:  one thread per (pair, point): the point's pixel and float32 sub-pixel distance; an atomic minimum
//                 of the distance bits per pixel (plane 1 of the output).
//   project_pick: the same projection again; per pixel one atomic maximum of a code that ranks, first, the points
//                 with d < m (fp64 d against the float32 minimum m) by largest index and, after them, the points with
//                 float32(d) = m by smallest index (plane 0 of the output).  That is the winner of the reference's
//                 in-order loop, which replaces the stored point when d < (double) stored.
//   columns:      one thread per (pair, column): the winner's float32 Z into plane 0 of each filled pixel, and the
//                 nearest filled row of every pixel (the lower row on ties) into the workspace.
//   rows:         one thread per (pair, row): the lower envelope of the column parabolas (c - q)^2 + (r - row_q)^2 in
//                 int32, the smaller column winning ties; every empty pixel takes its nearest filled pixel's depth and
//                 float32(sqrt(d2)), sqrt in fp64.  An image with no filled pixel gets scipy's index (-1, 0): depth
//                 0 and distance sqrt((r + 1)^2 + c^2).
//   records:      the fp64 voxel centres moved by Pc, intensity, and normals mapped NWU -> camera, as float32 [7, M].
//
// Every sum is evaluated in the association written below; the file is compiled with --fmad=false so that
// oracle_kitti_depth/ restates it bit for bit.
#include <math.h>

#include "common.cuh"

namespace dib {
namespace {

constexpr int kThreads = 256;
constexpr int kMaxT = 65535;
constexpr int kMaxSide = 32767;         // columns and rows fit the int16 workspace and the packed envelope
constexpr int kRowsPerBlock = 32;
constexpr int32_t kHi = 1 << 30;        // pick codes: kHi + i for d < m, kHi - 1 - i for float32(d) = m
constexpr uint32_t kEmpty = 0xFFFFFFFFu;

struct Hit {
  int pix;                              // -1: the point does not count
  double d;
};

// X, Y, Z = Pc (x, y, z, 1) as ((Pc0 x + Pc1 y) + Pc2 z) + Pc3; u, v, w = K (X, Y, Z) as (K0 X + K1 Y) + K2 Z.
// The point counts when Z > 0.1, w != 0 and rint(u / w), rint(v / w) (halves to even, as Python's round) land in
// the image.
__device__ __forceinline__ Hit project(const double* P, const float* K, double x, double y, double z, int H, int W) {
  Hit h{-1, 0.0};
  const double X = ((P[0] * x + P[1] * y) + P[2] * z) + P[3];
  const double Y = ((P[4] * x + P[5] * y) + P[6] * z) + P[7];
  const double Z = ((P[8] * x + P[9] * y) + P[10] * z) + P[11];
  if (!(Z > 0.1)) return h;
  const double u = ((double)K[0] * X + (double)K[1] * Y) + (double)K[2] * Z;
  const double v = ((double)K[3] * X + (double)K[4] * Y) + (double)K[5] * Z;
  const double w = ((double)K[6] * X + (double)K[7] * Y) + (double)K[8] * Z;
  if (w == 0.0) return h;
  const double px = u / w, py = v / w;
  const double rx = rint(px), ry = rint(py);
  if (!(rx >= 0.0 && rx <= (double)(W - 1) && ry >= 0.0 && ry <= (double)(H - 1))) return h;
  const double dx = px - rx, dy = py - ry;
  h.pix = (int)ry * W + (int)rx;
  h.d = sqrt(dx * dx + dy * dy);
  return h;
}

__device__ __forceinline__ double camera_z(const double* P, const float* xyz, int64_t n_stride, int i) {
  return ((P[8] * (double)xyz[i] + P[9] * (double)xyz[n_stride + i]) + P[10] * (double)xyz[2 * n_stride + i]) + P[11];
}

struct PairArgs {
  const float* xyz;
  int64_t n_stride;
  const int32_t* n_pts;
  const double* Pc;                     // [T][16]
  const float* K;                       // [T][9]
  int C;                                // cameras per scan: pair t reads scan t / C
  int H, W;
};

__global__ void __launch_bounds__(kThreads) project_min_kernel(PairArgs a, float* __restrict__ out) {
  const int t = blockIdx.y;
  const int s = t / a.C;
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= a.n_pts[s]) return;
  const float* p = a.xyz + (int64_t)s * 3 * a.n_stride;
  const Hit h = project(a.Pc + 16 * (int64_t)t, a.K + 9 * (int64_t)t, p[i], p[a.n_stride + i], p[2 * a.n_stride + i],
                        a.H, a.W);
  if (h.pix < 0) return;
  const int64_t plane = (int64_t)a.H * a.W;
  uint32_t* key = reinterpret_cast<uint32_t*>(out + (2 * t + 1) * plane);
  atomicMin(key + h.pix, __float_as_uint((float)h.d));
}

__global__ void __launch_bounds__(kThreads) project_pick_kernel(PairArgs a, float* __restrict__ out) {
  const int t = blockIdx.y;
  const int s = t / a.C;
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= a.n_pts[s]) return;
  const float* p = a.xyz + (int64_t)s * 3 * a.n_stride;
  const Hit h = project(a.Pc + 16 * (int64_t)t, a.K + 9 * (int64_t)t, p[i], p[a.n_stride + i], p[2 * a.n_stride + i],
                        a.H, a.W);
  if (h.pix < 0) return;
  const int64_t plane = (int64_t)a.H * a.W;
  const float m = __uint_as_float(reinterpret_cast<const uint32_t*>(out + (2 * t + 1) * plane)[h.pix]);
  int32_t code;
  if (h.d < (double)m)
    code = kHi + i;
  else if ((float)h.d == m)
    code = kHi - 1 - i;
  else
    return;
  atomicMax(reinterpret_cast<int32_t*>(out + 2 * t * plane) + h.pix, code);
}

__global__ void __launch_bounds__(kThreads) columns_kernel(PairArgs a, float* __restrict__ out,
                                                           int16_t* __restrict__ near_row) {
  const int t = blockIdx.y;
  const int c = blockIdx.x * kThreads + threadIdx.x;
  if (c >= a.W) return;
  const int W = a.W, H = a.H;
  const int64_t plane = (int64_t)H * W;
  float* depth = out + 2 * t * plane;
  const uint32_t* key = reinterpret_cast<const uint32_t*>(out + (2 * t + 1) * plane);
  int16_t* nr = near_row + t * plane;
  const double* P = a.Pc + 16 * (int64_t)t;
  const float* xyz = a.xyz + (int64_t)(t / a.C) * 3 * a.n_stride;
  const int n = a.n_pts[t / a.C];
  int above = -1;
  for (int r = 0; r < H; ++r) {
    const int64_t q = (int64_t)r * W + c;
    if (key[q] != kEmpty) {
      const int32_t code = reinterpret_cast<const int32_t*>(depth)[q];
      const int i = code >= kHi ? code - kHi : kHi - 1 - code;
      // A code outside the scan means out[] did not come from kitti_depth_project_f32: NaN, never a stray read.
      depth[q] = i >= 0 && i < n ? (float)camera_z(P, xyz, a.n_stride, i) : NAN;
      above = r;
    }
    nr[q] = (int16_t)above;
  }
  int below = -1;
  for (int r = H - 1; r >= 0; --r) {
    const int64_t q = (int64_t)r * W + c;
    const int up = nr[q];
    if (up == r) {
      below = r;
      continue;
    }
    if (below >= 0 && (up < 0 || below - r < r - up)) nr[q] = (int16_t)below;
  }
}

// The envelope entry: column (low 16 bits) and the first column where it is the nearest (high 16 bits).
__device__ __forceinline__ uint32_t pack(int col, int start) { return (uint32_t)col | ((uint32_t)start << 16); }

__global__ void rows_kernel(const int16_t* __restrict__ near_row, int T, int H, int W, float* __restrict__ out) {
  extern __shared__ uint32_t s_env[];
  const int R = blockDim.x;
  const int64_t row = (int64_t)blockIdx.x * R + threadIdx.x;
  if (row >= (int64_t)T * H) return;
  const int t = (int)(row / H), r = (int)(row % H);
  const int64_t plane = (int64_t)H * W;
  const int16_t* nr = near_row + t * plane + (int64_t)r * W;
  float* depth = out + 2 * t * plane;
  float* dist = depth + plane;
  uint32_t* env = s_env + threadIdx.x;                    // entry k at env[k * R]: lanes never share a bank
  int n = 0;
  for (int p = 0; p < W; ++p) {
    const int rp = nr[p];
    if (rp < 0) continue;
    const int fp = (r - rp) * (r - rp);
    while (n > 0) {                                       // pop while p strictly beats the top where the top starts
      const uint32_t e = env[(n - 1) * R];
      const int q = (int)(e & 0xFFFFu), z = (int)(e >> 16);
      const int rq = nr[q];
      const int fq = (r - rq) * (r - rq);
      if ((z - p) * (z - p) + fp < (z - q) * (z - q) + fq)
        --n;
      else
        break;
    }
    if (n == 0) {
      env[0] = pack(p, 0);
      n = 1;
      continue;
    }
    // The first column where p strictly beats the top q: c > num / (2 (p - q)), num >= 0 since p does not beat q at
    // q's start (>= 0).
    const int q = (int)(env[(n - 1) * R] & 0xFFFFu);
    const int rq = nr[q];
    const int num = ((r - rp) * (r - rp) + p * p) - ((r - rq) * (r - rq) + q * q);
    const int start = num / (2 * (p - q)) + 1;
    if (start < W) env[n++ * R] = pack(p, start);
  }
  float* drow = depth + (int64_t)r * W;
  float* trow = dist + (int64_t)r * W;
  if (n == 0) {                                           // no filled pixel in the image: scipy's index (-1, 0)
    for (int c = 0; c < W; ++c) {
      drow[c] = 0.0f;
      trow[c] = (float)sqrt((double)((r + 1) * (r + 1) + c * c));
    }
    return;
  }
  int k = 0;
  for (int c = 0; c < W; ++c) {
    while (k + 1 < n && (int)(env[(k + 1) * R] >> 16) <= c) ++k;
    const int q = (int)(env[k * R] & 0xFFFFu);
    const int rq = nr[q];
    const int d2 = (r - rq) * (r - rq) + (c - q) * (c - q);
    if (d2 == 0) continue;                                // a filled pixel keeps its depth and distance
    drow[c] = depth[(int64_t)rq * W + q];
    trow[c] = (float)sqrt((double)d2);
  }
}

__global__ void __launch_bounds__(kThreads) records_kernel(const double* __restrict__ xyz,
                                                           const double* __restrict__ nrm,
                                                           const float* __restrict__ inten,
                                                           const int32_t* __restrict__ m_pts, int64_t m_stride,
                                                           const double* __restrict__ Pc, int C,
                                                           float* __restrict__ out) {
  const int t = blockIdx.y;
  const int s = t / C;
  const int j = blockIdx.x * kThreads + threadIdx.x;
  if (j >= m_stride) return;
  float* o = out + (int64_t)t * 7 * m_stride + j;
  if (j >= m_pts[s]) {
    for (int q = 0; q < 7; ++q) o[q * m_stride] = 0.0f;
    return;
  }
  const double* p = xyz + (int64_t)s * 3 * m_stride;
  const double* nv = nrm + (int64_t)s * 3 * m_stride;
  const double* P = Pc + 16 * (int64_t)t;
  const double x = p[j], y = p[m_stride + j], z = p[2 * m_stride + j];
  for (int a = 0; a < 3; ++a)
    o[a * m_stride] = (float)(((P[4 * a] * x + P[4 * a + 1] * y) + P[4 * a + 2] * z) + P[4 * a + 3]);
  o[3 * m_stride] = inten[(int64_t)s * m_stride + j];
  o[4 * m_stride] = (float)(-nv[m_stride + j]);         // coordinate_NWU_to_cam: x <- -y, y <- -z, z <- x
  o[5 * m_stride] = (float)(-nv[2 * m_stride + j]);
  o[6 * m_stride] = (float)nv[j];
}

int rows_per_block(int W, int* R) {
  int dev = 0, optin = 0;
  DIB_CHECK_CUDA(cudaGetDevice(&dev));
  DIB_CHECK_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  const int r = optin / (W * (int)sizeof(uint32_t));
  *R = r < kRowsPerBlock ? r : kRowsPerBlock;
  DIB_REQUIRE(*R >= 1, "W = %d needs more shared memory per row than the device has", W);
  return 0;
}

// The envelope's squared distances and intercept numerators stay below (H-1)^2 + (W-1)^2, in int32.
bool valid_size(int H, int W) {
  return H >= 1 && H <= kMaxSide && W >= 1 && W <= kMaxSide &&
         (int64_t)(H - 1) * (H - 1) + (int64_t)(W - 1) * (W - 1) < ((int64_t)1 << 31);
}

bool valid_pairs(int S, int T) { return S >= 1 && T >= S && T <= kMaxT && T % S == 0; }

}  // namespace
}  // namespace dib

using namespace dib;

extern "C" {

size_t kitti_depth_fill_workspace_bytes(int T, int H, int W) {
  if (T < 0 || H < 0 || W < 0) return 0;
  return (size_t)T * H * W * sizeof(int16_t);
}

int kitti_depth_project_f32(const float* xyz, int64_t n_stride, const int32_t* n_pts, int S, const double* Pc,
                            const float* K, int T, int H, int W, float* out, dib_stream_t stream) {
  DIB_REQUIRE(valid_pairs(S, T), "T must be a positive multiple of S = %d, at most %d (got %d)", S, kMaxT, T);
  DIB_REQUIRE(valid_size(H, W), "H and W must be in [1, %d] with (H-1)^2 + (W-1)^2 < 2^31 (got %d x %d)", kMaxSide,
              H, W);
  DIB_REQUIRE(n_stride >= 1 && n_stride < kHi, "n_stride must be in [1, 2^30) (got %lld)", (long long)n_stride);
  DIB_REQUIRE(xyz && n_pts && Pc && K && out, "a required pointer is null");
  const PairArgs a{xyz, n_stride, n_pts, Pc, K, T / S, H, W};
  cudaStream_t cs = (cudaStream_t)stream;
  DIB_CHECK_CUDA(cudaMemsetAsync(out, 0xFF, (size_t)T * 2 * H * W * sizeof(float), cs));   // keys empty, codes -1
  const dim3 grid((unsigned)((n_stride + kThreads - 1) / kThreads), (unsigned)T);
  project_min_kernel<<<grid, kThreads, 0, cs>>>(a, out);
  DIB_CHECK_CUDA(cudaGetLastError());
  project_pick_kernel<<<grid, kThreads, 0, cs>>>(a, out);
  DIB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int kitti_depth_fill_f32(const float* xyz, int64_t n_stride, const int32_t* n_pts, int S, const double* Pc,
                         const float* K, int T, int H, int W, float* out, void* workspace, size_t workspace_bytes,
                         dib_stream_t stream) {
  DIB_REQUIRE(valid_pairs(S, T), "T must be a positive multiple of S = %d, at most %d (got %d)", S, kMaxT, T);
  DIB_REQUIRE(valid_size(H, W), "H and W must be in [1, %d] with (H-1)^2 + (W-1)^2 < 2^31 (got %d x %d)", kMaxSide,
              H, W);
  DIB_REQUIRE(n_stride >= 1 && n_stride < kHi, "n_stride must be in [1, 2^30) (got %lld)", (long long)n_stride);
  DIB_REQUIRE(xyz && n_pts && Pc && K && out && workspace, "a required pointer is null");
  const size_t need = kitti_depth_fill_workspace_bytes(T, H, W);
  if (workspace_bytes < need) {
    set_error("kitti_depth_fill: workspace is %zu bytes, %zu needed", workspace_bytes, need);
    return DIB_ENOMEM;
  }
  int R = 0;
  const int rc = rows_per_block(W, &R);
  if (rc) return rc;
  const PairArgs a{xyz, n_stride, n_pts, Pc, K, T / S, H, W};
  int16_t* near_row = (int16_t*)workspace;
  cudaStream_t cs = (cudaStream_t)stream;
  columns_kernel<<<dim3((unsigned)((W + kThreads - 1) / kThreads), (unsigned)T), kThreads, 0, cs>>>(a, out, near_row);
  DIB_CHECK_CUDA(cudaGetLastError());
  const int smem = R * W * (int)sizeof(uint32_t);
  DIB_CHECK_CUDA(cudaFuncSetAttribute(rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const int64_t rows = (int64_t)T * H;
  rows_kernel<<<(unsigned)((rows + R - 1) / R), R, smem, cs>>>(near_row, T, H, W, out);
  DIB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int kitti_depth_records_f32(const double* xyz, const double* nrm, const float* intensity, const int32_t* m_pts,
                            int64_t m_stride, int S, const double* Pc, int T, float* out, dib_stream_t stream) {
  DIB_REQUIRE(valid_pairs(S, T), "T must be a positive multiple of S = %d, at most %d (got %d)", S, kMaxT, T);
  DIB_REQUIRE(m_stride >= 1 && m_stride < INT32_MAX, "m_stride must be in [1, 2^31) (got %lld)", (long long)m_stride);
  DIB_REQUIRE(xyz && nrm && intensity && m_pts && Pc && out, "a required pointer is null");
  cudaStream_t cs = (cudaStream_t)stream;
  records_kernel<<<dim3((unsigned)((m_stride + kThreads - 1) / kThreads), (unsigned)T), kThreads, 0, cs>>>(
      xyz, nrm, intensity, m_pts, m_stride, Pc, T / S, out);
  DIB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
