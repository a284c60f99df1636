// KITTI accumulated-frame records (data/kitti/frame_accumulation.py accumulate_sequence, the body of its per-frame
// loop) for B output frames at once, from a ragged scan store.  DESIGN.md 4.29 states the contract.
//
//   count:   one block per (output, stride record) pair counts the record's points outside the ego box and their
//            largest intensity; one thread per output then lays its pairs out in window order and takes the
//            output's maximum.
//   scatter: one block per pair writes P (x, y, z, 1) and P (nx, ny, nz, 1) in fp64 (the reference moves the normals
//            with the translation too) and float32 intensity / max, in window order, then point order (a block-wide
//            order-preserving scan of the ego flags).
//   finish:  after voxel_downsample_batch_f64, one block per output keeps the voxels with sqrt(x x + y y) < radius
//            in order and rounds (x, y, z, colour * max, nx, ny, nz) to a float32 [7, M] record.
//
// Every sum is evaluated in the association written below; the file is compiled with --fmad=false so that
// oracle_kitti_build/ restates it bit for bit.
#include <math.h>

#include "common.cuh"

namespace dib {
namespace {

constexpr int kMaxB = 65535;
constexpr int kScanThreads = 256;

struct Box4 {
  float x_lo, x_hi, y_lo, y_hi;
};

// The reference's inside_mask: both comparisons strict, in float32 against the float32-rounded borders.
__device__ __forceinline__ bool outside_box(float x, float y, const Box4& b) {
  return !((x < b.x_hi && x > b.x_lo) && (y < b.y_hi && y > b.y_lo));
}

// An order-preserving block scan step: returns the flagged thread's index among this chunk's flagged threads and
// sets *total to their number.  Every thread of the block must call it.
__device__ __forceinline__ int block_rank(bool f, int* s_warp, int* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const unsigned bal = __ballot_sync(0xffffffffu, f);
  if (lane == 0) s_warp[w] = __popc(bal);
  __syncthreads();
  int before = 0, t = 0;
  for (int q = 0; q < kScanThreads / 32; ++q) {
    before += q < w ? s_warp[q] : 0;
    t += s_warp[q];
  }
  __syncthreads();
  *total = t;
  return before + __popc(bal & ((1u << lane) - 1u));
}

__global__ void __launch_bounds__(kScanThreads) count_kernel(const float* __restrict__ planes, int64_t ps,
                                                             const int64_t* __restrict__ offset,
                                                             const int32_t* __restrict__ npts, Box4 box,
                                                             int32_t* __restrict__ pcount,
                                                             float* __restrict__ pmax) {
  const int t = blockIdx.x;
  const float* x = planes + offset[t];
  const float* y = x + ps;
  const float* it = x + 3 * ps;
  const int n = npts[t];
  int cnt = 0;
  float mx = -INFINITY;
  for (int i = threadIdx.x; i < n; i += kScanThreads)
    if (outside_box(x[i], y[i], box)) {
      ++cnt;
      mx = fmaxf(mx, it[i]);
    }
  __shared__ int s_cnt[kScanThreads / 32];
  __shared__ float s_max[kScanThreads / 32];
  for (int off = 16; off; off >>= 1) {
    cnt += __shfl_down_sync(0xffffffffu, cnt, off);
    mx = fmaxf(mx, __shfl_down_sync(0xffffffffu, mx, off));
  }
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) {
    s_cnt[w] = cnt;
    s_max[w] = mx;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int q = 1; q < kScanThreads / 32; ++q) {
      cnt += s_cnt[q];
      mx = fmaxf(mx, s_max[q]);
    }
    pcount[t] = cnt;
    pmax[t] = mx;
  }
}

__global__ void layout_kernel(const int32_t* __restrict__ first, int B, const int32_t* __restrict__ pcount,
                              const float* __restrict__ pmax, int64_t* __restrict__ pos, int64_t* __restrict__ n_pts,
                              float* __restrict__ omax) {
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= B) return;
  int64_t acc = 0;
  float mx = -INFINITY;
  for (int t = first[o]; t < first[o + 1]; ++t) {
    pos[t] = acc;
    acc += pcount[t];
    mx = fmaxf(mx, pmax[t]);
  }
  n_pts[o] = acc;
  omax[o] = mx;
}

__device__ __forceinline__ double affine_row(const double* P, int r, double x, double y, double z) {
  return ((P[4 * r] * x + P[4 * r + 1] * y) + P[4 * r + 2] * z) + P[4 * r + 3];
}

__global__ void __launch_bounds__(kScanThreads) scatter_kernel(
    const float* __restrict__ planes, int64_t ps, const int64_t* __restrict__ offset, const int32_t* __restrict__ npts,
    const int32_t* __restrict__ pair_out, const double* __restrict__ P_all, Box4 box, const int64_t* __restrict__ pos,
    const float* __restrict__ omax, int64_t n_stride, double* __restrict__ xyz_out, double* __restrict__ attr_out) {
  const int t = blockIdx.x;
  const int o = pair_out[t];
  const float* x = planes + offset[t];
  const int n = npts[t];
  double P[12];
  for (int q = 0; q < 12; ++q) P[q] = P_all[16 * (int64_t)t + q];
  const float mx = omax[o];
  double* ox = xyz_out + (int64_t)o * 3 * n_stride;
  double* oa = attr_out + (int64_t)o * 4 * n_stride;
  __shared__ int s_warp[kScanThreads / 32];
  int64_t base = pos[t];
  for (int c = 0; c < n; c += kScanThreads) {
    const int i = c + threadIdx.x;
    const bool f = i < n && outside_box(x[i], x[ps + i], box);
    int total;
    const int r = block_rank(f, s_warp, &total);
    if (f) {
      const int64_t d = base + r;
      const double px = x[i], py = x[ps + i], pz = x[2 * ps + i];
      const double nx = x[4 * ps + i], ny = x[5 * ps + i], nz = x[6 * ps + i];
      for (int a = 0; a < 3; ++a) {
        ox[a * n_stride + d] = affine_row(P, a, px, py, pz);
        oa[(a + 1) * n_stride + d] = affine_row(P, a, nx, ny, nz);
      }
      oa[d] = (double)(x[3 * ps + i] / mx);
    }
    base += total;
  }
}

__global__ void __launch_bounds__(kScanThreads) finish_kernel(const double* __restrict__ xyz,
                                                              const double* __restrict__ attr,
                                                              const int32_t* __restrict__ m_pts,
                                                              const float* __restrict__ omax, double radius,
                                                              int64_t n_stride, int64_t m_stride,
                                                              float* __restrict__ out, int32_t* __restrict__ count) {
  const int o = blockIdx.x;
  const int m = m_pts[o];
  const double* p = xyz + (int64_t)o * 3 * n_stride;
  const double* a = attr + (int64_t)o * 4 * n_stride;
  float* os = out + (int64_t)o * 7 * m_stride;
  const double mx = (double)omax[o];
  __shared__ int s_warp[kScanThreads / 32];
  int64_t base = 0;
  for (int c = 0; c < m; c += kScanThreads) {
    const int j = c + threadIdx.x;
    double px = 0.0, py = 0.0;
    if (j < m) {
      px = p[j];
      py = p[n_stride + j];
    }
    const bool f = j < m && sqrt(px * px + py * py) < radius;
    int total;
    const int r = block_rank(f, s_warp, &total);
    if (f) {
      const int64_t d = base + r;
      os[d] = (float)px;
      os[m_stride + d] = (float)py;
      os[2 * m_stride + d] = (float)p[2 * n_stride + j];
      os[3 * m_stride + d] = (float)(a[j] * mx);
      for (int q = 1; q < 4; ++q) os[(3 + q) * m_stride + d] = (float)a[q * n_stride + j];
    }
    base += total;
  }
  for (int64_t j = base + threadIdx.x; j < m_stride; j += kScanThreads)
    for (int q = 0; q < 7; ++q) os[q * m_stride + j] = 0.0f;
  if (threadIdx.x == 0) count[o] = (int32_t)base;
}

bool valid_box(const float* b) {
  return b && isfinite(b[0]) && isfinite(b[1]) && isfinite(b[2]) && isfinite(b[3]) && b[0] <= b[1] && b[2] <= b[3];
}

}  // namespace
}  // namespace dib

using namespace dib;

extern "C" {

size_t kitti_build_count_workspace_bytes(int T) {
  if (T < 0) return 0;
  return ((size_t)T * sizeof(int32_t) + 255) / 256 * 256 + (size_t)T * sizeof(float);
}

int kitti_build_count_f32(const float* planes, int64_t plane_stride, const int64_t* offset, const int32_t* npts,
                          int T, const int32_t* first, int B, const float* box, int64_t* pos, int64_t* n_pts,
                          float* omax, void* workspace, size_t workspace_bytes, dib_stream_t stream) {
  DIB_REQUIRE(B >= 0 && B <= kMaxB, "B must be in [0, %d] (got %d)", kMaxB, B);
  DIB_REQUIRE(T >= 0 && T <= INT32_MAX / 2, "T must be in [0, 2^30] (got %d)", T);
  DIB_REQUIRE(plane_stride >= 0, "plane_stride must be >= 0");
  DIB_REQUIRE(valid_box(box), "the ego box must be four finite numbers (x_lo, x_hi, y_lo, y_hi), lo <= hi");
  if (B == 0) return 0;
  DIB_REQUIRE(first && pos && n_pts && omax, "a required pointer is null");
  DIB_REQUIRE(T == 0 || (planes && offset && npts && workspace), "a required pointer is null");
  const size_t need = kitti_build_count_workspace_bytes(T);
  if (workspace_bytes < need) {
    set_error("kitti_build_count: workspace is %zu bytes, %zu needed", workspace_bytes, need);
    return DIB_ENOMEM;
  }
  int32_t* pcount = (int32_t*)workspace;
  float* pmax = (float*)((char*)workspace + ((size_t)T * sizeof(int32_t) + 255) / 256 * 256);
  const Box4 b{box[0], box[1], box[2], box[3]};
  cudaStream_t cs = (cudaStream_t)stream;
  if (T > 0) {
    count_kernel<<<T, kScanThreads, 0, cs>>>(planes, plane_stride, offset, npts, b, pcount, pmax);
    DIB_CHECK_CUDA(cudaGetLastError());
  }
  layout_kernel<<<(B + 127) / 128, 128, 0, cs>>>(first, B, pcount, pmax, pos, n_pts, omax);
  DIB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int kitti_build_scatter_f64(const float* planes, int64_t plane_stride, const int64_t* offset, const int32_t* npts,
                            const int32_t* pair_out, const double* P, int T, int B, const float* box,
                            const int64_t* pos, const float* omax, int64_t n_stride, double* xyz_out,
                            double* attr_out, dib_stream_t stream) {
  DIB_REQUIRE(B >= 0 && B <= kMaxB, "B must be in [0, %d] (got %d)", kMaxB, B);
  DIB_REQUIRE(T >= 0 && T <= INT32_MAX / 2, "T must be in [0, 2^30] (got %d)", T);
  DIB_REQUIRE(plane_stride >= 0, "plane_stride must be >= 0");
  DIB_REQUIRE(n_stride >= 16 && n_stride % 16 == 0, "n_stride must be a positive multiple of 16 (got %lld)",
              (long long)n_stride);
  DIB_REQUIRE(valid_box(box), "the ego box must be four finite numbers (x_lo, x_hi, y_lo, y_hi), lo <= hi");
  if (T == 0 || B == 0) return 0;
  DIB_REQUIRE(planes && offset && npts && pair_out && P && pos && omax && xyz_out && attr_out,
              "a required pointer is null");
  const Box4 b{box[0], box[1], box[2], box[3]};
  cudaStream_t cs = (cudaStream_t)stream;
  scatter_kernel<<<T, kScanThreads, 0, cs>>>(planes, plane_stride, offset, npts, pair_out, P, b, pos, omax, n_stride,
                                             xyz_out, attr_out);
  DIB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int kitti_build_finish_f32(const double* xyz, const double* attr, const int32_t* m_pts, const float* omax, int B,
                           double radius, int64_t n_stride, int64_t m_stride, float* out, int32_t* count,
                           dib_stream_t stream) {
  DIB_REQUIRE(B >= 0 && B <= kMaxB, "B must be in [0, %d] (got %d)", kMaxB, B);
  DIB_REQUIRE(n_stride >= 1 && m_stride >= 1, "n_stride and m_stride must be positive");
  DIB_REQUIRE(isfinite(radius), "the radius must be finite");
  if (B == 0) return 0;
  DIB_REQUIRE(xyz && attr && m_pts && omax && out && count, "a required pointer is null");
  cudaStream_t cs = (cudaStream_t)stream;
  finish_kernel<<<B, kScanThreads, 0, cs>>>(xyz, attr, m_pts, omax, radius, n_stride, m_stride, out, count);
  DIB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
