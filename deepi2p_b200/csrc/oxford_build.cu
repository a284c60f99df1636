// Oxford RobotCar point-cloud build (data/oxford/build_dataset.py: my_build_pointcloud, downsample and the output
// transform of save_pc_img_for_traversal) for S clouds of one traversal at once.  DESIGN.md 4.24 states the contract.
//
//   plan:    one thread per cloud walks its window of LMS scans in order: rel_i = M_c P_i, the skip test against the
//            last kept scan (its inverse by fixed-order Gauss-Jordan) and T_i = rel_i G_posesource_laser.
//   count:   one block per (kept scan, cloud) counts the points with x < threshold and their largest reflectance;
//            one thread per cloud then lays the kept scans out in order and takes the cloud's exact maximum.
//   scatter: one block per (kept scan, cloud) writes T_i (x, y, 0, 1) in fp64 and reflectance / max in scan order,
//            then point order (a block-wide order-preserving scan of the mask flags).
//   pack:    the output transform O (x, y, z, 1) of the voxel centres in fp64, reflectance * max, both to float32.
//
// Every sum is evaluated in the association written below; the file is compiled with --fmad=false so that
// oracle_oxford_build/ restates it bit for bit.
#include <math.h>

#include "common.cuh"

namespace dib {
namespace {

constexpr int kMaxS = 65535;
constexpr int kPlanThreads = 32;
constexpr int kScanThreads = 128;
constexpr int kPackThreads = 256;

struct Mat16 {
  double m[16];
};

// One thread's 4x4 (or 4x8) matrix in the plan kernel's shared memory: element k of thread t is at
// base[k * kPlanThreads + t], so the 32 threads of a warp reading the same element touch 32 consecutive doubles and
// never share a bank.
struct Lane {
  double* p;
  __device__ __forceinline__ double& operator[](int k) const { return p[k * kPlanThreads]; }
};

// ((a0 b0 + a1 b1) + a2 b2) + a3 b3 for row r of A and column c of B (both row-major 4x4).
template <class MA, class MB>
__device__ __forceinline__ double dot4(const MA& A, int r, const MB& B, int c) {
  return ((A[4 * r] * B[c] + A[4 * r + 1] * B[4 + c]) + A[4 * r + 2] * B[8 + c]) + A[4 * r + 3] * B[12 + c];
}

// Gauss-Jordan inverse of a (row-major 4x4) with partial pivoting: column c's pivot is the first row r >= c with the
// largest |a[r][c]|; the pivot row is divided by the pivot, then every other row r (ascending) has a[r][c] times it
// subtracted, over all eight columns of [a | I].  aug is scratch of 32 doubles; inv receives 16.
__device__ void gj_inverse(const Lane& a, const Lane& aug, const Lane& inv) {
  for (int r = 0; r < 4; ++r)
    for (int j = 0; j < 8; ++j) aug[8 * r + j] = j < 4 ? a[4 * r + j] : (j - 4 == r ? 1.0 : 0.0);
  for (int c = 0; c < 4; ++c) {
    int p = c;
    double best = fabs(aug[8 * c + c]);
    for (int r = c + 1; r < 4; ++r) {
      const double v = fabs(aug[8 * r + c]);
      if (v > best) {
        best = v;
        p = r;
      }
    }
    if (p != c)
      for (int j = 0; j < 8; ++j) {
        const double t = aug[8 * c + j];
        aug[8 * c + j] = aug[8 * p + j];
        aug[8 * p + j] = t;
      }
    const double piv = aug[8 * c + c];
    for (int j = 0; j < 8; ++j) aug[8 * c + j] = aug[8 * c + j] / piv;
    for (int r = 0; r < 4; ++r) {
      if (r == c) continue;
      const double f = aug[8 * r + c];
      for (int j = 0; j < 8; ++j) aug[8 * r + j] = aug[8 * r + j] - f * aug[8 * c + j];
    }
  }
  for (int r = 0; r < 4; ++r)
    for (int j = 0; j < 4; ++j) inv[4 * r + j] = aug[8 * r + 4 + j];
}

__global__ void __launch_bounds__(kPlanThreads) plan_kernel(const double* __restrict__ poses,
                                                            const uint8_t* __restrict__ present, int64_t n_lms,
                                                            const int64_t* __restrict__ win,
                                                            const double* __restrict__ centre_inv, int S, Mat16 G,
                                                            double skip_threshold, int w_stride,
                                                            int32_t* __restrict__ kept_scan,
                                                            double* __restrict__ kept_T, int32_t* __restrict__ n_kept,
                                                            int32_t* __restrict__ n_skipped) {
  __shared__ double s_rel[16][kPlanThreads];
  __shared__ double s_inv[16][kPlanThreads];
  __shared__ double s_aug[32][kPlanThreads];
  __shared__ double s_M[16][kPlanThreads];
  const int s = blockIdx.x * kPlanThreads + threadIdx.x;
  if (s >= S) return;
  const Lane rel{&s_rel[0][threadIdx.x]}, inv{&s_inv[0][threadIdx.x]}, aug{&s_aug[0][threadIdx.x]};
  const Lane M{&s_M[0][threadIdx.x]};
  for (int k = 0; k < 16; ++k) M[k] = centre_inv[16 * (int64_t)s + k];
  const int64_t lo = win[2 * (int64_t)s], hi = win[2 * (int64_t)s + 1];
  if (lo < 0 || hi < lo || hi > n_lms || hi - lo > w_stride) {   // the host checks windows; never read past them
    n_kept[s] = 0;
    n_skipped[s] = -1;
    return;
  }
  int kept = 0, skipped = 0;
  bool have_prev = false;
  for (int64_t i = lo; i < hi; ++i) {
    if (!present[i]) continue;
    const double* P = poses + 16 * i;
    for (int r = 0; r < 4; ++r)
      for (int c = 0; c < 4; ++c) rel[4 * r + c] = dot4(M, r, P, c);
    if (have_prev) {
      double d[3];
      for (int r = 0; r < 3; ++r) d[r] = dot4(inv, r, rel, 3);
      const double norm = sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]);
      if (norm < skip_threshold) {
        ++skipped;
        continue;
      }
    }
    const int64_t o = (int64_t)s * w_stride + kept;
    kept_scan[o] = (int32_t)i;
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 4; ++c) kept_T[12 * o + 4 * r + c] = dot4(rel, r, G.m, c);
    gj_inverse(rel, aug, inv);
    have_prev = true;
    ++kept;
  }
  n_kept[s] = kept;
  n_skipped[s] = skipped;
}

__device__ __forceinline__ bool keep_point(double x, int use_mask, double thr) { return !use_mask || x < thr; }

__global__ void __launch_bounds__(kScanThreads) count_kernel(const double* __restrict__ x,
                                                             const double* __restrict__ r,
                                                             const int64_t* __restrict__ offsets,
                                                             const int32_t* __restrict__ kept_scan,
                                                             const int32_t* __restrict__ n_kept, int w_stride,
                                                             int use_mask, double thr, int32_t* __restrict__ pcount,
                                                             double* __restrict__ pmax) {
  const int s = blockIdx.y, k = blockIdx.x;
  if (k >= n_kept[s]) return;
  const int64_t o = (int64_t)s * w_stride + k;
  const int j = kept_scan[o];
  const int64_t b = offsets[j], e = offsets[j + 1];
  int cnt = 0;
  double mx = -INFINITY;
  for (int64_t i = b + threadIdx.x; i < e; i += kScanThreads)
    if (keep_point(x[i], use_mask, thr)) {
      ++cnt;
      mx = r[i] > mx ? r[i] : mx;
    }
  __shared__ int s_cnt[kScanThreads / 32];
  __shared__ double s_max[kScanThreads / 32];
  for (int off = 16; off; off >>= 1) {
    cnt += __shfl_down_sync(0xffffffffu, cnt, off);
    const double v = __shfl_down_sync(0xffffffffu, mx, off);
    mx = v > mx ? v : mx;
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
      mx = s_max[q] > mx ? s_max[q] : mx;
    }
    pcount[o] = cnt;
    pmax[o] = mx;
  }
}

__global__ void layout_kernel(const int32_t* __restrict__ n_kept, int S, int w_stride,
                              const int32_t* __restrict__ pcount, const double* __restrict__ pmax,
                              int32_t* __restrict__ pos, int32_t* __restrict__ n_pts, double* __restrict__ rmax) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= S) return;
  int64_t acc = 0;
  double mx = -INFINITY;
  for (int k = 0; k < n_kept[s]; ++k) {
    const int64_t o = (int64_t)s * w_stride + k;
    pos[o] = (int32_t)(acc < INT32_MAX ? acc : INT32_MAX);
    acc += pcount[o];
    mx = pmax[o] > mx ? pmax[o] : mx;
  }
  n_pts[s] = (int32_t)(acc < INT32_MAX ? acc : INT32_MAX);    // the host refuses a cloud this large
  rmax[s] = mx;
}

__global__ void __launch_bounds__(kScanThreads) scatter_kernel(
    const double* __restrict__ x, const double* __restrict__ y, const double* __restrict__ r,
    const int64_t* __restrict__ offsets, const int32_t* __restrict__ kept_scan, const double* __restrict__ kept_T,
    const int32_t* __restrict__ n_kept, const int32_t* __restrict__ pos, const double* __restrict__ rmax,
    int w_stride, int use_mask, double thr, int n_stride, double* __restrict__ xyz_out,
    double* __restrict__ attr_out) {
  const int s = blockIdx.y, k = blockIdx.x;
  if (k >= n_kept[s]) return;
  const int64_t o = (int64_t)s * w_stride + k;
  const int j = kept_scan[o];
  const int64_t b = offsets[j], e = offsets[j + 1];
  double T[12];
  for (int q = 0; q < 12; ++q) T[q] = kept_T[12 * o + q];
  const double mx = rmax[s];
  double* ox = xyz_out + (int64_t)s * 3 * n_stride;
  double* oa = attr_out + (int64_t)s * n_stride;
  __shared__ int s_warp[kScanThreads / 32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int64_t base = pos[o];
  for (int64_t c = b; c < e; c += kScanThreads) {
    const int64_t i = c + threadIdx.x;
    const bool f = i < e && keep_point(x[i], use_mask, thr);
    const unsigned bal = __ballot_sync(0xffffffffu, f);
    if (lane == 0) s_warp[w] = __popc(bal);
    __syncthreads();
    int before = 0, total = 0;
    for (int q = 0; q < kScanThreads / 32; ++q) {
      before += q < w ? s_warp[q] : 0;
      total += s_warp[q];
    }
    if (f) {
      const int64_t d = base + before + __popc(bal & ((1u << lane) - 1u));
      const double px = x[i], py = y[i], pz = 0.0;
      for (int a = 0; a < 3; ++a)
        ox[(int64_t)a * n_stride + d] = ((T[4 * a] * px + T[4 * a + 1] * py) + T[4 * a + 2] * pz) + T[4 * a + 3];
      oa[d] = r[i] / mx;
    }
    base += total;
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kPackThreads) pack_kernel(const double* __restrict__ xyz,
                                                            const double* __restrict__ attr,
                                                            const int32_t* __restrict__ m_pts,
                                                            const double* __restrict__ rmax, Mat16 O, int n_stride,
                                                            int m_stride, float* __restrict__ out) {
  const int s = blockIdx.y;
  const int j = blockIdx.x * kPackThreads + threadIdx.x;
  if (j >= m_stride) return;
  float* os = out + (int64_t)s * 4 * m_stride;
  if (j >= m_pts[s]) {
    for (int a = 0; a < 4; ++a) os[(int64_t)a * m_stride + j] = 0.0f;
    return;
  }
  const double* p = xyz + (int64_t)s * 3 * n_stride;
  const double px = p[j], py = p[n_stride + j], pz = p[2 * (int64_t)n_stride + j];
  for (int a = 0; a < 3; ++a)
    os[(int64_t)a * m_stride + j] =
        (float)(((O.m[4 * a] * px + O.m[4 * a + 1] * py) + O.m[4 * a + 2] * pz) + O.m[4 * a + 3]);
  os[3 * (int64_t)m_stride + j] = (float)(attr[(int64_t)s * n_stride + j] * rmax[s]);
}

bool finite16(const double* m) {
  for (int k = 0; k < 16; ++k)
    if (!isfinite(m[k])) return false;
  return true;
}

}  // namespace
}  // namespace dib

using namespace dib;

extern "C" {

int oxford_build_plan_f64(const double* lms_poses, const uint8_t* present, int64_t n_lms, const int64_t* windows,
                          const double* centre_inv, int S, const double* G, double skip_threshold, int w_stride,
                          int32_t* kept_scan, double* kept_T, int32_t* n_kept, int32_t* n_skipped,
                          dib_stream_t stream) {
  DIB_REQUIRE(S >= 0 && S <= kMaxS, "S must be in [0, %d] (got %d)", kMaxS, S);
  DIB_REQUIRE(n_lms >= 0 && n_lms < INT32_MAX, "n_lms must be in [0, 2^31 - 1) (got %lld)", (long long)n_lms);
  DIB_REQUIRE(w_stride >= 1, "w_stride must be positive (got %d)", w_stride);
  DIB_REQUIRE((int64_t)S * w_stride < INT32_MAX, "S * w_stride must be below 2^31");
  DIB_REQUIRE(G && finite16(G), "G_posesource_laser must be 16 finite numbers");
  DIB_REQUIRE(isfinite(skip_threshold) && skip_threshold >= 0, "skip_threshold must be finite and >= 0");
  if (S == 0) return 0;
  DIB_REQUIRE((lms_poses || n_lms == 0) && (present || n_lms == 0) && windows && centre_inv && kept_scan && kept_T &&
                  n_kept && n_skipped,
              "a required pointer is null");
  Mat16 g;
  for (int k = 0; k < 16; ++k) g.m[k] = G[k];
  cudaStream_t cs = (cudaStream_t)stream;
  plan_kernel<<<(S + kPlanThreads - 1) / kPlanThreads, kPlanThreads, 0, cs>>>(
      lms_poses, present, n_lms, windows, centre_inv, S, g, skip_threshold, w_stride, kept_scan, kept_T, n_kept,
      n_skipped);
  DIB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

size_t oxford_build_count_workspace_bytes(int S, int w_stride) {
  if (S < 0 || w_stride < 1) return 0;
  const size_t n = (size_t)S * (size_t)w_stride;
  return ((n * sizeof(int32_t) + 255) / 256 * 256) + n * sizeof(double);
}

int oxford_build_count_f64(const double* x, const double* r, const int64_t* offsets, const int32_t* kept_scan,
                           const int32_t* n_kept, int S, int w_stride, int use_mask, double threshold, int32_t* pos,
                           int32_t* n_pts, double* rmax, void* workspace, size_t workspace_bytes,
                           dib_stream_t stream) {
  DIB_REQUIRE(S >= 0 && S <= kMaxS, "S must be in [0, %d] (got %d)", kMaxS, S);
  DIB_REQUIRE(w_stride >= 1 && w_stride <= INT32_MAX / 2, "w_stride must be positive (got %d)", w_stride);
  DIB_REQUIRE((int64_t)S * w_stride < INT32_MAX, "S * w_stride must be below 2^31");
  DIB_REQUIRE(!use_mask || isfinite(threshold), "the ground threshold must be finite");
  if (S == 0) return 0;
  DIB_REQUIRE(x && r && offsets && kept_scan && n_kept && pos && n_pts && rmax && workspace,
              "a required pointer is null");
  const size_t need = oxford_build_count_workspace_bytes(S, w_stride);
  if (workspace_bytes < need) {
    set_error("oxford_build_count: workspace is %zu bytes, %zu needed", workspace_bytes, need);
    return DIB_ENOMEM;
  }
  const size_t n = (size_t)S * (size_t)w_stride;
  int32_t* pcount = (int32_t*)workspace;
  double* pmax = (double*)((char*)workspace + (n * sizeof(int32_t) + 255) / 256 * 256);
  cudaStream_t cs = (cudaStream_t)stream;
  count_kernel<<<dim3(w_stride, S), kScanThreads, 0, cs>>>(x, r, offsets, kept_scan, n_kept, w_stride, use_mask,
                                                           threshold, pcount, pmax);
  DIB_CHECK_CUDA(cudaGetLastError());
  layout_kernel<<<(S + 127) / 128, 128, 0, cs>>>(n_kept, S, w_stride, pcount, pmax, pos, n_pts, rmax);
  DIB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int oxford_build_scatter_f64(const double* x, const double* y, const double* r, const int64_t* offsets,
                             const int32_t* kept_scan, const double* kept_T, const int32_t* n_kept,
                             const int32_t* pos, const double* rmax, int S, int w_stride, int use_mask,
                             double threshold, int n_stride, double* xyz_out, double* attr_out,
                             dib_stream_t stream) {
  DIB_REQUIRE(S >= 0 && S <= kMaxS, "S must be in [0, %d] (got %d)", kMaxS, S);
  DIB_REQUIRE(w_stride >= 1 && w_stride <= INT32_MAX / 2, "w_stride must be positive (got %d)", w_stride);
  DIB_REQUIRE(n_stride >= 16 && n_stride % 16 == 0, "n_stride must be a positive multiple of 16 (got %d)", n_stride);
  DIB_REQUIRE((int64_t)S * 3 * n_stride < INT32_MAX, "S * 3 * n_stride must be below 2^31");
  DIB_REQUIRE(!use_mask || isfinite(threshold), "the ground threshold must be finite");
  if (S == 0) return 0;
  DIB_REQUIRE(x && y && r && offsets && kept_scan && kept_T && n_kept && pos && rmax && xyz_out && attr_out,
              "a required pointer is null");
  cudaStream_t cs = (cudaStream_t)stream;
  scatter_kernel<<<dim3(w_stride, S), kScanThreads, 0, cs>>>(x, y, r, offsets, kept_scan, kept_T, n_kept, pos, rmax,
                                                             w_stride, use_mask, threshold, n_stride, xyz_out,
                                                             attr_out);
  DIB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int oxford_build_pack_f32(const double* xyz, const double* attr, const int32_t* m_pts, const double* rmax,
                          const double* O, int S, int n_stride, int m_stride, float* out, dib_stream_t stream) {
  DIB_REQUIRE(S >= 0 && S <= kMaxS, "S must be in [0, %d] (got %d)", kMaxS, S);
  DIB_REQUIRE(n_stride >= 1 && m_stride >= 1 && m_stride <= n_stride, "need 1 <= m_stride <= n_stride (got %d, %d)",
              m_stride, n_stride);
  DIB_REQUIRE((int64_t)S * 4 * n_stride < INT32_MAX, "S * 4 * n_stride must be below 2^31");
  DIB_REQUIRE(O && finite16(O), "the output transform must be 16 finite numbers");
  if (S == 0) return 0;
  DIB_REQUIRE(xyz && attr && m_pts && rmax && out, "a required pointer is null");
  Mat16 o;
  for (int k = 0; k < 16; ++k) o.m[k] = O[k];
  cudaStream_t cs = (cudaStream_t)stream;
  pack_kernel<<<dim3((m_stride + kPackThreads - 1) / kPackThreads, S), kPackThreads, 0, cs>>>(
      xyz, attr, m_pts, rmax, o, n_stride, m_stride, out);
  DIB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
