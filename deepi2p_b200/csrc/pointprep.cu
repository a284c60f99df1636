// Batched LiDAR scan preparation: the Open3D steps of data/kitti/kitti_pc_bin_to_npy_with_downsample_sn.py:48-74 and
// of the loaders' downsample_with_intensity_sn / downsample_with_reflectance, restated for many clouds at once.
// DESIGN.md "Scan preparation" states the contract; oracle_prep/prep_oracle.cpp is its serial CPU restatement.
//
// voxel downsample (per call)
//   bbox      (one CTA per cloud)  bounding box in the coordinates' type (float32 or fp64); read back to the host,
//             which rejects clouds of 2^21 or more voxels along an axis and sizes the sort key from the largest voxel
//             index of the batch
//   key       voxel (ix, iy, iz) = floor((p - min_bound) / v) in fp64, packed into bx + by + bz bits
//   sort      stable cub radix sorts: by voxel key, then by cloud (padding last), so each voxel's points are
//             contiguous and in ascending original index
//   rank      voxel heads, an inclusive scan gives each point its voxel's rank
//   mean      one thread per voxel sums its points (and C attribute channels) sequentially, then divides by the count
// normal estimation (per call)
//   index     icp.cu's Morton box tree over each cloud (morton_index.cuh)
//   normal    one thread per point (in Morton order): the min(max_nn, c) nearest points with d2 < r^2, ties to the lower
//             index; covariance from moments about the point in (d2, index) order; smallest eigenvector by the
//             Jacobi solver of sym3_eig.cuh; orientation toward a reference direction
// nearest
//   index     as above; one thread per fp64 query, exact nearest float32 point, ties to the lowest index
// The file is compiled with --fmad=false (build.py NOFMA_SOURCES), so every operation rounds as the oracle's does.
#include <cfloat>
#include <climits>
#include <cmath>
#include <vector>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "morton_index.cuh"
#include "sym3_eig.cuh"

namespace dib {
namespace prep {

using icp::clamp_n;

constexpr int kMaxS = 65535;
constexpr int kMaxC = 64;             // attribute channels of a voxel downsample
constexpr int kMaxNN = 64;
constexpr int kVoxelBits = 21;        // voxel index range per axis: [0, 2^21)

inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }
inline size_t sort_reserve(size_t N) { return 8 * N + ((size_t)4 << 20); }

// ---------------------------------------------------------------------------------------------------------------
// Voxel downsample.

struct VoxWork {
  void* bbox;                           // [S][6] in the coordinates' type
  unsigned long long *key0, *key1;      // [N] voxel keys
  uint32_t *ck0, *ck1;                  // [N] cloud keys
  int32_t *val0, *val1;                 // [N] global point index s * n_stride + j
  int32_t* cnt;                         // [S + 1]
  int32_t* off;                         // [S + 1] first sorted position of each cloud; off[S] = total
  int32_t* head;                        // [N]
  int32_t* rank;                        // [N]
  void* tmp;
  size_t tmp_bytes;
};

size_t carve_vox(char* base, int S, int n_stride, VoxWork* wk) {
  const size_t N = (size_t)S * n_stride;
  size_t off = 0;
  auto take = [&](size_t bytes) { char* p = base ? base + off : nullptr; off += align256(bytes); return p; };
  VoxWork w;
  w.bbox = take((size_t)S * 6 * 8);
  w.key0 = (unsigned long long*)take(N * 8); w.key1 = (unsigned long long*)take(N * 8);
  w.ck0 = (uint32_t*)take(N * 4); w.ck1 = (uint32_t*)take(N * 4);
  w.val0 = (int32_t*)take(N * 4); w.val1 = (int32_t*)take(N * 4);
  w.cnt = (int32_t*)take(((size_t)S + 1) * 4);
  w.off = (int32_t*)take(((size_t)S + 1) * 4);
  w.head = (int32_t*)take(N * 4);
  w.rank = (int32_t*)take(N * 4);
  w.tmp_bytes = sort_reserve(N);
  w.tmp = take(w.tmp_bytes);
  if (wk) *wk = w;
  return off;
}

struct VoxKey {
  double v;
  int bz, byz;                          // bits of iz, and of (iy, iz)
};

// The voxel of point j of cloud s: floor(((double)p - min_bound) / v) per axis, min_bound = (double)lo - 0.5 * v.
template <typename T>
__device__ __forceinline__ unsigned long long voxel_key(const T* X, int n_stride, const T* bb, int j, const VoxKey& k) {
  unsigned long long c[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double mb = (double)bb[a] - 0.5 * k.v;
    const double f = floor(((double)X[(size_t)a * n_stride + j] - mb) / k.v);
    c[a] = f > 0.0 ? (unsigned long long)f : 0ull;    // >= 0 for every finite coordinate of the cloud
  }
  return (c[0] << k.byz) | (c[1] << k.bz) | c[2];
}

// The float32 clouds' box is icp.cu's bbox_kernel; fp64 clouds get this one (min / max are exact in any order).
__global__ void __launch_bounds__(256) bbox_f64_kernel(const double* __restrict__ X, const int32_t* __restrict__ n_pts,
                                                       int n_stride, double* __restrict__ bbox) {
  const int s = blockIdx.x;
  const int n = clamp_n(n_pts, s, n_stride);
  const double* P = X + (size_t)s * 3 * n_stride;
  double lo[3] = {DBL_MAX, DBL_MAX, DBL_MAX}, hi[3] = {-DBL_MAX, -DBL_MAX, -DBL_MAX};
  for (int j = threadIdx.x; j < n; j += blockDim.x)
    for (int a = 0; a < 3; ++a) {
      const double v = P[(size_t)a * n_stride + j];
      lo[a] = fmin(lo[a], v);
      hi[a] = fmax(hi[a], v);
    }
  __shared__ double red[6][8];
  for (int a = 0; a < 3; ++a)
    for (int o = 16; o > 0; o >>= 1) {
      lo[a] = fmin(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
      hi[a] = fmax(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
    }
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0)
    for (int a = 0; a < 3; ++a) red[a][w] = lo[a], red[3 + a][w] = hi[a];
  __syncthreads();
  if (threadIdx.x < 6) {
    double v = red[threadIdx.x][0];
    for (int q = 1; q < (int)(blockDim.x >> 5); ++q)
      v = threadIdx.x < 3 ? fmin(v, red[threadIdx.x][q]) : fmax(v, red[threadIdx.x][q]);
    bbox[s * 6 + threadIdx.x] = v;
  }
}

template <typename T>
__global__ void vox_key_kernel(const T* __restrict__ xyz, const int32_t* __restrict__ n_pts, int n_stride, int S,
                               const T* __restrict__ bbox, VoxKey k, unsigned long long* __restrict__ key,
                               int32_t* __restrict__ val) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)S * n_stride) return;
  const int s = (int)(g / n_stride), j = (int)(g - (long long)s * n_stride);
  key[g] = j < clamp_n(n_pts, s, n_stride) ? voxel_key(xyz + (size_t)s * 3 * n_stride, n_stride, bbox + s * 6, j, k)
                                           : 0ull;
  val[g] = (int32_t)g;
}

// Cloud key of each sorted point (padding: S, after every cloud); counts per cloud (cnt[S] = 0).
__global__ void vox_cloud_kernel(const int32_t* __restrict__ n_pts, int n_stride, int S,
                                 const int32_t* __restrict__ val, uint32_t* __restrict__ ck, int32_t* __restrict__ cnt) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g <= S) cnt[g] = g < S ? clamp_n(n_pts, (int)g, n_stride) : 0;
  if (g >= (long long)S * n_stride) return;
  const int v = val[g], s = v / n_stride, j = v - s * n_stride;
  ck[g] = j < clamp_n(n_pts, s, n_stride) ? (uint32_t)s : (uint32_t)S;
}

template <typename T>
__global__ void vox_head_kernel(const T* __restrict__ xyz, int n_stride, long long N, const T* __restrict__ bbox, VoxKey k,
                                const int32_t* __restrict__ val, const int32_t* __restrict__ off, int S, int32_t* __restrict__ head) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  int h = 0;
  if (i < off[S]) {
    const int v = val[i], s = v / n_stride, j = v - s * n_stride;
    h = 1;
    if (i > off[s]) {
      const int u = val[i - 1], ju = u - s * n_stride;     // same cloud
      const T* X = xyz + (size_t)s * 3 * n_stride;
      h = voxel_key(X, n_stride, bbox + s * 6, j, k) != voxel_key(X, n_stride, bbox + s * 6, ju, k);
    }
  }
  head[i] = h;
}

// One thread per voxel head: sequential sums over the voxel's points in ascending original index, then / count.
template <typename T>
__global__ void vox_mean_kernel(const T* __restrict__ xyz, const double* __restrict__ attr, int C, int n_stride,
                                long long N, const int32_t* __restrict__ n_pts, const int32_t* __restrict__ val,
                                const int32_t* __restrict__ off, const int32_t* __restrict__ head,
                                const int32_t* __restrict__ rank, int S, double* __restrict__ xyz_out,
                                double* __restrict__ attr_out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N || i >= off[S] || !head[i]) return;
  const int s = val[i] / n_stride;
  const int end = off[s] + clamp_n(n_pts, s, n_stride);
  const int o = rank[i] - rank[off[s]];
  int e = (int)i + 1;
  while (e < end && !head[e]) ++e;
  const double cnt = (double)(e - (int)i);
  const T* X = xyz + (size_t)s * 3 * n_stride;
  for (int a = 0; a < 3; ++a) {
    double sum = 0.0;
    for (int t = (int)i; t < e; ++t) sum += (double)X[(size_t)a * n_stride + (val[t] - s * n_stride)];
    xyz_out[((size_t)s * 3 + a) * n_stride + o] = sum / cnt;
  }
  for (int c = 0; c < C; ++c) {
    const double* A = attr + ((size_t)s * C + c) * n_stride;
    double sum = 0.0;
    for (int t = (int)i; t < e; ++t) sum += A[val[t] - s * n_stride];
    attr_out[((size_t)s * C + c) * n_stride + o] = sum / cnt;
  }
}

__global__ void vox_count_kernel(const int32_t* __restrict__ n_pts, int n_stride, int S,
                                 const int32_t* __restrict__ off, const int32_t* __restrict__ rank,
                                 int32_t* __restrict__ m_out) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= S) return;
  const int n = clamp_n(n_pts, s, n_stride);
  m_out[s] = n > 0 ? rank[off[s] + n - 1] - rank[off[s]] + 1 : 0;
}

inline int bits_of(unsigned long long x) {
  int b = 0;
  while (b < 64 && (x >> b) != 0) ++b;
  return b;
}

int check_stride(int stride, int S, const char* name) {
  DIB_REQUIRE(S >= 0 && S <= kMaxS, "S=%d must be in [0, %d] (larger batches: split them)", S, kMaxS);
  DIB_REQUIRE(stride >= 16 && stride % 16 == 0, "%s=%d must be a positive multiple of 16", name, stride);
  DIB_REQUIRE((long long)S * stride < (1LL << 31), "S * %s must be below 2^31", name);
  return DIB_OK;
}

template <typename T>
int voxel_downsample(const T* xyz, const int32_t* n_pts, int n_stride, int S, const double* attr, int C,
                     double voxel_size, double* xyz_out, double* attr_out, int32_t* m_pts_out, void* workspace,
                     size_t workspace_bytes, cudaStream_t st) {
  DIB_REQUIRE(xyz && xyz_out && m_pts_out, "NULL argument (xyz, xyz_out, m_pts_out)");
  int rc = check_stride(n_stride, S, "n_stride");
  if (rc != DIB_OK) return rc;
  DIB_REQUIRE(C >= 0 && C <= kMaxC, "C=%d must be in [0, %d]", C, kMaxC);
  DIB_REQUIRE(C == 0 || (attr && attr_out), "NULL argument (attr, attr_out with C=%d)", C);
  DIB_REQUIRE(std::isfinite(voxel_size) && voxel_size > 0.0, "voxel_size must be positive (got %g)", voxel_size);
  const size_t need = carve_vox(nullptr, S, n_stride, nullptr);
  DIB_REQUIRE(workspace && workspace_bytes >= need, "workspace too small (%zu < %zu)", workspace_bytes, need);
  DIB_REQUIRE(((uintptr_t)workspace & 255) == 0, "workspace must be 256-byte aligned");
  if (S == 0) return DIB_OK;
  VoxWork wk;
  carve_vox((char*)workspace, S, n_stride, &wk);
  T* bbox = (T*)wk.bbox;
  if constexpr (sizeof(T) == 4)
    icp::cloud_bbox(xyz, n_pts, n_stride, S, bbox, st);
  else
    bbox_f64_kernel<<<S, 256, 0, st>>>(xyz, n_pts, n_stride, bbox);
  DIB_CHECK_CUDA(cudaGetLastError());
  // The limit on the voxel count depends on the data, so the boxes come back to the host before the sort.
  std::vector<T> bb((size_t)S * 6);
  DIB_CHECK_CUDA(cudaMemcpyAsync(bb.data(), bbox, bb.size() * sizeof(T), cudaMemcpyDeviceToHost, st));
  DIB_CHECK_CUDA(cudaStreamSynchronize(st));
  unsigned long long top[3] = {0, 0, 0};
  for (int s = 0; s < S; ++s) {
    if (bb[s * 6] > bb[s * 6 + 3]) continue;             // empty cloud
    for (int a = 0; a < 3; ++a) {
      const double lo = (double)bb[s * 6 + a], hi = (double)bb[s * 6 + 3 + a];
      DIB_REQUIRE(std::isfinite(lo) && std::isfinite(hi), "cloud %d has a non-finite coordinate", s);
      const double mb = lo - 0.5 * voxel_size;
      const double f = std::floor((hi - mb) / voxel_size);
      DIB_REQUIRE(f < (double)(1 << kVoxelBits), "cloud %d spans 2^%d or more voxels along axis %d", s, kVoxelBits,
                  a);
      if ((unsigned long long)f > top[a]) top[a] = (unsigned long long)f;
    }
  }
  const VoxKey k{voxel_size, bits_of(top[2]), bits_of(top[1]) + bits_of(top[2])};
  const int kb = bits_of(top[0]) + k.byz;
  const long long N = (long long)S * n_stride;
  const int nb = (int)((N + 255) / 256);
  vox_key_kernel<T><<<nb, 256, 0, st>>>(xyz, n_pts, n_stride, S, bbox, k, wk.key0, wk.val0);
  DIB_CHECK_CUDA(cudaGetLastError());
  cub::DoubleBuffer<unsigned long long> keys(wk.key0, wk.key1);
  cub::DoubleBuffer<int32_t> vals(wk.val0, wk.val1);
  size_t tmp = 0;
  if (kb > 0) {                                           // kb == 0: one voxel per cloud, the order is already right
    DIB_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp, keys, vals, (int)N, 0, kb, st));
    if (tmp > wk.tmp_bytes) {
      set_error("voxel_downsample: the radix sort needs %zu bytes of scratch, %zu reserved", tmp, wk.tmp_bytes);
      return DIB_ENOMEM;
    }
    DIB_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(wk.tmp, tmp, keys, vals, (int)N, 0, kb, st));
  }
  const int nb1 = (int)((N + 1 + 255) / 256);             // one more thread for cnt[S]
  vox_cloud_kernel<<<nb1, 256, 0, st>>>(n_pts, n_stride, S, vals.Current(), wk.ck0, wk.cnt);
  DIB_CHECK_CUDA(cudaGetLastError());
  cub::DoubleBuffer<uint32_t> cks(wk.ck0, wk.ck1);
  const int fb = bits_of((unsigned long long)S);
  DIB_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp, cks, vals, (int)N, 0, fb, st));
  if (tmp > wk.tmp_bytes) {
    set_error("voxel_downsample: the radix sort needs %zu bytes of scratch, %zu reserved", tmp, wk.tmp_bytes);
    return DIB_ENOMEM;
  }
  DIB_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(wk.tmp, tmp, cks, vals, (int)N, 0, fb, st));
  DIB_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp, wk.cnt, wk.off, S + 1, st));
  DIB_REQUIRE(tmp <= wk.tmp_bytes, "voxel_downsample: scan scratch %zu exceeds %zu", tmp, wk.tmp_bytes);
  DIB_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(wk.tmp, tmp, wk.cnt, wk.off, S + 1, st));
  vox_head_kernel<T><<<nb, 256, 0, st>>>(xyz, n_stride, N, bbox, k, vals.Current(), wk.off, S, wk.head);
  DIB_CHECK_CUDA(cudaGetLastError());
  DIB_CHECK_CUDA(cub::DeviceScan::InclusiveSum(nullptr, tmp, wk.head, wk.rank, (int)N, st));
  DIB_REQUIRE(tmp <= wk.tmp_bytes, "voxel_downsample: scan scratch %zu exceeds %zu", tmp, wk.tmp_bytes);
  DIB_CHECK_CUDA(cub::DeviceScan::InclusiveSum(wk.tmp, tmp, wk.head, wk.rank, (int)N, st));
  vox_mean_kernel<T><<<nb, 256, 0, st>>>(xyz, attr, C, n_stride, N, n_pts, vals.Current(), wk.off, wk.head, wk.rank, S,
                                      xyz_out, attr_out);
  vox_count_kernel<<<(S + 127) / 128, 128, 0, st>>>(n_pts, n_stride, S, wk.off, wk.rank, m_pts_out);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Normal estimation and nearest point.

struct NormArgs {
  const float* xyz;
  const int32_t* m_pts;
  int m_stride;
  double r2;
  int max_nn;
  double o[3];
  double* normals;          // [S][3][m_stride]
  int32_t* count;           // [S][m_stride] or NULL
};

// One thread per point, in the index's Morton order (neighbouring threads search neighbouring boxes).
template <int K>
__global__ void __launch_bounds__(128) normals_kernel(NormArgs a, icp::Levels L, icp::Index ix, int S) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)S * a.m_stride) return;
  const int s = (int)(g / a.m_stride), k = (int)(g - (long long)s * a.m_stride);
  const int m = clamp_n(a.m_pts, s, a.m_stride);
  if (k >= m) return;
  int root = 0;
  while (icp::level_count(m, root) > 1) ++root;
  const float4* pts = ix.pts + (size_t)s * a.m_stride;
  const float4 p = pts[k];
  const int i = __float_as_int(p.w);
  const double qx = p.x, qy = p.y, qz = p.z;
  double d2s[K];
  int js[K];
  const int cnt = icp::knn<K>(pts, ix.lo + (size_t)s * L.per_frame, ix.hi + (size_t)s * L.per_frame, L, m, root, qx,
                              qy, qz, a.r2, a.max_nn, d2s, js);
  const float* X = a.xyz + (size_t)s * 3 * a.m_stride;
  double n[3] = {0.0, 0.0, 1.0};
  if (cnt >= 3) {
    double c[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};   // d, dx dx, dx dy, dx dz, dy dy, dy dz, dz dz
    for (int t = 0; t < cnt; ++t) {
      const int j = js[t];
      const double dx = (double)X[j] - qx, dy = (double)X[(size_t)a.m_stride + j] - qy,
                   dz = (double)X[(size_t)2 * a.m_stride + j] - qz;
      c[0] += dx; c[1] += dy; c[2] += dz;
      c[3] += dx * dx; c[4] += dx * dy; c[5] += dx * dz;
      c[6] += dy * dy; c[7] += dy * dz; c[8] += dz * dz;
    }
    const double fc = (double)cnt;
    for (int q = 0; q < 9; ++q) c[q] = c[q] / fc;
    double C[9];
    C[0] = c[3] - c[0] * c[0];
    C[4] = c[6] - c[1] * c[1];
    C[8] = c[8] - c[2] * c[2];
    C[1] = C[3] = c[4] - c[0] * c[1];
    C[2] = C[6] = c[5] - c[0] * c[2];
    C[5] = C[7] = c[7] - c[1] * c[2];
    if (C[0] == 0.0 && C[4] == 0.0 && C[8] == 0.0 && C[1] == 0.0 && C[2] == 0.0 && C[5] == 0.0) {
      n[0] = n[1] = n[2] = 0.0;
    } else {
      double lam[3], E[9];
      sym3_eig_desc(C, lam, E);
      const double e0 = E[2], e1 = E[5], e2 = E[8];
      const double nn = sqrt((e0 * e0 + e1 * e1) + e2 * e2);
      n[0] = e0 / nn; n[1] = e1 / nn; n[2] = e2 / nn;
    }
  }
  if (n[0] == 0.0 && n[1] == 0.0 && n[2] == 0.0) {
    n[0] = a.o[0]; n[1] = a.o[1]; n[2] = a.o[2];
  } else if ((n[0] * a.o[0] + n[1] * a.o[1]) + n[2] * a.o[2] < 0.0) {
    n[0] = -n[0]; n[1] = -n[1]; n[2] = -n[2];
  }
  for (int q = 0; q < 3; ++q) a.normals[((size_t)s * 3 + q) * a.m_stride + i] = n[q];
  if (a.count) a.count[(size_t)s * a.m_stride + i] = cnt;
}

__global__ void __launch_bounds__(128) nearest_kernel(const double* __restrict__ q, const int32_t* __restrict__ q_pts,
                                                      int q_stride, const int32_t* __restrict__ m_pts, int m_stride,
                                                      int S, icp::Levels L, icp::Index ix, int32_t* __restrict__ out) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)S * q_stride) return;
  const int s = (int)(g / q_stride), k = (int)(g - (long long)s * q_stride);
  if (k >= clamp_n(q_pts, s, q_stride)) return;
  const int m = clamp_n(m_pts, s, m_stride);
  int root = 0;
  while (icp::level_count(m, root) > 1) ++root;
  const double* Q = q + (size_t)s * 3 * q_stride;
  icp::Hit h;
  h.d2 = 0.5 * DBL_MAX;     // finite and below DBL_MAX, which the descent uses for a missing sibling box
  unsigned long long evals = 0;
  icp::nearest(ix.pts + (size_t)s * m_stride, ix.lo + (size_t)s * L.per_frame, ix.hi + (size_t)s * L.per_frame, L, m,
               root, Q[k], Q[(size_t)q_stride + k], Q[(size_t)2 * q_stride + k], h, evals);
  out[g] = h.j == INT_MAX ? -1 : h.j;
}

int check_index(const float* xyz, int m_stride, int S, void* workspace, size_t workspace_bytes) {
  DIB_REQUIRE(xyz, "NULL argument (xyz)");
  const int rc = check_stride(m_stride, S, "m_stride");
  if (rc != DIB_OK) return rc;
  DIB_REQUIRE(icp::make_levels(m_stride).n <= icp::kMaxLevels, "m_stride=%d is too large for the index", m_stride);
  const size_t need = icp::carve_index(nullptr, 0, S, m_stride, nullptr);
  DIB_REQUIRE(workspace && workspace_bytes >= need, "workspace too small (%zu < %zu)", workspace_bytes, need);
  DIB_REQUIRE(((uintptr_t)workspace & 255) == 0, "workspace must be 256-byte aligned");
  return DIB_OK;
}

int estimate_normals(const float* xyz, const int32_t* m_pts, int m_stride, int S, double radius, int max_nn,
                     const double* orient3, double* normals_out, int32_t* count_out, void* workspace,
                     size_t workspace_bytes, cudaStream_t st) {
  DIB_REQUIRE(normals_out && orient3, "NULL argument (normals_out, orient3)");
  DIB_REQUIRE(std::isfinite(radius) && radius > 0.0, "radius must be positive (got %g)", radius);
  DIB_REQUIRE(max_nn >= 1 && max_nn <= kMaxNN, "max_nn=%d must be in [1, %d]", max_nn, kMaxNN);
  DIB_REQUIRE(std::isfinite(orient3[0]) && std::isfinite(orient3[1]) && std::isfinite(orient3[2]),
              "orient3 must be finite");
  const int rc = check_index(xyz, m_stride, S, workspace, workspace_bytes);
  if (rc != DIB_OK) return rc;
  if (S == 0) return DIB_OK;
  icp::Index ix;
  icp::carve_index((char*)workspace, 0, S, m_stride, &ix);
  const icp::Levels L = icp::make_levels(m_stride);
  const int rb = icp::build_index(xyz, m_pts, m_stride, S, L, ix, st);
  if (rb != DIB_OK) return rb;
  const NormArgs a{xyz, m_pts, m_stride, radius * radius, max_nn, {orient3[0], orient3[1], orient3[2]},
                   normals_out, count_out};
  const long long N = (long long)S * m_stride;
  const int nb = (int)((N + 127) / 128);
  if (max_nn <= 16)
    normals_kernel<16><<<nb, 128, 0, st>>>(a, L, ix, S);
  else if (max_nn <= 32)
    normals_kernel<32><<<nb, 128, 0, st>>>(a, L, ix, S);
  else
    normals_kernel<64><<<nb, 128, 0, st>>>(a, L, ix, S);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

int nearest_batch(const double* q, const int32_t* q_pts, int q_stride, const float* xyz, const int32_t* m_pts,
                  int m_stride, int S, int32_t* idx_out, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  DIB_REQUIRE(q && idx_out, "NULL argument (q, idx_out)");
  int rc = check_stride(q_stride, S, "q_stride");
  if (rc != DIB_OK) return rc;
  rc = check_index(xyz, m_stride, S, workspace, workspace_bytes);
  if (rc != DIB_OK) return rc;
  if (S == 0) return DIB_OK;
  icp::Index ix;
  icp::carve_index((char*)workspace, 0, S, m_stride, &ix);
  const icp::Levels L = icp::make_levels(m_stride);
  const int rb = icp::build_index(xyz, m_pts, m_stride, S, L, ix, st);
  if (rb != DIB_OK) return rb;
  const long long N = (long long)S * q_stride;
  nearest_kernel<<<(int)((N + 127) / 128), 128, 0, st>>>(q, q_pts, q_stride, m_pts, m_stride, S, L, ix, idx_out);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

// Test hook: sym3_eig_desc on n independent 3x3 matrices, one thread each, compiled as its callers are (--fmad=false).
__global__ void __launch_bounds__(128) sym3_eig_kernel(const double* __restrict__ C, int n, double* __restrict__ lam,
                                                       double* __restrict__ E) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  double c[9], l[3], e[9];
  for (int q = 0; q < 9; ++q) c[q] = C[(size_t)t * 9 + q];
  sym3_eig_desc(c, l, e);
  for (int q = 0; q < 3; ++q) lam[(size_t)t * 3 + q] = l[q];
  for (int q = 0; q < 9; ++q) E[(size_t)t * 9 + q] = e[q];
}

}  // namespace prep
}  // namespace dib

extern "C" {

size_t voxel_downsample_workspace_bytes(int S, int n_stride, int C) {
  (void)C;
  if (S < 0 || S > dib::prep::kMaxS || n_stride < 16) return 0;
  return dib::prep::carve_vox(nullptr, S, n_stride, nullptr);
}

int voxel_downsample_batch_f32(const float* xyz, const int32_t* n_pts, int n_stride, int S, const double* attr, int C,
                               double voxel_size, double* xyz_out, double* attr_out, int32_t* m_pts_out,
                               void* workspace, size_t workspace_bytes, dib_stream_t stream) {
  return dib::prep::voxel_downsample<float>(xyz, n_pts, n_stride, S, attr, C, voxel_size, xyz_out, attr_out,
                                            m_pts_out, workspace, workspace_bytes, (cudaStream_t)stream);
}

int voxel_downsample_batch_f64(const double* xyz, const int32_t* n_pts, int n_stride, int S, const double* attr, int C,
                               double voxel_size, double* xyz_out, double* attr_out, int32_t* m_pts_out,
                               void* workspace, size_t workspace_bytes, dib_stream_t stream) {
  return dib::prep::voxel_downsample<double>(xyz, n_pts, n_stride, S, attr, C, voxel_size, xyz_out, attr_out,
                                             m_pts_out, workspace, workspace_bytes, (cudaStream_t)stream);
}

size_t estimate_normals_workspace_bytes(int S, int m_stride) {
  if (S < 0 || S > dib::prep::kMaxS || m_stride < 16) return 0;
  return dib::icp::carve_index(nullptr, 0, S, m_stride, nullptr);
}

int estimate_normals_batch_f32(const float* xyz, const int32_t* m_pts, int m_stride, int S, double radius, int max_nn,
                               const double* orient3, double* normals_out, int32_t* count_out, void* workspace,
                               size_t workspace_bytes, dib_stream_t stream) {
  return dib::prep::estimate_normals(xyz, m_pts, m_stride, S, radius, max_nn, orient3, normals_out, count_out,
                                     workspace, workspace_bytes, (cudaStream_t)stream);
}

int nearest_batch_f32(const double* q, const int32_t* q_pts, int q_stride, const float* xyz, const int32_t* m_pts,
                      int m_stride, int S, int32_t* idx_out, void* workspace, size_t workspace_bytes,
                      dib_stream_t stream) {
  return dib::prep::nearest_batch(q, q_pts, q_stride, xyz, m_pts, m_stride, S, idx_out, workspace, workspace_bytes,
                                  (cudaStream_t)stream);
}

int sym3_eig_batch_f64(const double* C, int n, double* lam, double* E, dib_stream_t stream) {
  DIB_REQUIRE(C && lam && E, "NULL argument (C, lam, E)");
  DIB_REQUIRE(n >= 0, "bad sizes (n=%d)", n);
  if (n == 0) return DIB_OK;
  dib::prep::sym3_eig_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(C, n, lam, E);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

}  // extern "C"
