// Batched assembly of the classifier's point inputs: the part of the KITTI / Oxford loaders' __getitem__ after the
// scan records are read (data/kitti_pc_img_pose_loader.py:199-446, data/oxford_pc_img_pose_loader.py:262-352).
// DESIGN.md "Batch assembly" states the contract; oracle_assemble/ is its numpy restatement.
//
// accumulate  one thread per (frame, point): p' = T p in fp64 with a fixed association, rounded once to float32 (or
//             kept in fp64: assemble_accumulate_f64); normals get the rotation only; an optional float32 x / y
//             exclusion box on the source coordinates and an optional float32 range mask (x'^2 + z'^2 < r^2); a scan
//             over the keep flags compacts every sample's frames into one cloud in (frame, index) order
// resample    a 64-bit Philox key per point, a stable segmented radix sort by key (ties: ascending index); output o
//             takes o mod n while o < r n (the fixed repeats of downsample_np) and the (o - r n)-th point in key order
//             after that; float32 jitter from Box-Muller on Philox words; p' = M p in fp64, rounded to float32
// candidates  the 8 M smallest-key points of a sample, in ascending key order
// fps         farthest-point sampling: fp64 d2 = (dx dx + dy dy) + dz dz, running minimum, arg-max with the lowest
//             index on ties.  One CTA per set of up to 8192 points; larger sets (up to 65536) run on a thread-block
//             cluster of up to 8 CTAs that exchange each round's winner through distributed shared memory.
// Philox4x32-10 (common.cuh): key = seed, counter = (position, sample, stream id, 0); the stream ids are below.
// The file is compiled with --fmad=false (build.py NOFMA_SOURCES), so every operation rounds as the oracle's does.
#include <cfloat>
#include <climits>
#include <cmath>

#include <cooperative_groups.h>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_segmented_radix_sort.cuh>

#include "common.cuh"

namespace cg = cooperative_groups;

namespace dib {
namespace asmb {

// Philox stream ids (counter word 2).  DESIGN.md "Batch assembly" keeps the same table.
constexpr uint32_t kStreamResample = 1;
constexpr uint32_t kStreamJitterPc = 2;
constexpr uint32_t kStreamJitterSn = 3;
constexpr uint32_t kStreamNodeA = 4;
constexpr uint32_t kStreamNodeB = 5;
constexpr uint32_t kStreamJitterIntensity = 6;

constexpr int kMaxS = 65535;
constexpr int kSlice = 8192;          // FPS points per CTA
constexpr int kMaxCluster = 8;        // portable cluster size
constexpr int kMaxFps = kSlice * kMaxCluster;
constexpr int kPPT = 8;               // FPS points per thread
constexpr int kJitterPc = 1, kJitterSn = 2, kJitterIntensity = 4;

__host__ __device__ inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }
constexpr size_t kScratch = (size_t)4 << 20;   // cub scan / segmented-sort scratch (a few KB in practice)

__device__ __forceinline__ int clamp_count(const int32_t* n, int s, int stride) {
  if (!n) return stride;
  const int v = n[s];
  return v < 0 ? 0 : (v > stride ? stride : v);
}

__device__ __forceinline__ void philox(uint32_t w[4], uint32_t pos, uint32_t s, uint32_t stream, uint64_t seed) {
  w[0] = pos; w[1] = s; w[2] = stream; w[3] = 0u;
  philox4x32_10(w, (uint32_t)seed, (uint32_t)(seed >> 32));
}

// (w + 0.5) 2^-32: a uniform in (0, 1), never 0 or 1.
__device__ __forceinline__ double unit(uint32_t w) { return ((double)w + 0.5) * 2.3283064365386963e-10; }

// Box-Muller on the four words of one Philox call: z0 = r0 cos(t0), z1 = r0 sin(t0), z2 = r1 cos(t1), with
// r_i = sqrt(-2 log u(w_2i)), t_i = 2 pi u(w_2i+1).
__device__ __forceinline__ void normals3(const uint32_t w[4], double z[3]) {
  const double r0 = sqrt(-2.0 * log(unit(w[0]))), t0 = 6.283185307179586 * unit(w[1]);
  const double r1 = sqrt(-2.0 * log(unit(w[2]))), t1 = 6.283185307179586 * unit(w[3]);
  z[0] = r0 * cos(t0);
  z[1] = r0 * sin(t0);
  z[2] = r1 * cos(t1);
}

// np.clip(sigma * z, -clip, clip).astype(float32)
__device__ __forceinline__ float jitter_of(double z, double sigma, double clip) {
  double j = sigma * z;
  j = j < -clip ? -clip : (j > clip ? clip : j);
  return (float)j;
}

__device__ __forceinline__ double affine_row(const double* M, int r, double x, double y, double z) {
  return ((M[r * 4] * x + M[r * 4 + 1] * y) + M[r * 4 + 2] * z) + M[r * 4 + 3];
}
__device__ __forceinline__ double rot_row(const double* M, int r, double x, double y, double z) {
  return (M[r * 4] * x + M[r * 4 + 1] * y) + M[r * 4 + 2] * z;
}

// ---------------------------------------------------------------------------------------------------------------
// Accumulation.

struct AccWork {
  int32_t* flag;        // [T * n_stride + 1]
  int32_t* pos;         // [T * n_stride + 1] exclusive scan of flag
  int32_t* first;       // [S + 1] first frame of each sample (lower bound in frame_sample)
  void* tmp;
};

size_t carve_acc(char* base, int T, int n_stride, int S, AccWork* wk) {
  const size_t N = (size_t)T * n_stride + 1;
  size_t off = 0;
  auto take = [&](size_t bytes) { char* p = base ? base + off : nullptr; off += align256(bytes); return p; };
  AccWork w;
  w.flag = (int32_t*)take(N * 4);
  w.pos = (int32_t*)take(N * 4);
  w.first = (int32_t*)take(((size_t)S + 1) * 4);
  w.tmp = take(kScratch);
  if (wk) *wk = w;
  return off;
}

struct AccArgs {
  const float *xyz, *intensity, *sn;
  const int32_t* n_pts;
  int n_stride, T;
  const int32_t* frame_sample;
  const double* frame_T;     // [T][16]
  int S;
  float range2;              // <= 0: no mask
  bool box;                  // drop source points with x_lo < x < x_hi and y_lo < y < y_hi (float32 compares)
  float x_lo, x_hi, y_lo, y_hi;
  float *xyz_out, *intensity_out, *sn_out;
  double* xyz64_out;         // the fp64 variant's coordinates (instead of xyz_out; no sn)
  int out_stride;
};

__device__ __forceinline__ void acc_point(const AccArgs& a, int t, int j, double p[3]) {
  const double* M = a.frame_T + (size_t)t * 16;
  const float* X = a.xyz + (size_t)t * 3 * a.n_stride;
  const double x = X[j], y = X[(size_t)a.n_stride + j], z = X[(size_t)2 * a.n_stride + j];
  for (int r = 0; r < 3; ++r) p[r] = affine_row(M, r, x, y, z);
}

__global__ void acc_flag_kernel(AccArgs a, int32_t* __restrict__ flag) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long N = (long long)a.T * a.n_stride;
  if (g > N) return;
  int f = 0;
  if (g < N) {
    const int t = (int)(g / a.n_stride), j = (int)(g - (long long)t * a.n_stride);
    const int s = a.frame_sample[t];
    if (j < clamp_count(a.n_pts, t, a.n_stride) && s >= 0 && s < a.S) {
      f = 1;
      if (a.box) {
        const float* X = a.xyz + (size_t)t * 3 * a.n_stride;
        const float x = X[j], y = X[(size_t)a.n_stride + j];
        f = !(x > a.x_lo && x < a.x_hi && y > a.y_lo && y < a.y_hi);
      }
      if (f && a.range2 > 0.0f) {
        double p[3];
        acc_point(a, t, j, p);
        const float px = (float)p[0], pz = (float)p[2];
        f = px * px + pz * pz < a.range2;
      }
    }
  }
  flag[g] = f;
}

// first[s] = the first frame whose sample is >= s (frame_sample is non-decreasing); first[S] = T.
__global__ void acc_first_kernel(const int32_t* __restrict__ frame_sample, int T, int S, int32_t* __restrict__ first) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s > S) return;
  int lo = 0, hi = T;
  while (lo < hi) {
    const int m = (lo + hi) >> 1;
    if (frame_sample[m] < s) lo = m + 1; else hi = m;
  }
  first[s] = s == S ? T : lo;
}

template <bool F64>
__global__ void acc_scatter_kernel(AccArgs a, const int32_t* __restrict__ flag, const int32_t* __restrict__ pos,
                                   const int32_t* __restrict__ first, int32_t* __restrict__ count_out) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g < a.S) {
    const int s = (int)g;
    count_out[s] = pos[(size_t)first[s + 1] * a.n_stride] - pos[(size_t)first[s] * a.n_stride];
  }
  if (g >= (long long)a.T * a.n_stride || !flag[g]) return;
  const int t = (int)(g / a.n_stride), j = (int)(g - (long long)t * a.n_stride);
  const int s = a.frame_sample[t];
  const int o = pos[g] - pos[(size_t)first[s] * a.n_stride];
  if (o < 0 || o >= a.out_stride) return;
  double p[3];
  acc_point(a, t, j, p);
  for (int r = 0; r < 3; ++r) {
    if constexpr (F64)
      a.xyz64_out[((size_t)s * 3 + r) * a.out_stride + o] = p[r];
    else
      a.xyz_out[((size_t)s * 3 + r) * a.out_stride + o] = (float)p[r];
  }
  a.intensity_out[(size_t)s * a.out_stride + o] = a.intensity[(size_t)t * a.n_stride + j];
  if (a.sn) {
    const double* M = a.frame_T + (size_t)t * 16;
    const float* Nn = a.sn + (size_t)t * 3 * a.n_stride;
    const double x = Nn[j], y = Nn[(size_t)a.n_stride + j], z = Nn[(size_t)2 * a.n_stride + j];
    for (int r = 0; r < 3; ++r) a.sn_out[((size_t)s * 3 + r) * a.out_stride + o] = (float)rot_row(M, r, x, y, z);
  }
}

template <bool F64>
int accumulate(const AccArgs& a, int32_t* count_out, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  DIB_REQUIRE(a.xyz && a.intensity && a.frame_sample && a.frame_T && (F64 ? (void*)a.xyz64_out : (void*)a.xyz_out) &&
              a.intensity_out && count_out,
              "NULL argument (xyz, intensity, frame_sample, frame_T, xyz_out, intensity_out, count_out)");
  DIB_REQUIRE(!a.sn || a.sn_out, "NULL argument (sn_out with sn)");
  DIB_REQUIRE(!a.box || (std::isfinite(a.x_lo) && std::isfinite(a.x_hi) && std::isfinite(a.y_lo) &&
                         std::isfinite(a.y_hi) && a.x_lo <= a.x_hi && a.y_lo <= a.y_hi),
              "exclude_box must be finite with x_lo <= x_hi and y_lo <= y_hi");
  DIB_REQUIRE(a.T >= 0 && a.S >= 0 && a.S <= kMaxS, "T=%d, S=%d: need T >= 0 and 0 <= S <= %d", a.T, a.S, kMaxS);
  DIB_REQUIRE(a.n_stride >= 1 && a.out_stride >= 1, "n_stride and out_stride must be positive");
  DIB_REQUIRE((long long)a.T * a.n_stride < (1LL << 31) - 1 && (long long)a.S * a.out_stride < (1LL << 31),
              "T * n_stride and S * out_stride must be below 2^31");
  const size_t need = carve_acc(nullptr, a.T, a.n_stride, a.S, nullptr);
  DIB_REQUIRE(workspace && workspace_bytes >= need, "workspace too small (%zu < %zu)", workspace_bytes, need);
  DIB_REQUIRE(((uintptr_t)workspace & 255) == 0, "workspace must be 256-byte aligned");
  if (a.S == 0) return DIB_OK;
  AccWork wk;
  carve_acc((char*)workspace, a.T, a.n_stride, a.S, &wk);
  const long long N = (long long)a.T * a.n_stride + 1;
  const int nb = (int)((N + 255) / 256);
  acc_flag_kernel<<<nb, 256, 0, st>>>(a, wk.flag);
  acc_first_kernel<<<(a.S + 1 + 127) / 128, 128, 0, st>>>(a.frame_sample, a.T, a.S, wk.first);
  DIB_CHECK_CUDA(cudaGetLastError());
  size_t tmp = 0;
  DIB_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp, wk.flag, wk.pos, (int)N, st));
  DIB_REQUIRE(tmp <= kScratch, "accumulate: scan scratch %zu exceeds %zu", tmp, kScratch);
  DIB_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(wk.tmp, tmp, wk.flag, wk.pos, (int)N, st));
  const long long M = N - 1 > a.S ? N - 1 : a.S;
  acc_scatter_kernel<F64><<<(int)((M + 255) / 256), 256, 0, st>>>(a, wk.flag, wk.pos, wk.first, count_out);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Key order: per sample, the points sorted by (64-bit Philox key, index).

struct SortWork {
  unsigned long long *key0, *key1;
  int32_t *val0, *val1;
  int32_t* seg;           // [S + 1] segment offsets s * n_stride
  void* tmp;
};

size_t carve_sort(char* base, int S, int n_stride, SortWork* wk) {
  const size_t N = (size_t)S * n_stride;
  size_t off = 0;
  auto take = [&](size_t bytes) { char* p = base ? base + off : nullptr; off += align256(bytes); return p; };
  SortWork w;
  w.key0 = (unsigned long long*)take(N * 8); w.key1 = (unsigned long long*)take(N * 8);
  w.val0 = (int32_t*)take(N * 4); w.val1 = (int32_t*)take(N * 4);
  w.seg = (int32_t*)take(((size_t)S + 1) * 4);
  w.tmp = take(kScratch);
  if (wk) *wk = w;
  return off;
}

// Padding entries (j >= n) get the largest key and sort after the sample's points (a point whose key is also
// ~0 keeps its place before them: the sort is stable and the points come first in index order).
__global__ void key_kernel(const int32_t* __restrict__ n_pts, int n_stride, int S, uint64_t seed, uint32_t stream,
                           unsigned long long* __restrict__ key, int32_t* __restrict__ val, int32_t* __restrict__ seg) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g <= S) seg[g] = (int32_t)(g * n_stride);
  if (g >= (long long)S * n_stride) return;
  const int s = (int)(g / n_stride), j = (int)(g - (long long)s * n_stride);
  unsigned long long k = ~0ull;
  if (j < clamp_count(n_pts, s, n_stride)) {
    uint32_t w[4];
    philox(w, (uint32_t)j, (uint32_t)s, stream, seed);
    k = ((unsigned long long)w[0] << 32) | w[1];
  }
  key[g] = k;
  val[g] = j;
}

// Returns the sorted local indices (val) of every sample at [s * n_stride, (s + 1) * n_stride).
int key_order(const int32_t* n_pts, int n_stride, int S, uint64_t seed, uint32_t stream, const SortWork& wk,
              const int32_t** sorted, cudaStream_t st) {
  const long long N = (long long)S * n_stride;
  key_kernel<<<(int)((N + 1 + 255) / 256), 256, 0, st>>>(n_pts, n_stride, S, seed, stream, wk.key0, wk.val0, wk.seg);
  DIB_CHECK_CUDA(cudaGetLastError());
  cub::DoubleBuffer<unsigned long long> keys(wk.key0, wk.key1);
  cub::DoubleBuffer<int32_t> vals(wk.val0, wk.val1);
  size_t tmp = 0;
  DIB_CHECK_CUDA(cub::DeviceSegmentedRadixSort::SortPairs(nullptr, tmp, keys, vals, (int)N, S, wk.seg, wk.seg + 1, 0,
                                                          64, st));
  if (tmp > kScratch) {
    set_error("assemble: the segmented sort needs %zu bytes of scratch, %zu reserved", tmp, kScratch);
    return DIB_ENOMEM;
  }
  DIB_CHECK_CUDA(cub::DeviceSegmentedRadixSort::SortPairs(wk.tmp, tmp, keys, vals, (int)N, S, wk.seg, wk.seg + 1, 0,
                                                          64, st));
  *sorted = vals.Current();
  return DIB_OK;
}

int check_sort_shape(int S, int n_stride, void* workspace, size_t workspace_bytes) {
  DIB_REQUIRE(S >= 0 && S <= kMaxS, "S=%d must be in [0, %d]", S, kMaxS);
  DIB_REQUIRE(n_stride >= 1 && (long long)S * n_stride < (1LL << 31) - 1, "S * n_stride must be below 2^31");
  const size_t need = carve_sort(nullptr, S, n_stride, nullptr);
  DIB_REQUIRE(workspace && workspace_bytes >= need, "workspace too small (%zu < %zu)", workspace_bytes, need);
  DIB_REQUIRE(((uintptr_t)workspace & 255) == 0, "workspace must be 256-byte aligned");
  return DIB_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Resample + jitter + transform.

struct ResArgs {
  const float *xyz, *intensity, *sn;
  const int32_t* n_pts;
  int n_stride, S, N;
  uint64_t seed;
  const double* M;            // [S][16]
  double sigma, clip;
  int jitter;
  float *xyz_out, *intensity_out, *sn_out;
  int32_t* src_out;
};

__global__ void resample_kernel(ResArgs a, const int32_t* __restrict__ sorted) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)a.S * a.N) return;
  const int s = (int)(g / a.N), o = (int)(g - (long long)s * a.N);
  const int n = clamp_count(a.n_pts, s, a.n_stride);
  if (n < 1) {
    a.src_out[g] = -1;
    return;
  }
  int j;
  if (n >= a.N) {
    j = sorted[(size_t)s * a.n_stride + o];
  } else {
    const int r = (a.N + n - 1) / n - 1;         // smallest r >= 1 with (r + 1) n >= N
    j = o < r * n ? o % n : sorted[(size_t)s * a.n_stride + (o - r * n)];
  }
  a.src_out[g] = j;
  const double* M = a.M + (size_t)s * 16;
  const float* X = a.xyz + (size_t)s * 3 * a.n_stride;
  float p[3] = {X[j], X[(size_t)a.n_stride + j], X[(size_t)2 * a.n_stride + j]};
  uint32_t w[4];
  double z[3];
  if (a.jitter & kJitterPc) {
    philox(w, (uint32_t)o, (uint32_t)s, kStreamJitterPc, a.seed);
    normals3(w, z);
    for (int r = 0; r < 3; ++r) p[r] = p[r] + jitter_of(z[r], a.sigma, a.clip);
  }
  for (int r = 0; r < 3; ++r)
    a.xyz_out[((size_t)s * 3 + r) * a.N + o] = (float)affine_row(M, r, p[0], p[1], p[2]);
  float in = a.intensity[(size_t)s * a.n_stride + j];
  if (a.jitter & kJitterIntensity) {
    philox(w, (uint32_t)o, (uint32_t)s, kStreamJitterIntensity, a.seed);
    normals3(w, z);
    in = in + jitter_of(z[0], a.sigma, a.clip);
  }
  a.intensity_out[g] = in;
  if (a.sn_out) {
    float q[3] = {0.0f, 0.0f, 0.0f};
    if (a.sn) {
      const float* Nn = a.sn + (size_t)s * 3 * a.n_stride;
      q[0] = Nn[j]; q[1] = Nn[(size_t)a.n_stride + j]; q[2] = Nn[(size_t)2 * a.n_stride + j];
      if (a.jitter & kJitterSn) {
        philox(w, (uint32_t)o, (uint32_t)s, kStreamJitterSn, a.seed);
        normals3(w, z);
        for (int r = 0; r < 3; ++r) q[r] = q[r] + jitter_of(z[r], a.sigma, a.clip);
      }
    }
    for (int r = 0; r < 3; ++r)
      a.sn_out[((size_t)s * 3 + r) * a.N + o] = (float)rot_row(M, r, q[0], q[1], q[2]);
  }
}

int resample(const ResArgs& a, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  DIB_REQUIRE(a.xyz && a.intensity && a.M && a.xyz_out && a.intensity_out && a.src_out,
              "NULL argument (xyz, intensity, M16, xyz_out, intensity_out, src_out)");
  DIB_REQUIRE(a.N >= 1, "input_pt_num=%d must be at least 1", a.N);
  DIB_REQUIRE((long long)a.S * a.N < (1LL << 31), "S * input_pt_num must be below 2^31");
  DIB_REQUIRE(a.jitter >= 0 && a.jitter <= 7, "jitter=%d is a mask of 1 (pc), 2 (sn), 4 (intensity)", a.jitter);
  DIB_REQUIRE(!(a.jitter & kJitterSn) || a.sn, "sn jitter needs sn");
  DIB_REQUIRE(std::isfinite(a.sigma) && std::isfinite(a.clip) && a.clip > 0.0, "sigma, clip must be finite, clip > 0");
  const int rc = check_sort_shape(a.S, a.n_stride, workspace, workspace_bytes);
  if (rc != DIB_OK) return rc;
  if (a.S == 0) return DIB_OK;
  SortWork wk;
  carve_sort((char*)workspace, a.S, a.n_stride, &wk);
  const int32_t* sorted = nullptr;
  const int rs = key_order(a.n_pts, a.n_stride, a.S, a.seed, kStreamResample, wk, &sorted, st);
  if (rs != DIB_OK) return rs;
  const long long G = (long long)a.S * a.N;
  resample_kernel<<<(int)((G + 255) / 256), 256, 0, st>>>(a, sorted);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Candidate sets: the m smallest-key points of each sample.

__global__ void candidates_kernel(const float* __restrict__ pc, int N, int S, int m, const int32_t* __restrict__ sorted,
                                  int32_t* __restrict__ idx_out, float* __restrict__ xyz_out) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)S * m) return;
  const int s = (int)(g / m), c = (int)(g - (long long)s * m);
  const int j = sorted[(size_t)s * N + c];
  idx_out[g] = j;
  for (int r = 0; r < 3; ++r) xyz_out[((size_t)s * 3 + r) * m + c] = pc[((size_t)s * 3 + r) * N + j];
}

int candidates(const float* pc, int N, int S, uint64_t seed, int node_set, int m, int32_t* idx_out, float* xyz_out,
               void* workspace, size_t workspace_bytes, cudaStream_t st) {
  DIB_REQUIRE(pc && idx_out && xyz_out, "NULL argument (pc, idx_out, xyz_out)");
  DIB_REQUIRE(node_set == 0 || node_set == 1, "node_set=%d must be 0 (node_a) or 1 (node_b)", node_set);
  DIB_REQUIRE(N >= 1 && m >= 1 && m <= N, "need 1 <= m (%d) <= N (%d)", m, N);
  const int rc = check_sort_shape(S, N, workspace, workspace_bytes);
  if (rc != DIB_OK) return rc;
  if (S == 0) return DIB_OK;
  SortWork wk;
  carve_sort((char*)workspace, S, N, &wk);
  const int32_t* sorted = nullptr;
  const int rs = key_order(nullptr, N, S, seed, node_set ? kStreamNodeB : kStreamNodeA, wk, &sorted, st);
  if (rs != DIB_OK) return rs;
  const long long G = (long long)S * m;
  candidates_kernel<<<(int)((G + 255) / 256), 256, 0, st>>>(pc, N, S, m, sorted, idx_out, xyz_out);
  DIB_CHECK_CUDA(cudaGetLastError());
  return DIB_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Farthest-point sampling.

template <typename T>
struct Winner {
  double d;
  int i;
  T p[3];
};

__device__ __forceinline__ bool beats(double d, int i, double bd, int bi) { return d > bd || (d == bd && i < bi); }

// Set s runs on blockIdx.y; with CLUSTER the cluster of gridDim.x CTAs splits it into slices of kSlice points.
// Each thread keeps the running minima of its kPPT points in registers; coordinates live in shared memory.
template <typename T, bool CLUSTER>
__global__ void __launch_bounds__(1024) fps_kernel(const T* __restrict__ xyz, const int32_t* __restrict__ n_pts,
                                                   int n_stride, int k, int cap, const int32_t* __restrict__ start,
                                                   int32_t* __restrict__ idx_out, T* __restrict__ nodes_out) {
  extern __shared__ __align__(16) unsigned char smem[];
  T* sp = reinterpret_cast<T*>(smem);                                       // [3][cap]
  Winner<T>* slot = reinterpret_cast<Winner<T>*>(smem + align256((size_t)3 * cap * sizeof(T)));   // [2]
  double* wd = reinterpret_cast<double*>(slot + 2);                         // [2][32]
  int* wi = reinterpret_cast<int*>(wd + 64);                                // [2][32]
  const int s = blockIdx.y;
  const int rank = CLUSTER ? (int)cg::this_cluster().block_rank() : 0;
  const int nc = CLUSTER ? (int)gridDim.x : 1;
  const int n = clamp_count(n_pts, s, n_stride);
  const int lo = rank * cap;
  const int cnt = max(0, min(n - lo, cap));
  const T* X = xyz + (size_t)s * 3 * n_stride;
  const int tid = threadIdx.x, bd = blockDim.x, lane = tid & 31, warp = tid >> 5, nw = (bd + 31) >> 5;
  if (n < 1) {                  // uniform over the cluster: no barrier is skipped by part of it
    if (rank == 0)
      for (int i = tid; i < k; i += bd) {
        idx_out[(size_t)s * k + i] = -1;
        for (int r = 0; r < 3; ++r) nodes_out[((size_t)s * 3 + r) * k + i] = T(0);
      }
    return;
  }
  for (int li = tid; li < cnt; li += bd)
    for (int r = 0; r < 3; ++r) sp[r * cap + li] = X[(size_t)r * n_stride + lo + li];
  double dmin[kPPT];
#pragma unroll
  for (int q = 0; q < kPPT; ++q) dmin[q] = DBL_MAX;
  int w = start ? start[s] : 0;
  if (w < 0 || w >= n) w = 0;
  T wp[3] = {X[w], X[(size_t)n_stride + w], X[(size_t)2 * n_stride + w]};
  __syncthreads();
  for (int i = 0;; ++i) {
    if (rank == 0 && tid == 0) {
      idx_out[(size_t)s * k + i] = w;
      for (int r = 0; r < 3; ++r) nodes_out[((size_t)s * 3 + r) * k + i] = wp[r];
    }
    if (i == k - 1) break;
    const int par = i & 1;
    const double px = (double)wp[0], py = (double)wp[1], pz = (double)wp[2];
    double bd_ = -1.0;
    int bi = INT_MAX;
#pragma unroll
    for (int q = 0; q < kPPT; ++q) {
      const int li = tid + q * bd;
      if (li < cnt) {
        const double dx = px - (double)sp[li], dy = py - (double)sp[cap + li], dz = pz - (double)sp[2 * cap + li];
        const double d = (dx * dx + dy * dy) + dz * dz;
        dmin[q] = d < dmin[q] ? d : dmin[q];
        if (dmin[q] > bd_) { bd_ = dmin[q]; bi = lo + li; }
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const double od = __shfl_down_sync(0xffffffffu, bd_, off);
      const int oi = __shfl_down_sync(0xffffffffu, bi, off);
      if (beats(od, oi, bd_, bi)) { bd_ = od; bi = oi; }
    }
    if (lane == 0) { wd[par * 32 + warp] = bd_; wi[par * 32 + warp] = bi; }
    __syncthreads();
    bd_ = wd[par * 32]; bi = wi[par * 32];
    for (int v = 1; v < nw; ++v)
      if (beats(wd[par * 32 + v], wi[par * 32 + v], bd_, bi)) { bd_ = wd[par * 32 + v]; bi = wi[par * 32 + v]; }
    if constexpr (CLUSTER) {
      cg::cluster_group cl = cg::this_cluster();
      if (tid == 0) {
        Winner<T>& my = slot[par];
        my.d = bd_; my.i = bi;
        const int li = bi == INT_MAX ? 0 : bi - lo;
        for (int r = 0; r < 3; ++r) my.p[r] = sp[r * cap + li];
      }
      cl.sync();
      int from = 0;
      for (int c = 0; c < nc; ++c) {
        const Winner<T>* o = cl.map_shared_rank(&slot[par], c);
        const double od = o->d;
        const int oi = o->i;
        if (c == 0 || beats(od, oi, bd_, bi)) { bd_ = od; bi = oi; from = c; }
      }
      const Winner<T>* o = cl.map_shared_rank(&slot[par], from);
      for (int r = 0; r < 3; ++r) wp[r] = o->p[r];
    } else {
      for (int r = 0; r < 3; ++r) wp[r] = sp[r * cap + bi];
    }
    w = bi;
  }
  if constexpr (CLUSTER) cg::this_cluster().sync();     // peers may still read this CTA's last winner
}

inline int fps_threads(int cap) {
  int t = (cap + kPPT - 1) / kPPT;
  t = (t + 31) / 32 * 32;
  return t < 32 ? 32 : (t > 1024 ? 1024 : t);
}

template <typename T>
size_t fps_smem(int cap) {
  return align256((size_t)3 * cap * sizeof(T)) + 2 * sizeof(Winner<T>) + 64 * sizeof(double) + 64 * sizeof(int);
}

template <typename T>
int fps(const T* xyz, const int32_t* n_pts, int n_stride, int S, int k, const int32_t* start, int32_t* idx_out,
        T* nodes_out, cudaStream_t st) {
  DIB_REQUIRE(xyz && idx_out && nodes_out, "NULL argument (xyz, idx_out, nodes_out)");
  DIB_REQUIRE(S >= 0 && S <= kMaxS, "S=%d must be in [0, %d]", S, kMaxS);
  DIB_REQUIRE(n_stride >= 1 && n_stride <= kMaxFps, "n_stride=%d: farthest-point sampling takes 1 to %d points",
              n_stride, kMaxFps);
  DIB_REQUIRE(k >= 1 && k <= n_stride, "k=%d must be in [1, n_stride=%d]", k, n_stride);
  if (S == 0) return DIB_OK;
  if (n_stride <= kSlice) {
    const int cap = n_stride;
    const size_t sm = fps_smem<T>(cap);
    auto kern = fps_kernel<T, false>;
    DIB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
    kern<<<dim3(1, S), fps_threads(cap), sm, st>>>(xyz, n_pts, n_stride, k, cap, start, idx_out, nodes_out);
    DIB_CHECK_CUDA(cudaGetLastError());
    return DIB_OK;
  }
  const int nc = (n_stride + kSlice - 1) / kSlice;
  const int cap = kSlice;
  const size_t sm = fps_smem<T>(cap);
  auto kern = fps_kernel<T, true>;
  DIB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(nc, S);
  cfg.blockDim = dim3(fps_threads(cap));
  cfg.dynamicSmemBytes = sm;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = nc;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  DIB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kern, xyz, n_pts, n_stride, k, cap, start, idx_out, nodes_out));
  return DIB_OK;
}

}  // namespace asmb
}  // namespace dib

extern "C" {

size_t assemble_accumulate_workspace_bytes(int T, int n_stride, int S) {
  if (T < 0 || n_stride < 1 || S < 0 || S > dib::asmb::kMaxS) return 0;
  return dib::asmb::carve_acc(nullptr, T, n_stride, S, nullptr);
}

int assemble_accumulate_f32(const float* xyz, const float* intensity, const float* sn, const int32_t* n_pts,
                            int n_stride, int T, const int32_t* frame_sample, const double* frame_T16, int S,
                            double range_max, float* xyz_out, float* intensity_out, float* sn_out, int out_stride,
                            int32_t* count_out, void* workspace, size_t workspace_bytes, dib_stream_t stream) {
  DIB_REQUIRE(std::isfinite(range_max), "range_max must be finite (<= 0: no range mask)");
  const float r2 = range_max > 0.0 ? (float)(range_max * range_max) : 0.0f;
  const dib::asmb::AccArgs a{xyz, intensity, sn, n_pts, n_stride, T, frame_sample, frame_T16, S, r2, false,
                             0.0f, 0.0f, 0.0f, 0.0f, xyz_out, intensity_out, sn_out, nullptr, out_stride};
  return dib::asmb::accumulate<false>(a, count_out, workspace, workspace_bytes, (cudaStream_t)stream);
}

size_t assemble_accumulate_f64_workspace_bytes(int T, int n_stride, int S) {
  return assemble_accumulate_workspace_bytes(T, n_stride, S);
}

int assemble_accumulate_f64(const float* xyz, const float* intensity, const int32_t* n_pts, int n_stride, int T,
                            const int32_t* frame_sample, const double* frame_T16, int S, double range_max,
                            const float* exclude_box, double* xyz_out, float* intensity_out, int out_stride,
                            int32_t* count_out, void* workspace, size_t workspace_bytes, dib_stream_t stream) {
  DIB_REQUIRE(std::isfinite(range_max), "range_max must be finite (<= 0: no range mask)");
  const float r2 = range_max > 0.0 ? (float)(range_max * range_max) : 0.0f;
  const float* b = exclude_box;
  const dib::asmb::AccArgs a{xyz, intensity, nullptr, n_pts, n_stride, T, frame_sample, frame_T16, S, r2, b != nullptr,
                             b ? b[0] : 0.0f, b ? b[1] : 0.0f, b ? b[2] : 0.0f, b ? b[3] : 0.0f, nullptr,
                             intensity_out, nullptr, xyz_out, out_stride};
  return dib::asmb::accumulate<true>(a, count_out, workspace, workspace_bytes, (cudaStream_t)stream);
}

size_t assemble_resample_workspace_bytes(int S, int n_stride) {
  if (S < 0 || S > dib::asmb::kMaxS || n_stride < 1) return 0;
  return dib::asmb::carve_sort(nullptr, S, n_stride, nullptr);
}

int assemble_resample_f32(const float* xyz, const float* intensity, const float* sn, const int32_t* n_pts,
                          int n_stride, int S, int input_pt_num, uint64_t seed, const double* M16, double sigma,
                          double clip, int jitter, float* xyz_out, float* intensity_out, float* sn_out,
                          int32_t* src_out, void* workspace, size_t workspace_bytes, dib_stream_t stream) {
  const dib::asmb::ResArgs a{xyz, intensity, sn, n_pts, n_stride, S, input_pt_num, seed, M16, sigma, clip, jitter,
                             xyz_out, intensity_out, sn_out, src_out};
  return dib::asmb::resample(a, workspace, workspace_bytes, (cudaStream_t)stream);
}

size_t assemble_candidates_workspace_bytes(int S, int N) {
  if (S < 0 || S > dib::asmb::kMaxS || N < 1) return 0;
  return dib::asmb::carve_sort(nullptr, S, N, nullptr);
}

int assemble_candidates_f32(const float* pc, int N, int S, uint64_t seed, int node_set, int m, int32_t* idx_out,
                            float* xyz_out, void* workspace, size_t workspace_bytes, dib_stream_t stream) {
  return dib::asmb::candidates(pc, N, S, seed, node_set, m, idx_out, xyz_out, workspace, workspace_bytes,
                               (cudaStream_t)stream);
}

int fps_batch_f32(const float* xyz, const int32_t* n_pts, int n_stride, int S, int k, const int32_t* start,
                  int32_t* idx_out, float* nodes_out, dib_stream_t stream) {
  return dib::asmb::fps<float>(xyz, n_pts, n_stride, S, k, start, idx_out, nodes_out, (cudaStream_t)stream);
}

int fps_batch_f64(const double* xyz, const int32_t* n_pts, int n_stride, int S, int k, const int32_t* start,
                  int32_t* idx_out, double* nodes_out, dib_stream_t stream) {
  return dib::asmb::fps<double>(xyz, n_pts, n_stride, S, k, start, idx_out, nodes_out, (cudaStream_t)stream);
}

}  // extern "C"
