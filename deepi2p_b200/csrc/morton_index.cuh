// Exact nearest-neighbour index over batched float32 clouds, shared by icp.cu (correspondences) and pointprep.cu
// (normal estimation and intensity transfer).  The build kernels live in icp.cu; this header declares them and holds
// the device-side descents.
//
// Per cloud s: the points are sorted by 48-bit Morton code within the cloud's box (one radix sort for the whole
// batch; the order only affects speed, never a result), stored as float4 (x, y, z, original index), and covered by an
// implicit binary tree of boxes: leaf k holds sorted points [16k, 16k + 16), node k of level l covers nodes 2k and
// 2k + 1 of level l - 1.  Counts follow from m alone: ceil(m / (16 << l)).
#pragma once
#include <cfloat>
#include <climits>

#include "common.cuh"

namespace dib {
namespace icp {

constexpr int kLeaf = 16;             // sorted points per leaf box
constexpr int kLeafShift = 4;
constexpr int kMaxLevels = 28;
constexpr int kStack = 32;
// A descent pushes at most two children per popped node and pops one, so the stack never holds more than one entry
// per level plus the root's.
static_assert(kStack > kMaxLevels + 1, "the descent stack must hold one entry per level");
static_assert(kMaxLevels <= 32, "a stack entry keeps the level in 5 bits");

struct Levels {
  int n;                    // levels of a full cloud (m = m_stride)
  int off[kMaxLevels];      // first node of level l within a cloud's node array
  int per_frame;            // nodes per cloud
};

// The index's device buffers (carved from a caller's workspace).
struct Index {
  float* bbox;              // [S][6]
  unsigned long long *key0, *key1;
  int32_t *val0, *val1;
  float4* pts;              // [S][m_stride]
  float4 *lo, *hi;          // [S][per_frame]
  void* sort_tmp;
  size_t sort_tmp_bytes;
};

__host__ __device__ inline int level_count(int m, int l) {
  return (int)(((long long)m + ((long long)kLeaf << l) - 1) >> (kLeafShift + l));
}

__device__ __forceinline__ int clamp_n(const int32_t* n, int s, int stride) {
  if (!n) return stride;
  const int v = n[s];
  return v < 0 ? 0 : (v > stride ? stride : v);
}

Levels make_levels(int m_stride);
// Per-cloud bounding box (lo xyz, hi xyz) of the first n_pts[s] points into bbox [S][6]; an empty cloud gives
// lo = FLT_MAX, hi = -FLT_MAX.  Enqueued on st.
void cloud_bbox(const float* X, const int32_t* n_pts, int stride, int S, float* bbox, cudaStream_t st);
// Carves the index of S clouds of m_stride points from base + off (base may be NULL); returns the offset after it.
size_t carve_index(char* base, size_t off, int S, int m_stride, Index* ix);
// bbox, Morton keys, radix sort, gather, one launch per tree level; enqueued on st.
int build_index(const float* tgt, const int32_t* m_pts, int m_stride, int S, const Levels& L, Index& ix,
                cudaStream_t st);

// ---------------------------------------------------------------------------------------------------------------
// Exact searches.  A box's lower bound is formed from its float corners with the same operations as d2, so it never
// exceeds the d2 of a point inside it (rounding is monotone); a box is skipped only when its bound is strictly above
// the search's bound, so an equally distant point of lower index is still found.

__device__ __forceinline__ double box_lb(const float4& lo, const float4& hi, double qx, double qy, double qz) {
  const double dx = fmax(fmax((double)lo.x - qx, qx - (double)hi.x), 0.0);
  const double dy = fmax(fmax((double)lo.y - qy, qy - (double)hi.y), 0.0);
  const double dz = fmax(fmax((double)lo.z - qz, qz - (double)hi.z), 0.0);
  return (dx * dx + dy * dy) + dz * dz;
}

struct Hit {
  double d2;
  int j;
  float x, y, z;
};

// The nearest point (ties -> lowest index) with d2 <= the caller's bound h.d2; h.j = INT_MAX when there is none.
__device__ __forceinline__ void nearest(const float4* __restrict__ pts, const float4* __restrict__ lo,
                                        const float4* __restrict__ hi, const Levels& L, int m, int root, double qx,
                                        double qy, double qz, Hit& h, unsigned long long& evals) {
  h.j = INT_MAX;            // h.d2 holds the caller's bound (r^2): nothing at or beyond it can be a correspondence
  if (m <= 0) return;
  unsigned st_node[kStack];   // (node << 5) | level: node < 2^27 and level < 32 for every admitted m_stride
  double st_lb[kStack];
  int sp = 0;
  st_node[sp] = (unsigned)root;
  st_lb[sp++] = box_lb(lo[L.off[root]], hi[L.off[root]], qx, qy, qz);
  while (sp > 0) {
    --sp;
    if (st_lb[sp] > h.d2) continue;
    const int l = (int)(st_node[sp] & 31u), k = (int)(st_node[sp] >> 5);
    if (l == 0) {
      const int e = k * kLeaf + min(kLeaf, m - k * kLeaf);
      for (int i = k * kLeaf; i < e; ++i) {
        const float4 p = pts[i];
        const double dx = qx - (double)p.x, dy = qy - (double)p.y, dz = qz - (double)p.z;
        const double d2 = (dx * dx + dy * dy) + dz * dz;
        const int j = __float_as_int(p.w);
        ++evals;
        if (d2 < h.d2 || (d2 == h.d2 && j < h.j)) {
          h.d2 = d2; h.j = j; h.x = p.x; h.y = p.y; h.z = p.z;
        }
      }
      continue;
    }
    const int c0 = 2 * k, nc = level_count(m, l - 1), o = L.off[l - 1];
    const double lb0 = box_lb(lo[o + c0], hi[o + c0], qx, qy, qz);
    const double lb1 = c0 + 1 < nc ? box_lb(lo[o + c0 + 1], hi[o + c0 + 1], qx, qy, qz) : DBL_MAX;
    const bool first1 = lb1 < lb0;           // nearer child on top of the stack
    const int cn = first1 ? c0 + 1 : c0, cf = first1 ? c0 : c0 + 1;
    const double ln = first1 ? lb1 : lb0, lf = first1 ? lb0 : lb1;
    if (lf <= h.d2) { st_node[sp] = ((unsigned)cf << 5) | (unsigned)(l - 1); st_lb[sp++] = lf; }
    if (ln <= h.d2) { st_node[sp] = ((unsigned)cn << 5) | (unsigned)(l - 1); st_lb[sp++] = ln; }
  }
}

// The k nearest points with d2 < r2, in ascending (d2, index) order, into d2s[0 .. cnt) and js[0 .. cnt); returns
// cnt <= k.  The same descent as nearest() with the bound generalised from the best d2 to the k-th best: while fewer
// than k points are held it is r2 (strict), then the k-th (d2, index) pair.  K is the capacity of the lists.
template <int K>
__device__ __forceinline__ int knn(const float4* __restrict__ pts, const float4* __restrict__ lo,
                                   const float4* __restrict__ hi, const Levels& L, int m, int root, double qx,
                                   double qy, double qz, double r2, int k, double (&d2s)[K], int (&js)[K]) {
  int cnt = 0;
  if (m <= 0) return 0;
  double bound = r2;        // boxes with a lower bound strictly above it are skipped
  unsigned st_node[kStack];
  double st_lb[kStack];
  int sp = 0;
  st_node[sp] = (unsigned)root;
  st_lb[sp++] = box_lb(lo[L.off[root]], hi[L.off[root]], qx, qy, qz);
  while (sp > 0) {
    --sp;
    if (st_lb[sp] > bound) continue;
    const int l = (int)(st_node[sp] & 31u), nk = (int)(st_node[sp] >> 5);
    if (l == 0) {
      const int e = nk * kLeaf + min(kLeaf, m - nk * kLeaf);
      for (int i = nk * kLeaf; i < e; ++i) {
        const float4 p = pts[i];
        const double dx = qx - (double)p.x, dy = qy - (double)p.y, dz = qz - (double)p.z;
        const double d2 = (dx * dx + dy * dy) + dz * dz;
        if (!(d2 < r2)) continue;
        const int j = __float_as_int(p.w);
        if (cnt == k && !(d2 < d2s[k - 1] || (d2 == d2s[k - 1] && j < js[k - 1]))) continue;
        int at = cnt < k ? cnt++ : k - 1;     // insertion from the back; the k-th entry drops out when full
        while (at > 0 && (d2 < d2s[at - 1] || (d2 == d2s[at - 1] && j < js[at - 1]))) {
          d2s[at] = d2s[at - 1];
          js[at] = js[at - 1];
          --at;
        }
        d2s[at] = d2;
        js[at] = j;
        if (cnt == k) bound = d2s[k - 1];
      }
      continue;
    }
    const int c0 = 2 * nk, nc = level_count(m, l - 1), o = L.off[l - 1];
    const double lb0 = box_lb(lo[o + c0], hi[o + c0], qx, qy, qz);
    const double lb1 = c0 + 1 < nc ? box_lb(lo[o + c0 + 1], hi[o + c0 + 1], qx, qy, qz) : DBL_MAX;
    const bool first1 = lb1 < lb0;
    const int cn = first1 ? c0 + 1 : c0, cf = first1 ? c0 : c0 + 1;
    const double ln = first1 ? lb1 : lb0, lf = first1 ? lb0 : lb1;
    if (lf <= bound) { st_node[sp] = ((unsigned)cf << 5) | (unsigned)(l - 1); st_lb[sp++] = lf; }
    if (ln <= bound) { st_node[sp] = ((unsigned)cn << 5) | (unsigned)(l - 1); st_lb[sp++] = ln; }
  }
  return cnt;
}

}  // namespace icp
}  // namespace dib
