// Batched baseline JPEG encoding (4:2:0, standard Huffman tables, no restart markers) of imageprep.pack_images' HWC
// RGB frames, bit for bit with OpenCV 4.13's cv2.imencode(".jpg") on libjpeg-turbo 3.1.  DESIGN.md 4.25 states the
// contract; deepi2p_b200/jpeg_encode.py builds the tables and the markers, oracle_oxford_images/ restates every stage.
//
// jpege_block_kernel  8 threads per 8 x 8 block, 32 blocks per CTA: the block's samples straight from the RGB frame
//                     (jccolor.c's fixed-point RGB -> YCbCr, h2v2_downsample with the bias 1, 2, 1, 2, ... and
//                     libjpeg's edge replication), jfdctint.c's islow DCT (thread per row, then per column through
//                     shared memory) and the rounding division by 8 q; coefficients in coding order (six blocks per
//                     MCU: Y00 Y01 Y10 Y11 Cb Cr)
// jpege_dummy_kernel  thread per MCU: jccoefct.c's dummy luma blocks past the image's last block column or row take
//                     the DC of the block before them in the MCU (AC zero)
// jpege_length_kernel thread per block: the bit length of its Huffman code (DC difference to the previous block of
//                     its component, AC run lengths with ZRL / EOB); an exclusive scan gives every block its bit
//                     offset in its image's stream
// jpege_emit_kernel   thread per block: writes its codes at its offset; words wholly inside the block are stored,
//                     the first and last word (shared with the neighbours) are OR-ed atomically, so the bits are
//                     disjoint and the result is independent of the order; the image's last block adds the 1-bit
//                     padding to the byte
// jpege_count_kernel  CTA per image: the byte count and the number of 0xFF bytes (read back by the caller)
// jpege_stuff_kernel  CTA per image: copies the bytes to the caller's compact output with a 0x00 after every 0xFF
//                     (a block-wide scan of the 0xFF counts per tile)
//
// Integer arithmetic only; the only atomics are integer ORs of disjoint bits, so a stream is identical across runs.
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>
#include <cub/device/device_scan.cuh>

#include <vector>

#include "common.cuh"

namespace dib {
namespace jpege {

constexpr int kMaxS = 65535;
constexpr int kBlocksPerCta = 32;
constexpr int kMaxBlockBytes = 208;      // jpeg_encode.MAX_BLOCK_BYTES: 1660 bits at most per block
constexpr int kTile = 16;                // bytes per thread per stuffing tile
constexpr int kStuffThreads = 256;
enum { kIn = 0, kH, kW, kBlk0, kEnt, kNblk };   // descriptor slots (caller: 0..2; library: 3..5)
static_assert(kNblk < DIB_JPEGE_DESC, "descriptor slots");

__host__ __device__ inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

struct Layout {
  size_t desc, first, quant, huff, coef, bits, scan_tmp, scan_tmp_bytes, ent, out_off, total;
  int64_t blocks, ent_bytes;
};

// Fills the library's descriptor slots and returns the workspace layout.
inline Layout layout(std::vector<int64_t>& d, int S, std::vector<int64_t>& first) {
  int64_t blocks = 0, ent = 0;
  first.assign((size_t)S + 1, 0);
  for (int s = 0; s < S; ++s) {
    int64_t* q = d.data() + (size_t)s * DIB_JPEGE_DESC;
    const int64_t n = 6 * ((q[kW] + 15) / 16) * ((q[kH] + 15) / 16);
    q[kBlk0] = blocks;
    q[kNblk] = n;
    q[kEnt] = ent;
    first[s] = blocks;
    blocks += n;
    ent += (int64_t)align256((size_t)(n * kMaxBlockBytes));
  }
  first[S] = blocks;
  Layout L;
  L.blocks = blocks;
  L.ent_bytes = ent;
  size_t tmp = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tmp, (const int64_t*)nullptr, (int64_t*)nullptr, (int)(blocks + 1));
  L.scan_tmp_bytes = tmp;
  L.desc = 0;
  L.first = align256((size_t)S * DIB_JPEGE_DESC * sizeof(int64_t));
  L.quant = L.first + align256(((size_t)S + 1) * sizeof(int64_t));
  L.huff = L.quant + align256(128 * sizeof(int32_t));
  L.coef = L.huff + align256(4 * 256 * sizeof(int32_t));
  L.bits = L.coef + align256((size_t)blocks * 64 * sizeof(int16_t));
  L.scan_tmp = L.bits + align256(((size_t)blocks + 1) * 2 * sizeof(int64_t));   // lengths, then their scan
  L.ent = L.scan_tmp + align256(tmp);
  L.out_off = L.ent + (size_t)ent;
  L.total = L.out_off + align256((size_t)S * sizeof(int64_t));
  return L;
}

__device__ __forceinline__ int find_image(const int64_t* __restrict__ first, int S, int64_t b) {
  int lo = 0, hi = S - 1;                                           // the last s with first[s] <= b
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (first[mid] <= b) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// jccolor.c rgb_ycc_convert with its tables' constants: FIX(x) = (int)(x * 65536 + 0.5).
__device__ __forceinline__ int rgb_y(int r, int g, int b) { return (19595 * r + 38470 * g + 7471 * b + 32768) >> 16; }
__device__ __forceinline__ int rgb_cb(int r, int g, int b) {
  return (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16;
}
__device__ __forceinline__ int rgb_cr(int r, int g, int b) {
  return (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16;
}

__device__ __forceinline__ int chroma_at(const uint8_t* __restrict__ img, int W, int r, int c, int comp) {
  const uint8_t* p = img + ((size_t)r * W + c) * 3;
  return comp == 1 ? rgb_cb(p[0], p[1], p[2]) : rgb_cr(p[0], p[1], p[2]);
}

__device__ __forceinline__ long long descale(long long x, int n) { return (x + (1ll << (n - 1))) >> n; }

// One jfdctint.c pass (CONST_BITS 13, PASS1_BITS 2) over d[0..7], in place.
__device__ __forceinline__ void fdct_1d(long long d[8], bool last) {
  const long long t0 = d[0] + d[7], t7 = d[0] - d[7], t1 = d[1] + d[6], t6 = d[1] - d[6];
  const long long t2 = d[2] + d[5], t5 = d[2] - d[5], t3 = d[3] + d[4], t4 = d[3] - d[4];
  const long long t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  const int sh = last ? 15 : 11;
  if (last) {
    d[0] = descale(t10 + t11, 2);
    d[4] = descale(t10 - t11, 2);
  } else {
    d[0] = (t10 + t11) << 2;
    d[4] = (t10 - t11) << 2;
  }
  long long z1 = (t12 + t13) * 4433;
  d[2] = descale(z1 + t13 * 6270, sh);
  d[6] = descale(z1 + t12 * -15137, sh);
  z1 = t4 + t7;
  long long z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7;
  const long long z5 = (z3 + z4) * 9633;
  const long long u4 = t4 * 2446, u5 = t5 * 16819, u6 = t6 * 25172, u7 = t7 * 12299;
  z1 *= -7373;
  z2 *= -20995;
  z3 = z3 * -16069 + z5;
  z4 = z4 * -3196 + z5;
  d[7] = descale(u4 + z1 + z3, sh);
  d[5] = descale(u5 + z2 + z4, sh);
  d[3] = descale(u6 + z2 + z3, sh);
  d[1] = descale(u7 + z1 + z4, sh);
}

__global__ void __launch_bounds__(8 * kBlocksPerCta) jpege_block_kernel(const uint8_t* __restrict__ rgb,
                                                                        const int64_t* __restrict__ desc,
                                                                        const int64_t* __restrict__ first, int S,
                                                                        int64_t blocks,
                                                                        const int32_t* __restrict__ quant,
                                                                        int16_t* __restrict__ coef) {
  __shared__ long long tile[kBlocksPerCta][8][9];
  const int g = threadIdx.x >> 3, row = threadIdx.x & 7;
  const int64_t gb = (int64_t)blockIdx.x * kBlocksPerCta + g;
  const bool valid = gb < blocks;
  int comp = 0;
  if (valid) {
    const int s = find_image(first, S, gb);
    const int64_t* q = desc + (size_t)s * DIB_JPEGE_DESC;
    const int H = (int)q[kH], W = (int)q[kW];
    const int mcux = (W + 15) / 16;
    const int64_t b = gb - q[kBlk0], m = b / 6;
    const int k = (int)(b % 6), mr = (int)(m / mcux), mc = (int)(m % mcux);
    const uint8_t* img = rgb + q[kIn];
    long long d[8];
    if (k < 4) {                                                    // luma: the last row and column replicated
      const int r = min(16 * mr + 8 * (k >> 1) + row, H - 1);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = min(16 * mc + 8 * (k & 1) + j, W - 1);
        const uint8_t* p = img + ((size_t)r * W + c) * 3;
        d[j] = rgb_y(p[0], p[1], p[2]) - 128;
      }
    } else {                                                        // chroma: h2v2 of the edge-replicated rows
      comp = k - 3;
      const int crow = min(8 * mr + row, (H + 1) / 2 - 1);
      const int r0 = min(2 * crow, H - 1), r1 = min(2 * crow + 1, H - 1);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int cx = 8 * mc + j;
        const int c0 = min(2 * cx, W - 1), c1 = min(2 * cx + 1, W - 1);
        const int v = chroma_at(img, W, r0, c0, comp) + chroma_at(img, W, r0, c1, comp) +
                      chroma_at(img, W, r1, c0, comp) + chroma_at(img, W, r1, c1, comp) + (j & 1 ? 2 : 1);
        d[j] = (v >> 2) - 128;
      }
    }
    fdct_1d(d, false);
#pragma unroll
    for (int j = 0; j < 8; ++j) tile[g][row][j] = d[j];
  }
  __syncthreads();
  if (!valid) return;
  const int col = row;
  long long d[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) d[i] = tile[g][i][col];
  fdct_1d(d, true);
  const int32_t* qt = quant + (comp ? 64 : 0);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int div = 8 * qt[i * 8 + col];                            // |d| < 2^16: 32-bit division is exact
    const int a = (int)(d[i] < 0 ? -d[i] : d[i]);
    const int v = (a + (div >> 1)) / div;
    coef[gb * 64 + i * 8 + col] = (int16_t)(d[i] < 0 ? -v : v);
  }
}

__global__ void jpege_dummy_kernel(const int64_t* __restrict__ desc, const int64_t* __restrict__ first, int S,
                                   int64_t mcus, int16_t* __restrict__ coef) {
  const int64_t gm = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gm >= mcus) return;
  const int s = find_image(first, S, 6 * gm);
  const int64_t* q = desc + (size_t)s * DIB_JPEGE_DESC;
  const int H = (int)q[kH], W = (int)q[kW];
  const int mcux = (W + 15) / 16, mcuy = (H + 15) / 16;
  const int64_t m = gm - q[kBlk0] / 6;
  const bool right = (int)(m % mcux) == mcux - 1 && ((W + 7) / 8) % 2 == 1;
  const bool bottom = (int)(m / mcux) == mcuy - 1 && ((H + 7) / 8) % 2 == 1;
  if (!right && !bottom) return;
  int16_t* c = coef + 6 * gm * 64;
  auto dummy = [&](int k, int from) {
    for (int i = 1; i < 64; ++i) c[k * 64 + i] = 0;
    c[k * 64] = c[from * 64];
  };
  if (right) {
    dummy(1, 0);
    dummy(3, 2);
  }
  if (bottom) {
    dummy(2, 1);
    dummy(3, 1);
  }
}

// jpeg_natural_order: zig-zag position -> natural (row-major) index.
__constant__ uint8_t kZigzag[64] = {0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

__device__ __forceinline__ int nbits(int v) { return v ? 32 - __clz(v < 0 ? -v : v) : 0; }

// The previous block of the same component in coding order, or -1 for the component's first block.
__device__ __forceinline__ int64_t prev_block(int64_t b) {
  const int k = (int)(b % 6);
  if (k >= 1 && k <= 3) return b - 1;
  if (b < 6) return -1;
  return k == 0 ? b - 3 : b - 6;
}

// Calls put(code, length) for every code of block gb of an image whose first block is b0.
template <class Put>
__device__ __forceinline__ void code_block(const int16_t* __restrict__ coef, const int32_t* __restrict__ huff,
                                           int64_t gb, int64_t b0, Put put) {
  const int64_t b = gb - b0;
  const int k = (int)(b % 6);
  const int32_t* dct = huff + (k < 4 ? 0 : 512);
  const int32_t* act = dct + 256;
  const int16_t* c = coef + gb * 64;
  const int64_t pb = prev_block(b);
  const int diff = (int)c[0] - (pb < 0 ? 0 : (int)coef[(b0 + pb) * 64]);
  int n = nbits(diff);
  put(dct[n] & 0xFFFF, dct[n] >> 16);
  if (n) put((uint32_t)(diff < 0 ? diff - 1 : diff) & ((1u << n) - 1), n);
  int run = 0;
  for (int z = 1; z < 64; ++z) {
    const int v = c[kZigzag[z]];
    if (v == 0) {
      ++run;
      continue;
    }
    while (run > 15) {
      put(act[0xF0] & 0xFFFF, act[0xF0] >> 16);
      run -= 16;
    }
    n = nbits(v);
    const int sym = (run << 4) + n;
    put(act[sym] & 0xFFFF, act[sym] >> 16);
    put((uint32_t)(v < 0 ? v - 1 : v) & ((1u << n) - 1), n);
    run = 0;
  }
  if (run) put(act[0] & 0xFFFF, act[0] >> 16);
}

__global__ void __launch_bounds__(256) jpege_length_kernel(const int16_t* __restrict__ coef,
                                                           const int32_t* __restrict__ huff,
                                                           const int64_t* __restrict__ first, int S, int64_t blocks,
                                                           int64_t* __restrict__ bits) {
  const int64_t gb = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gb > blocks) return;
  if (gb == blocks) {
    bits[gb] = 0;
    return;
  }
  const int s = find_image(first, S, gb);
  int64_t n = 0;
  code_block(coef, huff, gb, first[s], [&](uint32_t, int len) { n += len; });
  bits[gb] = n;
}

struct BitSink {
  uint32_t* buf;
  int64_t w, first_w;
  uint32_t cur;
  int fill;
  __device__ __forceinline__ void flush_word(bool shared) {
    const uint32_t v = __byte_perm(cur, 0, 0x0123);                 // the stream is big-endian
    if (shared) atomicOr(buf + w, v);
    else buf[w] = v;
  }
  __device__ __forceinline__ void put(uint32_t code, int n) {
    while (n > 0) {
      const int take = min(n, 32 - fill);
      const uint32_t v = (code >> (n - take)) & (take == 32 ? 0xFFFFFFFFu : ((1u << take) - 1));
      cur |= v << (32 - fill - take);
      fill += take;
      n -= take;
      if (fill == 32) {
        flush_word(w == first_w);
        ++w;
        cur = 0;
        fill = 0;
      }
    }
  }
};

__global__ void __launch_bounds__(256) jpege_emit_kernel(const int16_t* __restrict__ coef,
                                                         const int32_t* __restrict__ huff,
                                                         const int64_t* __restrict__ desc,
                                                         const int64_t* __restrict__ first, int S, int64_t blocks,
                                                         const int64_t* __restrict__ pos, uint8_t* ent) {
  const int64_t gb = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gb >= blocks) return;
  const int s = find_image(first, S, gb);
  const int64_t* q = desc + (size_t)s * DIB_JPEGE_DESC;
  const int64_t b0 = q[kBlk0];
  const int64_t p = pos[gb] - pos[b0];
  BitSink sink{(uint32_t*)(ent + q[kEnt]), p >> 5, p >> 5, 0u, (int)(p & 31)};
  code_block(coef, huff, gb, b0, [&](uint32_t code, int len) { sink.put(code, len); });
  if (gb == b0 + q[kNblk] - 1) {                                    // the image's last block: pad with 1 bits
    const int64_t total = pos[b0 + q[kNblk]] - pos[b0];
    const int pad = (int)((8 - (total & 7)) & 7);
    if (pad) sink.put((1u << pad) - 1, pad);
  }
  if (sink.fill) sink.flush_word(true);
}

__global__ void __launch_bounds__(kStuffThreads) jpege_count_kernel(const int64_t* __restrict__ desc,
                                                                    const int64_t* __restrict__ pos,
                                                                    const uint8_t* __restrict__ ent,
                                                                    int64_t* __restrict__ counts) {
  using Reduce = cub::BlockReduce<long long, kStuffThreads>;
  __shared__ typename Reduce::TempStorage tmp;
  const int s = blockIdx.x;
  const int64_t* q = desc + (size_t)s * DIB_JPEGE_DESC;
  const int64_t nbytes = (pos[q[kBlk0] + q[kNblk]] - pos[q[kBlk0]] + 7) >> 3;
  const uint8_t* e = ent + q[kEnt];
  long long ff = 0;
  for (int64_t i = threadIdx.x; i < nbytes; i += kStuffThreads) ff += e[i] == 0xFF;
  ff = Reduce(tmp).Sum(ff);
  if (threadIdx.x == 0) {
    counts[2 * s] = nbytes;
    counts[2 * s + 1] = ff;
  }
}

__global__ void __launch_bounds__(kStuffThreads) jpege_stuff_kernel(const int64_t* __restrict__ desc,
                                                                    const int64_t* __restrict__ pos,
                                                                    const uint8_t* __restrict__ ent,
                                                                    const int64_t* __restrict__ out_off,
                                                                    uint8_t* __restrict__ out, size_t out_bytes) {
  using Scan = cub::BlockScan<int, kStuffThreads>;
  __shared__ typename Scan::TempStorage tmp;
  const int s = blockIdx.x;
  const int64_t* q = desc + (size_t)s * DIB_JPEGE_DESC;
  const int64_t nbytes = (pos[q[kBlk0] + q[kNblk]] - pos[q[kBlk0]] + 7) >> 3;
  const uint8_t* e = ent + q[kEnt];
  uint8_t* o = out + out_off[s];
  const int64_t room = (int64_t)out_bytes - out_off[s];             // never write past the caller's buffer
  int64_t carry = 0;                                                // 0xFF bytes in earlier tiles
  for (int64_t t0 = 0; t0 < nbytes; t0 += (int64_t)kTile * kStuffThreads) {
    const int64_t i0 = t0 + (int64_t)threadIdx.x * kTile;
    uint8_t v[kTile];
    int ff = 0;
#pragma unroll
    for (int j = 0; j < kTile; ++j) {
      v[j] = i0 + j < nbytes ? e[i0 + j] : 0;
      ff += v[j] == 0xFF;
    }
    int before, total;
    Scan(tmp).ExclusiveSum(ff, before, total);
    __syncthreads();
    int64_t dst = i0 + carry + before;
#pragma unroll
    for (int j = 0; j < kTile; ++j) {
      if (i0 + j < nbytes) {
        if (dst < room) o[dst] = v[j];
        ++dst;
        if (v[j] == 0xFF) {
          if (dst < room) o[dst] = 0;
          ++dst;
        }
      }
    }
    carry += total;
  }
}

int prepare(const int64_t* desc, int S, size_t rgb_bytes, std::vector<int64_t>& d, std::vector<int64_t>& first,
            Layout& L) {
  DIB_REQUIRE(S >= 0 && S <= kMaxS, "S must be in [0, %d] (got %d)", kMaxS, S);
  DIB_REQUIRE(S == 0 || desc, "desc is null");
  d.assign(desc, desc + (size_t)S * DIB_JPEGE_DESC);
  for (int s = 0; s < S; ++s) {
    const int64_t* q = d.data() + (size_t)s * DIB_JPEGE_DESC;
    DIB_REQUIRE(q[kH] >= 1 && q[kW] >= 1 && q[kH] <= 65500 && q[kW] <= 65500, "image %d: size %lld x %lld", s,
                (long long)q[kH], (long long)q[kW]);
    DIB_REQUIRE(q[kIn] >= 0 && (size_t)(q[kIn] + 3 * q[kH] * q[kW]) <= rgb_bytes, "image %d: outside the input", s);
  }
  L = layout(d, S, first);
  DIB_REQUIRE(L.blocks < (int64_t)1 << 30, "too many blocks in one batch (%lld)", (long long)L.blocks);
  return 0;
}

int entropy(const uint8_t* rgb, size_t rgb_bytes, const int64_t* desc, int S, const int32_t* quant,
            const int32_t* huff, int64_t* counts, void* workspace, size_t workspace_bytes, cudaStream_t cs) {
  std::vector<int64_t> d, first;
  Layout L;
  const int rc = prepare(desc, S, rgb_bytes, d, first, L);
  if (rc) return rc;
  if (S == 0) return 0;
  DIB_REQUIRE(rgb && quant && huff && counts && workspace, "a required pointer is null");
  for (int i = 0; i < 128; ++i) DIB_REQUIRE(quant[i] >= 1 && quant[i] <= 255, "quant[%d] = %d", i, quant[i]);
  if (workspace_bytes < L.total) {
    set_error("jpeg_encode: workspace is %zu bytes, %zu needed", workspace_bytes, L.total);
    return DIB_ENOMEM;
  }
  unsigned char* ws = (unsigned char*)workspace;
  DIB_CHECK_CUDA(cudaMemcpyAsync(ws + L.desc, d.data(), d.size() * sizeof(int64_t), cudaMemcpyHostToDevice, cs));
  DIB_CHECK_CUDA(
      cudaMemcpyAsync(ws + L.first, first.data(), first.size() * sizeof(int64_t), cudaMemcpyHostToDevice, cs));
  DIB_CHECK_CUDA(cudaMemcpyAsync(ws + L.quant, quant, 128 * sizeof(int32_t), cudaMemcpyHostToDevice, cs));
  DIB_CHECK_CUDA(cudaMemcpyAsync(ws + L.huff, huff, 1024 * sizeof(int32_t), cudaMemcpyHostToDevice, cs));
  DIB_CHECK_CUDA(cudaMemsetAsync(ws + L.ent, 0, (size_t)L.ent_bytes, cs));
  const int64_t* dd = (const int64_t*)(ws + L.desc);
  const int64_t* fd = (const int64_t*)(ws + L.first);
  int16_t* coef = (int16_t*)(ws + L.coef);
  int64_t* bits = (int64_t*)(ws + L.bits);
  int64_t* pos = bits + L.blocks + 1;
  const int32_t* hd = (const int32_t*)(ws + L.huff);
  const int64_t nb = L.blocks;
  jpege_block_kernel<<<(unsigned)((nb + kBlocksPerCta - 1) / kBlocksPerCta), 8 * kBlocksPerCta, 0, cs>>>(
      rgb, dd, fd, S, nb, (const int32_t*)(ws + L.quant), coef);
  DIB_CHECK_CUDA(cudaGetLastError());
  jpege_dummy_kernel<<<(unsigned)((nb / 6 + 255) / 256), 256, 0, cs>>>(dd, fd, S, nb / 6, coef);
  DIB_CHECK_CUDA(cudaGetLastError());
  jpege_length_kernel<<<(unsigned)((nb + 1 + 255) / 256), 256, 0, cs>>>(coef, hd, fd, S, nb, bits);
  DIB_CHECK_CUDA(cudaGetLastError());
  size_t tmp = L.scan_tmp_bytes;
  DIB_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(ws + L.scan_tmp, tmp, bits, pos, (int)(nb + 1), cs));
  jpege_emit_kernel<<<(unsigned)((nb + 255) / 256), 256, 0, cs>>>(coef, hd, dd, fd, S, nb, pos, ws + L.ent);
  DIB_CHECK_CUDA(cudaGetLastError());
  jpege_count_kernel<<<S, kStuffThreads, 0, cs>>>(dd, pos, ws + L.ent, counts);
  DIB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

int stuff(const int64_t* desc, int S, const int64_t* out_off, uint8_t* out, size_t out_bytes, void* workspace,
          size_t workspace_bytes, cudaStream_t cs) {
  std::vector<int64_t> d, first;
  Layout L;
  const int rc = prepare(desc, S, SIZE_MAX / 4, d, first, L);
  if (rc) return rc;
  if (S == 0) return 0;
  DIB_REQUIRE(out_off && workspace && (out || out_bytes == 0), "a required pointer is null");
  for (int s = 0; s < S; ++s)
    DIB_REQUIRE(out_off[s] >= 0 && (size_t)out_off[s] <= out_bytes, "image %d: output offset outside the buffer", s);
  if (workspace_bytes < L.total) {
    set_error("jpeg_encode: workspace is %zu bytes, %zu needed", workspace_bytes, L.total);
    return DIB_ENOMEM;
  }
  unsigned char* ws = (unsigned char*)workspace;
  DIB_CHECK_CUDA(cudaMemcpyAsync(ws + L.out_off, out_off, (size_t)S * sizeof(int64_t), cudaMemcpyHostToDevice, cs));
  const int64_t* pos = (const int64_t*)(ws + L.bits) + L.blocks + 1;
  jpege_stuff_kernel<<<S, kStuffThreads, 0, cs>>>((const int64_t*)(ws + L.desc), pos, ws + L.ent,
                                                  (const int64_t*)(ws + L.out_off), out, out_bytes);
  DIB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace jpege
}  // namespace dib

extern "C" {

size_t jpeg_encode_workspace_bytes(const int64_t* desc, int S) {
  std::vector<int64_t> d, first;
  dib::jpege::Layout L;
  if (dib::jpege::prepare(desc, S, SIZE_MAX / 4, d, first, L)) return 0;
  return L.total;
}

int jpeg_encode_entropy_u8(const uint8_t* rgb, size_t rgb_bytes, const int64_t* desc, int S, const int32_t* quant,
                           const int32_t* huff, int64_t* counts, void* workspace, size_t workspace_bytes,
                           dib_stream_t stream) {
  return dib::jpege::entropy(rgb, rgb_bytes, desc, S, quant, huff, counts, workspace, workspace_bytes,
                             (cudaStream_t)stream);
}

int jpeg_encode_stuff_u8(const int64_t* desc, int S, const int64_t* out_off, uint8_t* out, size_t out_bytes,
                         void* workspace, size_t workspace_bytes, dib_stream_t stream) {
  return dib::jpege::stuff(desc, S, out_off, out, out_bytes, workspace, workspace_bytes, (cudaStream_t)stream);
}

}  // extern "C"
