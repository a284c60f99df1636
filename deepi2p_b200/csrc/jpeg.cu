// Batched sequential-Huffman JPEG decoding, bit for bit with libjpeg-turbo as Pillow 12.2 runs it (ISLOW IDCT, fancy
// upsampling), straight into imageprep.pack_images' HWC buffer.  DESIGN.md 4.19 states the contract; oracle_jpeg/ is
// its sequential restatement, and deepi2p_b200/jpeg.py parses the headers and packs the tables on the host.
//
// jpeg_unstuff_kernel    CTA per image: removes FF 00 stuffing and FF fill bytes from the entropy-coded data in
//                        8 KB tiles (one block scan per tile), records where each restart interval starts, and checks
//                        that the data ends in EOI with the interval count the DRI implies
// jpeg_huffman_kernel    CTA of 512 threads per image: self-synchronising decoding (Weissenberger & Schmidt, ICPP 2018).  Each
//                        restart interval is cut into windows of window_bits bits; every window is decoded from a
//                        guessed state (its first bit, block 0 of an MCU, DC next), then each round re-decodes the
//                        windows whose entry state differs from their predecessor's exit state, until none does.  The
//                        first window of an interval starts from its true state, so round r fixes window r at the
//                        latest: the loop ends, in the worst case after as many rounds as the longest interval has
//                        windows.  A scan over the windows' completed-block counts places each window's output; a
//                        last pass writes the coefficients (DC as differences) and a segmented scan per component
//                        turns the differences into DC values, reset at each interval
// jpeg_idct_kernel       thread per 8x8 block: dequantisation and jidctint.c's jpeg_idct_islow into the component's
//                        sample plane
// jpeg_color_kernel      thread per output pixel: jdsample.c's upsampling of each component (fancy h2v1 / h2v2 /
//                        h1v2, box replication when the downsampled width is <= 2) and jdcolor.c's ycc_rgb_convert,
//                        written as HWC uint8; grey is replicated to three channels
//
// Everything is integer arithmetic without atomics, so a decode is bit-identical across runs and streams.
#include <cub/block/block_scan.cuh>

#include <vector>

#include "common.cuh"

namespace dib {
namespace jpg {

constexpr int kThreads = 1024;
constexpr int kUnstuffPerThread = 8;
constexpr int kTile = kThreads * kUnstuffPerThread;
constexpr int kMaxS = 65535;
constexpr int kHuffWords = 356;                 // lut u16[512] (256 words), maxcode[18], valoff[18], vals u8[256]
// A window at least as long as the longest symbol (a 16-bit code and 15 extra bits) starts at least one symbol, so a
// corrected entry state reaches the next window in one round; shorter windows would pass states on one per round.
constexpr int kMinWindowBits = 32;
constexpr int kHuffThreads = 512;              // 128 registers per thread for the decode loop
constexpr int kIdctThreads = 128, kColorThreads = 256;

// Descriptor slots (int64), DIB_JPEG_DESC of them per image; the caller fills the first block, the library the rest.
enum {
  kStreamOff = 0, kStreamLen, kOutOff, kW, kH, kNc, kRi, kMcux, kMcuy, kBpm, kNblk, kHmax, kVmax,
  kComp = 16,            // per component c: kComp + 8 c + {h, v, bw, bh, dw, dh, plane_off, block_off}
  kCoefOff = 40, kSegOff, kSegCap, kWinOff, kWinCap, kCompOfBlk,   // kCompOfBlk: 4 bits per MCU block
};
static_assert(kCompOfBlk < DIB_JPEG_DESC, "descriptor slots");

__host__ __device__ inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

struct Layout {
  size_t desc, ustream, seg, info, wb0, wb1, wseg, entry, exit_, nblk, flag, base, coef, planes, total;
};

// Per-image totals on the host from the caller's descriptors: the library's own slots are filled in `d`.
inline Layout layout(std::vector<int64_t>& d, int S, size_t stream_bytes, int window_bits) {
  int64_t seg = 0, win = 0, blocks = 0, plane = 0;
  for (int s = 0; s < S; ++s) {
    int64_t* q = d.data() + (size_t)s * DIB_JPEG_DESC;
    const int64_t n_mcu = q[kNc] == 1 ? q[kNblk] : q[kMcux] * q[kMcuy];
    const int64_t seg_cap = q[kRi] ? (n_mcu + q[kRi] - 1) / q[kRi] : 1;
    q[kSegOff] = seg;
    q[kSegCap] = seg_cap;
    seg += seg_cap + 1;
    q[kWinOff] = win;
    q[kWinCap] = (q[kStreamLen] * 8) / window_bits + seg_cap + 1;
    win += q[kWinCap];
    q[kCoefOff] = blocks;
    blocks += q[kNblk];
    for (int c = 0; c < q[kNc]; ++c) {
      int64_t* cc = q + kComp + 8 * c;
      cc[6] = plane;
      plane += cc[2] * 8 * cc[3] * 8;
    }
  }
  Layout L;
  L.desc = 0;
  L.ustream = align256((size_t)S * DIB_JPEG_DESC * sizeof(int64_t));
  L.seg = L.ustream + align256(stream_bytes + 16);
  L.info = L.seg + align256((size_t)seg * sizeof(int32_t));
  L.wb0 = L.info + align256((size_t)S * 4 * sizeof(int32_t));
  L.wb1 = L.wb0 + align256((size_t)win * sizeof(int32_t));
  L.wseg = L.wb1 + align256((size_t)win * sizeof(int32_t));
  L.entry = L.wseg + align256((size_t)win * sizeof(int32_t));
  L.exit_ = L.entry + align256((size_t)win * sizeof(int64_t));
  L.nblk = L.exit_ + align256((size_t)win * sizeof(int64_t));
  L.flag = L.nblk + align256((size_t)win * sizeof(int32_t));
  L.base = L.flag + align256((size_t)win * sizeof(int32_t));
  L.coef = L.base + align256((size_t)win * sizeof(int32_t));
  L.planes = L.coef + align256((size_t)blocks * 64 * sizeof(int16_t));
  L.total = L.planes + align256((size_t)plane);
  return L;
}

// ---------------------------------------------------------------------------------------------------------------
// Unstuffing.  A byte is kept unless it is an FF followed by FF (fill), a 00 after FF (stuffing) or a marker code; an
// FF followed by 00 is one FF data byte.  FF D0..D7 starts a new restart interval; any other marker ends the data.
// info[s] = {intervals found, unstuffed bytes, ending marker code (256: none), -}.
__global__ void __launch_bounds__(kThreads) jpeg_unstuff_kernel(const uint8_t* __restrict__ src,
                                                                 const int64_t* __restrict__ desc, uint8_t* ustream,
                                                                 int32_t* seg_start, int32_t* info, int32_t* status) {
  using Scan = cub::BlockScan<uint32_t, kThreads>;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ int s_end;
  const int s = blockIdx.x;
  const int64_t* d = desc + (size_t)s * DIB_JPEG_DESC;
  const uint8_t* b = src + d[kStreamOff];
  const int64_t n = d[kStreamLen];
  uint8_t* out = ustream + d[kStreamOff];
  int32_t* seg = seg_start + d[kSegOff];
  const int64_t seg_cap = d[kSegCap];
  if (threadIdx.x == 0) seg[0] = 0;
  uint32_t kept_total = 0, rst_total = 0;
  int end_code = 256;
  for (int64_t t0 = 0; t0 < n; t0 += kTile) {
    if (threadIdx.x == 0) s_end = kTile;
    __syncthreads();
    const int64_t i0 = t0 + (int64_t)threadIdx.x * kUnstuffPerThread;
    uint8_t cur[kUnstuffPerThread + 2];   // cur[0] = byte i0 - 1, cur[1 + j] = byte i0 + j, cur[9] = byte i0 + 8
#pragma unroll
    for (int j = 0; j < kUnstuffPerThread + 2; ++j) {
      const int64_t i = i0 - 1 + j;
      cur[j] = (i >= 0 && i < n) ? b[i] : 0;
    }
    // the first byte (in stream order) that ends the data: an FF followed by a non-00, non-FF, non-RST byte, or an
    // FF that is the stream's last byte
#pragma unroll
    for (int j = 0; j < kUnstuffPerThread; ++j) {
      const int64_t i = i0 + j;
      if (i >= n) break;
      const uint8_t x = cur[1 + j], nx = cur[2 + j];
      const bool last = i + 1 == n;
      if (x == 0xFF && (last || (nx != 0x00 && nx != 0xFF && !(nx >= 0xD0 && nx <= 0xD7)))) {
        atomicMin(&s_end, (int)(i - t0));
        break;
      }
    }
    __syncthreads();
    const int end_local = s_end;
    uint32_t keep_mask = 0, rst_mask = 0;
#pragma unroll
    for (int j = 0; j < kUnstuffPerThread; ++j) {
      const int64_t i = i0 + j;
      if (i >= n || i - t0 >= end_local) break;
      const uint8_t p = cur[j], x = cur[1 + j], nx = cur[2 + j];
      if (x == 0xFF) {
        if (nx == 0x00) keep_mask |= 1u << j;
        else if (nx >= 0xD0 && nx <= 0xD7) rst_mask |= 1u << j;
      } else if (p != 0xFF || i == 0) {
        keep_mask |= 1u << j;
      }
    }
    const uint32_t mine = (uint32_t)__popc(rst_mask) << 16 | (uint32_t)__popc(keep_mask);
    uint32_t excl, agg;
    Scan(tmp).ExclusiveSum(mine, excl, agg);
    uint32_t kept = kept_total + (excl & 0xFFFF), rsts = rst_total + (excl >> 16);
#pragma unroll
    for (int j = 0; j < kUnstuffPerThread; ++j) {
      if (keep_mask >> j & 1) out[kept++] = cur[1 + j];
      if (rst_mask >> j & 1) {
        ++rsts;
        if (rsts <= (uint32_t)seg_cap) seg[rsts] = (int32_t)kept;
      }
    }
    kept_total += agg & 0xFFFF;
    rst_total += agg >> 16;
    if (end_local < kTile) {
      const int64_t e = t0 + end_local;
      end_code = e + 1 < n ? b[e + 1] : 256;
      break;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const uint32_t nseg = rst_total + 1;
    int st = 0;
    if (end_code == 256) st = DIB_JPEG_TRUNCATED;
    else if (end_code != 0xD9) st = DIB_JPEG_MARKER;
    else if (nseg != (uint32_t)seg_cap) st = DIB_JPEG_RESTARTS;
    else seg[nseg] = (int32_t)kept_total;
    info[4 * s + 0] = (int32_t)nseg;
    info[4 * s + 1] = (int32_t)kept_total;
    info[4 * s + 2] = end_code;
    status[2 * s] = st;
    status[2 * s + 1] = 0;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Huffman decoding
struct HuffT {
  uint16_t lut[512];
  int32_t maxcode[18];
  int32_t valoff[18];
  uint8_t vals[256];
};
static_assert(sizeof(HuffT) == kHuffWords * 4, "Huffman table layout");

// State at a symbol boundary: bit position << 16 | block-in-MCU << 8 | zig-zag index (0: the DC comes next).
__device__ __forceinline__ int64_t pack_state(int32_t pos, int blk, int k) {
  return (int64_t)pos << 16 | (int64_t)(blk << 8) | (int64_t)k;
}

enum { kFlagEnd = 1, kFlagBad = 2 };

__device__ const uint8_t d_natural[64] = {
    0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

struct Ctx {
  const uint8_t* u;          // the image's unstuffed data
  const uint8_t* natural;    // jpeg_natural_order (shared memory)
  const HuffT* tabs;         // [2 c] DC, [2 c + 1] AC
  const uint8_t* comp_of;    // MCU block -> component
  int bpm;
};

// A 64-bit bit buffer over [pos, end) (bits), zero-filled beyond end.
struct Bits {
  const uint8_t* u;
  uint64_t acc;
  int nacc;
  int32_t next;              // next byte to load
  int32_t end_byte;
  __device__ __forceinline__ void init(const uint8_t* base, int32_t pos, int32_t end_bits) {
    u = base;
    end_byte = (end_bits + 7) >> 3;
    next = pos >> 3;
    acc = 0;
    nacc = 0;
    refill();
    const int skip = pos & 7;
    acc <<= skip;
    nacc -= skip;
  }
  __device__ __forceinline__ void refill() {
    while (nacc <= 56) {
      const uint64_t byte = next < end_byte ? __ldg(u + next) : 0;
      acc |= byte << (56 - nacc);
      nacc += 8;
      ++next;
    }
  }
  __device__ __forceinline__ void skip(int n) {
    acc <<= n;
    nacc -= n;
  }
};

// Decode from `entry` while the position is below b1 (or until the interval's data ends).  With `coef` set, the
// coefficients go to the blocks base, base + 1, ... (decode order); DC as the difference.
template <bool kWrite>
__device__ void decode_window(const Ctx& cx, int64_t entry, int32_t b1, int32_t seg_end, int64_t* exit_state,
                              int32_t* nblk_out, int32_t* flag_out, int16_t* coef_img, const int64_t* d,
                              int32_t base) {
  int32_t pos = (int32_t)(entry >> 16);
  int blk = (int)(entry >> 8) & 0xFF, k = (int)entry & 0xFF;
  int32_t done = 0;
  int flag = 0;
  Bits br;
  br.init(cx.u, pos, seg_end);
  int16_t* blkp = nullptr;
  auto locate = [&](int32_t g) -> int16_t* {
    if (g >= d[kNblk]) return nullptr;
    int c, by, bx;
    if (d[kNc] == 1) {
      const int bw = (int)d[kComp + 2];
      c = 0;
      by = g / bw;
      bx = g - by * bw;
    } else {
      const int bpm = (int)d[kBpm];
      const int mcu = g / bpm, b = g - mcu * bpm;
      const int mcux = (int)d[kMcux];
      const int my = mcu / mcux, mx = mcu - my * mcux;
      c = cx.comp_of[b];
      int first = 0;
      for (int e = 0; e < c; ++e) first += (int)(d[kComp + 8 * e] * d[kComp + 8 * e + 1]);
      const int h = (int)d[kComp + 8 * c], r = b - first;
      by = my * (int)d[kComp + 8 * c + 1] + r / h;
      bx = mx * h + r % h;
    }
    const int64_t* cc = d + kComp + 8 * c;
    return coef_img + (cc[7] + (int64_t)by * cc[2] + bx) * 64;
  };
  if (kWrite) blkp = locate(base);
  while (pos < b1) {
    br.refill();
    const uint32_t p16 = (uint32_t)(br.acc >> 48);
    const HuffT& t = cx.tabs[2 * cx.comp_of[blk] + (k ? 1 : 0)];
    const uint32_t e = t.lut[p16 >> 7];
    int len = 0, sym = 0;
    if (e) {
      len = (int)(e >> 8);
      sym = (int)(e & 255);
    } else {
      for (int l = 10; l <= 16; ++l) {
        const int32_t code = (int32_t)(p16 >> (16 - l));
        if (code <= t.maxcode[l]) {
          len = l;
          sym = t.vals[(code + t.valoff[l]) & 255];
          break;
        }
      }
      if (!len) {
        if (seg_end - pos < 16) {        // the zero fill past the interval's end: its data ends here
          flag |= kFlagEnd;
          break;
        }
        // An invalid code.  Decoding from a guessed state meets these all the time; stopping would hand the next
        // window a stale state and serialise the synchronisation, so step one bit and go on.  From a true state it
        // is corrupt data, and the flag fails the image.
        flag |= kFlagBad;
        br.skip(1);
        ++pos;
        continue;
      }
    }
    const int s = k ? (sym & 15) : sym;
    if (pos + len + s > seg_end) {
      flag |= kFlagEnd;
      break;
    }
    br.skip(len);
    int v = 0;
    if (s) {
      const uint32_t r = (uint32_t)(br.acc >> (64 - s));
      br.skip(s);
      v = (r >> (s - 1)) ? (int)r : (int)r - (1 << s) + 1;
    }
    pos += len + s;
    if (k == 0) {
      if (kWrite && blkp) blkp[0] = (int16_t)v;
      k = 1;
    } else {
      const int r = sym >> 4;
      if (s) {
        k += r;
        if (kWrite && blkp) blkp[k > 63 ? 63 : cx.natural[k]] = (int16_t)v;
        ++k;
      } else if (r == 15) {
        k += 16;
      } else {
        k = 64;
      }
    }
    if (k >= 64) {
      k = 0;
      ++done;
      if (++blk == cx.bpm) blk = 0;
      if (kWrite) blkp = locate(base + done);
    }
  }
  *exit_state = pack_state(pos, blk, k);
  *nblk_out = done;
  *flag_out = flag;
}

struct SegPair {
  int32_t flag, val;
};
struct SegOp {
  __device__ __forceinline__ SegPair operator()(const SegPair& a, const SegPair& b) const {
    return SegPair{a.flag | b.flag, b.flag ? b.val : (int32_t)((uint32_t)a.val + (uint32_t)b.val)};
  }
};
template <typename T, typename Op>
struct RunningPrefix {
  T running;
  Op op;
  __device__ T operator()(T agg) {
    const T old = running;
    running = op(running, agg);
    return old;
  }
};

__global__ void __launch_bounds__(kHuffThreads) jpeg_huffman_kernel(const int64_t* __restrict__ desc,
                                                                 const int32_t* __restrict__ huff,
                                                                 const uint8_t* __restrict__ ustream,
                                                                 const int32_t* __restrict__ seg_start,
                                                                 int window_bits, int32_t* wb0, int32_t* wb1,
                                                                 int32_t* wseg, int64_t* entry, int64_t* exit_state,
                                                                 int32_t* nblk, int32_t* flag, int32_t* wbase,
                                                                 int16_t* coef, int32_t* status) {
  using IntScan = cub::BlockScan<int32_t, kHuffThreads>;
  using PairScan = cub::BlockScan<SegPair, kHuffThreads>;
  __shared__ union {
    typename IntScan::TempStorage i;
    typename PairScan::TempStorage p;
  } tmp;
  __shared__ HuffT tabs[6];
  __shared__ uint8_t comp_of[16], natural[64];
  __shared__ int32_t s_carry, s_bad;
  const int s = blockIdx.x;
  if (status[2 * s] != 0) return;
  const int64_t* d = desc + (size_t)s * DIB_JPEG_DESC;
  const int nc = (int)d[kNc];
  {
    const int32_t* src = huff + (size_t)s * 6 * kHuffWords;
    int32_t* dst = reinterpret_cast<int32_t*>(tabs);
    for (int i = threadIdx.x; i < 2 * nc * kHuffWords; i += blockDim.x) dst[i] = src[i];
    if (threadIdx.x < 64) natural[threadIdx.x] = d_natural[threadIdx.x];
    if (threadIdx.x < 16) comp_of[threadIdx.x] = (uint8_t)((d[kCompOfBlk] >> (4 * threadIdx.x)) & 15);
  }
  const int32_t* seg = seg_start + d[kSegOff];
  const int nseg = (int)d[kSegCap];
  const int64_t woff = d[kWinOff];
  int32_t* b0 = wb0 + woff;
  int32_t* b1 = wb1 + woff;
  int32_t* ws = wseg + woff;
  int64_t* en = entry + woff;
  int64_t* ex = exit_state + woff;
  int32_t* nb = nblk + woff;
  int32_t* fl = flag + woff;
  int32_t* wbs = wbase + woff;
  // 1. windows: interval i is cut into max(1, ceil(bits / window_bits)) windows
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (int t0 = 0; t0 < nseg; t0 += kHuffThreads) {
    const int i = t0 + threadIdx.x;
    int32_t nw = 0, bits = 0;
    if (i < nseg) {
      bits = (seg[i + 1] - seg[i]) * 8;
      nw = bits > 0 ? (bits + window_bits - 1) / window_bits : 1;
    }
    int32_t excl, agg;
    IntScan(tmp.i).ExclusiveSum(nw, excl, agg);
    const int32_t first = s_carry + excl;
    if (i < nseg && first + nw <= d[kWinCap]) {
      for (int w = 0; w < nw; ++w) {
        b0[first + w] = seg[i] * 8 + w * window_bits;
        b1[first + w] = min(seg[i] * 8 + (w + 1) * window_bits, seg[i + 1] * 8);
        ws[first + w] = i;
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) s_carry += agg;
    __syncthreads();
  }
  const int nwin = s_carry;
  if (nwin > d[kWinCap]) {          // cannot happen for a descriptor the library sized; kept as a guard
    if (threadIdx.x == 0) status[2 * s] = DIB_JPEG_MCUS;
    return;
  }
  const Ctx cx{ustream + d[kStreamOff], natural, tabs, comp_of, nc == 1 ? 1 : (int)d[kBpm]};
  // 2. speculative decode of every window from its guessed state
  for (int w = threadIdx.x; w < nwin; w += blockDim.x) {
    en[w] = pack_state(b0[w], 0, 0);
    decode_window<false>(cx, en[w], b1[w], seg[ws[w] + 1] * 8, ex + w, nb + w, fl + w, nullptr, d, 0);
  }
  __syncthreads();
  // 3. synchronisation rounds
  int rounds = 0;
  for (;;) {
    int dirty_any = 0;
    for (int w = threadIdx.x; w < nwin; w += blockDim.x) {
      if (w > 0 && ws[w - 1] == ws[w]) {
        const int64_t e = ex[w - 1];
        if (e != en[w]) {
          en[w] = e;
          fl[w] = -1;                  // dirty marker, replaced by the re-decode below
          dirty_any = 1;
        }
      }
    }
    if (!__syncthreads_or(dirty_any)) break;
    ++rounds;
    for (int w = threadIdx.x; w < nwin; w += blockDim.x)
      if (fl[w] == -1)
        decode_window<false>(cx, en[w], b1[w], seg[ws[w] + 1] * 8, ex + w, nb + w, fl + w, nullptr, d, 0);
    __syncthreads();
  }
  // 4. block index of each window's first block; check every interval
  if (threadIdx.x == 0) {
    s_carry = 0;
    s_bad = 0;
  }
  __syncthreads();
  for (int t0 = 0; t0 < nwin; t0 += kHuffThreads) {
    const int w = t0 + threadIdx.x;
    const int32_t v = w < nwin ? nb[w] : 0;
    int32_t excl, agg;
    IntScan(tmp.i).ExclusiveSum(v, excl, agg);
    if (w < nwin) wbs[w] = s_carry + excl;
    __syncthreads();
    if (threadIdx.x == 0) s_carry += agg;
    __syncthreads();
  }
  const int64_t Ri = d[kRi];
  const int64_t bpm = cx.bpm;
  const int64_t n_units = d[kNblk] / bpm;      // MCUs (or blocks of a one-component scan)
  for (int w = threadIdx.x; w < nwin; w += blockDim.x) {
    if (fl[w] & kFlagBad) atomicMax(&s_bad, 2);
    if (w + 1 == nwin || ws[w + 1] != ws[w]) {   // the interval's last window: blocks so far, and a whole MCU
      const int64_t end_unit = Ri ? min((int64_t)(ws[w] + 1) * Ri, n_units) : n_units;
      if ((int64_t)wbs[w] + nb[w] != end_unit * bpm || (ex[w] & 0xFFFF) != 0) atomicMax(&s_bad, 1);
    }
  }
  __syncthreads();
  if (s_bad) {
    if (threadIdx.x == 0) {
      status[2 * s] = s_bad == 2 ? DIB_JPEG_HUFFMAN : DIB_JPEG_MCUS;
      status[2 * s + 1] = rounds;
    }
    return;
  }
  // 5. coefficients
  int16_t* ci = coef + d[kCoefOff] * 64;
  for (int w = threadIdx.x; w < nwin; w += blockDim.x) {
    int64_t xs;
    int32_t xn, xf;
    decode_window<true>(cx, en[w], b1[w], seg[ws[w] + 1] * 8, &xs, &xn, &xf, ci, d, wbs[w]);
  }
  __syncthreads();
  // 6. DC: per component, a segmented inclusive scan of the differences over the blocks in decode order
  const int64_t nblk_img = d[kNblk];
  const int64_t interval_blocks = Ri ? Ri * bpm : nblk_img;
  for (int c = 0; c < nc; ++c) {
    RunningPrefix<SegPair, SegOp> pre{SegPair{1, 0}, SegOp{}};
    for (int64_t t0 = 0; t0 < nblk_img; t0 += kHuffThreads) {
      const int64_t g = t0 + threadIdx.x;
      int16_t* p = nullptr;
      SegPair v{0, 0};
      if (g < nblk_img) {
        const int b = (int)(g % bpm);
        v.flag = g % interval_blocks == 0;
        if (comp_of[b] == c) {
          // the block's storage (decode order -> component plane)
          int by, bx;
          if (nc == 1) {
            by = (int)(g / d[kComp + 2]);
            bx = (int)(g - (int64_t)by * d[kComp + 2]);
          } else {
            const int64_t mcu = g / bpm;
            const int my = (int)(mcu / d[kMcux]), mx = (int)(mcu - (int64_t)my * d[kMcux]);
            int first = 0;
            for (int e = 0; e < c; ++e) first += (int)(d[kComp + 8 * e] * d[kComp + 8 * e + 1]);
            const int h = (int)d[kComp + 8 * c], r = b - first;
            by = my * (int)d[kComp + 8 * c + 1] + r / h;
            bx = mx * h + r % h;
          }
          const int64_t* cc = d + kComp + 8 * c;
          p = ci + (cc[7] + (int64_t)by * cc[2] + bx) * 64;
          v.val = p[0];
        }
      }
      SegPair out;
      PairScan(tmp.p).InclusiveScan(v, out, SegOp{}, pre);
      __syncthreads();
      if (p) p[0] = (int16_t)out.val;
    }
  }
  if (threadIdx.x == 0) status[2 * s + 1] = rounds;
}

// ---------------------------------------------------------------------------------------------------------------
// jidctint.c jpeg_idct_islow
constexpr int kConstBits = 13, kPass1Bits = 2;
constexpr int32_t F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299,
                  F1847 = 15137, F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;

__device__ __forceinline__ void idct_1d(int32_t i0, int32_t i1, int32_t i2, int32_t i3, int32_t i4, int32_t i5,
                                        int32_t i6, int32_t i7, int32_t o[8], int shift) {
  int32_t z1 = (i2 + i6) * F0541;
  const int32_t tmp2 = z1 + i6 * -F1847;
  const int32_t tmp3 = z1 + i2 * F0765;
  const int32_t tmp0 = (i0 + i4) * (1 << kConstBits);
  const int32_t tmp1 = (i0 - i4) * (1 << kConstBits);
  const int32_t t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
  int32_t a0 = i7, a1 = i5, a2 = i3, a3 = i1;
  z1 = a0 + a3;
  int32_t z2 = a1 + a2, z3 = a0 + a2, z4 = a1 + a3;
  const int32_t z5 = (z3 + z4) * F1175;
  a0 *= F0298;
  a1 *= F2053;
  a2 *= F3072;
  a3 *= F1501;
  z1 *= -F0899;
  z2 *= -F2562;
  z3 *= -F1961;
  z4 *= -F0390;
  z3 += z5;
  z4 += z5;
  a0 += z1 + z3;
  a1 += z2 + z4;
  a2 += z2 + z3;
  a3 += z1 + z4;
  const int32_t rnd = 1 << (shift - 1);
  o[0] = (t10 + a3 + rnd) >> shift;
  o[7] = (t10 - a3 + rnd) >> shift;
  o[1] = (t11 + a2 + rnd) >> shift;
  o[6] = (t11 - a2 + rnd) >> shift;
  o[2] = (t12 + a1 + rnd) >> shift;
  o[5] = (t12 - a1 + rnd) >> shift;
  o[3] = (t13 + a0 + rnd) >> shift;
  o[4] = (t13 - a0 + rnd) >> shift;
}

// IDCT_range_limit[x & RANGE_MASK]: wrap x to 10 bits, then clamp x + 128 to [0, 255].
__device__ __forceinline__ uint32_t range_limit(int32_t x) {
  const int32_t t = x & 1023;
  const int32_t v = (t >= 512 ? t - 1024 : t) + 128;
  return (uint32_t)min(max(v, 0), 255);
}

__global__ void __launch_bounds__(kIdctThreads) jpeg_idct_kernel(const int64_t* __restrict__ desc,
                                                                  const int32_t* __restrict__ status,
                                                                  const int32_t* __restrict__ quant,
                                                                  const int16_t* __restrict__ coef, uint8_t* planes) {
  const int s = blockIdx.y;
  if (status[2 * s] != 0) return;
  const int64_t* d = desc + (size_t)s * DIB_JPEG_DESC;
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= d[kNblk]) return;
  int c = 0;
  while (c + 1 < d[kNc] && g >= d[kComp + 8 * (c + 1) + 7]) ++c;
  const int64_t* cc = d + kComp + 8 * c;
  const int64_t r = g - cc[7];
  const int bw = (int)cc[2];
  const int by = (int)(r / bw), bx = (int)(r - (int64_t)by * bw);
  const int16_t* in = coef + (d[kCoefOff] + g) * 64;
  const int32_t* q = quant + ((size_t)s * 3 + c) * 64;
  int32_t blk[64];
  {
    const int4* v = reinterpret_cast<const int4*>(in);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int4 x = v[j];
      const int32_t w4[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
      for (int h = 0; h < 4; ++h) {
        blk[8 * j + 2 * h] = (int16_t)(w4[h] & 0xFFFF) * __ldg(q + 8 * j + 2 * h);
        blk[8 * j + 2 * h + 1] = (int16_t)((uint32_t)w4[h] >> 16) * __ldg(q + 8 * j + 2 * h + 1);
      }
    }
  }
  int32_t ws[64];
#pragma unroll
  for (int col = 0; col < 8; ++col) {
    int32_t o[8];
    idct_1d(blk[col], blk[8 + col], blk[16 + col], blk[24 + col], blk[32 + col], blk[40 + col], blk[48 + col],
            blk[56 + col], o, kConstBits - kPass1Bits);
#pragma unroll
    for (int rr = 0; rr < 8; ++rr) ws[8 * rr + col] = o[rr];
  }
  uint8_t* dst = planes + cc[6] + (int64_t)(by * 8) * (bw * 8) + bx * 8;
#pragma unroll
  for (int row = 0; row < 8; ++row) {
    int32_t o[8];
    idct_1d(ws[8 * row], ws[8 * row + 1], ws[8 * row + 2], ws[8 * row + 3], ws[8 * row + 4], ws[8 * row + 5],
            ws[8 * row + 6], ws[8 * row + 7], o, kConstBits + kPass1Bits + 3);
    uint2 pk;
    pk.x = range_limit(o[0]) | range_limit(o[1]) << 8 | range_limit(o[2]) << 16 | range_limit(o[3]) << 24;
    pk.y = range_limit(o[4]) | range_limit(o[5]) << 8 | range_limit(o[6]) << 16 | range_limit(o[7]) << 24;
    *reinterpret_cast<uint2*>(dst + (int64_t)row * bw * 8) = pk;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Upsampling and colour
__device__ __forceinline__ int upsampled(const uint8_t* pl, int stride, int dw, int dh, int rh, int rv, int x, int y) {
  if (rh == 1 && rv == 1) return pl[(int64_t)y * stride + x];
  if (rh == 2 && dw <= 2) return pl[(int64_t)(rv == 2 ? y >> 1 : y) * stride + (x >> 1)];   // box replication
  if (rh == 1) {                                                                                 // h1v2
    const int i = y >> 1, odd = y & 1;
    const int i1 = odd ? min(i + 1, dh - 1) : max(i - 1, 0);
    return (3 * pl[(int64_t)i * stride + x] + pl[(int64_t)i1 * stride + x] + (odd ? 2 : 1)) >> 2;
  }
  const int j = x >> 1, right = x & 1;
  const int jn = right ? j + 1 : j - 1;           // the further column
  const bool edge = right ? j == dw - 1 : j == 0;
  if (rv == 1) {                                  // h2v1
    const uint8_t* row = pl + (int64_t)y * stride;
    if (edge) return row[j];
    return (3 * row[j] + row[jn] + (right ? 2 : 1)) >> 2;
  }
  const int i = y >> 1, odd = y & 1;              // h2v2
  const int i1 = odd ? min(i + 1, dh - 1) : max(i - 1, 0);
  const uint8_t* r0 = pl + (int64_t)i * stride;
  const uint8_t* r1 = pl + (int64_t)i1 * stride;
  const int cs = 3 * r0[j] + r1[j];
  if (edge) return (4 * cs + (right ? 7 : 8)) >> 4;
  const int cn = 3 * r0[jn] + r1[jn];
  return (3 * cs + cn + (right ? 7 : 8)) >> 4;
}

// jdcolor.c build_ycc_rgb_table (SCALEBITS 16): FIX(1.40200) = 91881, FIX(1.77200) = 116130, FIX(0.71414) = 46802,
// FIX(0.34414) = 22554, ONE_HALF = 1 << 15; the tables' entries, computed in place.
__device__ __forceinline__ int cr_r(int i) { return (91881 * (i - 128) + 32768) >> 16; }
__device__ __forceinline__ int cb_b(int i) { return (116130 * (i - 128) + 32768) >> 16; }
__device__ __forceinline__ int cr_g(int i) { return -46802 * (i - 128); }
__device__ __forceinline__ int cb_g(int i) { return -22554 * (i - 128) + 32768; }

__global__ void __launch_bounds__(kColorThreads) jpeg_color_kernel(const int64_t* __restrict__ desc,
                                                                    const int32_t* __restrict__ status,
                                                                    const uint8_t* __restrict__ planes,
                                                                    uint8_t* out) {
  const int s = blockIdx.y;
  if (status[2 * s] != 0) return;
  const int64_t* d = desc + (size_t)s * DIB_JPEG_DESC;
  const int W = (int)d[kW], H = (int)d[kH];
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= (int64_t)W * H) return;
  const int y = (int)(p / W), x = (int)(p - (int64_t)y * W);
  uint8_t* o = out + d[kOutOff] + 3 * p;
  const int64_t* c0 = d + kComp;
  const int Y = upsampled(planes + c0[6], (int)c0[2] * 8, (int)c0[4], (int)c0[5], (int)(d[kHmax] / c0[0]),
                          (int)(d[kVmax] / c0[1]), x, y);
  if (d[kNc] == 1) {
    o[0] = o[1] = o[2] = (uint8_t)Y;
    return;
  }
  const int64_t* c1 = d + kComp + 8;
  const int64_t* c2 = d + kComp + 16;
  const int cb = upsampled(planes + c1[6], (int)c1[2] * 8, (int)c1[4], (int)c1[5], (int)(d[kHmax] / c1[0]),
                           (int)(d[kVmax] / c1[1]), x, y);
  const int cr = upsampled(planes + c2[6], (int)c2[2] * 8, (int)c2[4], (int)c2[5], (int)(d[kHmax] / c2[0]),
                           (int)(d[kVmax] / c2[1]), x, y);
  const int r = Y + cr_r(cr);
  const int g = Y + ((cb_g(cb) + cr_g(cr)) >> 16);
  const int b = Y + cb_b(cb);
  o[0] = (uint8_t)min(max(r, 0), 255);
  o[1] = (uint8_t)min(max(g, 0), 255);
  o[2] = (uint8_t)min(max(b, 0), 255);
}

int check_desc(const int64_t* q, int s, size_t stream_bytes, size_t out_bytes) {
  DIB_REQUIRE(q[kW] >= 1 && q[kH] >= 1 && q[kW] <= 65535 && q[kH] <= 65535, "image %d: size %lld x %lld", s,
              (long long)q[kW], (long long)q[kH]);
  DIB_REQUIRE(q[kNc] == 1 || q[kNc] == 3, "image %d: %lld components", s, (long long)q[kNc]);
  DIB_REQUIRE(q[kStreamOff] >= 0 && q[kStreamLen] >= 0 && q[kStreamLen] < (1 << 28) &&
                  (size_t)(q[kStreamOff] + q[kStreamLen]) <= stream_bytes,
              "image %d: entropy data [%lld, +%lld) outside the %zu-byte stream", s, (long long)q[kStreamOff],
              (long long)q[kStreamLen], stream_bytes);
  DIB_REQUIRE(q[kOutOff] >= 0 && (size_t)(q[kOutOff] + 3 * q[kW] * q[kH]) <= out_bytes,
              "image %d: output outside the %zu-byte buffer", s, out_bytes);
  DIB_REQUIRE(q[kRi] >= 0 && q[kRi] <= 65535 && q[kHmax] >= 1 && q[kHmax] <= 2 && q[kVmax] >= 1 && q[kVmax] <= 2,
              "image %d: restart interval or sampling factors out of range", s);
  int64_t bpm = 0, nblk = 0;
  for (int c = 0; c < q[kNc]; ++c) {
    const int64_t* cc = q + kComp + 8 * c;
    DIB_REQUIRE(cc[0] >= 1 && cc[1] >= 1 && q[kHmax] % cc[0] == 0 && q[kVmax] % cc[1] == 0,
                "image %d: component %d sampling factors", s, c);
    DIB_REQUIRE(cc[4] == (q[kW] * cc[0] + q[kHmax] - 1) / q[kHmax] && cc[5] == (q[kH] * cc[1] + q[kVmax] - 1) / q[kVmax],
                "image %d: component %d size", s, c);
    DIB_REQUIRE(cc[2] * 8 >= cc[4] && cc[3] * 8 >= cc[5] && cc[7] == nblk, "image %d: component %d block grid", s, c);
    if (q[kNc] == 3)
      DIB_REQUIRE(cc[2] == q[kMcux] * cc[0] && cc[3] == q[kMcuy] * cc[1], "image %d: component %d block grid", s, c);
    bpm += cc[0] * cc[1];
    nblk += cc[2] * cc[3];
  }
  DIB_REQUIRE(q[kNblk] == nblk && (q[kNc] == 1 ? q[kBpm] == 1 : q[kBpm] == bpm && bpm <= 10),
              "image %d: block counts", s);
  DIB_REQUIRE(nblk < (1 << 27), "image %d: too many blocks", s);
  return 0;
}

int decode(const uint8_t* stream, size_t stream_bytes, const int64_t* desc, const int32_t* huff,
           const int32_t* quant, int S, int window_bits, uint8_t* out, size_t out_bytes, int32_t* status,
           void* workspace, size_t workspace_bytes, cudaStream_t cs) {
  DIB_REQUIRE(S >= 0 && S <= kMaxS, "S must be in [0, %d] (got %d)", kMaxS, S);
  DIB_REQUIRE(window_bits >= kMinWindowBits && window_bits <= (1 << 20), "window_bits must be in [%d, 2^20] (got %d)",
              kMinWindowBits, window_bits);
  if (S == 0) return 0;
  DIB_REQUIRE(stream && desc && huff && quant && out && status && workspace, "a required pointer is null");
  std::vector<int64_t> d(desc, desc + (size_t)S * DIB_JPEG_DESC);
  for (int s = 0; s < S; ++s) {
    const int rc = check_desc(d.data() + (size_t)s * DIB_JPEG_DESC, s, stream_bytes, out_bytes);
    if (rc) return rc;
  }
  const Layout L = layout(d, S, stream_bytes, window_bits);
  if (workspace_bytes < L.total) {
    set_error("jpeg_decode: workspace is %zu bytes, %zu needed", workspace_bytes, L.total);
    return DIB_ENOMEM;
  }
  int64_t max_blocks = 0, max_pixels = 0;
  for (int s = 0; s < S; ++s) {
    const int64_t* q = d.data() + (size_t)s * DIB_JPEG_DESC;
    max_blocks = q[kNblk] > max_blocks ? q[kNblk] : max_blocks;
    max_pixels = q[kW] * q[kH] > max_pixels ? q[kW] * q[kH] : max_pixels;
  }
  unsigned char* ws = (unsigned char*)workspace;
  DIB_CHECK_CUDA(cudaMemcpyAsync(ws + L.desc, d.data(), d.size() * sizeof(int64_t), cudaMemcpyHostToDevice, cs));
  const int64_t* dd = (const int64_t*)(ws + L.desc);
  int16_t* coef = (int16_t*)(ws + L.coef);
  DIB_CHECK_CUDA(cudaMemsetAsync(coef, 0, L.planes - L.coef, cs));
  jpeg_unstuff_kernel<<<S, kThreads, 0, cs>>>(stream, dd, ws + L.ustream, (int32_t*)(ws + L.seg),
                                              (int32_t*)(ws + L.info), status);
  DIB_CHECK_CUDA(cudaGetLastError());
  jpeg_huffman_kernel<<<S, kHuffThreads, 0, cs>>>(dd, huff, ws + L.ustream, (const int32_t*)(ws + L.seg), window_bits,
                                              (int32_t*)(ws + L.wb0), (int32_t*)(ws + L.wb1),
                                              (int32_t*)(ws + L.wseg), (int64_t*)(ws + L.entry),
                                              (int64_t*)(ws + L.exit_), (int32_t*)(ws + L.nblk),
                                              (int32_t*)(ws + L.flag), (int32_t*)(ws + L.base), coef, status);
  DIB_CHECK_CUDA(cudaGetLastError());
  const dim3 gi((unsigned)((max_blocks + kIdctThreads - 1) / kIdctThreads), S);
  jpeg_idct_kernel<<<gi, kIdctThreads, 0, cs>>>(dd, status, quant, coef, ws + L.planes);
  DIB_CHECK_CUDA(cudaGetLastError());
  const dim3 gc((unsigned)((max_pixels + kColorThreads - 1) / kColorThreads), S);
  jpeg_color_kernel<<<gc, kColorThreads, 0, cs>>>(dd, status, ws + L.planes, out);
  DIB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace jpg
}  // namespace dib

extern "C" {

size_t jpeg_decode_workspace_bytes(const int64_t* desc, int S, size_t stream_bytes, int window_bits) {
  if (S < 0 || S > dib::jpg::kMaxS || window_bits < dib::jpg::kMinWindowBits || window_bits > (1 << 20) || (S && !desc)) return 0;
  std::vector<int64_t> d(desc, desc + (size_t)S * DIB_JPEG_DESC);
  for (int s = 0; s < S; ++s)
    if (dib::jpg::check_desc(d.data() + (size_t)s * DIB_JPEG_DESC, s, stream_bytes, SIZE_MAX)) return 0;
  return dib::jpg::layout(d, S, stream_bytes, window_bits).total;
}

int jpeg_decode_batch_u8(const uint8_t* stream, size_t stream_bytes, const int64_t* desc, const int32_t* huff,
                         const int32_t* quant, int S, int window_bits, uint8_t* out, size_t out_bytes,
                         int32_t* status, void* workspace, size_t workspace_bytes, dib_stream_t stream_) {
  return dib::jpg::decode(stream, stream_bytes, desc, huff, quant, S, window_bits, out, out_bytes, status, workspace,
                          workspace_bytes, (cudaStream_t)stream_);
}

}  // extern "C"
