// Batched PNG decoding (8-bit truecolour, not interlaced), bit for bit with OpenCV 4.13 / libpng, straight into
// imageprep.pack_images' HWC buffer; 8-bit greyscale too when the descriptor's bytes-per-pixel slot says 1 (the
// RobotCar Bayer mosaics, imageprep.decode_grey_png_batch, DESIGN.md 4.25).  DESIGN.md 4.23 states the contract;
// oracle_png/ is its CPU restatement, and deepi2p_b200/png.py walks the chunks, checks the small critical chunks and
// packs the IDAT payloads on the host.
//
// png_crc_kernel       warp per piece (at most kPiece bytes of one IDAT chunk): CRC-32 of the piece, each lane over a
//                      contiguous slice, the slices combined in GF(2) (x^(8n) mod P, as zlib's crc32_combine does)
// png_chunk_kernel     thread per IDAT chunk: combines CRC("IDAT") with its pieces' CRCs and compares the result with
//                      the stored CRC
// png_inflate_kernel   warp per image: the zlib stream, block by block.  Every lane runs the same bit decode (the bit
//                      buffer in registers, refilled from a shared-memory stage the warp loads 1 KB at a time, table
//                      lookups broadcast from shared memory), so the control flow is warp-uniform; dynamic tables are
//                      built by the warp in shared memory (9-bit / 6-bit first level plus subtables, zlib's
//                      inflate_table rules), literals are staged in shared memory and written in runs of 32, and LZ77
//                      copies are spread over the lanes, an overlapping copy repeating its period.  The output is the
//                      filtered scanlines, h x (1 + 3w) bytes, in the workspace
// png_unfilter_kernel  CTA per image: the Adler-32 of the inflated data (sum and position-weighted sum, exact in
//                      64 bits per thread at any supported size, reduced mod 65521 before the block sum), the
//                      filter-byte check, then a row wavefront (thread per row and channel, row r one pixel behind
//                      row r - 1) that undoes the five filters into HWC RGB (or H x W grey)
//
// Every input read is bounded by the packed data, every output write by the image's descriptor; a corrupt stream ends
// in a status code.  Integer arithmetic only and no atomics, so a decode is bit-identical across runs and streams.
#include <cub/block/block_reduce.cuh>

#include <vector>

#include "common.cuh"

namespace dib {
namespace png {

constexpr int kMaxS = 65535;
constexpr int kPiece = 8192;                   // CRC piece length: one warp, 256 bytes per lane
constexpr int kWarps = 4;                      // inflate warps (images) per CTA
constexpr int kRows = 256;                     // unfilter wavefront rows per pass
constexpr int kUnfThreads = 3 * kRows;
constexpr int kLitRoot = 9, kDistRoot = 6, kClenRoot = 7;
constexpr int kLitCap = 852, kDistCap = 592;   // zlib's ENOUGH_LENS / ENOUGH_DISTS for these roots
constexpr int kStage = 2048;                   // input stage ring, loaded kStage / 2 bytes at a time
constexpr uint32_t kPoly = 0xEDB88320u;
constexpr uint32_t kCrcIdat = 0x35AF061Eu;     // CRC-32 of the chunk type "IDAT"

// Descriptor slots (int64), DIB_PNG_DESC of them per image; the caller fills 0..7, 9 and 10, the library 8.  kBpp is
// the bytes per pixel: 0 (the default) or 3 for RGB, 1 for grey.
enum { kInOff = 0, kInLen, kOutOff, kW, kH, kChunk0, kWbits, kSkip, kRawOff, kNChunk, kBpp };
static_assert(kBpp < DIB_PNG_DESC, "descriptor slots");
// Library chunk records in the workspace: the caller's four slots, then the chunk's first piece and piece count.
constexpr int kChunkSlots = 6;

__host__ __device__ inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

struct Layout {
  size_t desc, chunks, pieces, piece_crc, adler, raw, total;
};

__host__ __device__ inline int64_t bpp(const int64_t* q) { return q[kBpp] ? q[kBpp] : 3; }

__host__ __device__ inline int64_t raw_bytes(const int64_t* q) { return q[kSkip] ? 0 : q[kH] * (1 + bpp(q) * q[kW]); }

// Fills the library's slots (raw offsets) and the piece list, and returns the workspace layout.
inline Layout layout(std::vector<int64_t>& d, int S, std::vector<int64_t>& ch, int C, std::vector<int64_t>& pieces) {
  int64_t raw = 0;
  for (int s = 0; s < S; ++s) {
    int64_t* q = d.data() + (size_t)s * DIB_PNG_DESC;
    q[kRawOff] = raw;
    raw += (int64_t)align256((size_t)raw_bytes(q));
  }
  pieces.clear();
  for (int c = 0; c < C; ++c) {
    int64_t* r = ch.data() + (size_t)c * kChunkSlots;
    r[4] = (int64_t)(pieces.size() / 4);
    for (int64_t o = 0; o < r[2]; o += kPiece) {
      const int64_t n = r[2] - o < kPiece ? r[2] - o : kPiece;
      pieces.insert(pieces.end(), {r[1] + o, n, r[2] - o - n, 0});   // data offset, length, bytes after it
    }
    r[5] = (int64_t)(pieces.size() / 4) - r[4];
  }
  const size_t P = pieces.size() / 4;
  Layout L;
  L.desc = 0;
  L.chunks = align256((size_t)S * DIB_PNG_DESC * sizeof(int64_t));
  L.pieces = L.chunks + align256((size_t)C * kChunkSlots * sizeof(int64_t));
  L.piece_crc = L.pieces + align256(P * 4 * sizeof(int64_t));
  L.adler = L.piece_crc + align256(P * sizeof(uint32_t));
  L.raw = L.adler + align256((size_t)S * sizeof(uint32_t));
  L.total = L.raw + (size_t)raw;
  return L;
}

// ---------------------------------------------------------------------------------------------------------------
// CRC-32.  multmodp / x2nmodp are the GF(2) product modulo P and x^(n 2^k) mod P in the reflected representation
// (x^0 is bit 31); crc(A || B) = x^(8 |B|) crc(A) + crc(B).

__device__ __forceinline__ uint32_t multmodp(uint32_t a, uint32_t b) {
  uint32_t p = 0;
  for (uint32_t m = 1u << 31; m; m >>= 1) {
    if (a & m) p ^= b;
    b = (b & 1) ? (b >> 1) ^ kPoly : b >> 1;
  }
  return p;
}

// x2n[k] = x^(2^k) mod P.
__device__ void init_crc_tables(uint32_t* table, uint32_t* x2n) {
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    uint32_t c = (uint32_t)i;
    for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ kPoly : c >> 1;
    table[i] = c;
  }
  for (int k = threadIdx.x; k < 32; k += blockDim.x) {
    uint32_t p = 1u << 30;                                          // x^1
    for (int j = 0; j < k; ++j) p = multmodp(p, p);
    x2n[k] = p;
  }
  __syncthreads();
}

__device__ __forceinline__ uint32_t crc_combine(const uint32_t* x2n, uint32_t a, uint32_t b, int64_t len_b) {
  uint32_t p = 1u << 31;                                            // x^0
  for (int k = 3; len_b; len_b >>= 1, ++k)
    if (len_b & 1) p = multmodp(x2n[k & 31], p);
  return multmodp(p, a) ^ b;
}

__global__ void __launch_bounds__(256) png_crc_kernel(const uint8_t* __restrict__ data, size_t data_bytes,
                                                      const int64_t* __restrict__ pieces, int P,
                                                      uint32_t* __restrict__ piece_crc) {
  __shared__ uint32_t table[256], x2n[32];
  init_crc_tables(table, x2n);
  const int lane = threadIdx.x & 31;
  const int p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (p >= P) return;
  const int64_t off = pieces[4 * p], len = pieces[4 * p + 1];
  const int64_t per = (len + 31) >> 5;
  int64_t lo = min((int64_t)lane * per, len), hi = min(lo + per, len);
  if (off < 0 || (size_t)(off + len) > data_bytes) lo = hi = 0;     // the host checked; never read outside
  uint32_t c = 0xFFFFFFFFu;
  for (int64_t i = lo; i < hi; ++i) c = table[(c ^ data[off + i]) & 255] ^ (c >> 8);
  c ^= 0xFFFFFFFFu;
  int64_t n = hi - lo;
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t rc = __shfl_down_sync(0xFFFFFFFFu, c, d);
    const int64_t rn = __shfl_down_sync(0xFFFFFFFFu, n, d);
    if ((lane & (2 * d - 1)) == 0 && lane + d < 32) {
      c = crc_combine(x2n, c, rc, rn);
      n += rn;
    }
  }
  if (lane == 0) piece_crc[p] = c;
}

__global__ void __launch_bounds__(128) png_chunk_kernel(const int64_t* __restrict__ chunks, int C,
                                                        const uint32_t* __restrict__ piece_crc,
                                                        int32_t* __restrict__ status) {
  __shared__ uint32_t table[256], x2n[32];
  init_crc_tables(table, x2n);
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const int64_t* r = chunks + (size_t)c * kChunkSlots;
  uint32_t crc = kCrcIdat;
  int64_t left = r[2];
  for (int64_t i = 0; i < r[5]; ++i) {
    const int64_t n = left < kPiece ? left : kPiece;
    crc = crc_combine(x2n, crc, piece_crc[r[4] + i], n);
    left -= n;
  }
  if (crc != (uint32_t)r[3]) status[4 * r[0] + 1] = DIB_PNG_CRC;  // every writer stores the same value
}

// ---------------------------------------------------------------------------------------------------------------
// Inflate.  A table entry is 0 (no code), a symbol (bit 25 set, length in bits 16..20, symbol in 0..15) or a
// subtable pointer (bit 24 set, subtable bits in 16..20, offset in 0..15).

constexpr uint32_t kValid = 1u << 25, kPtr = 1u << 24;

__constant__ uint16_t kLenBase[29] = {3,  4,  5,  6,  7,  8,  9,  10, 11,  13,  15,  17,  19,  23, 27,
                                      31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t kLenExtra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t kDistBase[30] = {1,   2,   3,   4,   5,   7,    9,    13,   17,   25,   33,   49,   65,    97,    129,
                                       193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t kDistExtra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t kClenOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

struct alignas(16) WarpSmem {
  uint32_t lit[kLitCap];
  uint32_t dist[kDistCap];
  uint32_t clen[1 << kClenRoot];
  uint32_t count[16], start[16], code[16];
  uint16_t sorted[320];
  uint8_t lens[352];
  alignas(16) uint8_t stage[kStage];   // stage_load writes it 16 bytes at a time
  uint8_t litbuf[32];
  int next;          // build_table: the number of coded symbols
  int err;
};

enum Kind { kCodes = 0, kLens = 1, kDists = 2 };

__device__ __forceinline__ uint32_t bitrev(uint32_t code, int len) { return __brev(code) >> (32 - len); }

// zlib's inflate_table rules: over-subscribed sets are invalid; an incomplete set is valid only for literal/length or
// distance codes whose longest code has length 1; a set of all-zero lengths is valid and codes nothing.  Returns 0 or
// DIB_PNG_LENGTHS.  Called by the whole warp.
__device__ int build_table(WarpSmem& sm, const uint8_t* lens, int n, int root, uint32_t* table, int cap, int kind,
                           int lane) {
  for (int i = lane; i < cap; i += 32) table[i] = 0;
  __syncwarp();
  if (lane == 0) {
    int err = 0;
    for (int l = 0; l < 16; ++l) sm.count[l] = 0;
    for (int s = 0; s < n; ++s) sm.count[lens[s]]++;
    int max = 15;
    while (max > 0 && sm.count[max] == 0) --max;
    int left = 1;
    for (int l = 1; l <= 15; ++l) {
      left = (left << 1) - (int)sm.count[l];
      if (left < 0) err = DIB_PNG_LENGTHS;
    }
    if (kind == kCodes ? (max == 0 || left > 0) : (left > 0 && max > 1)) err = DIB_PNG_LENGTHS;
    uint32_t off = 0, code = 0;
    for (int l = 1; l <= 15; ++l) {
      sm.start[l] = off;
      sm.code[l] = code;
      off += sm.count[l];
      code = (code + sm.count[l]) << 1;
    }
    if (!err) {
      uint32_t fill[16];
      for (int l = 1; l <= 15; ++l) fill[l] = sm.start[l];
      for (int s = 0; s < n; ++s)
        if (lens[s]) sm.sorted[fill[lens[s]]++] = (uint16_t)s;
      // Subtables: the codes sharing a root prefix are contiguous in canonical order, and the last of a group is its
      // longest, so it sets the group's subtable size.
      int next = 1 << root;
      for (int i = 0; i < (int)off && !err; ++i) {
        const int l = lens[sm.sorted[i]];
        if (l <= root) continue;
        const uint32_t prefix = (sm.code[l] + (uint32_t)(i - (int)sm.start[l])) >> (l - root);
        bool last = i + 1 == (int)off;
        if (!last) {
          const int l2 = lens[sm.sorted[i + 1]];
          last = ((sm.code[l2] + (uint32_t)(i + 1 - (int)sm.start[l2])) >> (l2 - root)) != prefix;
        }
        if (!last) continue;
        if (next + (1 << (l - root)) > cap) {
          err = DIB_PNG_LENGTHS;
        } else {
          table[bitrev(prefix, root)] = kPtr | ((uint32_t)(l - root) << 16) | (uint32_t)next;
          next += 1 << (l - root);
        }
      }
    }
    sm.next = (int)off;
    sm.err = err;
  }
  __syncwarp();
  if (sm.err) return sm.err;
  const int nsym = sm.next;
  for (int i = lane; i < nsym; i += 32) {
    const int sym = sm.sorted[i];
    const int l = lens[sym];
    const uint32_t rev = bitrev(sm.code[l] + (uint32_t)(i - (int)sm.start[l]), l);
    if (l <= root) {
      const uint32_t e = kValid | ((uint32_t)l << 16) | (uint32_t)sym;
      for (uint32_t k = rev; k < (1u << root); k += 1u << l) table[k] = e;
    } else {
      const uint32_t p = table[rev & ((1u << root) - 1)];
      const int sb = (p >> 16) & 31, l2 = l - root;
      const uint32_t e = kValid | ((uint32_t)l2 << 16) | (uint32_t)sym;
      for (uint32_t k = rev >> root; k < (1u << sb); k += 1u << l2) table[(p & 0xFFFF) + k] = e;
    }
  }
  __syncwarp();
  return 0;
}

static_assert(sizeof(WarpSmem) % 16 == 0 && offsetof(WarpSmem, stage) % 16 == 0, "stage alignment");

struct Bits {
  uint64_t bb;
  int bc;
  int64_t inpos;      // next input byte to enter bb, relative to the image's IDAT data
  int64_t stage_hi;   // input bytes [stage_hi - kStage, stage_hi) are in the stage ring
};

__device__ __forceinline__ void stage_load(WarpSmem& sm, Bits& b, const uint8_t* in, int64_t in_abs, size_t data_bytes,
                                           int lane) {
  const int64_t base = b.stage_hi + lane * 32;
  uint4 v[2];
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int64_t g = in_abs + base + 16 * k;
    if (g >= 0 && (size_t)(g + 16) <= data_bytes) {
      v[k] = __ldg((const uint4*)(in + g));
    } else {                                                        // the buffer's last partial vector, byte by byte
      uint32_t wd[4] = {0, 0, 0, 0};
      for (int j = 0; j < 16; ++j)
        if (g + j >= 0 && (size_t)(g + j) < data_bytes) wd[j >> 2] |= (uint32_t)in[g + j] << (8 * (j & 3));
      v[k] = make_uint4(wd[0], wd[1], wd[2], wd[3]);
    }
  }
  uint4* dst = (uint4*)(sm.stage + ((b.stage_hi + lane * 32) & (kStage - 1)));
  dst[0] = v[0];
  dst[1] = v[1];
  b.stage_hi += kStage / 2;
  __syncwarp();
}

__device__ __forceinline__ void refill(WarpSmem& sm, Bits& b, const uint8_t* in, int64_t in_abs, size_t data_bytes,
                                       int lane) {
  if (b.bc >= 32) return;
  while (b.inpos + 4 > b.stage_hi) stage_load(sm, b, in, in_abs, data_bytes, lane);
  const uint32_t w = (uint32_t)sm.stage[b.inpos & (kStage - 1)] | ((uint32_t)sm.stage[(b.inpos + 1) & (kStage - 1)] << 8) |
                     ((uint32_t)sm.stage[(b.inpos + 2) & (kStage - 1)] << 16) |
                     ((uint32_t)sm.stage[(b.inpos + 3) & (kStage - 1)] << 24);
  b.bb |= (uint64_t)w << b.bc;
  b.bc += 32;
  b.inpos += 4;
}

__device__ __forceinline__ uint32_t take(Bits& b, int n) {   // n <= 16
  const uint32_t v = (uint32_t)b.bb & ((1u << n) - 1);
  b.bb >>= n;
  b.bc -= n;
  return v;
}

// One symbol: the root entry, then the subtable entry if it points to one.  Returns 0 for no code.
__device__ __forceinline__ uint32_t decode(Bits& b, const uint32_t* table, int root) {
  uint32_t e = table[(uint32_t)b.bb & ((1u << root) - 1)];
  if (e & kPtr) {
    const int sb = (e >> 16) & 31;
    const uint32_t sub = table[(e & 0xFFFF) + (((uint32_t)(b.bb >> root)) & ((1u << sb) - 1))];
    if (!(sub & kValid)) return 0;
    take(b, root);
    e = sub;
  }
  if (!(e & kValid)) return 0;
  take(b, (e >> 16) & 31);
  return e;
}

__global__ void __launch_bounds__(32 * kWarps) png_inflate_kernel(const uint8_t* __restrict__ in, size_t data_bytes,
                                                                  const int64_t* __restrict__ desc, int S,
                                                                  uint8_t* raw_all, uint32_t* __restrict__ adler,
                                                                  int32_t* __restrict__ status) {
  __shared__ WarpSmem smem[kWarps];
  const int lane = threadIdx.x & 31;
  const int s = blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (s >= S) return;
  WarpSmem& sm = smem[threadIdx.x >> 5];
  const int64_t* q = desc + (size_t)s * DIB_PNG_DESC;
  if (q[kSkip]) return;
  const int64_t in_abs = q[kInOff], lim = q[kInLen] * 8;
  const int64_t raw_n = raw_bytes(q), window = (int64_t)1 << q[kWbits];
  uint8_t* raw = raw_all + q[kRawOff];
  Bits b{0, 0, 2, 0};                                               // the zlib header was checked on the host
  b.stage_hi = 0;
  int64_t outpos = 0;                                               // bytes produced, staged literals included
  int nlit = 0, err = 0, fixed_built = 0;
  auto flush = [&]() {
    __syncwarp();
    if (lane < nlit) raw[outpos - nlit + lane] = sm.litbuf[lane];
    nlit = 0;
    __syncwarp();
  };
  for (;;) {
    refill(sm, b, in, in_abs, data_bytes, lane);
    const uint32_t hdr = take(b, 3);
    if (b.inpos * 8 - b.bc > lim) { err = DIB_PNG_TRUNCATED; break; }
    const int type = hdr >> 1;
    if (type == 3) { err = DIB_PNG_BLOCK_TYPE; break; }
    if (type == 0) {
      take(b, b.bc & 7);                                            // to the byte boundary
      refill(sm, b, in, in_abs, data_bytes, lane);
      const uint32_t ln = take(b, 16), nl = take(b, 16);
      const int64_t at = b.inpos - b.bc / 8;                        // first stored byte
      if (at * 8 > lim) { err = DIB_PNG_TRUNCATED; break; }
      if (ln != (~nl & 0xFFFF)) { err = DIB_PNG_STORED; break; }
      if ((at + ln) * 8 > lim) { err = DIB_PNG_TRUNCATED; break; }
      if (outpos + ln > raw_n) { err = DIB_PNG_TOO_MUCH; break; }
      flush();
      for (uint32_t k = lane; k < ln; k += 32) raw[outpos + k] = in[in_abs + at + k];
      outpos += ln;
      __syncwarp();
      b.bb = 0;
      b.bc = 0;
      b.inpos = at + ln;
      b.stage_hi = b.inpos & ~(int64_t)(kStage / 2 - 1);
    } else {
      if (type == 1) {
        if (!fixed_built) {
          if (lane == 0)
            for (int i = 0; i < 320; ++i) sm.lens[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : i < 288 ? 8 : 5;
          __syncwarp();
          build_table(sm, sm.lens, 288, kLitRoot, sm.lit, kLitCap, kLens, lane);
          build_table(sm, sm.lens + 288, 32, kDistRoot, sm.dist, kDistCap, kDists, lane);
          fixed_built = 1;
        }
      } else {
        fixed_built = 0;
        refill(sm, b, in, in_abs, data_bytes, lane);
        const int hlit = (int)take(b, 5) + 257, hdist = (int)take(b, 5) + 1, hclen = (int)take(b, 4) + 4;
        if (b.inpos * 8 - b.bc > lim) { err = DIB_PNG_TRUNCATED; break; }
        if (hlit > 286 || hdist > 30) { err = DIB_PNG_SYMBOLS; break; }
        if (lane == 0)
          for (int i = 0; i < 19; ++i) sm.lens[i] = 0;
        __syncwarp();
        for (int i = 0; i < hclen; ++i) {
          refill(sm, b, in, in_abs, data_bytes, lane);
          const uint32_t v = take(b, 3);
          if (lane == 0) sm.lens[kClenOrder[i]] = (uint8_t)v;
        }
        __syncwarp();
        if (b.inpos * 8 - b.bc > lim) { err = DIB_PNG_TRUNCATED; break; }
        if ((err = build_table(sm, sm.lens, 19, kClenRoot, sm.clen, 1 << kClenRoot, kCodes, lane))) break;
        const int total = hlit + hdist;
        int n = 0, prev = -1;
        uint8_t* lens = sm.lens + 32;                               // past the code-length code's own lengths
        while (n < total) {
          refill(sm, b, in, in_abs, data_bytes, lane);
          const uint32_t e = decode(b, sm.clen, kClenRoot);
          if (b.inpos * 8 - b.bc > lim) { err = DIB_PNG_TRUNCATED; break; }
          if (!e) { err = DIB_PNG_LENGTHS; break; }
          const int sym = e & 0xFFFF;
          int rep = 1, val = sym;
          if (sym == 16) {
            if (prev < 0) { err = DIB_PNG_REPEAT; break; }
            rep = 3 + (int)take(b, 2);
            val = prev;
          } else if (sym == 17) {
            rep = 3 + (int)take(b, 3);
            val = 0;
          } else if (sym == 18) {
            rep = 11 + (int)take(b, 7);
            val = 0;
          }
          if (n + rep > total) { err = DIB_PNG_OVERRUN; break; }
          if (lane == 0)
            for (int r = 0; r < rep; ++r) lens[n + r] = (uint8_t)val;
          n += rep;
          prev = val;
          if (b.inpos * 8 - b.bc > lim) { err = DIB_PNG_TRUNCATED; break; }
        }
        if (err) break;
        __syncwarp();
        if (lens[256] == 0) { err = DIB_PNG_NO_EOB; break; }
        // The tables' own lengths move to the front so build_table's scratch (sm.lens) is not overwritten.
        if ((err = build_table(sm, lens, hlit, kLitRoot, sm.lit, kLitCap, kLens, lane))) break;
        if ((err = build_table(sm, lens + hlit, hdist, kDistRoot, sm.dist, kDistCap, kDists, lane))) break;
      }
      for (;;) {
        refill(sm, b, in, in_abs, data_bytes, lane);
        const uint32_t e = decode(b, sm.lit, kLitRoot);
        if (b.inpos * 8 - b.bc > lim) { err = DIB_PNG_TRUNCATED; break; }
        if (!e) { err = DIB_PNG_LITLEN; break; }
        const int sym = e & 0xFFFF;
        if (sym < 256) {
          if (outpos >= raw_n) { err = DIB_PNG_TOO_MUCH; break; }
          if (lane == 0) sm.litbuf[nlit] = (uint8_t)sym;
          ++nlit;
          ++outpos;
          if (nlit == 32) flush();
          continue;
        }
        if (sym == 256) break;
        if (sym > 285) { err = DIB_PNG_LITLEN; break; }
        const int li = sym - 257;
        const int len = kLenBase[li] + (int)take(b, kLenExtra[li]);
        refill(sm, b, in, in_abs, data_bytes, lane);
        const uint32_t de = decode(b, sm.dist, kDistRoot);
        if (b.inpos * 8 - b.bc > lim) { err = DIB_PNG_TRUNCATED; break; }
        if (!de || (de & 0xFFFF) >= 30) { err = DIB_PNG_DISTANCE; break; }
        const int di = de & 0xFFFF;
        refill(sm, b, in, in_abs, data_bytes, lane);
        const int64_t dist = kDistBase[di] + (int64_t)take(b, kDistExtra[di]);
        if (b.inpos * 8 - b.bc > lim) { err = DIB_PNG_TRUNCATED; break; }
        if (dist > outpos) { err = DIB_PNG_FAR; break; }
        if (dist > window) { err = DIB_PNG_WINDOW; break; }
        if (outpos + len > raw_n) { err = DIB_PNG_TOO_MUCH; break; }
        flush();
        // Sources lie before outpos: an overlapping copy (dist < len) repeats its period of dist bytes.
        for (int k = lane; k < len; k += 32) raw[outpos + k] = raw[outpos - dist + (k < dist ? k : k % dist)];
        outpos += len;
        __syncwarp();
      }
      if (err) break;
    }
    if (hdr & 1) break;
  }
  if (!err) {
    flush();
    if (outpos != raw_n) {
      err = DIB_PNG_SHORT;
    } else {
      take(b, b.bc & 7);
      refill(sm, b, in, in_abs, data_bytes, lane);
      const uint32_t lo = take(b, 16), hi = take(b, 16);
      if (b.inpos * 8 - b.bc > lim) err = DIB_PNG_NO_ADLER;
      else if (lane == 0) adler[s] = __byte_perm(lo | (hi << 16), 0, 0x0123);   // stored big-endian
    }
  }
  if (err && lane == 0) status[4 * s] = err;
}

// ---------------------------------------------------------------------------------------------------------------
// Adler-32, the filter-byte check and the unfilter wavefront.

// The largest inflated size (OpenCV's limits: 2^20 per side, 2^30 pixels) and one thread's position-weighted sum at
// that size: below 2^64, so the per-thread Adler-32 sums need no reduction inside the loop.
constexpr unsigned long long kMaxRaw = 3ull * (1ull << 30) + (1ull << 20);
constexpr unsigned long long kAdlerBound = (kMaxRaw + kUnfThreads - 1) / kUnfThreads * kMaxRaw * 255ull;
static_assert(kAdlerBound / 255ull / kMaxRaw == (kMaxRaw + kUnfThreads - 1) / kUnfThreads &&
                  kAdlerBound < (1ull << 63), "per-thread Adler-32 sums must not wrap");

__global__ void __launch_bounds__(kUnfThreads) png_unfilter_kernel(const int64_t* __restrict__ desc,
                                                                   const uint8_t* __restrict__ raw_all,
                                                                   const uint32_t* __restrict__ adler, uint8_t* out,
                                                                   int32_t* __restrict__ status) {
  using Reduce = cub::BlockReduce<unsigned long long, kUnfThreads>;
  __shared__ typename Reduce::TempStorage tmp;
  const int s = blockIdx.x;
  const int64_t* q = desc + (size_t)s * DIB_PNG_DESC;
  if (q[kSkip] || status[4 * s]) return;                            // block-uniform
  const int64_t w = q[kW], h = q[kH], B = bpp(q), stride = 1 + B * w, n = h * stride;
  const uint8_t* raw = raw_all + q[kRawOff];
  unsigned long long s1 = 0, s2 = 0;
  for (int64_t i = threadIdx.x; i < n; i += kUnfThreads) {
    const unsigned long long v = raw[i];
    s1 += v;
    s2 += (unsigned long long)(n - i) * v;
  }
  // Each thread's sums are exact (kAdlerBound) and reduced mod 65521 before the block sum, which then stays exact.
  s1 %= 65521;
  s2 %= 65521;
  s1 = Reduce(tmp).Sum(s1);
  __syncthreads();
  s2 = Reduce(tmp).Sum(s2);
  int bad = 0;
  for (int64_t r = threadIdx.x; r < h; r += kUnfThreads) bad |= raw[r * stride] > 4;
  bad = __syncthreads_or(bad);
  if (threadIdx.x == 0) {
    const uint32_t a = (uint32_t)((1 + s1) % 65521), bsum = (uint32_t)(((unsigned long long)n + s2) % 65521);
    if (((bsum << 16) | a) != adler[s]) status[4 * s + 2] = DIB_PNG_ADLER;
    if (bad) status[4 * s + 3] = DIB_PNG_FILTER;
  }
  if (bad) return;
  uint8_t* o = out + q[kOutOff];
  const int t = threadIdx.x, c = t % (int)B, rows = kUnfThreads / (int)B;   // kRows rows of RGB, 3 kRows of grey
  for (int64_t r0 = 0; r0 < h; r0 += rows) {
    const int64_t r = r0 + t / B;
    const bool live = r < h;
    const int f = live ? raw[r * stride] : 0;
    const uint8_t* src = raw + r * stride + 1 + c;
    uint8_t* dst = o + r * B * w + c;
    int left = 0, upleft = 0;
    const int64_t steps = w + min((int64_t)rows, h - r0) - 1;
    for (int64_t k = 0; k < steps; ++k) {
      const int64_t x = k - t / B;
      if (live && x >= 0 && x < w) {
        const int v = src[B * x];
        const int up = r > 0 ? dst[B * x - B * w] : 0;
        int pred;
        switch (f) {
          case 0: pred = 0; break;
          case 1: pred = left; break;
          case 2: pred = up; break;
          case 3: pred = (left + up) >> 1; break;
          default: {
            const int p = left + up - upleft;
            const int pa = abs(p - left), pb = abs(p - up), pc = abs(p - upleft);
            pred = (pa <= pb && pa <= pc) ? left : pb <= pc ? up : upleft;
          }
        }
        const int val = (v + pred) & 255;
        dst[B * x] = (uint8_t)val;
        left = val;
        upleft = up;
      }
      __syncthreads();
    }
  }
}

int check_desc(const int64_t* q, int s, size_t data_bytes, size_t out_bytes, const int64_t* ch, int C) {
  if (q[kSkip]) return 0;
  DIB_REQUIRE(q[kW] >= 1 && q[kH] >= 1 && q[kW] <= (1 << 20) && q[kH] <= (1 << 20) && q[kW] * q[kH] <= (1ll << 30),
              "image %d: size %lld x %lld", s, (long long)q[kW], (long long)q[kH]);
  DIB_REQUIRE(q[kInOff] >= 0 && q[kInOff] % 16 == 0 && q[kInLen] >= 2 && (size_t)(q[kInOff] + q[kInLen]) <= data_bytes,
              "image %d: IDAT data [%lld, +%lld) outside the %zu-byte stream or not 16-byte aligned", s,
              (long long)q[kInOff], (long long)q[kInLen], data_bytes);
  DIB_REQUIRE(q[kBpp] == 0 || q[kBpp] == 1 || q[kBpp] == 3, "image %d: bytes per pixel %lld", s, (long long)q[kBpp]);
  DIB_REQUIRE(q[kOutOff] >= 0 && (size_t)(q[kOutOff] + bpp(q) * q[kW] * q[kH]) <= out_bytes,
              "image %d: output outside the %zu-byte buffer", s, out_bytes);
  DIB_REQUIRE(q[kWbits] >= 8 && q[kWbits] <= 15, "image %d: window bits %lld", s, (long long)q[kWbits]);
  DIB_REQUIRE(q[kChunk0] >= 0 && q[kNChunk] >= 1 && q[kChunk0] + q[kNChunk] <= C, "image %d: chunk range", s);
  int64_t pos = q[kInOff];
  for (int64_t c = q[kChunk0]; c < q[kChunk0] + q[kNChunk]; ++c) {
    const int64_t* r = ch + (size_t)c * 4;
    DIB_REQUIRE(r[0] == s && r[1] == pos && r[2] >= 0 && r[3] >= 0 && r[3] <= 0xFFFFFFFFll,
                "image %d: chunk %lld does not continue the image's IDAT data", s, (long long)c);
    pos += r[2];
  }
  DIB_REQUIRE(pos == q[kInOff] + q[kInLen], "image %d: chunk lengths do not add up to the IDAT data", s);
  return 0;
}

int prepare(const int64_t* desc, int S, const int64_t* chunks, int C, size_t data_bytes, size_t out_bytes,
            std::vector<int64_t>& d, std::vector<int64_t>& ch, std::vector<int64_t>& pieces, Layout& L) {
  DIB_REQUIRE(S >= 0 && S <= kMaxS, "S must be in [0, %d] (got %d)", kMaxS, S);
  DIB_REQUIRE(C >= 0 && (C == 0 || chunks), "chunks: bad count or null pointer");
  DIB_REQUIRE(S == 0 || desc, "desc is null");
  d.assign(desc, desc + (size_t)S * DIB_PNG_DESC);
  for (int s = 0; s < S; ++s) {
    const int rc = check_desc(d.data() + (size_t)s * DIB_PNG_DESC, s, data_bytes, out_bytes, chunks, C);
    if (rc) return rc;
  }
  ch.assign((size_t)C * kChunkSlots, 0);
  for (int c = 0; c < C; ++c)
    for (int k = 0; k < 4; ++k) ch[(size_t)c * kChunkSlots + k] = chunks[(size_t)c * 4 + k];
  L = layout(d, S, ch, C, pieces);
  return 0;
}

int decode_batch(const uint8_t* data, size_t data_bytes, const int64_t* desc, int S, const int64_t* chunks, int C,
                 uint8_t* out, size_t out_bytes, int32_t* status, void* workspace, size_t workspace_bytes,
                 cudaStream_t cs) {
  std::vector<int64_t> d, ch, pieces;
  Layout L;
  const int rc = prepare(desc, S, chunks, C, data_bytes, out_bytes, d, ch, pieces, L);
  if (rc) return rc;
  if (S == 0) return 0;
  DIB_REQUIRE(data && status && workspace && (out || out_bytes == 0), "a required pointer is null");
  if (workspace_bytes < L.total) {
    set_error("png_decode: workspace is %zu bytes, %zu needed", workspace_bytes, L.total);
    return DIB_ENOMEM;
  }
  unsigned char* ws = (unsigned char*)workspace;
  const int P = (int)(pieces.size() / 4);
  DIB_CHECK_CUDA(cudaMemcpyAsync(ws + L.desc, d.data(), d.size() * sizeof(int64_t), cudaMemcpyHostToDevice, cs));
  if (C) DIB_CHECK_CUDA(cudaMemcpyAsync(ws + L.chunks, ch.data(), ch.size() * sizeof(int64_t), cudaMemcpyHostToDevice, cs));
  if (P) DIB_CHECK_CUDA(cudaMemcpyAsync(ws + L.pieces, pieces.data(), pieces.size() * sizeof(int64_t), cudaMemcpyHostToDevice, cs));
  DIB_CHECK_CUDA(cudaMemsetAsync(status, 0, (size_t)S * 4 * sizeof(int32_t), cs));
  const int64_t* dd = (const int64_t*)(ws + L.desc);
  uint32_t* piece_crc = (uint32_t*)(ws + L.piece_crc);
  if (P) {
    png_crc_kernel<<<(P + 7) / 8, 256, 0, cs>>>(data, data_bytes, (const int64_t*)(ws + L.pieces), P, piece_crc);
    DIB_CHECK_CUDA(cudaGetLastError());
  }
  if (C) {
    png_chunk_kernel<<<(C + 127) / 128, 128, 0, cs>>>((const int64_t*)(ws + L.chunks), C, piece_crc, status);
    DIB_CHECK_CUDA(cudaGetLastError());
  }
  uint32_t* adler = (uint32_t*)(ws + L.adler);
  png_inflate_kernel<<<(S + kWarps - 1) / kWarps, 32 * kWarps, 0, cs>>>(data, data_bytes, dd, S, ws + L.raw, adler,
                                                                       status);
  DIB_CHECK_CUDA(cudaGetLastError());
  png_unfilter_kernel<<<S, kUnfThreads, 0, cs>>>(dd, ws + L.raw, adler, out, status);
  DIB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace png
}  // namespace dib

extern "C" {

size_t png_decode_workspace_bytes(const int64_t* desc, int S, const int64_t* chunks, int n_chunks, size_t data_bytes) {
  std::vector<int64_t> d, ch, pieces;
  dib::png::Layout L;
  if (dib::png::prepare(desc, S, chunks, n_chunks, data_bytes, SIZE_MAX / 4, d, ch, pieces, L)) return 0;
  return L.total;
}

int png_decode_batch_u8(const uint8_t* data, size_t data_bytes, const int64_t* desc, int S, const int64_t* chunks,
                        int n_chunks, uint8_t* out, size_t out_bytes, int32_t* status, void* workspace,
                        size_t workspace_bytes, dib_stream_t stream) {
  return dib::png::decode_batch(data, data_bytes, desc, S, chunks, n_chunks, out, out_bytes, status, workspace,
                                workspace_bytes, (cudaStream_t)stream);
}

}  // extern "C"
