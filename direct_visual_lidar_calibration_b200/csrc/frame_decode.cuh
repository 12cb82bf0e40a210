// frame_decode.cuh -- the format logic of the zstd (RFC 8878) and LZ4-frame decoders, written once as a __host__
// __device__ core: frame_decode.cu runs it on the GPU (one warp per frame, the tables in shared memory, the warp
// computing the CRC-32), tests/cpp/frame_decode_check.cu runs the same source on the CPU under the sanitizers.
//
// One call decodes one container frame (an MCAP or ROS 1 chunk, or one rosbag2 message): a run of concatenated zstd
// or LZ4 frames, skippable frames among them, into dst[0, cap).  Every read is checked against [src, src + n) and
// every write against [dst, dst + cap); nothing is read or written outside them whatever the input holds.
//
// zstd: everything but dictionaries.  Literals that are Huffman-coded (or RLE) are decoded into the tail of dst, as
// libzstd does: the bytes a block has still to write past its output position are at least its unread literals, so
// the literal area never meets the output of a frame that fits dst.  A match or literal that would run into it
// means the frame decodes to more than cap bytes (status kSize).  Back-references reach at most to the start of
// their zstd frame (frames are independent); the window size is not needed, since the whole output stays in dst.
// LZ4 frame: independent and linked blocks, uncompressed blocks, every checksum; a match reaches at most to the start
// of its block (independent) or of its frame (linked).
#pragma once

#include <cstdint>

#ifdef __CUDACC__
#define FD_HD __host__ __device__ __forceinline__
#else
#define FD_HD inline
#endif

// Constant tables, one copy for the host and one in the device's constant bank.
#ifdef __CUDACC__
#define FD_TABLE(T, name, ...) \
  static const T name##_h[] = __VA_ARGS__; \
  __constant__ const T name##_d[] = __VA_ARGS__;
#else
#define FD_TABLE(T, name, ...) static const T name##_h[] = __VA_ARGS__;
#endif
#ifdef __CUDA_ARCH__
#define FD_T(name) name##_d
#else
#define FD_T(name) name##_h
#endif

namespace vlcal {
namespace fd {

enum Status { kOk = 0, kCorrupt = 1, kChecksum = 2, kSize = 3, kUnsupported = 4 };
enum Codec { kZstd = 1, kLz4Frame = 2 };

// ---- checksums -----------------------------------------------------------------------------------------------------

FD_HD uint32_t rotl32(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }
FD_HD uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
FD_HD uint32_t le32(const uint8_t* p) { return uint32_t(p[0]) | (uint32_t(p[1]) << 8) | (uint32_t(p[2]) << 16) | (uint32_t(p[3]) << 24); }
FD_HD uint64_t le64(const uint8_t* p) { return uint64_t(le32(p)) | (uint64_t(le32(p + 4)) << 32); }

constexpr uint32_t kX32P1 = 0x9E3779B1u, kX32P2 = 0x85EBCA77u, kX32P3 = 0xC2B2AE3Du, kX32P4 = 0x27D4EB2Fu, kX32P5 = 0x165667B1u;

FD_HD uint32_t xxh32(const uint8_t* p, int64_t n, uint32_t seed) {
  const uint8_t* const end = p + n;
  uint32_t h;
  if (n >= 16) {
    uint32_t v1 = seed + kX32P1 + kX32P2, v2 = seed + kX32P2, v3 = seed, v4 = seed - kX32P1;
    for (; end - p >= 16; p += 16) {
      v1 = rotl32(v1 + le32(p) * kX32P2, 13) * kX32P1;
      v2 = rotl32(v2 + le32(p + 4) * kX32P2, 13) * kX32P1;
      v3 = rotl32(v3 + le32(p + 8) * kX32P2, 13) * kX32P1;
      v4 = rotl32(v4 + le32(p + 12) * kX32P2, 13) * kX32P1;
    }
    h = rotl32(v1, 1) + rotl32(v2, 7) + rotl32(v3, 12) + rotl32(v4, 18);
  } else {
    h = seed + kX32P5;
  }
  h += uint32_t(n);
  for (; end - p >= 4; p += 4) h = rotl32(h + le32(p) * kX32P3, 17) * kX32P4;
  for (; p < end; p++) h = rotl32(h + *p * kX32P5, 11) * kX32P1;
  h ^= h >> 15;
  h *= kX32P2;
  h ^= h >> 13;
  h *= kX32P3;
  return h ^ (h >> 16);
}

constexpr uint64_t kX64P1 = 0x9E3779B185EBCA87ull, kX64P2 = 0xC2B2AE3D27D4EB4Full, kX64P3 = 0x165667B19E3779F9ull, kX64P4 = 0x85EBCA77C2B2AE63ull,
                   kX64P5 = 0x27D4EB2F165667C5ull;

FD_HD uint64_t xxh64_round(uint64_t acc, uint64_t in) { return rotl64(acc + in * kX64P2, 31) * kX64P1; }
FD_HD uint64_t xxh64_merge(uint64_t h, uint64_t v) { return (h ^ xxh64_round(0, v)) * kX64P1 + kX64P4; }

FD_HD uint64_t xxh64(const uint8_t* p, int64_t n, uint64_t seed) {
  const uint8_t* const end = p + n;
  uint64_t h;
  if (n >= 32) {
    uint64_t v1 = seed + kX64P1 + kX64P2, v2 = seed + kX64P2, v3 = seed, v4 = seed - kX64P1;
    for (; end - p >= 32; p += 32) {
      v1 = xxh64_round(v1, le64(p));
      v2 = xxh64_round(v2, le64(p + 8));
      v3 = xxh64_round(v3, le64(p + 16));
      v4 = xxh64_round(v4, le64(p + 24));
    }
    h = rotl64(v1, 1) + rotl64(v2, 7) + rotl64(v3, 12) + rotl64(v4, 18);
    h = xxh64_merge(xxh64_merge(xxh64_merge(xxh64_merge(h, v1), v2), v3), v4);
  } else {
    h = seed + kX64P5;
  }
  h += uint64_t(n);
  for (; end - p >= 8; p += 8) h = rotl64(h ^ xxh64_round(0, le64(p)), 27) * kX64P1 + kX64P4;
  if (end - p >= 4) {
    h = rotl64(h ^ (uint64_t(le32(p)) * kX64P1), 23) * kX64P2 + kX64P3;
    p += 4;
  }
  for (; p < end; p++) h = rotl64(h ^ (*p * kX64P5), 11) * kX64P1;
  h ^= h >> 33;
  h *= kX64P2;
  h ^= h >> 29;
  h *= kX64P3;
  return h ^ (h >> 32);
}

// CRC-32 with the zlib polynomial (reflected 0xEDB88320), byte-wise from a 256-entry table of crc32_table_entry(i).
constexpr uint32_t kCrcPoly = 0xEDB88320u;

FD_HD uint32_t crc32_table_entry(uint32_t i) {
  uint32_t c = i;
  for (int k = 0; k < 8; k++) c = (c & 1) ? (c >> 1) ^ kCrcPoly : c >> 1;
  return c;
}

// crc: a finished CRC-32 of the bytes before p (0 for none); returns that of the bytes through p + n
FD_HD uint32_t crc32_update(const uint32_t* t, uint32_t crc, const uint8_t* p, int64_t n) {
  crc = ~crc;
  for (int64_t i = 0; i < n; i++) crc = t[(crc ^ p[i]) & 0xff] ^ (crc >> 8);
  return ~crc;
}

// a(x) b(x) mod P(x), both reflected (zlib's multmodp)
FD_HD uint32_t crc32_mulmod(uint32_t a, uint32_t b) {
  uint32_t p = 0;
  for (uint32_t m = 1u << 31; m; m >>= 1) {
    if (a & m) p ^= b;
    b = (b & 1) ? (b >> 1) ^ kCrcPoly : b >> 1;
  }
  return p;
}

// CRC-32 of A followed by B from crc(A), crc(B) and |B| (zlib's crc32_combine): crc(A) x^(8|B|) + crc(B)
FD_HD uint32_t crc32_combine(uint32_t crc_a, uint32_t crc_b, int64_t len_b) {
  uint32_t x = 1u << 31, sq = 1u << 23;  // x^0, x^8
  for (uint64_t n = uint64_t(len_b); n; n >>= 1) {
    if (n & 1) x = crc32_mulmod(sq, x);
    sq = crc32_mulmod(sq, sq);
  }
  return crc32_mulmod(x, crc_a) ^ crc_b;
}

// ---- bit readers ---------------------------------------------------------------------------------------------------

FD_HD int highbit32(uint32_t v) {  // v > 0
#ifdef __CUDA_ARCH__
  return 31 - __clz(v);
#else
  return 31 - __builtin_clz(v);
#endif
}

// up to 8 little-endian bytes of p[i..] that lie below n; zeros beyond
FD_HD uint64_t load_le_bounded(const uint8_t* p, int64_t n, int64_t i) {
  if (i + 8 <= n) return le64(p + i);
  uint64_t v = 0;
  for (int k = 0; k < 8 && i + k < n; k++) v |= uint64_t(p[i + k]) << (8 * k);
  return v;
}

// A zstd backward bitstream: read from the last byte's highest set bit (the end mark) down to bit 0.  Bits below
// bit 0 read as zeros; `bits` then goes negative, which the callers treat as corrupt at the end of the stream.
struct BackBits {
  const uint8_t* p;
  int64_t n;
  int64_t bits;  // bits not yet read, above bit 0

  FD_HD bool init(const uint8_t* p_, int64_t n_) {
    p = p_, n = n_;
    if (n < 1 || p[n - 1] == 0) return false;
    bits = (n - 1) * 8 + highbit32(p[n - 1]);
    return true;
  }
  FD_HD uint32_t peek(int k) const {  // k <= 32
    if (k == 0) return 0;
    const uint64_t mask = (uint64_t(1) << k) - 1;
    const int64_t lo = bits - k;
    if (lo >= 0) return uint32_t((load_le_bounded(p, n, lo >> 3) >> (lo & 7)) & mask);
    if (bits <= 0) return 0;
    return uint32_t(((load_le_bounded(p, n, 0) & ((uint64_t(1) << bits) - 1)) << (-lo)) & mask);
  }
  FD_HD uint32_t read(int k) {
    const uint32_t v = peek(k);
    bits -= k;
    return v;
  }
};

// ---- zstd ----------------------------------------------------------------------------------------------------------

struct FseEntry {
  uint16_t base;   // next state = base + the nbits read
  uint8_t symbol;
  uint8_t nbits;
};

constexpr int kLLMaxLog = 9, kMLMaxLog = 9, kOFMaxLog = 8, kHufMaxBits = 11, kBlockMax = 128 * 1024;

// Per-frame tables; the device keeps one per warp in shared memory (~10 KB).
struct ZstdTables {
  FseEntry ll[1 << kLLMaxLog], ml[1 << kMLMaxLog], of[1 << kOFMaxLog];
  uint16_t huf[1 << kHufMaxBits];  // (symbol << 8) | code length, indexed by the next huf_bits bits
  FseEntry wt[64];                 // the FSE table of FSE-compressed Huffman weights
  int16_t norm[64];
  uint16_t next[64];
  uint8_t weights[256];
  int8_t ll_log, ml_log, of_log;   // -1: no table yet in this frame (Repeat mode is corrupt)
  int8_t huf_bits;                 // 0: no Huffman table yet (Treeless literals are corrupt)
};

FD_TABLE(uint32_t, kLLBase, {0,  1,  2,  3,  4,  5,  6,  7,   8,   9,   10,  11,   12,   13,   14,   15,   16,    18,
                                  20, 22, 24, 28, 32, 40, 48, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536})
FD_TABLE(uint8_t, kLLBits, {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16})
FD_TABLE(uint32_t, kMLBase, {3,  4,  5,  6,  7,  8,  9,  10, 11, 12, 13, 14, 15, 16,  17,  18,  19,   20,   21,   22,   23,    24,    25,    26,    27,    28, 29,
                                  30, 31, 32, 33, 34, 35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195, 16387, 32771, 65539})
FD_TABLE(uint8_t, kMLBits, {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0,
                                 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16})
FD_TABLE(int16_t, kLLDefault, {4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1})
FD_TABLE(int16_t, kMLDefault, {1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1,
                                    1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1, -1, -1})
FD_TABLE(int16_t, kOFDefault, {1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1})

// FSE table from normalized counts norm[0..n_sym) of accuracy log `log` (RFC 8878 4.1.1); false when the counts do
// not spread over the table.  `next` is scratch of n_sym entries.
FD_HD bool fse_build(FseEntry* table, const int16_t* norm, int n_sym, int log, uint16_t* next) {
  const int size = 1 << log;
  int high = size - 1;
  for (int s = 0; s < n_sym; s++) {
    if (norm[s] == -1) {
      table[high--].symbol = uint8_t(s);
      next[s] = 1;
    } else {
      next[s] = uint16_t(norm[s]);
    }
  }
  const int step = (size >> 1) + (size >> 3) + 3, mask = size - 1;
  int pos = 0;
  for (int s = 0; s < n_sym; s++)
    for (int i = 0; i < norm[s]; i++) {
      table[pos].symbol = uint8_t(s);
      do pos = (pos + step) & mask;
      while (pos > high);
    }
  if (pos != 0) return false;
  for (int u = 0; u < size; u++) {
    const uint32_t x = next[table[u].symbol]++;
    const int nb = log - highbit32(x);
    table[u].nbits = uint8_t(nb);
    table[u].base = uint16_t((x << nb) - size);
  }
  return true;
}

// An FSE table description (the normalized counts, RFC 8878 4.1.1) at src[0, n): builds the table and returns the
// bytes it took, or -1 when it is corrupt.  At most max_sym + 1 symbols and an accuracy log of at most max_log.
FD_HD int64_t fse_read_table(const uint8_t* src, int64_t n, int max_sym, int max_log, FseEntry* table, int* log_out, ZstdTables& t) {
  int64_t bit = 0;
  auto peek = [&](int k) { return uint32_t((load_le_bounded(src, n, bit >> 3) >> (bit & 7)) & ((uint64_t(1) << k) - 1)); };
  const int log = int(peek(4)) + 5;
  bit += 4;
  if (log > max_log) return -1;
  int remaining = (1 << log) + 1, threshold = 1 << log, nbits = log + 1, sym = 0;
  bool prev0 = false;
  while (remaining > 1 && sym <= max_sym) {
    if (prev0) {
      int zeros = 0;
      uint32_t r;
      while ((r = peek(2)) == 3) {
        zeros += 3;
        bit += 2;
        if (bit > 8 * n) return -1;
      }
      zeros += int(r);
      bit += 2;
      if (sym + zeros > max_sym + 1) return -1;
      while (zeros--) t.norm[sym++] = 0;
      if (sym > max_sym) break;
    }
    const int max = 2 * threshold - 1 - remaining;
    int count;
    const uint32_t v = peek(nbits);
    if (int(v & uint32_t(threshold - 1)) < max) {
      count = int(v & uint32_t(threshold - 1));
      bit += nbits - 1;
    } else {
      count = int(v & uint32_t(2 * threshold - 1));
      if (count >= threshold) count -= max;
      bit += nbits;
    }
    count--;
    remaining -= count < 0 ? -count : count;
    t.norm[sym++] = int16_t(count);
    prev0 = count == 0;
    while (remaining < threshold) {
      nbits--;
      threshold >>= 1;
    }
    if (bit > 8 * n) return -1;
  }
  if (remaining != 1 || bit > 8 * n) return -1;
  if (!fse_build(table, t.norm, sym, log, t.next)) return -1;
  *log_out = log;
  return (bit + 7) >> 3;
}

FD_HD void fse_rle(FseEntry* table, int* log_out, uint8_t sym) {
  table[0].symbol = sym, table[0].nbits = 0, table[0].base = 0;
  *log_out = 0;
}

// The Huffman tree description at src[0, n) (RFC 8878 4.2.1): builds t.huf; returns the bytes it took or -1.
FD_HD int64_t huf_read_table(const uint8_t* src, int64_t n, ZstdTables& t) {
  if (n < 1) return -1;
  const int h = src[0];
  int count = 0;
  int64_t used;
  if (h >= 128) {  // h - 127 weights of 4 bits, two per byte, the first in the high nibble
    count = h - 127;
    used = 1 + (count + 1) / 2;
    if (used > n) return -1;
    for (int i = 0; i < count; i++) t.weights[i] = (src[1 + i / 2] >> ((i & 1) ? 0 : 4)) & 15;
  } else {  // FSE-compressed weights in h bytes: two interleaved states over one backward stream
    used = 1 + h;
    if (used > n) return -1;
    int log = 0;
    const int64_t th = fse_read_table(src + 1, h, kHufMaxBits, 6, t.wt, &log, t);
    if (th < 0 || th >= h) return -1;
    BackBits br;
    if (!br.init(src + 1 + th, h - th)) return -1;
    uint32_t s1 = br.read(log), s2 = br.read(log);
    if (br.bits < 0) return -1;
    for (;;) {
      if (count >= 255) return -1;
      t.weights[count++] = t.wt[s1].symbol;
      s1 = t.wt[s1].base + br.read(t.wt[s1].nbits);
      if (br.bits < 0) {
        if (count >= 255) return -1;
        t.weights[count++] = t.wt[s2].symbol;
        break;
      }
      if (count >= 255) return -1;
      t.weights[count++] = t.wt[s2].symbol;
      s2 = t.wt[s2].base + br.read(t.wt[s2].nbits);
      if (br.bits < 0) {
        if (count >= 255) return -1;
        t.weights[count++] = t.wt[s1].symbol;
        break;
      }
    }
  }
  // the last symbol's weight is implied: it completes the sum of 2^(w-1) to a power of two
  uint32_t total = 0;
  for (int i = 0; i < count; i++) {
    if (t.weights[i] > kHufMaxBits) return -1;
    if (t.weights[i]) total += 1u << (t.weights[i] - 1);
  }
  if (total == 0) return -1;
  const int max_bits = highbit32(total) + 1;
  if (max_bits > kHufMaxBits) return -1;
  const uint32_t left = (1u << max_bits) - total;
  if (left & (left - 1)) return -1;
  t.weights[count++] = uint8_t(highbit32(left) + 1);
  // codes by rising weight (longest codes first), each weight's symbols in symbol order
  uint32_t start[kHufMaxBits + 2] = {0};
  for (int i = 0; i < count; i++)
    if (t.weights[i]) start[t.weights[i]] += 1u << (t.weights[i] - 1);
  uint32_t pos = 0;
  for (int w = 1; w <= max_bits; w++) {
    const uint32_t c = start[w];
    start[w] = pos;
    pos += c;
  }
  for (int s = 0; s < count; s++) {
    const int w = t.weights[s];
    if (!w) continue;
    const uint16_t e = uint16_t((s << 8) | (max_bits + 1 - w));
    for (uint32_t k = 0; k < (1u << (w - 1)); k++) t.huf[start[w] + k] = e;
    start[w] += 1u << (w - 1);
  }
  t.huf_bits = int8_t(max_bits);
  return used;
}

// one Huffman stream src[0, n) into out[0, m); the stream must be consumed exactly
FD_HD bool huf_stream(const uint8_t* src, int64_t n, uint8_t* out, int64_t m, const ZstdTables& t) {
  BackBits br;
  if (!br.init(src, n)) return false;
  const int b = t.huf_bits;
  for (int64_t i = 0; i < m; i++) {
    const uint16_t e = t.huf[br.peek(b)];
    out[i] = uint8_t(e >> 8);
    br.bits -= e & 0xff;
  }
  return br.bits == 0;
}

FD_HD void copy_bytes(uint8_t* d, const uint8_t* s, int64_t n) {  // forward, byte by byte: overlapping matches repeat
  for (int64_t i = 0; i < n; i++) d[i] = s[i];
}

// Output state of one container frame.
struct Out {
  uint8_t* dst;
  int64_t cap;
  int64_t pos;    // bytes written
  int64_t floor;  // a back-reference may not reach below this (start of the zstd frame / LZ4 frame or block)
};

// One compressed block src[0, n) (RFC 8878 3.1.1.3).
FD_HD int zstd_block(const uint8_t* src, int64_t n, Out& o, ZstdTables& t, uint32_t rep[3]) {
  if (n < 1) return kCorrupt;
  // -- literals section
  const int ltype = src[0] & 3, sf = (src[0] >> 2) & 3;
  int64_t hsz, regen, csize = 0;
  int streams = 1;
  if (ltype < 2) {
    if (sf == 0 || sf == 2) hsz = 1, regen = src[0] >> 3;
    else if (sf == 1) hsz = 2, regen = n >= 2 ? (src[0] >> 4) + (int64_t(src[1]) << 4) : 0;
    else hsz = 3, regen = n >= 3 ? (src[0] >> 4) + (int64_t(src[1]) << 4) + (int64_t(src[2]) << 12) : 0;
  } else {
    hsz = sf < 2 ? 3 : sf == 2 ? 4 : 5;
    streams = sf == 0 ? 1 : 4;
    if (n < hsz) return kCorrupt;
    const uint32_t v = sf < 2 ? (src[0] | (src[1] << 8) | (uint32_t(src[2]) << 16)) : le32(src);
    if (sf < 2) regen = (v >> 4) & 0x3FF, csize = (v >> 14) & 0x3FF;
    else if (sf == 2) regen = (v >> 4) & 0x3FFF, csize = v >> 18;
    else regen = (v >> 4) & 0x3FFFF, csize = (v >> 22) | (int64_t(src[4]) << 10);
  }
  if (n < hsz || regen > kBlockMax) return kCorrupt;
  int64_t p = hsz;
  const uint8_t* lit;
  int64_t lit_pos = -1;  // offset of the literals in dst when they are decoded there, else -1
  if (ltype == 0) {
    if (p + regen > n) return kCorrupt;
    lit = src + p;
    p += regen;
  } else {
    if (regen > o.cap - o.pos) return kSize;
    lit_pos = o.cap - regen;
    uint8_t* lo = o.dst + lit_pos;
    if (ltype == 1) {
      if (p + 1 > n) return kCorrupt;
      for (int64_t i = 0; i < regen; i++) lo[i] = src[p];
      p += 1;
    } else {
      if (p + csize > n) return kCorrupt;
      const uint8_t* ls = src + p;
      int64_t lsz = csize;
      if (ltype == 2) {
        const int64_t th = huf_read_table(ls, lsz, t);
        if (th < 0) return kCorrupt;
        ls += th, lsz -= th;
      } else if (t.huf_bits == 0) {
        return kCorrupt;
      }
      if (streams == 1) {
        if (!huf_stream(ls, lsz, lo, regen, t)) return kCorrupt;
      } else {
        if (lsz < 6) return kCorrupt;
        const int64_t s1 = ls[0] | (ls[1] << 8), s2 = ls[2] | (ls[3] << 8), s3 = ls[4] | (ls[5] << 8);
        const int64_t s4 = lsz - 6 - s1 - s2 - s3, q = (regen + 3) / 4;
        if (s4 < 0 || regen < 3 * q) return kCorrupt;
        const uint8_t* b = ls + 6;
        if (!huf_stream(b, s1, lo, q, t) || !huf_stream(b + s1, s2, lo + q, q, t) || !huf_stream(b + s1 + s2, s3, lo + 2 * q, q, t) ||
            !huf_stream(b + s1 + s2 + s3, s4, lo + 3 * q, regen - 3 * q, t))
          return kCorrupt;
      }
      p += csize;
    }
    lit = o.dst + lit_pos;
  }
  // -- sequences section
  if (p >= n) return kCorrupt;
  int64_t nseq = src[p];
  if (nseq < 128) {
    p += 1;
  } else if (nseq < 255) {
    if (p + 2 > n) return kCorrupt;
    nseq = ((nseq - 128) << 8) + src[p + 1];
    p += 2;
  } else {
    if (p + 3 > n) return kCorrupt;
    nseq = src[p + 1] + (int64_t(src[p + 2]) << 8) + 0x7F00;
    p += 3;
  }
  const int64_t block_start = o.pos;
  int64_t lit_left = regen;
  if (nseq > 0) {
    if (p >= n) return kCorrupt;
    const int modes = src[p++];
    if (modes & 3) return kCorrupt;
    struct Spec {
      int mode;
      FseEntry* table;
      int8_t* log;
      int max_sym, max_log, def_log, n_def;
      const int16_t* def;
    };
    const Spec specs[3] = {{(modes >> 6) & 3, t.ll, &t.ll_log, 35, kLLMaxLog, 6, 36, FD_T(kLLDefault)},
                           {(modes >> 4) & 3, t.of, &t.of_log, 31, kOFMaxLog, 5, 29, FD_T(kOFDefault)},
                           {(modes >> 2) & 3, t.ml, &t.ml_log, 52, kMLMaxLog, 6, 53, FD_T(kMLDefault)}};
    for (int k = 0; k < 3; k++) {
      const Spec& s = specs[k];
      int log = 0;
      if (s.mode == 0) {
        for (int i = 0; i < s.n_def; i++) t.norm[i] = s.def[i];
        fse_build(s.table, t.norm, s.n_def, s.def_log, t.next);
        log = s.def_log;
      } else if (s.mode == 1) {
        if (p >= n || src[p] > s.max_sym) return kCorrupt;
        fse_rle(s.table, &log, src[p++]);
      } else if (s.mode == 2) {
        const int64_t used = fse_read_table(src + p, n - p, s.max_sym, s.max_log, s.table, &log, t);
        if (used < 0) return kCorrupt;
        p += used;
      } else {
        if (*s.log < 0) return kCorrupt;
        log = *s.log;
      }
      *s.log = int8_t(log);
    }
    BackBits br;
    if (!br.init(src + p, n - p)) return kCorrupt;
    uint32_t sll = br.read(t.ll_log), sof = br.read(t.of_log), sml = br.read(t.ml_log);
    for (int64_t i = 0; i < nseq; i++) {
      const FseEntry el = t.ll[sll], eo = t.of[sof], em = t.ml[sml];
      if (eo.symbol > 31 || el.symbol > 35 || em.symbol > 52) return kCorrupt;
      uint32_t ofv = (1u << eo.symbol) + br.read(eo.symbol);
      const int64_t ml = FD_T(kMLBase)[em.symbol] + br.read(FD_T(kMLBits)[em.symbol]);
      const int64_t ll = FD_T(kLLBase)[el.symbol] + br.read(FD_T(kLLBits)[el.symbol]);
      uint32_t off;
      if (ofv > 3) {
        off = ofv - 3;
        rep[2] = rep[1], rep[1] = rep[0], rep[0] = off;
      } else {
        if (ll == 0) ofv++;
        if (ofv == 1) {
          off = rep[0];
        } else {
          off = ofv == 2 ? rep[1] : ofv == 3 ? rep[2] : rep[0] - 1;
          if (ofv != 2) rep[2] = rep[1];
          rep[1] = rep[0], rep[0] = off;
        }
      }
      if (i + 1 < nseq) {
        sll = el.base + br.read(el.nbits);
        sml = em.base + br.read(em.nbits);
        sof = eo.base + br.read(eo.nbits);
      }
      if (br.bits < 0) return kCorrupt;
      // execute: ll literals, then ml bytes from `off` back
      if (ll > lit_left) return kCorrupt;
      if (o.pos + ll > o.cap) return kSize;
      copy_bytes(o.dst + o.pos, lit, ll);
      lit += ll, lit_left -= ll, o.pos += ll;
      if (lit_pos >= 0) lit_pos += ll;
      if (off == 0 || off > o.pos - o.floor) return kCorrupt;
      if (o.pos + ml > (lit_pos >= 0 ? lit_pos : o.cap)) return kSize;
      copy_bytes(o.dst + o.pos, o.dst + o.pos - off, ml);
      o.pos += ml;
    }
    if (br.bits != 0) return kCorrupt;
  } else if (p != n) {
    return kCorrupt;
  }
  if (o.pos + lit_left > o.cap) return kSize;
  copy_bytes(o.dst + o.pos, lit, lit_left);
  o.pos += lit_left;
  return o.pos - block_start > kBlockMax ? kCorrupt : kOk;
}

constexpr uint32_t kZstdMagic = 0xFD2FB528u, kLz4Magic = 0x184D2204u, kLz4LegacyMagic = 0x184C2102u;

FD_HD bool skippable_magic(uint32_t m) { return (m & 0xFFFFFFF0u) == 0x184D2A50u; }

// One zstd frame at src[0, n) (its magic included) -> o; *used: the bytes it took.
FD_HD int zstd_frame(const uint8_t* src, int64_t n, Out& o, ZstdTables& t, int64_t* used) {
  if (n < 6) return kCorrupt;
  const int fhd = src[4];
  const int fcs_flag = fhd >> 6, single = (fhd >> 5) & 1, checksum = (fhd >> 2) & 1, did_flag = fhd & 3;
  if (fhd & 8) return kCorrupt;  // reserved bit
  int64_t p = 5;
  if (!single) {
    const int wd = src[p++];
    if ((wd >> 3) + 10 > 31) return kUnsupported;  // a window above 2 GiB
  }
  const int did_bytes = did_flag == 3 ? 4 : did_flag;
  if (p + did_bytes > n) return kCorrupt;
  uint32_t did = 0;
  for (int i = 0; i < did_bytes; i++) did |= uint32_t(src[p + i]) << (8 * i);
  p += did_bytes;
  if (did != 0) return kUnsupported;
  const int fcs_bytes = fcs_flag == 0 ? single : fcs_flag == 1 ? 2 : fcs_flag == 2 ? 4 : 8;
  if (p + fcs_bytes > n) return kCorrupt;
  uint64_t fcs = 0;
  for (int i = 0; i < fcs_bytes; i++) fcs |= uint64_t(src[p + i]) << (8 * i);
  if (fcs_bytes == 2) fcs += 256;
  p += fcs_bytes;
  o.floor = o.pos;
  t.ll_log = t.ml_log = t.of_log = -1;
  t.huf_bits = 0;
  uint32_t rep[3] = {1, 4, 8};
  for (;;) {
    if (p + 3 > n) return kCorrupt;
    const uint32_t bh = src[p] | (src[p + 1] << 8) | (uint32_t(src[p + 2]) << 16);
    p += 3;
    const int last = bh & 1, type = (bh >> 1) & 3;
    const int64_t size = bh >> 3;
    if (type == 3 || size > kBlockMax) return kCorrupt;
    if (type == 1) {  // RLE: one byte, repeated size times
      if (p + 1 > n) return kCorrupt;
      if (size > o.cap - o.pos) return kSize;
      for (int64_t i = 0; i < size; i++) o.dst[o.pos + i] = src[p];
      o.pos += size;
      p += 1;
    } else {
      if (p + size > n) return kCorrupt;
      if (type == 0) {
        if (size > o.cap - o.pos) return kSize;
        copy_bytes(o.dst + o.pos, src + p, size);
        o.pos += size;
      } else {
        const int rc = zstd_block(src + p, size, o, t, rep);
        if (rc != kOk) return rc;
      }
      p += size;
    }
    if (last) break;
  }
  const int64_t produced = o.pos - o.floor;
  if ((fcs_bytes && uint64_t(produced) != fcs)) return kCorrupt;
  if (checksum) {
    if (p + 4 > n) return kCorrupt;
    if (uint32_t(xxh64(o.dst + o.floor, produced, 0)) != le32(src + p)) return kChecksum;
    p += 4;
  }
  *used = p;
  return kOk;
}

// ---- LZ4 -----------------------------------------------------------------------------------------------------------

// One LZ4 block src[0, n) -> o (the LZ4 block format: tokens, literals, 16-bit offsets).
FD_HD int lz4_block(const uint8_t* src, int64_t n, Out& o) {
  int64_t p = 0;
  for (;;) {
    if (p >= n) return kCorrupt;
    const int token = src[p++];
    int64_t ll = token >> 4;
    if (ll == 15) {
      int b;
      do {
        if (p >= n) return kCorrupt;
        b = src[p++];
        ll += b;
      } while (b == 255);
    }
    if (ll > n - p) return kCorrupt;
    if (ll > o.cap - o.pos) return kSize;
    copy_bytes(o.dst + o.pos, src + p, ll);
    o.pos += ll, p += ll;
    if (p == n) return kOk;  // the last sequence has literals only
    if (p + 2 > n) return kCorrupt;
    const int64_t off = src[p] | (src[p + 1] << 8);
    p += 2;
    int64_t ml = (token & 15) + 4;
    if ((token & 15) == 15) {
      int b;
      do {
        if (p >= n) return kCorrupt;
        b = src[p++];
        ml += b;
      } while (b == 255);
    }
    if (off == 0 || off > o.pos - o.floor) return kCorrupt;
    if (ml > o.cap - o.pos) return kSize;
    copy_bytes(o.dst + o.pos, o.dst + o.pos - off, ml);
    o.pos += ml;
  }
}

// One LZ4 frame at src[0, n) (its magic included) -> o; *used: the bytes it took.
FD_HD int lz4_frame(const uint8_t* src, int64_t n, Out& o, int64_t* used) {
  if (n < 7) return kCorrupt;
  const int flg = src[4], bd = src[5];
  if ((flg >> 6) != 1 || (flg & 2) || (bd & 0x8F)) return kCorrupt;
  const int indep = (flg >> 5) & 1, bsum = (flg >> 4) & 1, csize = (flg >> 3) & 1, csum = (flg >> 2) & 1, dict = flg & 1;
  const int bmax_code = (bd >> 4) & 7;
  if (bmax_code < 4) return kCorrupt;
  const int64_t bmax = int64_t(1) << (8 + 2 * bmax_code);
  const int64_t hlen = 2 + (csize ? 8 : 0) + (dict ? 4 : 0);
  if (4 + hlen + 1 > n) return kCorrupt;
  if ((xxh32(src + 4, hlen, 0) >> 8 & 0xff) != src[4 + hlen]) return kChecksum;
  if (dict) return kUnsupported;
  const uint64_t content = csize ? le64(src + 6) : 0;
  int64_t p = 4 + hlen + 1;
  const int64_t start = o.pos;
  o.floor = start;
  for (;;) {
    if (p + 4 > n) return kCorrupt;
    const uint32_t bs = le32(src + p);
    p += 4;
    if (bs == 0) break;
    const int64_t size = bs & 0x7FFFFFFFu;
    if (size > bmax || p + size + (bsum ? 4 : 0) > n) return kCorrupt;
    if (bsum && xxh32(src + p, size, 0) != le32(src + p + size)) return kChecksum;
    if (bs >> 31) {
      if (size > o.cap - o.pos) return kSize;
      copy_bytes(o.dst + o.pos, src + p, size);
      o.pos += size;
    } else {
      if (indep) o.floor = o.pos;
      const int64_t before = o.pos;
      const int rc = lz4_block(src + p, size, o);
      if (rc != kOk) return rc;
      if (o.pos - before > bmax) return kCorrupt;
    }
    p += size + (bsum ? 4 : 0);
  }
  if (csize && uint64_t(o.pos - start) != content) return kCorrupt;
  if (csum) {
    if (p + 4 > n) return kCorrupt;
    if (xxh32(o.dst + start, o.pos - start, 0) != le32(src + p)) return kChecksum;
    p += 4;
  }
  *used = p;
  return kOk;
}

// ---- a container frame ---------------------------------------------------------------------------------------------

// Decodes src[0, n) -- one or more frames of `codec`, skippable frames anywhere -- into dst[0, cap).  *produced: the
// bytes written (produced may be null).  Returns a Status; kSize when the frames hold more or fewer than cap bytes.
// Empty input is corrupt.
FD_HD int decode_frame(const uint8_t* src, int64_t n, uint8_t* dst, int64_t cap, int codec, ZstdTables& t, int64_t* produced) {
  Out o{dst, cap, 0, 0};
  if (produced) *produced = 0;
  if (codec != kZstd && codec != kLz4Frame) return kUnsupported;
  if (n <= 0) return kCorrupt;
  int64_t p = 0;
  while (p < n) {
    if (n - p < 4) return kCorrupt;
    const uint32_t magic = le32(src + p);
    int64_t used = 0;
    int rc;
    if (skippable_magic(magic)) {
      if (n - p < 8) return kCorrupt;
      const int64_t len = le32(src + p + 4);
      if (len > n - p - 8) return kCorrupt;
      used = 8 + len;
      rc = kOk;
    } else if (codec == kZstd && magic == kZstdMagic) {
      rc = zstd_frame(src + p, n - p, o, t, &used);
    } else if (codec == kLz4Frame && magic == kLz4Magic) {
      rc = lz4_frame(src + p, n - p, o, &used);
    } else if (codec == kLz4Frame && magic == kLz4LegacyMagic) {
      rc = kUnsupported;
    } else {
      rc = kCorrupt;
    }
    if (produced) *produced = o.pos;
    if (rc != kOk) return rc;
    p += used;
  }
  return o.pos == cap ? kOk : kSize;
}

}  // namespace fd
}  // namespace vlcal
