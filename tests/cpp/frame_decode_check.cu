// Host build of the frame decoder core (csrc/frame_decode.cuh, the source the GPU kernel runs), for
// tests/test_codec_host.py.  Built host-only under -fsanitize=address,undefined.
//
//   frame_decode_check decode FILE   FILE: records (u32 codec, u64 src_size, u64 dst_size, src bytes); prints one line
//                                    per record: status, bytes produced, CRC-32 of the dst_size output bytes
//   frame_decode_check hash FILE     FILE: records (u64 size, bytes); prints XXH32, XXH64 (seed 0), the CRC-32 byte by
//                                    byte and the CRC-32 of seven slices joined by crc32_combine
#include <cstdio>
#include <cstring>
#include <vector>

#include "frame_decode.cuh"

using namespace vlcal;

static bool read_exact(FILE* f, void* p, size_t n) { return fread(p, 1, n, f) == n; }

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  FILE* f = fopen(argv[2], "rb");
  if (!f) return 2;
  static uint32_t table[256];
  for (uint32_t i = 0; i < 256; i++) table[i] = fd::crc32_table_entry(i);
  fd::ZstdTables* t = new fd::ZstdTables;
  const bool decode = strcmp(argv[1], "decode") == 0;
  for (;;) {
    uint32_t codec = 0;
    uint64_t n = 0, cap = 0;
    if (decode && !read_exact(f, &codec, 4)) break;
    if (!read_exact(f, &n, 8)) break;
    if (decode && !read_exact(f, &cap, 8)) return 2;
    // exact-size heap buffers: any read or write past them is an AddressSanitizer report
    std::vector<uint8_t> src(n);
    if (n && !read_exact(f, src.data(), n)) return 2;
    uint8_t* in = new uint8_t[n ? n : 1];
    if (n) memcpy(in, src.data(), n);
    if (decode) {
      uint8_t* out = new uint8_t[cap ? cap : 1];
      memset(out, 0, cap);
      int64_t produced = 0;
      const int st = fd::decode_frame(in, int64_t(n), out, int64_t(cap), int(codec), *t, &produced);
      printf("%d %lld %u\n", st, (long long)produced, fd::crc32_update(table, 0, out, int64_t(cap)));
      delete[] out;
    } else {
      uint32_t joined = 0;
      const int64_t slice = int64_t(n) / 7 + 1;
      for (int64_t lo = 0; lo < int64_t(n); lo += slice) {
        const int64_t len = lo + slice < int64_t(n) ? slice : int64_t(n) - lo;
        joined = fd::crc32_combine(joined, fd::crc32_update(table, 0, in + lo, len), len);
      }
      printf("%u %llu %u %u\n", fd::xxh32(in, int64_t(n), 0), (unsigned long long)fd::xxh64(in, int64_t(n), 0), fd::crc32_update(table, 0, in, int64_t(n)), joined);
    }
    delete[] in;
  }
  delete t;
  return 0;
}
