// frame_decode.cu -- a batch of independent zstd / LZ4-frame container frames decoded on the GPU (DESIGN §4f).
//
// One warp per frame.  Frames are claimed largest first through an atomic counter, so the long frames start early and
// the short ones fill in behind them.  Lane 0 runs the format core of frame_decode.cuh (headers, the FSE and Huffman
// tables in the warp's slice of shared memory, literals, sequences, the XXH32 / XXH64 checksums the formats carry);
// then, for frames with a CRC-32 to check (MCAP chunks), the warp hashes 32 slices of the output in parallel and
// joins them with crc32_combine in a shuffle tree.
#include <algorithm>
#include <cstdint>
#include <numeric>
#include <string>
#include <vector>

#include "frame_decode.cuh"
#include "preprocess_common.cuh"

namespace vlcal {
namespace {

constexpr int kWarpsPerBlock = 4;  // 4 x ~10 KB of tables per block; 4 blocks per SM keep the core at 121 registers, unspilled

struct FrameDecodeArgs {
  const uint8_t* src;
  const vlcal_frame* frames;
  const int* order;  // frame indices, largest first
  int n_frames;
  uint8_t* dst;
  int32_t* status;
  int* next;         // the claim counter
};

__global__ void __launch_bounds__(kWarpsPerBlock * 32, 4) frame_decode_kernel(const __grid_constant__ FrameDecodeArgs a) {
  __shared__ fd::ZstdTables tables[kWarpsPerBlock];
  __shared__ uint32_t crc_table[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) crc_table[i] = fd::crc32_table_entry(i);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (;;) {
    int k = 0;
    if (lane == 0) k = atomicAdd(a.next, 1);
    k = __shfl_sync(0xffffffffu, k, 0);
    if (k >= a.n_frames) return;
    const int idx = a.order[k];
    const vlcal_frame f = a.frames[idx];
    uint8_t* const out = a.dst + f.dst_offset;
    int st = 0;
    if (lane == 0) st = fd::decode_frame(a.src + f.src_offset, f.src_size, out, f.dst_size, f.codec, tables[warp], nullptr);
    __syncwarp();  // lane 0's output writes are visible to the warp's CRC reads below
    st = __shfl_sync(0xffffffffu, st, 0);
    if (st == fd::kOk && f.has_crc32) {
      const int64_t slice = (f.dst_size + 31) / 32;
      const int64_t lo = min(lane * slice, f.dst_size);
      int64_t len = min(lo + slice, f.dst_size) - lo;
      uint32_t crc = fd::crc32_update(crc_table, 0, out + lo, len);
      for (int d = 1; d < 32; d <<= 1) {
        const uint32_t crc_b = __shfl_down_sync(0xffffffffu, crc, d);
        const int64_t len_b = __shfl_down_sync(0xffffffffu, len, d);
        if ((lane & (2 * d - 1)) == 0) {
          crc = fd::crc32_combine(crc, crc_b, len_b);
          len += len_b;
        }
      }
      if (crc != f.crc32) st = fd::kChecksum;
    }
    if (lane == 0) a.status[idx] = st;
  }
}

bool in_range(int64_t off, int64_t size, int64_t bytes) { return off >= 0 && size >= 0 && off <= bytes && size <= bytes - off; }

}  // namespace
}  // namespace vlcal

using namespace vlcal;

extern "C" int vlcal_decode_frames(int device, const uint8_t* src, int64_t src_bytes, const vlcal_frame* frames, int n_frames, uint8_t* dst, int64_t dst_bytes,
                                   int32_t* status_out, double* ms_out) {
  if (n_frames < 0 || src_bytes < 0 || dst_bytes < 0 || (n_frames > 0 && (!frames || !status_out)) || (src_bytes > 0 && !src) || (dst_bytes > 0 && !dst)) {
    set_last_error("decode_frames: invalid arguments (n_frames >= 0, buffer sizes >= 0, non-null buffers)");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  if (ms_out)
    for (int k = 0; k < 3; k++) ms_out[k] = 0.0;
  for (int i = 0; i < n_frames; i++) {
    const vlcal_frame& f = frames[i];
    if (f.codec != VLCAL_CODEC_ZSTD && f.codec != VLCAL_CODEC_LZ4_FRAME) {
      set_last_error("decode_frames: frame " + std::to_string(i) + ": unknown codec " + std::to_string(f.codec));
      return VLCAL_ERR_INVALID_ARGUMENT;
    }
    if (f.has_crc32 != 0 && f.has_crc32 != 1) {
      set_last_error("decode_frames: frame " + std::to_string(i) + ": has_crc32 must be 0 or 1");
      return VLCAL_ERR_INVALID_ARGUMENT;
    }
    if (!in_range(f.src_offset, f.src_size, src_bytes) || !in_range(f.dst_offset, f.dst_size, dst_bytes)) {
      set_last_error("decode_frames: frame " + std::to_string(i) + ": its src or dst range lies outside the buffer");
      return VLCAL_ERR_INVALID_ARGUMENT;
    }
  }
  // overlap: each non-empty range against the furthest end of all non-empty ranges that start at or before it
  std::vector<int> by_dst(n_frames);
  std::iota(by_dst.begin(), by_dst.end(), 0);
  std::sort(by_dst.begin(), by_dst.end(), [&](int x, int y) { return frames[x].dst_offset < frames[y].dst_offset; });
  int64_t reach = -1;
  int reach_frame = -1;
  for (int i : by_dst) {
    const vlcal_frame& q = frames[i];
    if (q.dst_size == 0) continue;
    if (reach_frame >= 0 && q.dst_offset < reach) {
      set_last_error("decode_frames: the dst ranges of frames " + std::to_string(reach_frame) + " and " + std::to_string(i) + " overlap");
      return VLCAL_ERR_INVALID_ARGUMENT;
    }
    reach = q.dst_offset + q.dst_size, reach_frame = i;
  }
  if (n_frames == 0) return VLCAL_OK;
  int rc = prepare_device(&device);
  if (rc != VLCAL_OK) return rc;

  std::vector<int> order(n_frames);
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return frames[x].dst_size + frames[x].src_size > frames[y].dst_size + frames[y].src_size; });
  Scratch s(device);
  uint8_t *d_src, *d_dst;
  vlcal_frame* d_frames;
  int *d_order, *d_next;
  int32_t* d_status;
  VL_CUDA(s.alloc(static_cast<size_t>(src_bytes), &d_src));
  VL_CUDA(s.alloc(static_cast<size_t>(dst_bytes), &d_dst));
  VL_CUDA(s.alloc(n_frames, &d_frames));
  VL_CUDA(s.alloc(n_frames, &d_order));
  VL_CUDA(s.alloc(n_frames, &d_status));
  VL_CUDA(s.alloc(1, &d_next));
  StageTimer timer(ms_out != nullptr);
  VL_CUDA(timer.mark());
  if (src_bytes) VL_CUDA(cudaMemcpy(d_src, src, static_cast<size_t>(src_bytes), cudaMemcpyHostToDevice));
  VL_CUDA(cudaMemcpy(d_frames, frames, sizeof(vlcal_frame) * n_frames, cudaMemcpyHostToDevice));
  VL_CUDA(cudaMemcpy(d_order, order.data(), sizeof(int) * n_frames, cudaMemcpyHostToDevice));
  VL_CUDA(cudaMemset(d_next, 0, sizeof(int)));
  VL_CUDA(timer.mark());
  int sms = 0;
  VL_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  FrameDecodeArgs a{d_src, d_frames, d_order, n_frames, d_dst, d_status, d_next};
  const int blocks = static_cast<int>(std::min<int64_t>((n_frames + kWarpsPerBlock - 1) / kWarpsPerBlock, int64_t(sms) * 8));
  frame_decode_kernel<<<blocks, kWarpsPerBlock * 32>>>(a);
  VL_CUDA(cudaGetLastError());
  VL_CUDA(timer.mark());
  // the frames' dst ranges back, adjacent ranges in one copy; bytes of dst outside every range are left as they were
  for (int i = 0; i < n_frames;) {
    const int64_t lo = frames[by_dst[i]].dst_offset;
    int64_t hi = lo + frames[by_dst[i]].dst_size;
    int j = i + 1;
    for (; j < n_frames && frames[by_dst[j]].dst_offset == hi; j++) hi += frames[by_dst[j]].dst_size;
    if (hi > lo) VL_CUDA(cudaMemcpy(dst + lo, d_dst + lo, static_cast<size_t>(hi - lo), cudaMemcpyDeviceToHost));
    i = j;
  }
  VL_CUDA(cudaMemcpy(status_out, d_status, sizeof(int32_t) * n_frames, cudaMemcpyDeviceToHost));
  VL_CUDA(timer.mark());
  VL_CUDA(timer.read(ms_out, 3));
  return VLCAL_OK;
}
