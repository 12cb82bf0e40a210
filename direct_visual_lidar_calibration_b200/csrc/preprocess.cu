// preprocess.cu -- the GPU stages of preprocess_map (reference: src/preprocess_map.cpp:34-214, src/vlcal/common/estimate_fov.cpp:53-91).
//
// Four pieces of the map preprocessing, each giving the reference's bits (DESIGN §4 "preprocess_map"):
//   1. pcl::ApproximateVoxelGrid<PointXYZI> (leaf float(voxel_resolution), 512 history slots, all fields averaged).  The
//      reference runs it sequentially over the points in file order; each of the 512 slots is an independent sequential
//      stream, so a stable sort by slot splits it into runs (a maximal stretch of one slot's points with one voxel key),
//      each run is summed by one thread in original order (the float bits of the sequential sums), and the runs are
//      emitted in the order the sequential loop flushes them: run r is flushed when the first point of the next run of
//      its slot arrives (time = that point's index), the last run of slot s at the end (time = N + s).  All times differ,
//      so a scatter by time and a compaction give the output order.
//   2. the rank equalisation (preprocess_map.cpp:158-167): stable radix sort of order-preserving keys of the float
//      intensities (-0.0 folded into +0.0, which the comparator treats as equal), ties by point index.
//   3. estimate_lidar_fov's pcl::VoxelGrid<PointXYZ> (0.2 m, with PCL's INT32_MAX fallback to the unfiltered input) and
//      the `norm() < 1.0` removal; voxel sums in point-index order.
//   4. the smallest pairwise cosine of the hull vertices' bearings (never-contracted double, Eigen's term order).
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <cfloat>
#include <climits>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "preprocess_common.cuh"

namespace vlcal {
namespace {

constexpr int kHistSize = 512;                     // ApproximateVoxelGrid::histsize_
constexpr long long kMaxPoints = 0x7fffffffLL - kHistSize;  // flush times N + slot must fit int32

// ------------------------------------------------------------------------------------------------------------------
// 1. ApproximateVoxelGrid
// ------------------------------------------------------------------------------------------------------------------

struct AvgArgs {
  const float4* points;  // (x, y, z, intensity)
  int n;
  float inv;              // 1.0f / float(leaf)
  int4* keys;             // (ix, iy, iz, -)
  unsigned int* slot;     // [n]
  int* index;             // [n] = i
  unsigned int* flags;    // [0]: non-finite seen, [1]: points with an axis index out of int range
};

__global__ void __launch_bounds__(256) avg_keys_kernel(const __grid_constant__ AvgArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  const float4 p = __ldg(a.points + i);
  if (!(finite_f(p.x) && finite_f(p.y) && finite_f(p.z) && finite_f(p.w))) atomicOr(a.flags, 1u);
  const float fx = floorf(__fmul_rn(p.x, a.inv)), fy = floorf(__fmul_rn(p.y, a.inv)), fz = floorf(__fmul_rn(p.z, a.inv));
  const int ix = float_to_int_x86(fx), iy = float_to_int_x86(fy), iz = float_to_int_x86(fz);
  if ((ix == INT_MIN && fx != -2147483648.0f) || (iy == INT_MIN && fy != -2147483648.0f) || (iz == INT_MIN && fz != -2147483648.0f)) atomicAdd(a.flags + 1, 1u);
  // (ix * 7171 + iy * 3079 + iz * 4231) & (histsize_ - 1): the reference's int arithmetic wraps; the low 9 bits are these
  const unsigned int h = static_cast<unsigned int>(ix) * 7171u + static_cast<unsigned int>(iy) * 3079u + static_cast<unsigned int>(iz) * 4231u;
  a.keys[i] = make_int4(ix, iy, iz, 0);
  a.slot[i] = h & (kHistSize - 1);
  a.index[i] = i;
}

// a run starts where the slot or the voxel key changes (positions in slot-sorted order)
__global__ void __launch_bounds__(256) avg_heads_kernel(const unsigned int* slot_sorted, const int* idx_sorted, const int4* keys, int n, unsigned char* head) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  bool h = p == 0;
  if (!h) {
    const int4 k = keys[idx_sorted[p]], q = keys[idx_sorted[p - 1]];
    h = slot_sorted[p] != slot_sorted[p - 1] || k.x != q.x || k.y != q.y || k.z != q.z;
  }
  head[p] = h ? 1 : 0;
}

// One thread per run: centroid += scratch in arrival order from zero, then centroid / float(count) (the flush), and the
// run's flush time.  The stable sort keeps a run's points in original order.  Worst case: one run holding the whole
// cloud is one thread's sequential loop.
__global__ void __launch_bounds__(256) avg_runs_kernel(
  const float4* points, const unsigned int* slot_sorted, const int* idx_sorted, const int* run_start, const int* n_runs_d, int n, float4* centroid,
  int* run_at_time, unsigned char* time_used) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  const int n_runs = *n_runs_d;
  if (r >= n_runs) return;
  const int s = run_start[r], e = r + 1 < n_runs ? run_start[r + 1] : n;
  float sx = 0.0f, sy = 0.0f, sz = 0.0f, sw = 0.0f;  // centroid.setZero()
  for (int p = s; p < e; p++) {
    const float4 v = __ldg(points + idx_sorted[p]);
    sx = __fadd_rn(sx, v.x);
    sy = __fadd_rn(sy, v.y);
    sz = __fadd_rn(sz, v.z);
    sw = __fadd_rn(sw, v.w);
  }
  const float c = __int2float_rn(e - s);  // static_cast<float>(count)
  centroid[r] = make_float4(__fdiv_rn(sx, c), __fdiv_rn(sy, c), __fdiv_rn(sz, c), __fdiv_rn(sw, c));
  const unsigned int slot = slot_sorted[s];
  const int t = (e < n && slot_sorted[e] == slot) ? idx_sorted[e] : n + static_cast<int>(slot);
  run_at_time[t] = r;
  time_used[t] = 1;
}

// ------------------------------------------------------------------------------------------------------------------
// 2. rank equalisation
// ------------------------------------------------------------------------------------------------------------------

// float -> uint32 with the order of `<` on floats; -0.0 is folded into +0.0 (they compare equal)
__device__ __forceinline__ unsigned int ordered_key(float v) {
  unsigned int u = __float_as_uint(v);
  if (u == 0x80000000u) u = 0u;
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__global__ void __launch_bounds__(256) eq_keys_kernel(const float* in, int n, unsigned int* key, int* index, unsigned int* bad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = in[i];
  if (!finite_f(v)) atomicOr(bad, 1u);
  key[i] = ordered_key(v);
  index[i] = i;
}

// intensities[idx[i]] = floor(bins * double(i) / N) / bins
__global__ void __launch_bounds__(256) eq_assign_kernel(const int* idx_sorted, int n, double* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  out[idx_sorted[i]] = __ddiv_rn(floor(__ddiv_rn(__dmul_rn(256.0, static_cast<double>(i)), static_cast<double>(n))), 256.0);
}

// ------------------------------------------------------------------------------------------------------------------
// 3. estimate_lidar_fov's VoxelGrid + norm filter
// ------------------------------------------------------------------------------------------------------------------

__device__ __forceinline__ unsigned int ord_f(float v) {
  const unsigned int u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __forceinline__ float unord_f(unsigned int k) {
  const unsigned int u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
  float v;
  std::memcpy(&v, &u, 4);
  return v;
}

// getMinMax3D as order-preserving uint32 (min x y z, max x y z); exact whatever the order
__global__ void __launch_bounds__(256) fov_minmax_kernel(const float* xyz, int n, unsigned int* mm, unsigned int* bad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned int lo[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, hi[3] = {0u, 0u, 0u};
  if (i < n) {
    for (int c = 0; c < 3; c++) {
      const float v = xyz[3 * static_cast<long long>(i) + c];
      if (!finite_f(v)) atomicOr(bad, 1u);
      lo[c] = hi[c] = ord_f(v);
    }
  }
  for (int c = 0; c < 3; c++) {
    for (int o = 16; o > 0; o >>= 1) {
      lo[c] = min(lo[c], __shfl_xor_sync(0xffffffffu, lo[c], o));
      hi[c] = max(hi[c], __shfl_xor_sync(0xffffffffu, hi[c], o));
    }
  }
  if ((threadIdx.x & 31) == 0) {
    for (int c = 0; c < 3; c++) {
      atomicMin(mm + c, lo[c]);
      atomicMax(mm + 3 + c, hi[c]);
    }
  }
}

struct FovGrid {
  float inv;
  int min_b[3];
  unsigned int mul1, mul2;  // divb_mul_[1], divb_mul_[2] (int arithmetic, wrapping)
};

// ijk = int(floor(p * inv) - float(min_b)), idx = ijk0 + ijk1 * div_x + ijk2 * div_x * div_y (voxel_grid.hpp)
__global__ void __launch_bounds__(256) fov_keys_kernel(const float* xyz, int n, const FovGrid g, unsigned int* key, int* index) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  unsigned int ijk[3];
  for (int c = 0; c < 3; c++) {
    const float v = xyz[3 * static_cast<long long>(i) + c];
    ijk[c] = static_cast<unsigned int>(float_to_int_x86(__fsub_rn(floorf(__fmul_rn(v, g.inv)), static_cast<float>(g.min_b[c]))));
  }
  key[i] = ijk[0] + ijk[1] * g.mul1 + ijk[2] * g.mul2;
  index[i] = i;
}

__global__ void __launch_bounds__(256) key_heads_kernel(const unsigned int* key_sorted, int n, unsigned char* head) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < n) head[p] = (p == 0 || key_sorted[p] != key_sorted[p - 1]) ? 1 : 0;
}

// `pt.getVector3fMap().norm() < 1.0` removes the point: sqrtf((x*x + y*y) + z*z), never contracted
__device__ __forceinline__ bool keep_by_norm(float x, float y, float z) {
  const float n2 = __fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z));
  return !(__fsqrt_rn(n2) < 1.0f);
}

// one thread per voxel: the sum of its points in index order, / float(count) (voxel_grid.hpp, downsample_all_data_ false)
__global__ void __launch_bounds__(256) fov_voxels_kernel(
  const float* xyz, const int* idx_sorted, const int* run_start, const int* n_runs_d, int n, float4* centroid, unsigned char* keep) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  const int n_runs = *n_runs_d;
  if (r >= n_runs) return;
  const int s = run_start[r], e = r + 1 < n_runs ? run_start[r + 1] : n;
  float sx = 0.0f, sy = 0.0f, sz = 0.0f;
  for (int p = s; p < e; p++) {
    const long long j = 3 * static_cast<long long>(idx_sorted[p]);
    sx = __fadd_rn(sx, xyz[j]);
    sy = __fadd_rn(sy, xyz[j + 1]);
    sz = __fadd_rn(sz, xyz[j + 2]);
  }
  const float c = __int2float_rn(e - s);
  const float cx = __fdiv_rn(sx, c), cy = __fdiv_rn(sy, c), cz = __fdiv_rn(sz, c);
  centroid[r] = make_float4(cx, cy, cz, 0.0f);
  keep[r] = keep_by_norm(cx, cy, cz) ? 1 : 0;
}

// PCL's fallback (the grid would overflow int32): the input itself, norm-filtered in input order
__global__ void __launch_bounds__(256) fov_passthrough_kernel(const float* xyz, int n, float4* centroid, unsigned char* keep) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long j = 3 * static_cast<long long>(i);
  centroid[i] = make_float4(xyz[j], xyz[j + 1], xyz[j + 2], 0.0f);
  keep[i] = keep_by_norm(xyz[j], xyz[j + 1], xyz[j + 2]) ? 1 : 0;
}

// ------------------------------------------------------------------------------------------------------------------
// 4. minimum bearing cosine
// ------------------------------------------------------------------------------------------------------------------

constexpr int kCosTile = 128;

// double -> uint64 with the order of `<`; the minimum of these is the minimum cosine whatever the order of the pairs
__host__ __device__ __forceinline__ unsigned long long ord_d(double v) {
  unsigned long long u;
#ifdef __CUDA_ARCH__
  u = static_cast<unsigned long long>(__double_as_longlong(v));
#else
  std::memcpy(&u, &v, 8);
#endif
  return (u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull);
}
__host__ __forceinline__ double unord_d(unsigned long long k) {
  const unsigned long long u = (k & 0x8000000000000000ull) ? (k & 0x7fffffffffffffffull) : ~k;
  double v;
  std::memcpy(&v, &u, 8);
  return v;
}

// dirs[i] = p.cast<double>().normalized(): p / sqrt((x*x + y*y) + z*z) when that is > 0
__global__ void __launch_bounds__(256) bearings_kernel(const float* xyz, int n, double3* dirs) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
  const double n2 = __dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z));
  if (n2 > 0.0) {
    const double nn = __dsqrt_rn(n2);
    dirs[i] = make_double3(__ddiv_rn(x, nn), __ddiv_rn(y, nn), __ddiv_rn(z, nn));
  } else {
    dirs[i] = make_double3(x, y, z);
  }
}

// tile (blockIdx.y, blockIdx.x) of the pair matrix, only pairs i < j; one atomicMin per block
__global__ void __launch_bounds__(256) min_cosine_kernel(const double3* dirs, int n, unsigned long long* result) {
  if (blockIdx.x < blockIdx.y) return;
  __shared__ double3 a[kCosTile], b[kCosTile];
  __shared__ unsigned long long warp_min[8];
  const int i0 = blockIdx.y * kCosTile, j0 = blockIdx.x * kCosTile;
  for (int t = threadIdx.x; t < kCosTile; t += blockDim.x) {
    if (i0 + t < n) a[t] = dirs[i0 + t];
    if (j0 + t < n) b[t] = dirs[j0 + t];
  }
  __syncthreads();
  unsigned long long best = ~0ull;
  for (int q = threadIdx.x; q < kCosTile * kCosTile; q += blockDim.x) {
    const int ti = q / kCosTile, tj = q % kCosTile;
    const int i = i0 + ti, j = j0 + tj;
    if (i >= n || j >= n || j <= i) continue;
    const double3 u = a[ti], v = b[tj];
    const double c = __dadd_rn(__dadd_rn(__dmul_rn(u.x, v.x), __dmul_rn(u.y, v.y)), __dmul_rn(u.z, v.z));  // dirs[i].dot(dirs[j])
    best = min(best, ord_d(c));
  }
  for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
  if ((threadIdx.x & 31) == 0) warp_min[threadIdx.x >> 5] = best;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < static_cast<int>(blockDim.x >> 5); w++) best = min(best, warp_min[w]);
    if (best != ~0ull) atomicMin(result, best);
  }
}

}  // namespace
}  // namespace vlcal

using namespace vlcal;

extern "C" int vlcal_approximate_voxel_grid(
  int device, const float* points_xyzi, int64_t n_points, double leaf_size, float* points_out, int64_t* n_out, int64_t* out_of_range_points, double* stage_ms_out) {
  const float leaf = static_cast<float>(leaf_size);  // setLeafSize(float, float, float)
  const float inv = 1.0f / leaf;                      // inverse_leaf_size_ = Ones / leaf_size_
  if (n_points < 0 || n_points > kMaxPoints || (n_points > 0 && (!points_xyzi || !points_out)) || !n_out) {
    set_last_error("approximate_voxel_grid: invalid arguments (0 <= n <= 2^31 - 513 points, non-null buffers)");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  if (!(leaf > 0.0f) || !finite_f(leaf) || !finite_f(inv)) {
    set_last_error("approximate_voxel_grid: the leaf size must be a positive float with a finite inverse");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  *n_out = 0;
  if (out_of_range_points) *out_of_range_points = 0;
  int rc = prepare_device(&device);
  if (rc != VLCAL_OK) return rc;
  if (n_points == 0) {
    if (stage_ms_out)
      for (int k = 0; k < 4; k++) stage_ms_out[k] = 0.0;
    return VLCAL_OK;
  }
  const int n = static_cast<int>(n_points);
  Scratch s(device);
  float4 *pts, *centroid;
  int4* keys;
  unsigned int *slot, *slot_sorted, *flags;
  int *index, *idx_sorted, *run_start, *n_runs, *run_at_time, *order, *n_order;
  unsigned char *head, *time_used;
  VL_CUDA(s.alloc(n, &pts));
  VL_CUDA(s.alloc(n, &keys));
  VL_CUDA(s.alloc(n, &slot));
  VL_CUDA(s.alloc(n, &slot_sorted));
  VL_CUDA(s.alloc(n, &index));
  VL_CUDA(s.alloc(n, &idx_sorted));
  VL_CUDA(s.alloc(n, &head));
  VL_CUDA(s.alloc(n, &run_start));
  VL_CUDA(s.alloc(n, &centroid));
  VL_CUDA(s.alloc(static_cast<size_t>(n) + kHistSize, &run_at_time));
  VL_CUDA(s.alloc(static_cast<size_t>(n) + kHistSize, &time_used));
  VL_CUDA(s.alloc(n, &order));
  VL_CUDA(s.alloc(4, &n_runs));
  n_order = n_runs + 1;
  VL_CUDA(s.alloc(2, &flags));
  size_t tmp_sort = 0, tmp_sel = 0, tmp_if = 0;
  VL_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_sort, slot, slot_sorted, index, idx_sorted, n, 0, 9));
  VL_CUDA(cub::DeviceSelect::Flagged(nullptr, tmp_sel, thrust::counting_iterator<int>(0), head, run_start, n_runs, n));
  VL_CUDA(cub::DeviceSelect::Flagged(nullptr, tmp_if, run_at_time, time_used, order, n_order, n + kHistSize));
  unsigned char* tmp;
  VL_CUDA(s.alloc(std::max(tmp_sort, std::max(tmp_sel, tmp_if)), &tmp));
  VL_CUDA(cudaMemcpy(pts, points_xyzi, sizeof(float4) * n, cudaMemcpyHostToDevice));
  VL_CUDA(cudaMemset(flags, 0, 2 * sizeof(unsigned int)));

  StageTimer timer(stage_ms_out != nullptr);
  VL_CUDA(timer.mark());
  AvgArgs a;
  a.points = pts, a.n = n, a.inv = inv, a.keys = keys, a.slot = slot, a.index = index, a.flags = flags;
  avg_keys_kernel<<<blocks_for(n, 256), 256>>>(a);
  VL_CUDA(cudaGetLastError());
  VL_CUDA(timer.mark());
  VL_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tmp_sort, slot, slot_sorted, index, idx_sorted, n, 0, 9));  // stable
  VL_CUDA(timer.mark());
  avg_heads_kernel<<<blocks_for(n, 256), 256>>>(slot_sorted, idx_sorted, keys, n, head);
  VL_CUDA(cudaGetLastError());
  VL_CUDA(cub::DeviceSelect::Flagged(tmp, tmp_sel, thrust::counting_iterator<int>(0), head, run_start, n_runs, n));
  VL_CUDA(cudaMemsetAsync(time_used, 0, static_cast<size_t>(n) + kHistSize, cudaStreamLegacy));
  avg_runs_kernel<<<blocks_for(n, 256), 256>>>(pts, slot_sorted, idx_sorted, run_start, n_runs, n, centroid, run_at_time, time_used);
  VL_CUDA(cudaGetLastError());
  VL_CUDA(timer.mark());
  VL_CUDA(cub::DeviceSelect::Flagged(tmp, tmp_if, run_at_time, time_used, order, n_order, n + kHistSize));
  gather_float4_kernel<<<blocks_for(n, 256), 256>>>(centroid, order, n_order, reinterpret_cast<float4*>(keys));  // keys are dead: reuse
  VL_CUDA(cudaGetLastError());
  VL_CUDA(timer.mark());
  int counts[2];
  unsigned int h_flags[2];
  VL_CUDA(cudaMemcpy(counts, n_runs, sizeof(counts), cudaMemcpyDeviceToHost));
  VL_CUDA(cudaMemcpy(h_flags, flags, sizeof(h_flags), cudaMemcpyDeviceToHost));
  if (h_flags[0]) {
    set_last_error("approximate_voxel_grid: non-finite coordinate or intensity in the input (the reference's behaviour is undefined there)");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  if (counts[0] != counts[1]) {
    set_last_error("approximate_voxel_grid: internal error: flush times are not distinct");
    return VLCAL_ERR_CUDA;
  }
  VL_CUDA(cudaMemcpy(points_out, keys, sizeof(float4) * counts[0], cudaMemcpyDeviceToHost));
  VL_CUDA(timer.read(stage_ms_out, 4));
  *n_out = counts[0];
  if (out_of_range_points) *out_of_range_points = h_flags[1];
  return VLCAL_OK;
}

extern "C" int vlcal_equalize_intensities(int device, const float* intensities, int64_t n_points, double* intensities_out, double* kernel_ms_out) {
  if (n_points < 0 || n_points > 0x7fffffffLL || (n_points > 0 && (!intensities || !intensities_out))) {
    set_last_error("equalize_intensities: invalid arguments (0 <= n <= 2^31 - 1 points, non-null buffers)");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  int rc = prepare_device(&device);
  if (rc != VLCAL_OK) return rc;
  if (kernel_ms_out) *kernel_ms_out = 0.0;
  if (n_points == 0) return VLCAL_OK;
  const int n = static_cast<int>(n_points);
  Scratch s(device);
  float* in;
  unsigned int *key, *key_sorted, *bad;
  int *index, *idx_sorted;
  double* out;
  VL_CUDA(s.alloc(n, &in));
  VL_CUDA(s.alloc(n, &key));
  VL_CUDA(s.alloc(n, &key_sorted));
  VL_CUDA(s.alloc(n, &index));
  VL_CUDA(s.alloc(n, &idx_sorted));
  VL_CUDA(s.alloc(n, &out));
  VL_CUDA(s.alloc(1, &bad));
  size_t tmp_sort = 0;
  VL_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_sort, key, key_sorted, index, idx_sorted, n));
  unsigned char* tmp;
  VL_CUDA(s.alloc(tmp_sort, &tmp));
  VL_CUDA(cudaMemcpy(in, intensities, sizeof(float) * n, cudaMemcpyHostToDevice));
  VL_CUDA(cudaMemset(bad, 0, sizeof(unsigned int)));
  StageTimer timer(kernel_ms_out != nullptr);
  VL_CUDA(timer.mark());
  eq_keys_kernel<<<blocks_for(n, 256), 256>>>(in, n, key, index, bad);
  VL_CUDA(cudaGetLastError());
  VL_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tmp_sort, key, key_sorted, index, idx_sorted, n));  // stable: ties by index
  eq_assign_kernel<<<blocks_for(n, 256), 256>>>(idx_sorted, n, out);
  VL_CUDA(cudaGetLastError());
  VL_CUDA(timer.mark());
  unsigned int h_bad = 0;
  VL_CUDA(cudaMemcpy(&h_bad, bad, sizeof(h_bad), cudaMemcpyDeviceToHost));
  if (h_bad) {
    set_last_error("equalize_intensities: non-finite intensity in the input (the reference's comparator is undefined there)");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  VL_CUDA(cudaMemcpy(intensities_out, out, sizeof(double) * n, cudaMemcpyDeviceToHost));
  VL_CUDA(timer.read(kernel_ms_out, 1));
  return VLCAL_OK;
}

extern "C" int vlcal_lidar_fov_candidates(
  int device, const float* points_xyz, int64_t n_points, float* candidates_out, int64_t* n_out, int* unfiltered_out, double* kernel_ms_out) {
  if (n_points < 0 || n_points > 0x7fffffffLL || (n_points > 0 && (!points_xyz || !candidates_out)) || !n_out) {
    set_last_error("lidar_fov_candidates: invalid arguments (0 <= n <= 2^31 - 1 points, non-null buffers)");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  *n_out = 0;
  if (unfiltered_out) *unfiltered_out = 0;
  if (kernel_ms_out) *kernel_ms_out = 0.0;
  int rc = prepare_device(&device);
  if (rc != VLCAL_OK) return rc;
  if (n_points == 0) return VLCAL_OK;
  const int n = static_cast<int>(n_points);
  Scratch s(device);
  float* xyz;
  unsigned int *mm, *bad, *key, *key_sorted;
  int *index, *idx_sorted, *run_start, *n_runs;
  unsigned char *head, *keep;
  float4 *centroid, *selected;
  VL_CUDA(s.alloc(3 * static_cast<size_t>(n), &xyz));
  VL_CUDA(s.alloc(8, &mm));
  bad = mm + 6;
  VL_CUDA(s.alloc(n, &key));
  VL_CUDA(s.alloc(n, &key_sorted));
  VL_CUDA(s.alloc(n, &index));
  VL_CUDA(s.alloc(n, &idx_sorted));
  VL_CUDA(s.alloc(n, &run_start));
  VL_CUDA(s.alloc(4, &n_runs));
  VL_CUDA(s.alloc(n, &head));
  VL_CUDA(s.alloc(n, &keep));
  VL_CUDA(s.alloc(n, &centroid));
  VL_CUDA(s.alloc(n, &selected));
  VL_CUDA(cudaMemcpy(xyz, points_xyz, 3 * sizeof(float) * n, cudaMemcpyHostToDevice));
  const unsigned int mm_init[8] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u, 0u, 0u};
  VL_CUDA(cudaMemcpy(mm, mm_init, sizeof(mm_init), cudaMemcpyHostToDevice));
  StageTimer timer(kernel_ms_out != nullptr);
  VL_CUDA(timer.mark());
  fov_minmax_kernel<<<blocks_for(n, 256), 256>>>(xyz, n, mm, bad);
  VL_CUDA(cudaGetLastError());
  unsigned int h_mm[8];
  VL_CUDA(cudaMemcpy(h_mm, mm, sizeof(h_mm), cudaMemcpyDeviceToHost));
  if (h_mm[6]) {
    set_last_error("lidar_fov_candidates: non-finite coordinate in the input");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  // voxel_grid.hpp applyFilter: the grid extent check on int64, else min_b / div_b / divb_mul in int
  const float leaf = 0.2f;
  const float inv = 1.0f / leaf;
  float min_p[3], max_p[3];
  bool overflow = false;
  int64_t d[3];
  for (int c = 0; c < 3; c++) {
    min_p[c] = unord_f(h_mm[c]);
    max_p[c] = unord_f(h_mm[3 + c]);
    const float ext = (max_p[c] - min_p[c]) * inv;
    if (!(ext < 9.2e18f)) overflow = true;  // beyond int64 (PCL's cast is undefined there): the grid would overflow anyway
    else d[c] = static_cast<int64_t>(ext) + 1;
  }
  // (dx * dy * dz) > INT32_MAX in int64, wrapping as the reference's imul does (only extents beyond ~2^21 voxels per
  // axis wrap)
  if (!overflow) {
    const uint64_t prod = static_cast<uint64_t>(d[0]) * static_cast<uint64_t>(d[1]) * static_cast<uint64_t>(d[2]);
    overflow = static_cast<int64_t>(prod) > static_cast<int64_t>(INT32_MAX);
  }
  size_t tmp_sort = 0, tmp_sel = 0, tmp_keep = 0;
  VL_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_sort, key, key_sorted, index, idx_sorted, n));
  VL_CUDA(cub::DeviceSelect::Flagged(nullptr, tmp_sel, thrust::counting_iterator<int>(0), head, run_start, n_runs, n));
  VL_CUDA(cub::DeviceSelect::Flagged(nullptr, tmp_keep, centroid, keep, selected, n_runs + 1, n));
  unsigned char* tmp;
  VL_CUDA(s.alloc(std::max(tmp_sort, std::max(tmp_sel, tmp_keep)), &tmp));
  int n_voxels = n;
  if (overflow) {
    fov_passthrough_kernel<<<blocks_for(n, 256), 256>>>(xyz, n, centroid, keep);  // output = *input_
    VL_CUDA(cudaGetLastError());
  } else {
    FovGrid g;
    g.inv = inv;
    int div_b[3];
    for (int c = 0; c < 3; c++) {
      g.min_b[c] = float_to_int_x86(std::floor(min_p[c] * inv));
      const int max_b = float_to_int_x86(std::floor(max_p[c] * inv));
      div_b[c] = static_cast<int>(static_cast<unsigned int>(max_b) - static_cast<unsigned int>(g.min_b[c]) + 1u);
    }
    g.mul1 = static_cast<unsigned int>(div_b[0]);
    g.mul2 = static_cast<unsigned int>(div_b[0]) * static_cast<unsigned int>(div_b[1]);
    fov_keys_kernel<<<blocks_for(n, 256), 256>>>(xyz, n, g, key, index);
    VL_CUDA(cudaGetLastError());
    VL_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tmp_sort, key, key_sorted, index, idx_sorted, n));  // stable: index order
    key_heads_kernel<<<blocks_for(n, 256), 256>>>(key_sorted, n, head);
    VL_CUDA(cudaGetLastError());
    VL_CUDA(cub::DeviceSelect::Flagged(tmp, tmp_sel, thrust::counting_iterator<int>(0), head, run_start, n_runs, n));
    fov_voxels_kernel<<<blocks_for(n, 256), 256>>>(xyz, idx_sorted, run_start, n_runs, n, centroid, keep);
    VL_CUDA(cudaGetLastError());
    VL_CUDA(cudaMemcpy(&n_voxels, n_runs, sizeof(int), cudaMemcpyDeviceToHost));
  }
  VL_CUDA(cub::DeviceSelect::Flagged(tmp, tmp_keep, centroid, keep, selected, n_runs + 1, n_voxels));  // remove_if keeps the order
  VL_CUDA(timer.mark());
  int n_kept = 0;
  VL_CUDA(cudaMemcpy(&n_kept, n_runs + 1, sizeof(int), cudaMemcpyDeviceToHost));
  std::vector<float4> host(n_kept);
  if (n_kept) VL_CUDA(cudaMemcpy(host.data(), selected, sizeof(float4) * n_kept, cudaMemcpyDeviceToHost));
  for (int k = 0; k < n_kept; k++) {
    candidates_out[3 * k] = host[k].x;
    candidates_out[3 * k + 1] = host[k].y;
    candidates_out[3 * k + 2] = host[k].z;
  }
  VL_CUDA(timer.read(kernel_ms_out, 1));
  *n_out = n_kept;
  if (unfiltered_out) *unfiltered_out = overflow ? 1 : 0;
  return VLCAL_OK;
}

extern "C" int vlcal_min_bearing_cosine(int device, const float* vertices_xyz, int64_t n_vertices, double* min_cosine_out) {
  // 65535 tiles per grid axis
  if (n_vertices < 0 || n_vertices > 65535LL * kCosTile || (n_vertices > 0 && !vertices_xyz) || !min_cosine_out) {
    set_last_error("min_bearing_cosine: invalid arguments (0 <= n <= 8388480 vertices, non-null buffers)");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  for (int64_t i = 0; i < 3 * n_vertices; i++) {
    if (!std::isfinite(vertices_xyz[i])) {
      set_last_error("min_bearing_cosine: non-finite vertex coordinate");
      return VLCAL_ERR_INVALID_ARGUMENT;
    }
  }
  int rc = prepare_device(&device);
  if (rc != VLCAL_OK) return rc;
  const unsigned long long init = ord_d(M_PI);  // double min_cosine = M_PI
  if (n_vertices < 2) {
    *min_cosine_out = M_PI;
    return VLCAL_OK;
  }
  const int n = static_cast<int>(n_vertices);
  Scratch s(device);
  float* xyz;
  double3* dirs;
  unsigned long long* result;
  VL_CUDA(s.alloc(3 * static_cast<size_t>(n), &xyz));
  VL_CUDA(s.alloc(n, &dirs));
  VL_CUDA(s.alloc(1, &result));
  VL_CUDA(cudaMemcpy(xyz, vertices_xyz, 3 * sizeof(float) * n, cudaMemcpyHostToDevice));
  VL_CUDA(cudaMemcpy(result, &init, sizeof(init), cudaMemcpyHostToDevice));
  bearings_kernel<<<blocks_for(n, 256), 256>>>(xyz, n, dirs);
  VL_CUDA(cudaGetLastError());
  const unsigned int tiles = blocks_for(n, kCosTile);
  min_cosine_kernel<<<dim3(tiles, tiles), 256>>>(dirs, n, result);
  VL_CUDA(cudaGetLastError());
  unsigned long long h = 0;
  VL_CUDA(cudaMemcpy(&h, result, sizeof(h), cudaMemcpyDeviceToHost));
  *min_cosine_out = unord_d(h);
  return VLCAL_OK;
}
