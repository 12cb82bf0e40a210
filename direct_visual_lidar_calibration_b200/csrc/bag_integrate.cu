// bag_integrate.cu -- PointCloud2 decoding and the static point integration of `preprocess` on the GPU (reference:
// include/vlcal/common/ros_cloud_converter.hpp:62-175 extract_raw_points, src/vlcal/preprocess/preprocess.cpp:454-459
// the finiteness filter, src/vlcal/preprocess/static_point_cloud_integrator.cpp:25-62 insert_points / get_points).
//
// The reference walks every point of every accepted scan of a bag, in arrival order, into
// unordered_map<Vector3i, Vector4d>: voxelgrid[floor(p / voxel_resolution)] = (x, y, z, intensity), so the last point
// written to a voxel wins.  Here all scans of a bag are one launch (DESIGN §4c):
//   1. decode: one thread per point finds its scan (binary search over the scans' first point), reads x, y, z and the
//      intensity with byte loads (PointCloud2 offsets need not be aligned), drops non-finite points and points with
//      (x*x + y*y) + z*z rooted below min_distance (never-contracted double, Eigen's order), and writes the voxel key
//      floor(p / voxel_resolution) cast to int (x86's INT_MIN out of range) and the float-cast values of get_points.
//   2. the kept points' global indices (ascending: arrival order) are sorted by the 96-bit key with two stable radix
//      sorts (z, then x:y), so each run of equal keys holds its points in arrival order.
//   3. one thread per run: the last index of the run is the point that wins; it is written at the run's first index,
//      and a compaction in index order emits the winners in first-write order.  The reference's order is libstdc++'s
//      hash-table iteration order, which nothing downstream depends on.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <cmath>
#include <cstdint>
#include <string>

#include "preprocess_common.cuh"

namespace vlcal {
namespace {

// sensor_msgs/PointField datatypes
constexpr int kUint8 = 2, kUint16 = 4, kUint32 = 6, kFloat32 = 7, kFloat64 = 8;

__device__ __forceinline__ unsigned int load_u32(const unsigned char* p) {
  return static_cast<unsigned int>(p[0]) | (static_cast<unsigned int>(p[1]) << 8) | (static_cast<unsigned int>(p[2]) << 16) |
         (static_cast<unsigned int>(p[3]) << 24);
}

__device__ __forceinline__ double load_f64(const unsigned char* p) {
  const unsigned long long lo = load_u32(p), hi = load_u32(p + 4);
  return __longlong_as_double(static_cast<long long>(lo | (hi << 32)));
}

// x / y / z as get_vec4<float> or get_vec4<double> reads them (little-endian; big-endian clouds are refused on the host)
__device__ __forceinline__ double load_coord(const unsigned char* p, int type) {
  return type == kFloat32 ? static_cast<double>(__uint_as_float(load_u32(p))) : load_f64(p);
}

// ros_cloud_converter.hpp:150-165
__device__ __forceinline__ double load_intensity(const unsigned char* p, int type) {
  switch (type) {
    case kUint8: return static_cast<double>(p[0]);
    case kUint16: return static_cast<double>(static_cast<unsigned int>(p[0]) | (static_cast<unsigned int>(p[1]) << 8));
    case kUint32: return static_cast<double>(load_u32(p));
    case kFloat32: return static_cast<double>(__uint_as_float(load_u32(p)));
    default: return load_f64(p);
  }
}

// static_cast<int>(double) as x86-64 compiles it (cvttsd2si): INT_MIN out of range.  `d` is a floor result.
__device__ __forceinline__ int double_to_int_x86(double d) { return (d >= -2147483648.0 && d < 2147483648.0) ? static_cast<int>(d) : INT_MIN; }

__device__ __forceinline__ bool finite_d(double v) { return fabs(v) <= DBL_MAX; }

struct DecodeArgs {
  const unsigned char* data;
  const vlcal_scan_desc* scans;
  const long long* scan_first;  // [n_scans + 1], first global point index of each scan
  int n_scans;
  int n;                        // points in all scans
  double res, min_distance;
  int* kx;                      // [n] voxel keys
  int* ky;
  int* kz;
  float4* values;               // [n] (float(x), float(y), float(z), float(intensity))
  unsigned char* keep;          // [n]
  unsigned long long* out_of_range;
};

__global__ void __launch_bounds__(256) bag_decode_kernel(const __grid_constant__ DecodeArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  int lo = 0, hi = a.n_scans - 1;  // the last scan whose first point is <= i (empty scans are skipped over)
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(a.scan_first + mid) <= i) lo = mid;
    else hi = mid - 1;
  }
  const vlcal_scan_desc s = a.scans[lo];
  const unsigned char* p = a.data + s.byte_offset + static_cast<long long>(s.point_step) * (i - __ldg(a.scan_first + lo));
  // Vector4d(x, y, z, 1); z is read with x's datatype (the reference checks x against y twice and never looks at z's)
  const double x = load_coord(p + s.x_offset, s.xyz_type), y = load_coord(p + s.y_offset, s.xyz_type), z = load_coord(p + s.z_offset, s.xyz_type);
  const double w = load_intensity(p + s.intensity_offset, s.intensity_type);
  bool keep = finite_d(x) && finite_d(y) && finite_d(z);  // p.array().isFinite().all()
  // pt.head<3>().norm() < min_distance drops the point
  keep = keep && !(__dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z))) < a.min_distance);
  a.keep[i] = keep ? 1 : 0;
  if (!keep) return;
  const double fx = floor(__ddiv_rn(x, a.res)), fy = floor(__ddiv_rn(y, a.res)), fz = floor(__ddiv_rn(z, a.res));
  const int ix = double_to_int_x86(fx), iy = double_to_int_x86(fy), iz = double_to_int_x86(fz);
  if ((ix == INT_MIN && fx != -2147483648.0) || (iy == INT_MIN && fy != -2147483648.0) || (iz == INT_MIN && fz != -2147483648.0)) atomicAdd(a.out_of_range, 1ull);
  a.kx[i] = ix;
  a.ky[i] = iy;
  a.kz[i] = iz;
  a.values[i] = make_float4(__double2float_rn(x), __double2float_rn(y), __double2float_rn(z), __double2float_rn(w));  // get_points' casts
}

__global__ void __launch_bounds__(256) gather_z_kernel(const int* kz, const int* idx, const int* m_d, unsigned int* out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < *m_d) out[k] = static_cast<unsigned int>(kz[idx[k]]);
}

__global__ void __launch_bounds__(256) gather_xy_kernel(const int* kx, const int* ky, const int* idx, const int* m_d, unsigned long long* out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < *m_d) out[k] = (static_cast<unsigned long long>(static_cast<unsigned int>(kx[idx[k]])) << 32) | static_cast<unsigned int>(ky[idx[k]]);
}

// a run of equal (x, y, z) keys starts at sorted position p
__global__ void __launch_bounds__(256) bag_heads_kernel(const unsigned long long* xy_sorted, const int* kz, const int* idx_sorted, const int* m_d, unsigned char* head) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= *m_d) return;
  head[p] = (p == 0 || xy_sorted[p] != xy_sorted[p - 1] || kz[idx_sorted[p]] != kz[idx_sorted[p - 1]]) ? 1 : 0;
}

// one thread per run: the run's last (largest) index wins and is placed at its first (smallest) index
__global__ void __launch_bounds__(256) bag_runs_kernel(const int* idx_sorted, const int* run_start, const int* n_runs_d, const int* m_d, int* winner_at, unsigned char* used) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  const int n_runs = *n_runs_d;
  if (r >= n_runs) return;
  const int s = run_start[r], e = r + 1 < n_runs ? run_start[r + 1] : *m_d;
  const int first = idx_sorted[s];
  winner_at[first] = idx_sorted[e - 1];
  used[first] = 1;
}

int field_size(int type) { return type == kUint8 ? 1 : type == kUint16 ? 2 : (type == kUint32 || type == kFloat32) ? 4 : 8; }

}  // namespace
}  // namespace vlcal

using namespace vlcal;

extern "C" int vlcal_bag_integrate(
  int device, const uint8_t* data, int64_t data_bytes, const vlcal_scan_desc* scans, int64_t n_scans, double voxel_resolution, double min_distance,
  float* points_out, int64_t* n_out, int64_t* out_of_range_points, double* stage_ms_out) {
  if (!n_out || n_scans < 0 || n_scans > 0x7fffffffLL || data_bytes < 0 || (n_scans > 0 && !scans)) {
    set_last_error("bag_integrate: invalid arguments (0 <= n_scans < 2^31, non-null buffers)");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  if (!(voxel_resolution > 0.0) || !std::isfinite(voxel_resolution) || std::isnan(min_distance)) {
    set_last_error("bag_integrate: voxel_resolution must be a positive finite number and min_distance a number");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  *n_out = 0;
  if (out_of_range_points) *out_of_range_points = 0;
  if (stage_ms_out)
    for (int k = 0; k < 3; k++) stage_ms_out[k] = 0.0;
  std::vector<long long> first(n_scans + 1, 0);
  for (int64_t s = 0; s < n_scans; s++) {
    const vlcal_scan_desc& d = scans[s];
    const bool types_ok = (d.xyz_type == kFloat32 || d.xyz_type == kFloat64) &&
                          (d.intensity_type == kUint8 || d.intensity_type == kUint16 || d.intensity_type == kUint32 || d.intensity_type == kFloat32 ||
                           d.intensity_type == kFloat64);
    bool ok = types_ok && d.n_points >= 0 && d.byte_offset >= 0 && d.point_step >= 0 && d.x_offset >= 0 && d.y_offset >= 0 && d.z_offset >= 0 && d.intensity_offset >= 0;
    if (ok && d.n_points > 0) {
      // every field of the last point lies inside the data
      const int64_t last = d.byte_offset + static_cast<int64_t>(d.point_step) * (d.n_points - 1);
      const int64_t cs = field_size(d.xyz_type);
      const int64_t end = std::max(std::max(d.x_offset + cs, d.y_offset + cs), std::max(d.z_offset + cs, d.intensity_offset + static_cast<int64_t>(field_size(d.intensity_type))));
      ok = last + end <= data_bytes && data;
    }
    if (!ok) {
      set_last_error("bag_integrate: scan " + std::to_string(s) + ": unsupported datatype or a field beyond the data");
      return VLCAL_ERR_INVALID_ARGUMENT;
    }
    first[s + 1] = first[s] + d.n_points;
  }
  const long long total = first[n_scans];
  if (total > 0x7fffffffLL) {
    set_last_error("bag_integrate: more than 2^31 - 1 points in one bag");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  if (total > 0 && !points_out) {
    set_last_error("bag_integrate: points_out is null");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  int rc = prepare_device(&device);
  if (rc != VLCAL_OK) return rc;
  if (total == 0) return VLCAL_OK;
  const int n = static_cast<int>(total);

  Scratch s(device);
  unsigned char *d_data, *keep, *head, *used;
  vlcal_scan_desc* d_scans;
  long long* d_first;
  int *kx, *ky, *kz, *sel, *idx_a, *idx_b, *run_start, *winner_at, *order, *counts;
  unsigned int *z_in, *z_sorted;
  unsigned long long *xy_in, *xy_sorted, *oor;
  float4 *values, *out;
  VL_CUDA(s.alloc(static_cast<size_t>(data_bytes), &d_data));
  VL_CUDA(s.alloc(n_scans, &d_scans));
  VL_CUDA(s.alloc(n_scans + 1, &d_first));
  VL_CUDA(s.alloc(n, &kx));
  VL_CUDA(s.alloc(n, &ky));
  VL_CUDA(s.alloc(n, &kz));
  VL_CUDA(s.alloc(n, &values));
  VL_CUDA(s.alloc(n, &keep));
  VL_CUDA(s.alloc(n, &sel));
  VL_CUDA(s.alloc(n, &z_in));
  VL_CUDA(s.alloc(n, &z_sorted));
  VL_CUDA(s.alloc(n, &idx_a));
  VL_CUDA(s.alloc(n, &xy_in));
  VL_CUDA(s.alloc(n, &xy_sorted));
  VL_CUDA(s.alloc(n, &idx_b));
  VL_CUDA(s.alloc(n, &head));
  VL_CUDA(s.alloc(n, &run_start));
  VL_CUDA(s.alloc(n, &winner_at));
  VL_CUDA(s.alloc(n, &used));
  VL_CUDA(s.alloc(n, &order));
  VL_CUDA(s.alloc(n, &out));
  VL_CUDA(s.alloc(4, &counts));  // kept points, runs, emitted points
  VL_CUDA(s.alloc(1, &oor));
  // cub's temporary storage is sized for n items; the sorts run on the kept points only (m <= n, read from the device)
  size_t tmp_sel = 0, tmp_z = 0, tmp_xy = 0, tmp_runs = 0, tmp_out = 0;
  VL_CUDA(cub::DeviceSelect::Flagged(nullptr, tmp_sel, thrust::counting_iterator<int>(0), keep, sel, counts, n));
  VL_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_z, z_in, z_sorted, sel, idx_a, n));
  VL_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_xy, xy_in, xy_sorted, idx_a, idx_b, n));
  VL_CUDA(cub::DeviceSelect::Flagged(nullptr, tmp_runs, thrust::counting_iterator<int>(0), head, run_start, counts + 1, n));
  VL_CUDA(cub::DeviceSelect::Flagged(nullptr, tmp_out, winner_at, used, order, counts + 2, n));
  unsigned char* tmp;
  VL_CUDA(s.alloc(std::max(std::max(tmp_sel, tmp_z), std::max(tmp_xy, std::max(tmp_runs, tmp_out))), &tmp));
  if (data_bytes) VL_CUDA(cudaMemcpy(d_data, data, static_cast<size_t>(data_bytes), cudaMemcpyHostToDevice));
  VL_CUDA(cudaMemcpy(d_scans, scans, sizeof(vlcal_scan_desc) * n_scans, cudaMemcpyHostToDevice));
  VL_CUDA(cudaMemcpy(d_first, first.data(), sizeof(long long) * (n_scans + 1), cudaMemcpyHostToDevice));
  VL_CUDA(cudaMemset(oor, 0, sizeof(unsigned long long)));
  VL_CUDA(cudaMemset(used, 0, n));

  StageTimer timer(stage_ms_out != nullptr);
  VL_CUDA(timer.mark());
  DecodeArgs a;
  a.data = d_data, a.scans = d_scans, a.scan_first = d_first, a.n_scans = static_cast<int>(n_scans), a.n = n;
  a.res = voxel_resolution, a.min_distance = min_distance;
  a.kx = kx, a.ky = ky, a.kz = kz, a.values = values, a.keep = keep, a.out_of_range = oor;
  bag_decode_kernel<<<blocks_for(n, 256), 256>>>(a);
  VL_CUDA(cudaGetLastError());
  VL_CUDA(timer.mark());
  int m = 0;
  VL_CUDA(cub::DeviceSelect::Flagged(tmp, tmp_sel, thrust::counting_iterator<int>(0), keep, sel, counts, n));
  VL_CUDA(cudaMemcpy(&m, counts, sizeof(int), cudaMemcpyDeviceToHost));
  if (m > 0) {
    gather_z_kernel<<<blocks_for(m, 256), 256>>>(kz, sel, counts, z_in);
    VL_CUDA(cudaGetLastError());
    VL_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tmp_z, z_in, z_sorted, sel, idx_a, m));  // stable
    gather_xy_kernel<<<blocks_for(m, 256), 256>>>(kx, ky, idx_a, counts, xy_in);
    VL_CUDA(cudaGetLastError());
    VL_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tmp_xy, xy_in, xy_sorted, idx_a, idx_b, m));  // stable: runs in index order
  }
  VL_CUDA(timer.mark());
  int emitted = 0;
  if (m > 0) {
    bag_heads_kernel<<<blocks_for(m, 256), 256>>>(xy_sorted, kz, idx_b, counts, head);
    VL_CUDA(cudaGetLastError());
    VL_CUDA(cub::DeviceSelect::Flagged(tmp, tmp_runs, thrust::counting_iterator<int>(0), head, run_start, counts + 1, m));
    bag_runs_kernel<<<blocks_for(m, 256), 256>>>(idx_b, run_start, counts + 1, counts, winner_at, used);
    VL_CUDA(cudaGetLastError());
    VL_CUDA(cub::DeviceSelect::Flagged(tmp, tmp_out, winner_at, used, order, counts + 2, n));  // first-write order
    gather_float4_kernel<<<blocks_for(m, 256), 256>>>(values, order, counts + 2, out);
    VL_CUDA(cudaGetLastError());
    VL_CUDA(cudaMemcpy(&emitted, counts + 2, sizeof(int), cudaMemcpyDeviceToHost));
  }
  VL_CUDA(timer.mark());
  if (emitted) VL_CUDA(cudaMemcpy(points_out, out, sizeof(float4) * emitted, cudaMemcpyDeviceToHost));
  unsigned long long h_oor = 0;
  VL_CUDA(cudaMemcpy(&h_oor, oor, sizeof(h_oor), cudaMemcpyDeviceToHost));
  VL_CUDA(timer.read(stage_ms_out, 3));
  *n_out = emitted;
  if (out_of_range_points) *out_of_range_points = static_cast<int64_t>(h_oor);
  return VLCAL_OK;
}
