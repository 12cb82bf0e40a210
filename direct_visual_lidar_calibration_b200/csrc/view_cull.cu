// view_cull.cu -- K4: GPU ViewCulling (reference: src/vlcal/calib/view_culling.cpp:21-92).
//
// The reference removes hidden points before every inner solve with two serial passes over the cloud:
//   pass 1 (:43-68)  FoV test on the homogeneous 4-vector (:45), projection + truncation + bounds (:50-54), then a
//                    per-pixel running minimum of float-rounded ranges in a CV_32F map (:59-67)
//   pass 2 (:70-89)  keep candidates whose range is within +0.1 m of their pixel's minimum (:81)
// The final depth map is the per-pixel MIN over float(range) (float rounding is monotone), i.e. order independent,
// so pass 1 is one kernel with atomicMin on the bit pattern of the non-negative floats, pass 2 a flag kernel, and
// the stable (ascending original index) output a block-scan compaction.  Geometry uses the exact double path.
#include <algorithm>
#include <cstring>

#include "mem_pool.hpp"
#include "nid_context.cuh"

namespace vlcal {

constexpr int CULL_THREADS = 256;

struct CullArgs {
  const void* points;
  long long n;
  int width, height;
  double min_z;  // cos(estimate_camera_fov)  (:17)
  CameraParams cam;
  double pose[12];
  unsigned int* zbuf;  // H x W float bit patterns, initialised to +inf
  int* pix;            // [n] iy*W+ix of candidates, -1 otherwise
  double* dist;        // [n] |pt_camera.head<3>()|
  int depth;
  int tiles_x;         // image tiles of 32 x 8 pixels (tile-ordered compaction)
  int n_tiles;
  int keep_all;        // reorder mode: nothing is dropped, points outside the view go to one extra bucket
};

template <bool F32>
__device__ __forceinline__ void load_point(const void* points, long long i, double& x, double& y, double& z) {
  if constexpr (F32) {
    const float4 q = __ldg(static_cast<const float4*>(points) + i);
    x = q.x, y = q.y, z = q.z;
  } else {
    const double4 q = static_cast<const double4*>(points)[i];
    x = q.x, y = q.y, z = q.z;
  }
}

template <int MODEL, bool F32>
__global__ void __launch_bounds__(CULL_THREADS) cull_project_kernel(const __grid_constant__ CullArgs a) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  double x, y, z;
  load_point<F32>(a.points, i, x, y, z);
  const double* T = a.pose;
  const xd X(x), Y(y), Z(z);
  // :25-28 points_camera[i] = T * points[i]  (w = 1)
  const xd pcx = ((xd(T[0]) * X + xd(T[1]) * Y) + xd(T[2]) * Z) + xd(T[3]);
  const xd pcy = ((xd(T[4]) * X + xd(T[5]) * Y) + xd(T[6]) * Z) + xd(T[7]);
  const xd pcz = ((xd(T[8]) * X + xd(T[9]) * Y) + xd(T[10]) * Z) + xd(T[11]);
  // :45 pt_camera.normalized().head<3>().z(): the 4-vector (x,y,z,1) is normalised, w included
  const xd n4 = (pcx * pcx + pcy * pcy) + (pcz * pcz + xd(1.0));
  const xd nz = n4 > xd(0.0) ? pcz / xsqrt(n4) : pcz;
  int pix = -1;
  if (!(nz < xd(a.min_z))) {
    xd u, v;
    project_exact<MODEL>(a.cam, pcx, pcy, pcz, u, v);  // :50
    const int ix = cast_int_x86(u.v);
    const int iy = cast_int_x86(v.v);
    if (!(ix < 0 || iy < 0 || ix >= a.width || iy >= a.height)) {  // :51-54
      pix = iy * a.width + ix;
      const xd d = xsqrt(sqnorm3(pcx, pcy, pcz));  // :60
      a.dist[i] = d.v;
      if (a.depth) {
        atomicMin(a.zbuf + pix, __float_as_uint(__double2float_rn(d.v)));  // :61-65
      }
    }
  }
  a.pix[i] = pix;
}

__device__ __forceinline__ bool cull_keep(const CullArgs& a, long long i) {
  if (i >= a.n) return false;
  if (a.keep_all) return true;
  const int pix = a.pix[i];
  if (pix < 0) return false;
  if (!a.depth) return true;
  const double cell = static_cast<double>(__uint_as_float(a.zbuf[pix]));
  return !(a.dist[i] > __dadd_rn(cell, 0.1));  // :81
}

// ---- tile-ordered compaction (internal cost objects only) -----------------------------------------------------
// The NID histogram is integer, hence invariant under any permutation of the cloud.  Kept points are therefore
// written grouped by the 32x8-pixel image tile they project to at the culling pose (counting sort: per-tile counts,
// scan, atomic cursors), so that the 32 lanes of a warp of the cost kernel gather their image bins from a handful
// of 32-byte sectors instead of 32 scattered ones.  The public vlcal_view_cull keeps the reference's ascending order.
__device__ __forceinline__ int cull_tile_of(const CullArgs& a, int pix) {
  if (pix < 0) return a.n_tiles - 1;  // keep_all: not in view at this pose
  const int iy = pix / a.width, ix = pix - iy * a.width;
  return (iy >> 3) * a.tiles_x + (ix >> 5);
}

__global__ void __launch_bounds__(CULL_THREADS) cull_tile_count_kernel(const __grid_constant__ CullArgs a, int* tile_counts) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (cull_keep(a, i)) atomicAdd(&tile_counts[cull_tile_of(a, a.pix[i])], 1);
}

template <bool F32>
__global__ void __launch_bounds__(CULL_THREADS) cull_tile_scatter_kernel(const __grid_constant__ CullArgs a, const int* tile_offsets, int* tile_cursor, void* points_out) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (!cull_keep(a, i)) return;
  const int tile = cull_tile_of(a, a.pix[i]);
  const int dst = tile_offsets[tile] + atomicAdd(&tile_cursor[tile], 1);
  if constexpr (F32) {
    static_cast<float4*>(points_out)[dst] = static_cast<const float4*>(a.points)[i];
  } else {
    static_cast<double4*>(points_out)[dst] = static_cast<const double4*>(a.points)[i];
  }
}

__global__ void __launch_bounds__(CULL_THREADS) cull_count_kernel(const __grid_constant__ CullArgs a, int* block_counts) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int c = __syncthreads_count(cull_keep(a, i) ? 1 : 0);
  if (threadIdx.x == 0) block_counts[blockIdx.x] = c;
}

// exclusive scan of block_counts (single block), total -> *total_out
__global__ void __launch_bounds__(1024) cull_scan_kernel(int* block_counts, int num_blocks, long long* total_out) {
  __shared__ long long warp_tot[32];
  __shared__ long long carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < num_blocks; base += blockDim.x) {
    const int idx = base + threadIdx.x;
    const long long v = idx < num_blocks ? block_counts[idx] : 0;
    long long incl = v;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      long long w = warp_tot[lane];
      long long wi = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const long long t = __shfl_up_sync(0xffffffffu, wi, o);
        if (lane >= o) wi += t;
      }
      warp_tot[lane] = wi - w;  // exclusive prefix of warp totals
    }
    __syncthreads();
    const long long excl = carry + warp_tot[warp] + (incl - v);
    if (idx < num_blocks) block_counts[idx] = static_cast<int>(excl);  // total kept < 2^31 (indices are int32)
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) carry = excl + v;
    __syncthreads();
  }
  if (threadIdx.x == 0) *total_out = carry;
}

template <bool F32>
__global__ void __launch_bounds__(CULL_THREADS) cull_scatter_kernel(const __grid_constant__ CullArgs a, const int* block_offsets, int* indices_out, void* points_out) {
  __shared__ int warp_cnt[CULL_THREADS / 32];
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const bool keep = cull_keep(a, i);
  const unsigned int ballot = __ballot_sync(0xffffffffu, keep);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) warp_cnt[warp] = __popc(ballot);
  __syncthreads();
  int offset = block_offsets[blockIdx.x];
  for (int w = 0; w < warp; w++) offset += warp_cnt[w];
  if (keep) {
    const int dst = offset + __popc(ballot & ((1u << lane) - 1u));
    if (indices_out) indices_out[dst] = static_cast<int>(i);  // ascending original index (:56, :85)
    if (points_out) {                                         // sample(): frame_cpu.cpp:281-331
      if constexpr (F32) {
        static_cast<float4*>(points_out)[dst] = static_cast<const float4*>(a.points)[i];
      } else {
        static_cast<double4*>(points_out)[dst] = static_cast<const double4*>(a.points)[i];
      }
    }
  }
}

__global__ void fill_u32_kernel(unsigned int* p, size_t n, unsigned int v) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

using CullProjectKernel = void (*)(const CullArgs);

template <int MODEL>
static CullProjectKernel pick_cull_layout(bool f32) {
  return f32 ? cull_project_kernel<MODEL, true> : cull_project_kernel<MODEL, false>;
}

static CullProjectKernel pick_cull_kernel(int model, bool f32) {
  switch (model) {
    case CAM_PLUMB_BOB: return pick_cull_layout<CAM_PLUMB_BOB>(f32);
    case CAM_FISHEYE: return pick_cull_layout<CAM_FISHEYE>(f32);
    case CAM_ATAN: return pick_cull_layout<CAM_ATAN>(f32);
    case CAM_OMNIDIR: return pick_cull_layout<CAM_OMNIDIR>(f32);
    case CAM_EQUIRECTANGULAR: return pick_cull_layout<CAM_EQUIRECTANGULAR>(f32);
    case CAM_RATIONAL_POLYNOMIAL: return pick_cull_layout<CAM_RATIONAL_POLYNOMIAL>(f32);
    default: return nullptr;
  }
}

struct DevBuf {  // pooled scratch; returned to the pool after the culling pass has synchronised its stream
  void* p = nullptr;
  int device = 0;
  cudaError_t alloc(int dev, size_t bytes) {
    device = dev;
    return MemPool::instance().device_alloc(dev, bytes, &p);
  }
  ~DevBuf() { MemPool::instance().device_free(device, p); }
};

int view_cull_device(
  const CameraParams& cam, int width, int height, double max_fov, bool depth_culling, const DeviceCloud& cloud, const double T[16], cudaStream_t stream,
  std::shared_ptr<DeviceCloud>* culled_out, int32_t* indices_host_out, int64_t* n_kept, bool keep_all) {
  VL_CUDA(cudaSetDevice(cloud.device));
  const long long n = cloud.n;
  if (n == 0) {
    if (culled_out) {
      auto c = std::make_shared<DeviceCloud>();
      c->device = cloud.device, c->f32 = cloud.f32, c->n = 0;
      *culled_out = c;
    }
    if (n_kept) *n_kept = 0;
    return VLCAL_OK;
  }
  if (n > 0x7fffffffLL) {
    set_last_error("view culling supports at most 2^31-1 points (int32 indices, as std::vector<int> in the reference)");
    return VLCAL_ERR_UNSUPPORTED;
  }
  const int num_blocks = static_cast<int>((n + CULL_THREADS - 1) / CULL_THREADS);
  const size_t npix = static_cast<size_t>(width) * height;
  DevBuf zbuf, pix, dist, counts, total, idx;
  VL_CUDA(zbuf.alloc(cloud.device, sizeof(unsigned int) * npix));
  VL_CUDA(pix.alloc(cloud.device, sizeof(int) * n));
  VL_CUDA(dist.alloc(cloud.device, sizeof(double) * n));
  VL_CUDA(total.alloc(cloud.device, sizeof(long long)));
  // :40 dist_map filled with cv::Scalar(DBL_MAX) -> saturates to +inf in CV_32F
  fill_u32_kernel<<<static_cast<unsigned int>((npix + 255) / 256), 256, 0, stream>>>(static_cast<unsigned int*>(zbuf.p), npix, 0x7f800000u);
  VL_CUDA(cudaGetLastError());

  CullArgs a;
  std::memset(&a, 0, sizeof(a));
  a.points = cloud.d_points;
  a.n = n;
  a.width = width;
  a.height = height;
  a.min_z = std::cos(max_fov);
  a.cam = cam;
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 4; c++) a.pose[4 * r + c] = T[r + 4 * c];
  a.zbuf = static_cast<unsigned int*>(zbuf.p);
  a.pix = static_cast<int*>(pix.p);
  a.dist = static_cast<double*>(dist.p);
  a.depth = (depth_culling && !keep_all) ? 1 : 0;
  a.keep_all = keep_all ? 1 : 0;

  CullProjectKernel project = pick_cull_kernel(cam.model, cloud.f32);
  project<<<num_blocks, CULL_THREADS, 0, stream>>>(a);
  VL_CUDA(cudaGetLastError());

  const bool by_tile = culled_out != nullptr && indices_host_out == nullptr;  // internal cost object: order is free
  DevBuf cursor;
  int num_counts = num_blocks;
  if (by_tile) {
    a.tiles_x = (width + 31) / 32;
    num_counts = a.tiles_x * ((height + 7) / 8) + 1;  // + the out-of-view bucket of keep_all
    a.n_tiles = num_counts;
    VL_CUDA(counts.alloc(cloud.device, sizeof(int) * num_counts));
    VL_CUDA(cursor.alloc(cloud.device, sizeof(int) * num_counts));
    VL_CUDA(cudaMemsetAsync(counts.p, 0, sizeof(int) * num_counts, stream));
    VL_CUDA(cudaMemsetAsync(cursor.p, 0, sizeof(int) * num_counts, stream));
    cull_tile_count_kernel<<<num_blocks, CULL_THREADS, 0, stream>>>(a, static_cast<int*>(counts.p));
  } else {
    VL_CUDA(counts.alloc(cloud.device, sizeof(int) * num_counts));
    cull_count_kernel<<<num_blocks, CULL_THREADS, 0, stream>>>(a, static_cast<int*>(counts.p));
  }
  VL_CUDA(cudaGetLastError());
  cull_scan_kernel<<<1, 1024, 0, stream>>>(static_cast<int*>(counts.p), num_counts, static_cast<long long*>(total.p));
  VL_CUDA(cudaGetLastError());
  long long kept = 0;
  VL_CUDA(cudaMemcpyAsync(&kept, total.p, sizeof(long long), cudaMemcpyDeviceToHost, stream));
  VL_CUDA(cudaStreamSynchronize(stream));

  std::shared_ptr<DeviceCloud> culled;
  if (culled_out) {
    culled = std::make_shared<DeviceCloud>();
    culled->device = cloud.device;
    culled->f32 = cloud.f32;
    culled->n = kept;
    if (kept > 0) VL_CUDA(MemPool::instance().device_alloc(cloud.device, static_cast<size_t>(kept) * culled->bytes_per_point(), &culled->d_points));
  }
  if (indices_host_out && kept > 0) VL_CUDA(idx.alloc(cloud.device, sizeof(int) * kept));
  if (kept > 0 && by_tile) {
    if (cloud.f32) {
      cull_tile_scatter_kernel<true><<<num_blocks, CULL_THREADS, 0, stream>>>(a, static_cast<int*>(counts.p), static_cast<int*>(cursor.p), culled->d_points);
    } else {
      cull_tile_scatter_kernel<false><<<num_blocks, CULL_THREADS, 0, stream>>>(a, static_cast<int*>(counts.p), static_cast<int*>(cursor.p), culled->d_points);
    }
    VL_CUDA(cudaGetLastError());
    VL_CUDA(cudaStreamSynchronize(stream));
  } else if (kept > 0 && (culled_out || indices_host_out)) {
    if (cloud.f32) {
      cull_scatter_kernel<true><<<num_blocks, CULL_THREADS, 0, stream>>>(a, static_cast<int*>(counts.p), static_cast<int*>(idx.p), culled ? culled->d_points : nullptr);
    } else {
      cull_scatter_kernel<false><<<num_blocks, CULL_THREADS, 0, stream>>>(a, static_cast<int*>(counts.p), static_cast<int*>(idx.p), culled ? culled->d_points : nullptr);
    }
    VL_CUDA(cudaGetLastError());
    if (indices_host_out) VL_CUDA(cudaMemcpyAsync(indices_host_out, idx.p, sizeof(int) * kept, cudaMemcpyDeviceToHost, stream));
    VL_CUDA(cudaStreamSynchronize(stream));
  }
  if (culled_out) *culled_out = culled;
  if (n_kept) *n_kept = kept;
  return VLCAL_OK;
}

}  // namespace vlcal

using namespace vlcal;

extern "C" int vlcal_view_cull(
  int device,
  int camera_model,
  const double* intrinsics,
  int n_intrinsics,
  const double* distortion,
  int n_distortion,
  int width,
  int height,
  double max_fov_rad,
  int enable_depth_buffer_culling,
  const double* points_xyzw,
  int64_t n_points,
  const double T_camera_lidar[16],
  int32_t* indices_out,
  int64_t* n_kept) {
  if (width <= 0 || height <= 0 || n_points < 0 || (n_points > 0 && (!points_xyzw || !indices_out)) || !T_camera_lidar || !n_kept) {
    set_last_error("invalid arguments");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  CameraParams cam;
  int rc = make_camera(camera_model, intrinsics, n_intrinsics, distortion, n_distortion, &cam);
  if (rc != VLCAL_OK) return rc;
  if (vlcal_nid_device_count() == 0) {
    set_last_error("no CUDA device available: this library has no CPU fallback");
    return VLCAL_ERR_NO_DEVICE;
  }
  if (device < 0) VL_CUDA(cudaGetDevice(&device));
  VL_CUDA(cudaSetDevice(device));
  if (max_fov_rad < 0.0) max_fov_rad = estimate_camera_fov_host(cam, width, height);
  // culling never reads intensities: upload zeros so that the float4 layout test only looks at x,y,z
  std::vector<double> zeros(static_cast<size_t>(n_points), 0.0);
  std::shared_ptr<DeviceCloud> cloud;
  rc = upload_cloud(device, points_xyzw, zeros.data(), n_points, nullptr, &cloud);
  if (rc != VLCAL_OK) return rc;
  return view_cull_device(cam, width, height, max_fov_rad, enable_depth_buffer_culling != 0, *cloud, T_camera_lidar, nullptr, nullptr, indices_out, n_kept, false);
}

extern "C" int vlcal_debug_view_cull_points(
  int device,
  int camera_model,
  const double* intrinsics,
  int n_intrinsics,
  const double* distortion,
  int n_distortion,
  int width,
  int height,
  double max_fov_rad,
  int enable_depth_buffer_culling,
  int keep_all,
  const double* points_xyzw,
  const double* intensities,
  int64_t n_points,
  const double T_camera_lidar[16],
  double* points_out,
  int64_t* n_kept,
  int* points_are_f32) {
  if (width <= 0 || height <= 0 || n_points < 0 || (n_points > 0 && (!points_xyzw || !intensities || !points_out)) || !T_camera_lidar || !n_kept) {
    set_last_error("invalid arguments");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  CameraParams cam;
  int rc = make_camera(camera_model, intrinsics, n_intrinsics, distortion, n_distortion, &cam);
  if (rc != VLCAL_OK) return rc;
  if (vlcal_nid_device_count() == 0) {
    set_last_error("no CUDA device available: this library has no CPU fallback");
    return VLCAL_ERR_NO_DEVICE;
  }
  if (device < 0) VL_CUDA(cudaGetDevice(&device));
  VL_CUDA(cudaSetDevice(device));
  if (max_fov_rad < 0.0) max_fov_rad = estimate_camera_fov_host(cam, width, height);
  std::shared_ptr<DeviceCloud> cloud, culled;
  rc = upload_cloud(device, points_xyzw, intensities, n_points, nullptr, &cloud);
  if (rc != VLCAL_OK) return rc;
  if (points_are_f32) *points_are_f32 = cloud->f32 ? 1 : 0;
  // culled_out without an index list: the paths of the cost objects (tile-ordered counting sort, or the keep_all reorder)
  rc = view_cull_device(cam, width, height, max_fov_rad, enable_depth_buffer_culling != 0, *cloud, T_camera_lidar, nullptr, &culled, nullptr, n_kept, keep_all != 0);
  if (rc != VLCAL_OK) return rc;
  const size_t kept = static_cast<size_t>(culled->n);
  if (kept == 0) return VLCAL_OK;
  if (culled->f32) {
    std::vector<float4> h(kept);
    VL_CUDA(cudaMemcpy(h.data(), culled->d_points, sizeof(float4) * kept, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < kept; i++) {
      points_out[4 * i] = h[i].x, points_out[4 * i + 1] = h[i].y, points_out[4 * i + 2] = h[i].z, points_out[4 * i + 3] = h[i].w;
    }
  } else {
    VL_CUDA(cudaMemcpy(points_out, culled->d_points, sizeof(double4) * kept, cudaMemcpyDeviceToHost));
  }
  return VLCAL_OK;
}
