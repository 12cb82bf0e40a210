// lidar_image.cu -- K5: vlcal::generate_lidar_image on the GPU (reference: src/vlcal/preprocess/generate_lidar_image.cpp:8-41).
//
// The reference renders a LiDAR intensity image and a point-index map with one serial pass: a point is projected with the
// same FoV / projection / truncation / bounds decisions as the NID cost (:21-28 == cost_calculator_nid.cpp:32-38) and
// replaces the pixel's current winner unless the stored squared range is strictly smaller (:31-37) -- i.e. per pixel the
// smallest squared range wins, and of several points with the same squared range the LAST one.  Both rules are order
// independent, so three kernels reproduce the images exactly:
//   1. exact projection (exact_classify.cuh), squared range in Eigen's order, atomicMin on the bit pattern of the
//      non-negative double per pixel;
//   2. points whose squared range equals their pixel's minimum: atomicMax of the point index;
//   3. per pixel: intensity of the winning point (0 / -1 where nothing landed, :13-15).
// Passes 1 and 2 take a radius: a point then competes for the (2r+1)^2 square of pixels around its own, clipped to the
// image.  The reference's image is radius 0; the viewer's overlay (viewer.cu) draws with a larger one through the same
// routine, lidar_index_image_passes.
#include <cstring>

#include "exact_classify.cuh"
#include "mem_pool.hpp"
#include "nid_context.cuh"

namespace vlcal {

struct LidarImageArgs {
  const void* points;  // float4 (x, y, z, intensity) or double4
  long long n;
  int width, height;
  int radius;  // a point covers pixels within `radius` of its own in x and y (0: the reference's rendering)
  double cos_fov;
  CameraParams cam;
  double pose[12];
  unsigned long long* zmin;  // [H*W] bit patterns of the smallest squared range, initialised to DBL_MAX (:13)
  int* pix;                  // [n] pixel of every point, -1 if the reference skips it
  double* sq_dist;           // [n]
  int* index_image;          // [H*W], initialised to -1 (:15)
};

// f(pixel) for every pixel of the square of `radius` around pixel `pix`, clipped to the image
template <class F>
__device__ __forceinline__ void for_each_covered_pixel(int pix, int radius, int width, int height, F f) {
  if (radius == 0) {
    f(pix);
    return;
  }
  const int iy = pix / width, ix = pix - iy * width;
  const int x0 = max(ix - radius, 0), x1 = min(ix + radius, width - 1);
  const int y0 = max(iy - radius, 0), y1 = min(iy + radius, height - 1);
  for (int y = y0; y <= y1; y++)
    for (int x = x0; x <= x1; x++) f(y * width + x);
}

template <int MODEL, bool F32>
__global__ void __launch_bounds__(256) lidar_image_project_kernel(const __grid_constant__ LidarImageArgs a) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  double x, y, z;
  if constexpr (F32) {
    const float4 q = __ldg(static_cast<const float4*>(a.points) + i);
    x = q.x, y = q.y, z = q.z;
  } else {
    const double4 q = static_cast<const double4*>(a.points)[i];
    x = q.x, y = q.y, z = q.z;
  }
  const int pix = exact_pixel_hd<MODEL>(a.cam, a.cos_fov, a.width, a.height, a.pose, x, y, z);  // :19-28
  a.pix[i] = pix;
  if (pix < 0) return;
  const double* T = a.pose;
  const xd X(x), Y(y), Z(z);
  const xd pcx = ((xd(T[0]) * X + xd(T[1]) * Y) + xd(T[2]) * Z) + xd(T[3]);
  const xd pcy = ((xd(T[4]) * X + xd(T[5]) * Y) + xd(T[6]) * Z) + xd(T[7]);
  const xd pcz = ((xd(T[8]) * X + xd(T[9]) * Y) + xd(T[10]) * Z) + xd(T[11]);
  const double sq = sqnorm3(pcx, pcy, pcz).v;  // :30 head<3>().squaredNorm()
  a.sq_dist[i] = sq;
  // :31 `stored < sq_dist` keeps the stored one: the minimum wins (non-negative doubles order like their bit patterns; a point
  // at +inf never beats the initial DBL_MAX, exactly as in the reference)
  const unsigned long long key = static_cast<unsigned long long>(__double_as_longlong(sq));
  for_each_covered_pixel(pix, a.radius, a.width, a.height, [&](int p) { atomicMin(a.zmin + p, key); });
}

__global__ void __launch_bounds__(256) lidar_image_winner_kernel(const __grid_constant__ LidarImageArgs a) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  const int pix = a.pix[i];
  if (pix < 0) return;
  const unsigned long long key = static_cast<unsigned long long>(__double_as_longlong(a.sq_dist[i]));
  for_each_covered_pixel(pix, a.radius, a.width, a.height, [&](int p) {
    if (key == a.zmin[p]) atomicMax(a.index_image + p, static_cast<int>(i));  // ties: the last point wins
  });
}

template <bool F32>
__global__ void __launch_bounds__(256) lidar_image_gather_kernel(const void* points, const int* index_image, double* intensity_image, size_t npix) {
  const size_t p = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p >= npix) return;
  const int idx = index_image[p];
  double v = 0.0;  // :14
  if (idx >= 0) {
    if constexpr (F32) v = static_cast<double>(static_cast<const float4*>(points)[idx].w);  // lossless by construction of the float4 layout
    else v = static_cast<const double4*>(points)[idx].w;
  }
  intensity_image[p] = v;  // :36
}

__global__ void lidar_image_init_kernel(unsigned long long* zmin, int* index_image, size_t npix) {
  const size_t p = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p < npix) {
    zmin[p] = 0x7fefffffffffffffull;  // DBL_MAX (:13)
    index_image[p] = -1;              // :15
  }
}

using ProjectKernel = void (*)(const LidarImageArgs);

template <int MODEL>
static ProjectKernel pick_project_layout(bool f32) {
  return f32 ? lidar_image_project_kernel<MODEL, true> : lidar_image_project_kernel<MODEL, false>;
}

static ProjectKernel pick_project(int model, bool f32) {
  switch (model) {
    case CAM_PLUMB_BOB: return pick_project_layout<CAM_PLUMB_BOB>(f32);
    case CAM_FISHEYE: return pick_project_layout<CAM_FISHEYE>(f32);
    case CAM_ATAN: return pick_project_layout<CAM_ATAN>(f32);
    case CAM_OMNIDIR: return pick_project_layout<CAM_OMNIDIR>(f32);
    case CAM_EQUIRECTANGULAR: return pick_project_layout<CAM_EQUIRECTANGULAR>(f32);
    case CAM_RATIONAL_POLYNOMIAL: return pick_project_layout<CAM_RATIONAL_POLYNOMIAL>(f32);
    default: return nullptr;
  }
}

namespace {
struct DevBuf {
  void* p = nullptr;
  int device = 0;
  cudaError_t alloc(int dev, size_t bytes) {
    device = dev;
    return MemPool::instance().device_alloc(dev, bytes, &p);
  }
  ~DevBuf() { MemPool::instance().device_free(device, p); }
};
}  // namespace

// Passes 1 and 2 for a cloud on the device, enqueued on the legacy stream: d_index_image [H*W] receives the winning point
// of every pixel (-1: none).  Scratch from the caller: zmin [H*W], pix and sq_dist [max(n, 1)].
int lidar_index_image_passes(
  const CameraParams& cam, int width, int height, const double T_camera_lidar[16], const DeviceCloud& cloud, int radius, unsigned long long* zmin, int* pix, double* sq_dist,
  int* d_index_image) {
  LidarImageArgs a;
  std::memset(&a, 0, sizeof(a));
  a.points = cloud.d_points;
  a.n = cloud.n;
  a.width = width, a.height = height;
  a.radius = radius;
  a.cos_fov = std::cos(estimate_camera_fov_host(cam, width, height));  // :10-11
  a.cam = cam;
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 4; c++) a.pose[4 * r + c] = T_camera_lidar[r + 4 * c];
  a.zmin = zmin;
  a.pix = pix;
  a.sq_dist = sq_dist;
  a.index_image = d_index_image;
  const size_t npix = static_cast<size_t>(width) * height;
  lidar_image_init_kernel<<<static_cast<unsigned int>((npix + 255) / 256), 256>>>(a.zmin, a.index_image, npix);
  VL_CUDA(cudaGetLastError());
  if (cloud.n > 0) {
    const unsigned int pt_blocks = static_cast<unsigned int>((cloud.n + 255) / 256);
    pick_project(cam.model, cloud.f32)<<<pt_blocks, 256>>>(a);
    VL_CUDA(cudaGetLastError());
    lidar_image_winner_kernel<<<pt_blocks, 256>>>(a);
    VL_CUDA(cudaGetLastError());
  }
  return VLCAL_OK;
}

}  // namespace vlcal

using namespace vlcal;

extern "C" int vlcal_generate_lidar_image(
  int device, int camera_model, const double* intrinsics, int n_intrinsics, const double* distortion, int n_distortion, int width, int height, const double T_camera_lidar[16],
  const double* points_xyzw, const double* intensities, int64_t n_points, double* intensity_image_out, int32_t* index_image_out) {
  if (width <= 0 || height <= 0 || n_points < 0 || n_points > 0x7fffffffLL || (n_points > 0 && (!points_xyzw || !intensities)) || !T_camera_lidar || !intensity_image_out || !index_image_out) {
    set_last_error("invalid arguments (at most 2^31-1 points: the index map is CV_32SC1)");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  // pixel indices are int (exact_pixel_hd returns iy * width + ix): refused before anything is uploaded or allocated
  if (static_cast<int64_t>(width) * height > 0x7fffffffLL) {
    set_last_error("invalid arguments (at most 2^31-1 pixels: width * height = " + std::to_string(static_cast<int64_t>(width) * height) + ")");
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
  std::shared_ptr<DeviceCloud> cloud;
  rc = upload_cloud(device, points_xyzw, intensities, n_points, nullptr, &cloud);
  if (rc != VLCAL_OK) return rc;
  const size_t npix = static_cast<size_t>(width) * height;
  DevBuf zmin, pix, sq, index, inten;
  VL_CUDA(zmin.alloc(device, sizeof(unsigned long long) * npix));
  VL_CUDA(index.alloc(device, sizeof(int) * npix));
  VL_CUDA(inten.alloc(device, sizeof(double) * npix));
  VL_CUDA(pix.alloc(device, sizeof(int) * std::max<int64_t>(1, n_points)));
  VL_CUDA(sq.alloc(device, sizeof(double) * std::max<int64_t>(1, n_points)));
  int* d_index = static_cast<int*>(index.p);
  double* d_inten = static_cast<double*>(inten.p);
  rc = lidar_index_image_passes(cam, width, height, T_camera_lidar, *cloud, 0, static_cast<unsigned long long*>(zmin.p), static_cast<int*>(pix.p), static_cast<double*>(sq.p), d_index);
  if (rc != VLCAL_OK) return rc;
  const unsigned int pix_blocks = static_cast<unsigned int>((npix + 255) / 256);
  if (cloud->f32) lidar_image_gather_kernel<true><<<pix_blocks, 256>>>(cloud->d_points, d_index, d_inten, npix);
  else lidar_image_gather_kernel<false><<<pix_blocks, 256>>>(cloud->d_points, d_index, d_inten, npix);
  VL_CUDA(cudaGetLastError());
  VL_CUDA(cudaMemcpy(intensity_image_out, d_inten, sizeof(double) * npix, cudaMemcpyDeviceToHost));
  VL_CUDA(cudaMemcpy(index_image_out, d_index, sizeof(int) * npix, cudaMemcpyDeviceToHost));
  return VLCAL_OK;
}
