// viewer.cu -- the headless viewer's kernels: the reference's only validation is looking at the cloud coloured with the
// camera image through the estimated pose (src/viewer.cpp, src/vlcal/common/points_color_updater.cpp:37-61).
//
//   colorize_points_kernel  PointsColorUpdater::update: per point the exact projection of the cost (exact_classify.cuh)
//                           with the viewer's own, looser FoV threshold (:27,43), the uint8 pixel under it, and
//                           gray * w + turbo(intensity) * (1 - w) as float32 RGBA (:54-57); a skipped point keeps (0, 0, 0, 0) (:38).
//   overlay_compose_kernel  the cloud drawn into the camera image: per pixel the winner of generate_lidar_image's z-buffer
//                           passes (lidar_index_image_passes, with a point radius) coloured the same way, uint8 BGR.
//
// Arithmetic of the blend, as Eigen evaluates `color * blend_weight + intensity_colors[i] * (1.0 - blend_weight)` on
// Vector4f with a double blend_weight: a scalar factor is cast to the vector's scalar type, so w = float(blend_weight),
// 1 - w is formed in double and then rounded to float, and every product and sum is a float32 operation of its own.
// The kernels therefore use __fmul_rn / __fadd_rn / __fdiv_rn (never contracted into FMAs).
//
// turbo(x) stands in for glk::colormapf(TURBO, x) (Iridescence, not part of the reference's sources): entry
// clamp(int(float(x) * 255.0), 0, 255) of the published 256-entry table (turbo_colormap.hpp), NaN -> entry 0, each
// channel / 255.0f, alpha 1.
#include <cmath>
#include <cstring>

#include "exact_classify.cuh"
#include "preprocess_common.cuh"
#include "turbo_blend.cuh"
#include "turbo_colormap.hpp"

namespace vlcal {

static const unsigned char h_turbo_rgb[768] = {VLCAL_TURBO_RGB_BYTES};

struct ViewerArgs {
  const void* points;  // float4 (x, y, z, intensity) or double4
  long long n;
  int width, height;
  double cos_fov;
  CameraParams cam;
  double pose[12];
  const uint8_t* image;  // [H*W]
  float w, one_minus_w;
  float4* rgba;            // colourise: [n]
  const int* index_image;  // compose: [H*W]
  uint8_t* bgr;            // compose: [H*W*3]
};

template <int MODEL, bool F32>
__global__ void __launch_bounds__(256) colorize_points_kernel(const __grid_constant__ ViewerArgs a) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  double x, y, z;
  float intensity;
  if constexpr (F32) {
    const float4 q = __ldg(static_cast<const float4*>(a.points) + i);
    x = q.x, y = q.y, z = q.z, intensity = q.w;
  } else {
    const double4 q = static_cast<const double4*>(a.points)[i];
    x = q.x, y = q.y, z = q.z, intensity = __double2float_rn(q.w);
  }
  const int pix = exact_pixel_hd<MODEL>(a.cam, a.cos_fov, a.width, a.height, a.pose, x, y, z);  // :41-52
  a.rgba[i] = pix < 0 ? make_float4(0.0f, 0.0f, 0.0f, 0.0f) : blend_colors(__ldg(a.image + pix), intensity, a.w, a.one_minus_w);
}

template <bool F32>
__global__ void __launch_bounds__(256) overlay_compose_kernel(const __grid_constant__ ViewerArgs a) {
  const size_t p = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p >= static_cast<size_t>(a.width) * a.height) return;
  const int idx = a.index_image[p];
  const uint8_t pix = a.image[p];
  uint8_t b = pix, g = pix, r = pix;  // no point covers the pixel: the camera image
  if (idx >= 0) {
    float intensity;
    if constexpr (F32) intensity = static_cast<const float4*>(a.points)[idx].w;
    else intensity = __double2float_rn(static_cast<const double4*>(a.points)[idx].w);
    const float4 c = blend_colors(pix, intensity, a.w, a.one_minus_w);
    b = to_byte(c.z), g = to_byte(c.y), r = to_byte(c.x);
  }
  a.bgr[3 * p] = b, a.bgr[3 * p + 1] = g, a.bgr[3 * p + 2] = r;
}

using ViewerKernel = void (*)(const ViewerArgs);

template <int MODEL>
static ViewerKernel pick_colorize_layout(bool f32) {
  return f32 ? colorize_points_kernel<MODEL, true> : colorize_points_kernel<MODEL, false>;
}

static ViewerKernel pick_colorize(int model, bool f32) {
  switch (model) {
    case CAM_PLUMB_BOB: return pick_colorize_layout<CAM_PLUMB_BOB>(f32);
    case CAM_FISHEYE: return pick_colorize_layout<CAM_FISHEYE>(f32);
    case CAM_ATAN: return pick_colorize_layout<CAM_ATAN>(f32);
    case CAM_OMNIDIR: return pick_colorize_layout<CAM_OMNIDIR>(f32);
    case CAM_EQUIRECTANGULAR: return pick_colorize_layout<CAM_EQUIRECTANGULAR>(f32);
    case CAM_RATIONAL_POLYNOMIAL: return pick_colorize_layout<CAM_RATIONAL_POLYNOMIAL>(f32);
    default: return nullptr;
  }
}

namespace {

// argument rules shared by the two entry points (those of vlcal_generate_lidar_image, plus the image and the weight)
int check_viewer_args(int width, int height, const uint8_t* image, int row_stride, const double* T, const double* points_xyzw, const double* intensities, int64_t n_points, float blend_weight) {
  if (width <= 0 || height <= 0 || !image || row_stride < width || n_points < 0 || n_points > 0x7fffffffLL || (n_points > 0 && (!points_xyzw || !intensities)) || !T) {
    set_last_error("invalid arguments (at most 2^31-1 points; row_stride >= width)");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  if (static_cast<int64_t>(width) * height > 0x7fffffffLL) {
    set_last_error("invalid arguments (at most 2^31-1 pixels: width * height = " + std::to_string(static_cast<int64_t>(width) * height) + ")");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  if (!(blend_weight >= 0.0f && blend_weight <= 1.0f)) {
    set_last_error("invalid arguments (blend_weight must be in [0, 1])");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  return VLCAL_OK;
}

void fill_viewer_args(ViewerArgs* a, const CameraParams& cam, int width, int height, const double T[16], const DeviceCloud& cloud, const DeviceImage& image, float blend_weight) {
  std::memset(a, 0, sizeof(*a));
  a->points = cloud.d_points;
  a->n = cloud.n;
  a->width = width, a->height = height;
  a->cam = cam;
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 4; c++) a->pose[4 * r + c] = T[r + 4 * c];
  a->image = image.d_raw;
  a->w = blend_weight;
  a->one_minus_w = static_cast<float>(1.0 - static_cast<double>(blend_weight));  // :57
}

}  // namespace
}  // namespace vlcal

using namespace vlcal;

extern "C" int vlcal_turbo_colormap(uint8_t rgb_out[768]) {
  if (!rgb_out) {
    set_last_error("invalid arguments");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  std::memcpy(rgb_out, h_turbo_rgb, sizeof(h_turbo_rgb));
  return VLCAL_OK;
}

extern "C" int vlcal_colorize_points(
  int device, int camera_model, const double* intrinsics, int n_intrinsics, const double* distortion, int n_distortion, int width, int height, const uint8_t* image, int row_stride,
  const double T_camera_lidar[16], const double* points_xyzw, const double* intensities, int64_t n_points, float blend_weight, float* rgba_out, double* kernel_ms_out) {
  if (kernel_ms_out) *kernel_ms_out = 0.0;
  int rc = check_viewer_args(width, height, image, row_stride, T_camera_lidar, points_xyzw, intensities, n_points, blend_weight);
  if (rc != VLCAL_OK) return rc;
  if (n_points > 0 && !rgba_out) {
    set_last_error("invalid arguments (rgba_out is NULL)");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  CameraParams cam;
  rc = make_camera(camera_model, intrinsics, n_intrinsics, distortion, n_distortion, &cam);
  if (rc != VLCAL_OK) return rc;
  rc = prepare_device(&device);
  if (rc != VLCAL_OK || n_points == 0) return rc;
  std::shared_ptr<DeviceCloud> cloud;
  rc = upload_cloud(device, points_xyzw, intensities, n_points, nullptr, &cloud);
  if (rc != VLCAL_OK) return rc;
  std::shared_ptr<DeviceImage> dimg;
  rc = upload_image(device, image, width, height, row_stride, nullptr, &dimg);
  if (rc != VLCAL_OK) return rc;
  Scratch scratch(device);
  ViewerArgs a;
  fill_viewer_args(&a, cam, width, height, T_camera_lidar, *cloud, *dimg, blend_weight);
  a.cos_fov = std::cos(estimate_camera_fov_host(cam, width, height) + 0.5 * M_PI / 180.0);  // min_nz (:27)
  VL_CUDA(scratch.alloc(static_cast<size_t>(n_points), &a.rgba));
  StageTimer timer(kernel_ms_out != nullptr);
  VL_CUDA(timer.mark());
  pick_colorize(cam.model, cloud->f32)<<<blocks_for(n_points, 256), 256>>>(a);
  VL_CUDA(cudaGetLastError());
  VL_CUDA(timer.mark());
  VL_CUDA(cudaMemcpy(rgba_out, a.rgba, sizeof(float4) * static_cast<size_t>(n_points), cudaMemcpyDeviceToHost));
  VL_CUDA(timer.read(kernel_ms_out, 1));
  return VLCAL_OK;
}

extern "C" int vlcal_render_overlay(
  int device, int camera_model, const double* intrinsics, int n_intrinsics, const double* distortion, int n_distortion, int width, int height, const uint8_t* image, int row_stride,
  const double T_camera_lidar[16], const double* points_xyzw, const double* intensities, int64_t n_points, int point_radius, float blend_weight, uint8_t* bgr_out,
  int32_t* index_image_out, double* kernel_ms_out) {
  if (kernel_ms_out) *kernel_ms_out = 0.0;
  int rc = check_viewer_args(width, height, image, row_stride, T_camera_lidar, points_xyzw, intensities, n_points, blend_weight);
  if (rc != VLCAL_OK) return rc;
  if (!bgr_out || point_radius < 0 || point_radius > 8) {
    set_last_error("invalid arguments (bgr_out is NULL or point_radius outside [0, 8])");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  CameraParams cam;
  rc = make_camera(camera_model, intrinsics, n_intrinsics, distortion, n_distortion, &cam);
  if (rc != VLCAL_OK) return rc;
  rc = prepare_device(&device);
  if (rc != VLCAL_OK) return rc;
  std::shared_ptr<DeviceCloud> cloud;
  rc = upload_cloud(device, points_xyzw, intensities, n_points, nullptr, &cloud);
  if (rc != VLCAL_OK) return rc;
  std::shared_ptr<DeviceImage> dimg;
  rc = upload_image(device, image, width, height, row_stride, nullptr, &dimg);
  if (rc != VLCAL_OK) return rc;
  const size_t npix = static_cast<size_t>(width) * height;
  Scratch scratch(device);
  unsigned long long* zmin;
  int *pix, *index;
  double* sq;
  ViewerArgs a;
  fill_viewer_args(&a, cam, width, height, T_camera_lidar, *cloud, *dimg, blend_weight);
  VL_CUDA(scratch.alloc(npix, &zmin));
  VL_CUDA(scratch.alloc(npix, &index));
  VL_CUDA(scratch.alloc(npix * 3, &a.bgr));
  VL_CUDA(scratch.alloc(static_cast<size_t>(n_points), &pix));
  VL_CUDA(scratch.alloc(static_cast<size_t>(n_points), &sq));
  a.index_image = index;
  StageTimer timer(kernel_ms_out != nullptr);
  VL_CUDA(timer.mark());
  rc = lidar_index_image_passes(cam, width, height, T_camera_lidar, *cloud, point_radius, zmin, pix, sq, index);
  if (rc != VLCAL_OK) return rc;
  if (cloud->f32) overlay_compose_kernel<true><<<blocks_for(static_cast<long long>(npix), 256), 256>>>(a);
  else overlay_compose_kernel<false><<<blocks_for(static_cast<long long>(npix), 256), 256>>>(a);
  VL_CUDA(cudaGetLastError());
  VL_CUDA(timer.mark());
  VL_CUDA(cudaMemcpy(bgr_out, a.bgr, npix * 3, cudaMemcpyDeviceToHost));
  if (index_image_out) VL_CUDA(cudaMemcpy(index_image_out, index, sizeof(int) * npix, cudaMemcpyDeviceToHost));
  VL_CUDA(timer.read(kernel_ms_out, 1));
  return VLCAL_OK;
}
