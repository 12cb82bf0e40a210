// agreement.cu -- where in the image do the LiDAR and the camera disagree at a pose?  Per point, the pointwise mutual
// information of its joint bin in the NID histogram of that pose, splatted into the camera image.
//
//   agreement_hist_kernel     the reference's per-point decision (exact_pixel_hd, the arbiter of the persistent kernel's
//                             classifier, with calculate's FoV), the point's joint bin (image bin of the pixel, LiDAR bin of
//                             the intensity, cost_calculator_nid.cpp:43-49) and the joint histogram -- integer counts, so
//                             equal to calculate's histogram of the pose
//   agreement_pmi_kernel      log(p(a, b) / (p(a) p(b))) = log(c_ab * N / (c_a * c_b)) of every counted point from that
//                             histogram (NaN for a point the histogram does not count)
//   K5's z-buffer passes      the nearest point of every pixel (lidar_index_image_passes, the tie rule of
//                             generate_lidar_image, with a point radius)
//   agreement_compose_kernel  the winner's PMI as turbo(0.5 + PMI / (2 * VLCAL_AGREEMENT_PMI_RANGE)) blended over the
//                             camera image as the viewer's overlay blends its intensities (turbo_blend.cuh)
#include <cmath>
#include <cstring>

#include "exact_classify.cuh"
#include "nid_kernels.cuh"
#include "preprocess_common.cuh"
#include "turbo_blend.cuh"

namespace vlcal {

struct AgreementArgs {
  const void* points;  // float4 (x, y, z, intensity) or double4
  long long n;
  int width, height, bins;
  double cos_fov;
  CameraParams cam;
  double pose[12];
  const uint8_t* image;  // [H*W]
  int* jbin;             // [n] joint bin image_bin + lidar_bin * bins, -1: not counted
  int* hist;             // [bins * bins], zeroed
  double* pmi;           // [n]
  float* shade;          // [n] 0.5 + PMI / (2 * range), the colormap coordinate
  float w, one_minus_w;
  const int* index_image;  // [H*W]
  uint8_t* bgr;            // [H*W*3]
};

template <int MODEL, bool F32>
__global__ void __launch_bounds__(256) agreement_hist_kernel(const __grid_constant__ AgreementArgs a) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  double x, y, z, intensity;
  if constexpr (F32) {
    const float4 q = __ldg(static_cast<const float4*>(a.points) + i);
    x = q.x, y = q.y, z = q.z, intensity = q.w;
  } else {
    const double4 q = static_cast<const double4*>(a.points)[i];
    x = q.x, y = q.y, z = q.z, intensity = q.w;
  }
  const int pix = exact_pixel_hd<MODEL>(a.cam, a.cos_fov, a.width, a.height, a.pose, x, y, z);  // :31-38
  int j = -1;
  if (pix >= 0) {
    const double pixel = static_cast<double>(__ldg(a.image + pix)) / 255.0;  // :43
    int ib = cast_int_x86(pixel * a.bins);
    ib = ib < a.bins - 1 ? ib : a.bins - 1;
    ib = ib > 0 ? ib : 0;
    j = ib + lidar_bin_of(intensity, a.bins) * a.bins;  // :44-49
    atomicAdd(a.hist + j, 1);
  }
  a.jbin[i] = j;
}

__global__ void __launch_bounds__(256) agreement_pmi_kernel(const __grid_constant__ AgreementArgs a) {
  __shared__ int s_marg[2 * 32];  // image-bin marginal, then LiDAR-bin marginal (bins <= 32)
  __shared__ unsigned long long s_total;
  const int nb = a.bins * a.bins;
  if (threadIdx.x < 2 * a.bins) s_marg[threadIdx.x] = 0;
  if (threadIdx.x == 0) s_total = 0ull;
  __syncthreads();
  for (int k = threadIdx.x; k < nb; k += blockDim.x) {
    const int c = a.hist[k];
    if (c) {
      atomicAdd(&s_marg[k % a.bins], c);
      atomicAdd(&s_marg[a.bins + k / a.bins], c);
      atomicAdd(&s_total, static_cast<unsigned long long>(c));
    }
  }
  __syncthreads();
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  const int j = a.jbin[i];
  double v = NAN;
  if (j >= 0) {
    const double cab = a.hist[j], ca = s_marg[j % a.bins], cb = s_marg[a.bins + j / a.bins];
    v = log((cab * static_cast<double>(s_total)) / (ca * cb));  // every count < 2^31: the products are exact
  }
  a.pmi[i] = v;
  a.shade[i] = static_cast<float>(0.5 + v / (2.0 * VLCAL_AGREEMENT_PMI_RANGE));
}

__global__ void __launch_bounds__(256) agreement_compose_kernel(const __grid_constant__ AgreementArgs a) {
  const size_t p = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p >= static_cast<size_t>(a.width) * a.height) return;
  const int idx = a.index_image[p];
  const uint8_t pix = a.image[p];
  uint8_t b = pix, g = pix, r = pix;  // no point covers the pixel: the camera image
  if (idx >= 0) {
    const float4 c = blend_colors(pix, a.shade[idx], a.w, a.one_minus_w);
    b = to_byte(c.z), g = to_byte(c.y), r = to_byte(c.x);
  }
  a.bgr[3 * p] = b, a.bgr[3 * p + 1] = g, a.bgr[3 * p + 2] = r;
}

using AgreementKernel = void (*)(const AgreementArgs);

template <int MODEL>
static AgreementKernel pick_hist_layout(bool f32) {
  return f32 ? agreement_hist_kernel<MODEL, true> : agreement_hist_kernel<MODEL, false>;
}

static AgreementKernel pick_hist(int model, bool f32) {
  switch (model) {
    case CAM_PLUMB_BOB: return pick_hist_layout<CAM_PLUMB_BOB>(f32);
    case CAM_FISHEYE: return pick_hist_layout<CAM_FISHEYE>(f32);
    case CAM_ATAN: return pick_hist_layout<CAM_ATAN>(f32);
    case CAM_OMNIDIR: return pick_hist_layout<CAM_OMNIDIR>(f32);
    case CAM_EQUIRECTANGULAR: return pick_hist_layout<CAM_EQUIRECTANGULAR>(f32);
    case CAM_RATIONAL_POLYNOMIAL: return pick_hist_layout<CAM_RATIONAL_POLYNOMIAL>(f32);
    default: return nullptr;
  }
}

}  // namespace vlcal

using namespace vlcal;

extern "C" int vlcal_agreement_map(
  int device, int camera_model, const double* intrinsics, int n_intrinsics, const double* distortion, int n_distortion, int width, int height, const uint8_t* image, int row_stride,
  const double T_camera_lidar[16], const double* points_xyzw, const double* intensities, int64_t n_points, int bins, int point_radius, float blend_weight, double* pmi_out,
  int32_t* hist_out, uint8_t* bgr_out, int32_t* index_image_out) {
  if (width <= 0 || height <= 0 || !image || row_stride < width || n_points < 0 || n_points > 0x7fffffffLL || (n_points > 0 && (!points_xyzw || !intensities || !pmi_out)) ||
      !T_camera_lidar || !bgr_out || static_cast<int64_t>(width) * height > 0x7fffffffLL) {
    set_last_error("invalid arguments (at most 2^31-1 points and pixels; row_stride >= width; pmi_out and bgr_out required)");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  if (bins < 1 || bins > 32 || point_radius < 0 || point_radius > 8 || !(blend_weight >= 0.0f && blend_weight <= 1.0f)) {
    set_last_error("invalid arguments (bins in [1, 32], point_radius in [0, 8], blend_weight in [0, 1])");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  CameraParams cam;
  int rc = make_camera(camera_model, intrinsics, n_intrinsics, distortion, n_distortion, &cam);
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
  const size_t n = static_cast<size_t>(std::max<int64_t>(n_points, 1));
  Scratch scratch(device);
  AgreementArgs a;
  std::memset(&a, 0, sizeof(a));
  a.points = cloud->d_points;
  a.n = n_points;
  a.width = width, a.height = height, a.bins = bins;
  a.cos_fov = std::cos(estimate_camera_fov_host(cam, width, height));  // calculate's FoV (cost_calculator_nid.cpp:17,32)
  a.cam = cam;
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 4; c++) a.pose[4 * r + c] = T_camera_lidar[r + 4 * c];
  a.image = dimg->d_raw;
  a.w = blend_weight;
  a.one_minus_w = static_cast<float>(1.0 - static_cast<double>(blend_weight));
  unsigned long long* zmin;
  int *pix, *index;
  double* sq;
  VL_CUDA(scratch.alloc(n, &a.jbin));
  VL_CUDA(scratch.alloc(static_cast<size_t>(bins) * bins, &a.hist));
  VL_CUDA(scratch.alloc(n, &a.pmi));
  VL_CUDA(scratch.alloc(n, &a.shade));
  VL_CUDA(scratch.alloc(npix, &zmin));
  VL_CUDA(scratch.alloc(npix, &index));
  VL_CUDA(scratch.alloc(npix * 3, &a.bgr));
  VL_CUDA(scratch.alloc(n, &pix));
  VL_CUDA(scratch.alloc(n, &sq));
  a.index_image = index;
  VL_CUDA(cudaMemset(a.hist, 0, sizeof(int) * static_cast<size_t>(bins) * bins));
  if (n_points > 0) {
    pick_hist(cam.model, cloud->f32)<<<blocks_for(n_points, 256), 256>>>(a);
    agreement_pmi_kernel<<<blocks_for(n_points, 256), 256>>>(a);
    VL_CUDA(cudaGetLastError());
  }
  rc = lidar_index_image_passes(cam, width, height, T_camera_lidar, *cloud, point_radius, zmin, pix, sq, index);
  if (rc != VLCAL_OK) return rc;
  agreement_compose_kernel<<<blocks_for(static_cast<long long>(npix), 256), 256>>>(a);
  VL_CUDA(cudaGetLastError());
  if (n_points > 0) VL_CUDA(cudaMemcpy(pmi_out, a.pmi, sizeof(double) * static_cast<size_t>(n_points), cudaMemcpyDeviceToHost));
  if (hist_out) VL_CUDA(cudaMemcpy(hist_out, a.hist, sizeof(int) * static_cast<size_t>(bins) * bins, cudaMemcpyDeviceToHost));
  VL_CUDA(cudaMemcpy(bgr_out, a.bgr, npix * 3, cudaMemcpyDeviceToHost));
  if (index_image_out) VL_CUDA(cudaMemcpy(index_image_out, index, sizeof(int) * npix, cudaMemcpyDeviceToHost));
  return VLCAL_OK;
}
