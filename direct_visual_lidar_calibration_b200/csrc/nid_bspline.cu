// nid_bspline.cu -- host side of mode B: vlcal_nid_evaluate_bspline (reference: NIDCost::operator()<double>,
// include/vlcal/costs/nid_cost.hpp:36-107; constructed per bag at visual_camera_calibration.cpp:203-206).
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>

#include "mem_pool.hpp"
#include "nid_bspline_kernels.cuh"
#include "nid_context.cuh"

namespace vlcal {

using NidBKernel = void (*)(const NidBArgs);

template <int MODEL>
static NidBKernel pick_b_layout(bool f32) {
  return f32 ? nid_bspline_kernel<MODEL, true> : nid_bspline_kernel<MODEL, false>;
}

static NidBKernel pick_b_kernel(int model, bool f32) {
  switch (model) {
    case CAM_PLUMB_BOB: return pick_b_layout<CAM_PLUMB_BOB>(f32);
    case CAM_FISHEYE: return pick_b_layout<CAM_FISHEYE>(f32);
    case CAM_ATAN: return pick_b_layout<CAM_ATAN>(f32);
    case CAM_OMNIDIR: return pick_b_layout<CAM_OMNIDIR>(f32);
    case CAM_EQUIRECTANGULAR: return pick_b_layout<CAM_EQUIRECTANGULAR>(f32);
    case CAM_RATIONAL_POLYNOMIAL: return pick_b_layout<CAM_RATIONAL_POLYNOMIAL>(f32);
    default: return nullptr;
  }
}

using NidGKernel = void (*)(const NidGArgs);

template <int MODEL>
static NidGKernel pick_g_layout(bool f32) {
  return f32 ? nid_bspline_grad_kernel<MODEL, true> : nid_bspline_grad_kernel<MODEL, false>;
}

static NidGKernel pick_g_kernel(int model, bool f32) {
  switch (model) {
    case CAM_PLUMB_BOB: return pick_g_layout<CAM_PLUMB_BOB>(f32);
    case CAM_FISHEYE: return pick_g_layout<CAM_FISHEYE>(f32);
    case CAM_ATAN: return pick_g_layout<CAM_ATAN>(f32);
    case CAM_OMNIDIR: return pick_g_layout<CAM_OMNIDIR>(f32);
    case CAM_EQUIRECTANGULAR: return pick_g_layout<CAM_EQUIRECTANGULAR>(f32);
    case CAM_RATIONAL_POLYNOMIAL: return pick_g_layout<CAM_RATIONAL_POLYNOMIAL>(f32);
    default: return nullptr;
  }
}

// hist_points and the inlier total are int counters (as in mode A)
static int check_bspline_cloud(const vlcal_nid_ctx* ctx) {
  if (ctx->cloud->n > INT_MAX) {
    set_last_error("mode B counts inliers in 32-bit integers: clouds are limited to 2^31 - 1 points");
    return VLCAL_ERR_UNSUPPORTED;
  }
  return VLCAL_OK;
}

struct PoolBuf {
  void* p = nullptr;
  int device = 0;
  cudaError_t alloc(int dev, size_t bytes) {
    device = dev;
    return MemPool::instance().device_alloc(dev, bytes, &p);
  }
  ~PoolBuf() { MemPool::instance().device_free(device, p); }
};

// synchronises the stream when it goes out of scope (normal returns have already synchronised: this is free there)
struct StreamGuard {
  cudaStream_t stream;
  ~StreamGuard() {
    if (cudaStreamQuery(stream) == cudaErrorNotReady) cudaStreamSynchronize(stream);
    cudaGetLastError();
  }
};

}  // namespace vlcal

using namespace vlcal;

extern "C" int vlcal_nid_evaluate_bspline(vlcal_nid_ctx* ctx, const double* T_params, int n_poses, double* nid_out, int32_t* ok_out, double* hist_out) {
  if (!ctx || !T_params || n_poses <= 0 || !nid_out) {
    set_last_error("invalid arguments");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  if (ctx->mode != VLCAL_NID_MODE_BSPLINE) {
    set_last_error("context was created in histogram mode; create it with VLCAL_NID_MODE_BSPLINE");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  VL_CUDA(cudaSetDevice(ctx->device));
  if (const int rc = check_bspline_cloud(ctx); rc != VLCAL_OK) return rc;
  const int bins = ctx->bins, nb = bins * bins;
  const int fixed_bits = nidb_fixed_bits(ctx->cloud->n);
  {  // one pose's joint histogram (8 B per bin) + marginal must fit the shared memory K2 opts into
    constexpr size_t SMEM_OPT_IN_CHECK = 100 * 1024;
    if (static_cast<size_t>(nb) * 8 + static_cast<size_t>(bins) * 4 + 64 > SMEM_OPT_IN_CHECK) {
      set_last_error("bins too large for the mode-B kernel's shared-memory histogram (bins <= 112)");
      return VLCAL_ERR_UNSUPPORTED;
    }
  }
  PoolBuf gjoint, gpoints, counter, d_nid, d_ok, d_hist;
  StreamGuard guard{ctx->stream};  // declared last = destroyed first: no scratch goes back to the pool while launches may still run
  VL_CUDA(gjoint.alloc(ctx->device, sizeof(unsigned long long) * NIDB_MAX_POSES * nb));
  VL_CUDA(gpoints.alloc(ctx->device, sizeof(int) * NIDB_MAX_POSES * bins));
  VL_CUDA(counter.alloc(ctx->device, sizeof(unsigned int)));
  VL_CUDA(d_nid.alloc(ctx->device, sizeof(double) * n_poses));
  VL_CUDA(d_ok.alloc(ctx->device, sizeof(int) * n_poses));
  if (hist_out) VL_CUDA(d_hist.alloc(ctx->device, sizeof(double) * static_cast<size_t>(n_poses) * nb));
  VL_CUDA(cudaMemsetAsync(gjoint.p, 0, sizeof(unsigned long long) * NIDB_MAX_POSES * nb, ctx->stream));
  VL_CUDA(cudaMemsetAsync(gpoints.p, 0, sizeof(int) * NIDB_MAX_POSES * bins, ctx->stream));
  VL_CUDA(cudaMemsetAsync(counter.p, 0, sizeof(unsigned int), ctx->stream));

  NidBKernel kernel = pick_b_kernel(ctx->cam.model, ctx->cloud->f32);
  constexpr size_t SMEM_OPT_IN = 100 * 1024;
  VL_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(SMEM_OPT_IN)));
  const int max_poses = std::max(1, std::min<int>(NIDB_MAX_POSES, static_cast<int>((SMEM_OPT_IN - 20 * 1024) / (static_cast<size_t>(nb) * 8 + bins * 4))));
  static const double C6[4][4] = {{1.0, -3.0, 3.0, -1.0}, {4.0, 0.0, -6.0, 3.0}, {1.0, 3.0, 3.0, -3.0}, {0.0, 0.0, 0.0, 1.0}};  // nid_cost.hpp:29-32

  for (int p0 = 0; p0 < n_poses; p0 += max_poses) {
    const int pc = std::min(max_poses, n_poses - p0);
    NidBArgs a;
    std::memset(&a, 0, sizeof(a));
    a.points = ctx->cloud->d_points;
    a.bin_image = ctx->d_bin_image;
    a.n = ctx->cloud->n;
    a.width = ctx->image->width;
    a.height = ctx->image->height;
    a.bins = bins;
    a.nb = nb;
    a.n_poses = pc;
    a.cam = ctx->cam;
    for (int p = 0; p < pc; p++) std::memcpy(a.pose[p], T_params + 7 * static_cast<size_t>(p0 + p), 7 * sizeof(double));
    for (int i = 0; i < 4; i++)
      for (int j = 0; j < 4; j++) a.C[i][j] = C6[i][j] / 6.0;  // :33 spline_coeffs /= 6.0
    a.fixed_one = std::ldexp(1.0, fixed_bits);
    a.inv_one = std::ldexp(1.0, -fixed_bits);
    a.gjoint = static_cast<unsigned long long*>(gjoint.p);
    a.gpoints = static_cast<int*>(gpoints.p);
    a.counter = static_cast<unsigned int*>(counter.p);
    a.nid_out = static_cast<double*>(d_nid.p) + p0;
    a.ok_out = static_cast<int*>(d_ok.p) + p0;
    a.hist_out = hist_out ? static_cast<double*>(d_hist.p) + static_cast<size_t>(p0) * nb : nullptr;
    const size_t per_copy = static_cast<size_t>(pc) * nb * 8;
    a.copies = static_cast<int>(std::max<size_t>(1, std::min<size_t>(NIDB_THREADS / 32, (64 * 1024) / per_copy)));
    // joint copies + hist_points, and never less than the finalize scratch (8 warps x bins x 8 B)
    const size_t smem = std::max<size_t>(per_copy * a.copies + static_cast<size_t>(pc) * bins * 4, static_cast<size_t>(8) * bins * 8 + 64);
    int blocks_per_sm = 1;
    VL_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, kernel, NIDB_THREADS, smem));
    const long long want = (a.n + NIDB_THREADS - 1) / NIDB_THREADS;
    const int grid = static_cast<int>(std::max<long long>(1, std::min<long long>(want, static_cast<long long>(ctx->num_sms) * std::max(1, blocks_per_sm))));
    kernel<<<grid, NIDB_THREADS, smem, ctx->stream>>>(a);
    VL_CUDA(cudaGetLastError());
    ctx->launches++;
    ctx->poses_total += pc;
  }
  VL_CUDA(cudaMemcpyAsync(nid_out, d_nid.p, sizeof(double) * n_poses, cudaMemcpyDeviceToHost, ctx->stream));
  std::vector<int> ok_host(n_poses);
  VL_CUDA(cudaMemcpyAsync(ok_host.data(), d_ok.p, sizeof(int) * n_poses, cudaMemcpyDeviceToHost, ctx->stream));
  if (hist_out) VL_CUDA(cudaMemcpyAsync(hist_out, d_hist.p, sizeof(double) * static_cast<size_t>(n_poses) * nb, cudaMemcpyDeviceToHost, ctx->stream));
  VL_CUDA(cudaStreamSynchronize(ctx->stream));
  if (ok_out)
    for (int p = 0; p < n_poses; p++) ok_out[p] = ok_host[p];
  return VLCAL_OK;
}

// value + gradient of the mode-B cost (NIDCost::operator()<ceres::Jet<double, 7>>), one launch per pose
extern "C" int vlcal_nid_evaluate_bspline_grad(vlcal_nid_ctx* ctx, const double* T_params, int n_poses, double* nid_out, double* grad_out, int32_t* ok_out) {
  if (!ctx || !T_params || n_poses <= 0 || !nid_out || !grad_out) {
    set_last_error("invalid arguments");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  if (ctx->mode != VLCAL_NID_MODE_BSPLINE) {
    set_last_error("context was created in histogram mode; create it with VLCAL_NID_MODE_BSPLINE");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  VL_CUDA(cudaSetDevice(ctx->device));
  if (const int rc = check_bspline_cloud(ctx); rc != VLCAL_OK) return rc;
  const int bins = ctx->bins, nb = bins * bins;
  const int fixed_bits = nidb_fixed_bits(ctx->cloud->n);
  const size_t smem = static_cast<size_t>(nb) * 8 * 8 + static_cast<size_t>(bins) * 4 + 16;
  if (smem > 200 * 1024) {
    set_last_error("bins too large for the gradient kernel's shared-memory histogram (bins <= 56)");
    return VLCAL_ERR_UNSUPPORTED;
  }
  PoolBuf gjoint, gpart, gpoints, counter, d_out;
  StreamGuard guard{ctx->stream};
  VL_CUDA(gjoint.alloc(ctx->device, sizeof(unsigned long long) * nb));
  VL_CUDA(gpart.alloc(ctx->device, sizeof(double) * nb * 7));
  VL_CUDA(gpoints.alloc(ctx->device, sizeof(int) * bins));
  VL_CUDA(counter.alloc(ctx->device, sizeof(unsigned int)));
  VL_CUDA(d_out.alloc(ctx->device, sizeof(double) * 9 * n_poses));
  VL_CUDA(cudaMemsetAsync(gjoint.p, 0, sizeof(unsigned long long) * nb, ctx->stream));
  VL_CUDA(cudaMemsetAsync(gpart.p, 0, sizeof(double) * nb * 7, ctx->stream));
  VL_CUDA(cudaMemsetAsync(gpoints.p, 0, sizeof(int) * bins, ctx->stream));
  VL_CUDA(cudaMemsetAsync(counter.p, 0, sizeof(unsigned int), ctx->stream));

  NidGKernel kernel = pick_g_kernel(ctx->cam.model, ctx->cloud->f32);
  VL_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  int blocks_per_sm = 1;
  VL_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, kernel, NIDG_THREADS, smem));
  const long long want = (ctx->cloud->n + NIDG_THREADS - 1) / NIDG_THREADS;
  const int grid = static_cast<int>(std::max<long long>(1, std::min<long long>(want, static_cast<long long>(ctx->num_sms) * std::max(1, blocks_per_sm))));
  static const double C6[4][4] = {{1.0, -3.0, 3.0, -1.0}, {4.0, 0.0, -6.0, 3.0}, {1.0, 3.0, 3.0, -3.0}, {0.0, 0.0, 0.0, 1.0}};  // nid_cost.hpp:29-32
  for (int p = 0; p < n_poses; p++) {
    NidGArgs a;
    std::memset(&a, 0, sizeof(a));
    a.points = ctx->cloud->d_points;
    a.bin_image = ctx->d_bin_image;
    a.n = ctx->cloud->n;
    a.width = ctx->image->width;
    a.height = ctx->image->height;
    a.bins = bins;
    a.nb = nb;
    a.cam = ctx->cam;
    std::memcpy(a.pose, T_params + 7 * static_cast<size_t>(p), 7 * sizeof(double));
    for (int i = 0; i < 4; i++)
      for (int j = 0; j < 4; j++) a.C[i][j] = C6[i][j] / 6.0;
    a.fixed_one = std::ldexp(1.0, fixed_bits);
    a.inv_one = std::ldexp(1.0, -fixed_bits);
    a.gjoint = static_cast<unsigned long long*>(gjoint.p);
    a.gpart = static_cast<double*>(gpart.p);
    a.gpoints = static_cast<int*>(gpoints.p);
    a.counter = static_cast<unsigned int*>(counter.p);
    a.out = static_cast<double*>(d_out.p) + 9 * static_cast<size_t>(p);
    kernel<<<grid, NIDG_THREADS, smem, ctx->stream>>>(a);
    VL_CUDA(cudaGetLastError());
    ctx->launches++;
    ctx->poses_total += 1;
  }
  std::vector<double> host(static_cast<size_t>(9) * n_poses);
  VL_CUDA(cudaMemcpyAsync(host.data(), d_out.p, sizeof(double) * 9 * n_poses, cudaMemcpyDeviceToHost, ctx->stream));
  VL_CUDA(cudaStreamSynchronize(ctx->stream));
  for (int p = 0; p < n_poses; p++) {
    nid_out[p] = host[9 * static_cast<size_t>(p)];
    for (int k = 0; k < 7; k++) grad_out[7 * static_cast<size_t>(p) + k] = host[9 * static_cast<size_t>(p) + 1 + k];
    if (ok_out) ok_out[p] = host[9 * static_cast<size_t>(p) + 8] != 0.0 ? 1 : 0;
  }
  return VLCAL_OK;
}
