// nid_context.cu -- cost-object lifecycle and batched evaluation behind the C ABI (include/vlcal_nid.h).
//
// Plays the role of vlcal::CostCalculatorNID (reference: include/vlcal/calib/cost_calculator_nid.hpp:16-29,
// src/vlcal/calib/cost_calculator_nid.cpp:13-67): the constructor copies one bag (image + cloud) into HBM once,
// calculate() becomes a batched kernel launch on the context's own stream.
#include "nid_context.cuh"

#include <omp.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <map>
#include <thread>
#include <tuple>

#include "fast_filter.hpp"
#include "host_math.hpp"
#include "mem_pool.hpp"
#include "nid_kernels.cuh"
#include "nid_persistent.cuh"

namespace vlcal {

// ---------------------------------------------------------------------------------------------
// errors
// ---------------------------------------------------------------------------------------------

static thread_local std::string g_last_error;

void set_last_error(const std::string& msg) {
  g_last_error = msg;
}

int cuda_fail(cudaError_t e, const char* what, const char* file, int line) {
  char buf[1024];
  std::snprintf(buf, sizeof(buf), "CUDA error %d (%s) at %s:%d: %s", static_cast<int>(e), cudaGetErrorString(e), file, line, what);
  set_last_error(buf);
  cudaGetLastError();  // clear the sticky per-thread error
  if (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver || e == cudaErrorInvalidDevice) {
    return VLCAL_ERR_NO_DEVICE;
  }
  return VLCAL_ERR_CUDA;
}

// ---------------------------------------------------------------------------------------------
// camera factory rules + estimate_camera_fov
// ---------------------------------------------------------------------------------------------

int make_camera(int model, const double* intr, int n_intr, const double* dist, int n_dist, CameraParams* out) {
  int ni = 0, nd = 0;
  if (!camera_num_params(model, &ni, &nd)) {
    set_last_error("unknown camera model id " + std::to_string(model));  // create_camera.cpp:49-50
    return VLCAL_ERR_UNKNOWN_CAMERA_MODEL;
  }
  if (n_intr != ni || (ni > 0 && intr == nullptr)) {
    set_last_error("num of intrinsic parameters mismatch: model expects " + std::to_string(ni) + ", got " + std::to_string(n_intr));  // :19-22
    return VLCAL_ERR_INTRINSIC_COUNT;
  }
  std::memset(out, 0, sizeof(*out));
  out->model = model;
  out->n_intr = ni;
  out->n_dist = nd;
  for (int i = 0; i < ni; i++) out->intr[i] = intr[i];
  for (int i = 0; i < nd && i < n_dist && dist != nullptr; i++) out->dist[i] = dist[i];  // :24-27 zero-pad / truncate
  return VLCAL_OK;
}

// to_dir(x) = AngleAxisd(x0, UnitX) * AngleAxisd(x1, UnitY) * UnitZ  (estimate_fov.cpp:18-20), evaluated the way
// Eigen does: quaternion product, then Quaternion::_transformVector
static void fov_to_dir(const double x[2], double dir[3]) {
  const double ha = 0.5 * x[0], hb = 0.5 * x[1];
  const double aw = std::cos(ha), ax = std::sin(ha);
  const double bw = std::cos(hb), by = std::sin(hb);
  const double qw = aw * bw - ax * 0.0 - 0.0 * by - 0.0 * 0.0;
  const double qx = aw * 0.0 + ax * bw + 0.0 * 0.0 - 0.0 * by;
  const double qy = aw * by + 0.0 * bw + 0.0 * 0.0 - ax * 0.0;
  const double qz = aw * 0.0 + 0.0 * bw + ax * by - 0.0 * 0.0;
  const double v[3] = {0.0, 0.0, 1.0};
  double uv[3] = {qy * v[2] - qz * v[1], qz * v[0] - qx * v[2], qx * v[1] - qy * v[0]};
  uv[0] += uv[0], uv[1] += uv[1], uv[2] += uv[2];
  const double c[3] = {qy * uv[2] - qz * uv[1], qz * uv[0] - qx * uv[2], qx * uv[1] - qy * uv[0]};
  for (int i = 0; i < 3; i++) dir[i] = v[i] + qw * uv[i] + c[i];
}

double estimate_camera_fov_host(const CameraParams& cam, int width, int height) {
  // estimate_fov.cpp:37 (integer divisions), :39-48
  const double corners[3][2] = {{0.0, 0.0}, {static_cast<double>(width / 2), 0.0}, {0.0, static_cast<double>(height / 2)}};
  double max_fov = 0.0;
  for (int k = 0; k < 3; k++) {
    const double* target = corners[k];
    auto f = [&](const double* xs, int count, double* ys) {  // :22-26
      for (int i = 0; i < count; i++) {
        double dir[3], u, v;
        fov_to_dir(xs + 2 * i, dir);
        project_exact_dyn(cam, dir[0], dir[1], dir[2], &u, &v);
        const double ex = target[0] - u, ey = target[1] - v;
        const double err = ex * ex + ey * ey;
        ys[i] = std::isfinite(err) ? err : DBL_MAX;
      }
    };
    auto observe = [](const double*, double) {};
    const double x0[2] = {0.0, 0.0};
    host::NelderMeadParams p;  // :29 defaults
    const host::NelderMeadResult r = host::nelder_mead(2, f, observe, x0, p, /*speculate=*/false);
    double dir[3];
    fov_to_dir(r.x.data(), dir);  // :33
    const double n2 = (dir[0] * dir[0] + dir[1] * dir[1]) + dir[2] * dir[2];
    const double nz = n2 > 0.0 ? dir[2] / std::sqrt(n2) : dir[2];
    const double fov = std::acos(nz);  // :43
    if (fov > max_fov) max_fov = fov;
  }
  return max_fov;
}

// ---------------------------------------------------------------------------------------------
// device containers
// ---------------------------------------------------------------------------------------------

DeviceCloud::~DeviceCloud() {
  MemPool::instance().device_free(device, d_points);
}

DeviceImage::~DeviceImage() {
  MemPool::instance().device_free(device, d_raw);
}

// pinned staging buffers (cudaHostAlloc costs milliseconds; contexts are rebuilt every outer iteration).  A small pool
// rather than one buffer: the reference builds its cost objects from an OpenMP loop over bags
// (visual_camera_calibration.cpp:107 runs calculate() that way; constructors may be called from several threads too),
// and concurrent uploads -- to the same or to different devices -- must not serialise on one staging area.
struct PinnedStage {
  void* ptr = nullptr;
  size_t cap = 0;
  bool busy = false;
  int reserve(size_t bytes) {
    if (bytes <= cap) return VLCAL_OK;
    MemPool::instance().pinned_free(ptr);
    ptr = nullptr, cap = 0;
    const size_t want = std::max(bytes + bytes / 4, static_cast<size_t>(1) << 20);
    VL_CUDA(MemPool::instance().pinned_alloc(want, &ptr));
    cap = want;
    return VLCAL_OK;
  }
};

class StagePool {
public:
  // a free stage (the one with the largest capacity, so that steady-state callers never reallocate); grows on demand
  PinnedStage* acquire() {
    std::lock_guard<std::mutex> lock(mu_);
    PinnedStage* best = nullptr;
    for (auto& s : stages_)
      if (!s->busy && (!best || s->cap > best->cap)) best = s.get();
    if (!best) {
      stages_.emplace_back(new PinnedStage());
      best = stages_.back().get();
    }
    best->busy = true;
    return best;
  }
  void release(PinnedStage* s) {
    std::lock_guard<std::mutex> lock(mu_);
    s->busy = false;
  }

private:
  std::mutex mu_;
  std::vector<std::unique_ptr<PinnedStage>> stages_;
};
static StagePool g_stages;

struct StageLease {
  PinnedStage* s;
  StageLease() : s(g_stages.acquire()) {}
  ~StageLease() { g_stages.release(s); }
};

// threads of the copy-convert team.  NOT omp_get_max_threads(): launchers such as torch.distributed.run export
// OMP_NUM_THREADS=1 for every rank, which silently made the upload serial.
// The loop is memory-bound: a dozen threads saturate it, waking every core of a 128-core host costs more than it saves.
static int conversion_threads() {
  static const int n = [] {
    if (const char* e = std::getenv("VLCAL_UPLOAD_THREADS")) return std::max(1, std::min(64, std::atoi(e)));
    const unsigned hw = std::thread::hardware_concurrency();
    return static_cast<int>(std::max(1u, std::min(16u, hw ? hw : 1u)));
  }();
  return n;
}

int upload_cloud(int device, const double* points_xyzw, const double* intensities, int64_t n, cudaStream_t stream, std::shared_ptr<DeviceCloud>* out) {
  auto cloud = std::make_shared<DeviceCloud>();
  cloud->device = device;
  cloud->n = n;
  cloud->f32 = true;
  if (n == 0) {
    *out = cloud;
    return VLCAL_OK;
  }
  StageLease lease;
  PinnedStage& g_stage = *lease.s;
  {
    const int rc = g_stage.reserve(static_cast<size_t>(n) * 32);
    if (rc != VLCAL_OK) return rc;
  }
  // float4 (x,y,z,intensity) is lossless when the doubles came from a float32 PLY and intensity = k/256 (SURVEY D9).
  // Convert in a few chunks so that the H2D copy of chunk c overlaps the conversion of chunk c+1.
  float4* stage = static_cast<float4*>(g_stage.ptr);
  int lossless = 1, w_is_one = 1;
  const int conv_threads = conversion_threads();
  VL_CUDA(MemPool::instance().device_alloc(device, static_cast<size_t>(n) * 16, &cloud->d_points));
  constexpr int64_t CHUNK = 1 << 18;
  for (int64_t c0 = 0; c0 < n; c0 += CHUNK) {
    const int64_t c1 = std::min<int64_t>(n, c0 + CHUNK);
#pragma omp parallel for schedule(static) reduction(&& : lossless, w_is_one) num_threads(conv_threads)
    for (int64_t i = c0; i < c1; i++) {
      const double* p = points_xyzw + 4 * i;
      const float4 q = make_float4(static_cast<float>(p[0]), static_cast<float>(p[1]), static_cast<float>(p[2]), static_cast<float>(intensities[i]));
      stage[i] = q;
      lossless = lossless && (static_cast<double>(q.x) == p[0] || p[0] != p[0]) && (static_cast<double>(q.y) == p[1] || p[1] != p[1]) &&
                 (static_cast<double>(q.z) == p[2] || p[2] != p[2]) && (static_cast<double>(q.w) == intensities[i] || intensities[i] != intensities[i]);
      w_is_one = w_is_one && (p[3] == 1.0);
    }
    if (!lossless || !w_is_one) break;
    VL_CUDA(cudaMemcpyAsync(static_cast<float4*>(cloud->d_points) + c0, stage + c0, sizeof(float4) * static_cast<size_t>(c1 - c0), cudaMemcpyHostToDevice, stream));
  }
  VL_CUDA(cudaStreamSynchronize(stream));  // staging buffer is shared
  if (!w_is_one) {
    set_last_error("points_xyzw: homogeneous coordinate w must be 1 for every point (Frame::points, frame.hpp:66)");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  cloud->f32 = lossless != 0;
  if (!cloud->f32) {  // not float32-representable: 32-byte double layout (exact kernel only)
    for (int64_t i = 0; i < n; i++) {
      if (points_xyzw[4 * i + 3] != 1.0) {
        set_last_error("points_xyzw: homogeneous coordinate w must be 1 for every point (Frame::points, frame.hpp:66)");
        return VLCAL_ERR_INVALID_ARGUMENT;
      }
    }
    MemPool::instance().device_free(device, cloud->d_points);
    cloud->d_points = nullptr;
    double4* stage64 = static_cast<double4*>(g_stage.ptr);
#pragma omp parallel for schedule(static) num_threads(conv_threads)
    for (int64_t i = 0; i < n; i++) {
      const double* p = points_xyzw + 4 * i;
      stage64[i] = make_double4(p[0], p[1], p[2], intensities[i]);
    }
    const size_t bytes = static_cast<size_t>(n) * 32;
    VL_CUDA(MemPool::instance().device_alloc(device, bytes, &cloud->d_points));
    VL_CUDA(cudaMemcpyAsync(cloud->d_points, g_stage.ptr, bytes, cudaMemcpyHostToDevice, stream));
    VL_CUDA(cudaStreamSynchronize(stream));
  }
  *out = cloud;
  return VLCAL_OK;
}

int upload_image(int device, const uint8_t* image, int width, int height, int row_stride, cudaStream_t stream, std::shared_ptr<DeviceImage>* out) {
  auto img = std::make_shared<DeviceImage>();
  img->device = device;
  img->width = width;
  img->height = height;
  const size_t bytes = static_cast<size_t>(width) * height;
  VL_CUDA(MemPool::instance().device_alloc(device, bytes, reinterpret_cast<void**>(&img->d_raw)));
  VL_CUDA(cudaMemcpy2DAsync(img->d_raw, width, image, row_stride, width, height, cudaMemcpyHostToDevice, stream));
  VL_CUDA(cudaStreamSynchronize(stream));
  *out = img;
  return VLCAL_OK;
}

// ---------------------------------------------------------------------------------------------
// kernel dispatch
// ---------------------------------------------------------------------------------------------

using NidKernel = void (*)(const NidArgs);

// kind: 0 = fp32 filter + exact recheck (float4 layout only; 4 points/thread), 1 = exact fp64, 2 = verify (debug),
//       3 = fp32 filter with 2 points/thread (A/B measurement); devloop: device-resident solver-loop variant of 0 / 1
template <int MODEL>
static NidKernel pick_layout(bool f32, int kind, bool devloop) {
  if (devloop) {
    if (f32 && (kind == 0 || kind == 3)) return nid_hist_filter_kernel<MODEL, true, 4, true>;
    return f32 ? nid_hist_exact_kernel<MODEL, true, true> : nid_hist_exact_kernel<MODEL, false, true>;
  }
  if (f32 && kind == 0) return nid_hist_filter_kernel<MODEL, true, 4, false>;
  if (f32 && kind == 3) return nid_hist_filter_kernel<MODEL, true, 2, false>;
  if (f32 && kind == 2) return nid_filter_verify_kernel<MODEL, true>;
  return f32 ? nid_hist_exact_kernel<MODEL, true, false> : nid_hist_exact_kernel<MODEL, false, false>;
}

static NidKernel pick_kernel(int model, bool f32, int kind, bool devloop = false) {
  switch (model) {
    case CAM_PLUMB_BOB: return pick_layout<CAM_PLUMB_BOB>(f32, kind, devloop);
    case CAM_FISHEYE: return pick_layout<CAM_FISHEYE>(f32, kind, devloop);
    case CAM_ATAN: return pick_layout<CAM_ATAN>(f32, kind, devloop);
    case CAM_OMNIDIR: return pick_layout<CAM_OMNIDIR>(f32, kind, devloop);
    case CAM_EQUIRECTANGULAR: return pick_layout<CAM_EQUIRECTANGULAR>(f32, kind, devloop);
    case CAM_RATIONAL_POLYNOMIAL: return pick_layout<CAM_RATIONAL_POLYNOMIAL>(f32, kind, devloop);
    default: return nullptr;
  }
}

constexpr size_t NID_SMEM_OPT_IN = 100 * 1024;  // dynamic shared memory ceiling we opt into
constexpr size_t NID_SMEM_TARGET = 64 * 1024;   // privatised-copy budget per block

struct LaunchGeom {
  int copies;
  size_t smem;
  int blocks_per_sm;
  int finalize_split;
};

static std::mutex g_geom_mu;
// keyed by device too: function attributes (the dynamic shared memory opt-in) and occupancy are per device / context
static std::map<std::tuple<int, const void*, size_t>, int> g_occupancy_cache;

static int hist_copies_cap() {
  // warp-private copies bought nothing measurable over a couple of shared ones in a shared-atomic microbenchmark
  // (tools/microbench.cu), but every copy is zeroed and merged by every block on every launch; VLCAL_HIST_COPIES overrides for A/B
  static const int cap = [] {
    const char* e = std::getenv("VLCAL_HIST_COPIES");
    const int v = e ? std::atoi(e) : 2;
    return std::max(1, std::min(v, NID_THREADS / 32));
  }();
  return cap;
}

static int launch_geometry(int device, NidKernel kernel, int n_poses, int nb, int bins, LaunchGeom* g) {
  const size_t per_copy = static_cast<size_t>(n_poses) * nb * sizeof(int);
  int copies = static_cast<int>(NID_SMEM_TARGET / per_copy);
  copies = std::max(1, std::min(copies, hist_copies_cap()));
  g->copies = copies;
  g->smem = per_copy * copies;
  // room for nid_finalize to split one pose over several warps: 8 pose slots x (nb doubles + 2*bins ints)
  // 8 pose slots x (nb + 2*bins staged doubles + 2*bins marginal counts)
  const size_t split_need = static_cast<size_t>(NID_THREADS / 32) * (static_cast<size_t>(nb + 2 * bins) * 8 + static_cast<size_t>(bins) * 8);
  g->finalize_split = nb <= 1024;
  if (g->finalize_split) g->smem = std::max(g->smem, split_need);
  std::lock_guard<std::mutex> lock(g_geom_mu);
  const auto key = std::make_tuple(device, reinterpret_cast<const void*>(kernel), g->smem);
  auto it = g_occupancy_cache.find(key);
  if (it == g_occupancy_cache.end()) {
    VL_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(NID_SMEM_OPT_IN)));
    int nblk = 0;
    VL_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nblk, kernel, NID_THREADS, g->smem));
    it = g_occupancy_cache.emplace(key, std::max(1, nblk)).first;
  }
  g->blocks_per_sm = it->second;
  return VLCAL_OK;
}

// ---------------------------------------------------------------------------------------------
// context
// ---------------------------------------------------------------------------------------------

}  // namespace vlcal

vlcal_nid_ctx::~vlcal_nid_ctx() {
  cudaSetDevice(device);
  if (stream) cudaStreamSynchronize(stream);
  for (auto& e : events) {
    cudaEventDestroy(e.start);
    cudaEventDestroy(e.stop);
  }
  auto& pool = vlcal::MemPool::instance();
  pool.device_free(device, d_bin_image);
  pool.device_free(device, d_ghist);
  pool.device_free(device, d_counter);
  pool.device_free(device, d_nid);
  pool.device_free(device, d_hist_out);
  pool.pinned_free(h_nid);
  pool.pinned_free(h_flag);
  pool.pinned_free(h_timeline);
  if (stream) cudaStreamDestroy(stream);
}

namespace vlcal {

int nid_ctx_create(
  int device, int mode, const CameraParams& cam, std::shared_ptr<DeviceImage> image, std::shared_ptr<DeviceCloud> cloud, int bins, double max_fov, vlcal_nid_ctx** out) {
  if (mode != VLCAL_NID_MODE_HISTOGRAM && mode != VLCAL_NID_MODE_BSPLINE) {
    set_last_error("unknown NID mode");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  if (bins < 1 || bins > NID_MAX_BINS) {
    set_last_error("bins must be in [1, " + std::to_string(NID_MAX_BINS) + "]");
    return VLCAL_ERR_UNSUPPORTED;
  }
  VL_CUDA(cudaSetDevice(device));
  std::unique_ptr<vlcal_nid_ctx> ctx(new vlcal_nid_ctx());
  ctx->device = device;
  ctx->mode = mode;
  ctx->bins = bins;
  ctx->cam = cam;
  ctx->image = image;
  ctx->cloud = cloud;
  ctx->max_fov = max_fov;
  ctx->cos_fov = std::cos(max_fov);  // cost_calculator_nid.cpp:32
  ctx->fast = make_fast_cam(cam, image->width, image->height, max_fov);
  ctx->lean = make_lean_cam(cam, ctx->fast, image->width, image->height, max_fov);
  VL_CUDA(cudaDeviceGetAttribute(&ctx->num_sms, cudaDevAttrMultiProcessorCount, device));
  VL_CUDA(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));

  const int nb = bins * bins;
  ctx->max_poses = std::max(1, std::min<int>(NID_MAX_POSES, static_cast<int>((NID_SMEM_OPT_IN - 4096) / (static_cast<size_t>(nb) * sizeof(int)))));
  VL_CUDA(MemPool::instance().device_alloc(device, sizeof(int) * static_cast<size_t>(NID_MAX_POSES) * nb, reinterpret_cast<void**>(&ctx->d_ghist)));
  VL_CUDA(cudaMemsetAsync(ctx->d_ghist, 0, sizeof(int) * static_cast<size_t>(NID_MAX_POSES) * nb, ctx->stream));
  VL_CUDA(MemPool::instance().device_alloc(device, sizeof(unsigned int), reinterpret_cast<void**>(&ctx->d_counter)));
  VL_CUDA(cudaMemsetAsync(ctx->d_counter, 0, sizeof(unsigned int), ctx->stream));

  // image -> image-bin plane: image_bin = max(0, min(bins-1, int(u8/255.0 * bins)))  (cost_calculator_nid.cpp:43,46)
  uint8_t lut[256];
  for (int v = 0; v < 256; v++) {
    int b;
    if (mode == VLCAL_NID_MODE_HISTOGRAM) {
      const double pixel = v / 255.0;  // image.at<uint8_t>() / 255.0  (cost_calculator_nid.cpp:43)
      b = cast_int_x86(pixel * bins);
      b = b < bins - 1 ? b : bins - 1;
      b = b > 0 ? b : 0;
    } else {
      const double pix = v * (1.0 / 255.0);  // image.convertTo(CV_64FC1, 1.0 / 255.0)  (visual_camera_calibration.cpp:203-204)
      b = cast_int_x86(pix * bins);          // std::min<int>(pix * bins, bins - 1)  (nid_cost.hpp:79)
      b = b < bins - 1 ? b : bins - 1;
    }
    lut[v] = static_cast<uint8_t>(b);
  }
  uint8_t* d_lut = nullptr;
  VL_CUDA(MemPool::instance().device_alloc(device, 256, reinterpret_cast<void**>(&d_lut)));
  VL_CUDA(cudaMemcpyAsync(d_lut, lut, 256, cudaMemcpyHostToDevice, ctx->stream));
  const size_t npix = static_cast<size_t>(image->width) * image->height;
  VL_CUDA(MemPool::instance().device_alloc(device, std::max<size_t>(npix, 1), reinterpret_cast<void**>(&ctx->d_bin_image)));
  if (npix > 0) {
    const dim3 grid((image->width + 255) / 256, image->height);
    apply_lut_kernel<<<grid, 256, 0, ctx->stream>>>(image->d_raw, image->width, ctx->d_bin_image, image->width, image->height, d_lut);
    VL_CUDA(cudaGetLastError());
  }
  VL_CUDA(cudaStreamSynchronize(ctx->stream));
  MemPool::instance().device_free(device, d_lut);
  *out = ctx.release();
  return VLCAL_OK;
}

static int ensure_outputs(vlcal_nid_ctx* ctx, int n_poses, bool want_hist) {
  if (n_poses > ctx->d_nid_cap) {
    auto& pool = MemPool::instance();
    pool.device_free(ctx->device, ctx->d_nid);
    pool.pinned_free(ctx->h_nid);
    ctx->d_nid = nullptr, ctx->h_nid = nullptr, ctx->d_nid_cap = 0;
    const int cap = std::max(n_poses, 64);
    VL_CUDA(pool.device_alloc(ctx->device, sizeof(double) * cap, reinterpret_cast<void**>(&ctx->d_nid)));
    VL_CUDA(pool.pinned_alloc(sizeof(double) * cap, reinterpret_cast<void**>(&ctx->h_nid)));
    if (!ctx->h_flag) {
      VL_CUDA(pool.pinned_alloc(sizeof(unsigned long long), reinterpret_cast<void**>(&ctx->h_flag)));
      *ctx->h_flag = 0;
    }
    ctx->d_nid_cap = cap;
    ctx->h_nid_cap = cap;
  }
  if (want_hist) {
    const size_t need = static_cast<size_t>(n_poses) * ctx->bins * ctx->bins;
    if (need > ctx->d_hist_out_cap) {
      MemPool::instance().device_free(ctx->device, ctx->d_hist_out);
      ctx->d_hist_out = nullptr, ctx->d_hist_out_cap = 0;
      VL_CUDA(MemPool::instance().device_alloc(ctx->device, sizeof(int) * need, reinterpret_cast<void**>(&ctx->d_hist_out)));
      ctx->d_hist_out_cap = need;
    }
  }
  return VLCAL_OK;
}

// float copy of the poses for the fp32 filter: R, t rounded to nearest; max|t| rounded up
static void fill_pose32(NidArgs& a, int pc) {
  for (int p = 0; p < pc; p++) {
    const double* T = a.pose[p];
    float* P = a.pose32[p];
    for (int r = 0; r < 3; r++) {
      for (int c = 0; c < 3; c++) P[3 * r + c] = static_cast<float>(T[4 * r + c]);
      P[9 + r] = static_cast<float>(T[4 * r + 3]);
    }
    const double tmax = std::max(std::fabs(T[3]), std::max(std::fabs(T[7]), std::fabs(T[11])));
    P[12] = std::nextafter(static_cast<float>(tmax), INFINITY);
    P[13] = P[14] = P[15] = 0.f;
  }
}

// everything of NidArgs that does not depend on the batch
static void fill_common_args(vlcal_nid_ctx* ctx, NidArgs& a) {
  std::memset(&a, 0, sizeof(a));
  a.points = ctx->cloud->d_points;
  a.bin_image = ctx->d_bin_image;
  a.n = ctx->cloud->n;
  a.width = ctx->image->width;
  a.height = ctx->image->height;
  a.bins = ctx->bins;
  a.nb = ctx->bins * ctx->bins;
  a.cos_fov = ctx->cos_fov;
  a.cam = ctx->cam;
  a.fast = ctx->fast;
  a.timeline = ctx->h_timeline;
  if (ctx->p2p && ctx->p2p->connected && ctx->p2p->world > 1) {
    for (int r = 0; r < ctx->p2p->world; r++) a.peer_box[r] = ctx->p2p->peers[r];
    a.p2p_world = ctx->p2p->world;
    a.p2p_rank = ctx->p2p->rank;
    a.p2p_counter = ctx->p2p->d_counter;
    a.p2p_error = ctx->p2p->h_error;
  }
  a.ghist = ctx->d_ghist;
  a.counter = ctx->d_counter;
}

static NidKernel select_kernel(vlcal_nid_ctx* ctx, bool devloop = false) {
  // the fp32 filter needs the float4 layout, a camera/FoV it has bounds for, and 32-bit point indices
  const bool use_filter = ctx->variant != 1 && ctx->cloud->f32 && ctx->fast.enabled && ctx->cloud->n < 0x7fffffffLL;
  // points per lane and tile (tools/kernel_scaling.py measures the choice):
  //  * fisheye / equirectangular / atan carry transcendental calls and more live state per point: 2 points
  //  * plumb_bob / rational_polynomial / omnidir: 4 while a warp's share of the cloud is a few 128-point tiles; below one
  //    tile the 4-point path degenerates to single rows, and on long ranges (5 M points) the lighter register footprint
  //    of 2 wins again
  const bool heavy = ctx->cam.model == CAM_FISHEYE || ctx->cam.model == CAM_EQUIRECTANGULAR || ctx->cam.model == CAM_ATAN;
  const long long points_per_warp = ctx->cloud->n / (static_cast<long long>(ctx->num_sms) * 2 * (NID_THREADS / 32));
  const bool four = !heavy && points_per_warp >= 96 && points_per_warp <= 1100;
  const int filter_kind = ctx->variant == 2 ? 3 : (ctx->variant == 3 ? 0 : (four ? 0 : 3));
  return pick_kernel(ctx->cam.model, ctx->cloud->f32, use_filter ? filter_kind : 1, devloop);
}

constexpr int PROFILE_STRIDE = 4;

static int launch_one(vlcal_nid_ctx* ctx, NidKernel kernel, NidArgs& a, int geometry_poses, int profile_poses) {
  LaunchGeom g{1, 0, 1, 0};
  {
    const int rc = launch_geometry(ctx->device, kernel, geometry_poses, a.nb, a.bins, &g);
    if (rc != VLCAL_OK) return rc;
  }
  a.copies = g.copies;
  a.finalize_split = g.finalize_split;
  const long long want_blocks = (a.n + NID_THREADS - 1) / NID_THREADS;
  const int grid = static_cast<int>(std::max<long long>(1, std::min<long long>(want_blocks, static_cast<long long>(ctx->num_sms) * g.blocks_per_sm)));
  ProfileEvents* ev = nullptr;
  // event pairs cost host time per launch on the Nelder-Mead critical path: sample one launch in four
  if (ctx->profiling && (ctx->launch_counter++ % PROFILE_STRIDE) == 0) {
    if (ctx->events_used == ctx->events.size()) {
      ProfileEvents e;
      VL_CUDA(cudaEventCreate(&e.start));
      VL_CUDA(cudaEventCreate(&e.stop));
      e.poses = 0;
      ctx->events.push_back(e);
    }
    ev = &ctx->events[ctx->events_used++];
    ev->poses = profile_poses;
    VL_CUDA(cudaEventRecord(ev->start, ctx->stream));
  }
  kernel<<<grid, NID_THREADS, g.smem, ctx->stream>>>(a);
  VL_CUDA(cudaGetLastError());
  if (ev) VL_CUDA(cudaEventRecord(ev->stop, ctx->stream));
  return VLCAL_OK;
}

int nid_evaluate_async(vlcal_nid_ctx* ctx, const double* T_colmajor, int n_poses, bool want_hist) {
  if (ctx->in_flight) {
    set_last_error("an evaluation is already in flight on this context");
    return VLCAL_ERR_BUSY;
  }
  if (ctx->mode != VLCAL_NID_MODE_HISTOGRAM) {
    set_last_error("context was created in B-spline mode; use vlcal_nid_evaluate_bspline");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  VL_CUDA(cudaSetDevice(ctx->device));
  {
    const int rc = ensure_outputs(ctx, n_poses, want_hist);
    if (rc != VLCAL_OK) return rc;
  }
  const int nb = ctx->bins * ctx->bins;
  NidKernel kernel = select_kernel(ctx);
  for (int p0 = 0; p0 < n_poses; p0 += ctx->max_poses) {
    const int pc = std::min(ctx->max_poses, n_poses - p0);
    NidArgs a;
    fill_common_args(ctx, a);
    a.n_poses = pc;
    for (int p = 0; p < pc; p++) {
      const double* T = T_colmajor + 16 * static_cast<size_t>(p0 + p);
      for (int r = 0; r < 3; r++)
        for (int c = 0; c < 4; c++) a.pose[p][4 * r + c] = T[r + 4 * c];
    }
    fill_pose32(a, pc);
    a.nid_out = ctx->d_nid + p0;
    a.nid_host = ctx->h_nid + p0;  // UVA: pinned host memory is directly addressable from the device
    const bool last_chunk = p0 + pc >= n_poses;
    a.done_flag = last_chunk ? ctx->h_flag : nullptr;
    a.done_seq = ctx->seq + 1;
    a.hist_out = want_hist ? ctx->d_hist_out + static_cast<size_t>(p0) * nb : nullptr;
    const int rc = launch_one(ctx, kernel, a, pc, pc);
    if (rc != VLCAL_OK) return rc;
    ctx->launches++;
    ctx->passes++;
    ctx->poses_total += pc;
  }
  ctx->seq += 1;
  ctx->in_flight = true;
  ctx->in_flight_poses = n_poses;
  return VLCAL_OK;
}

int nid_enqueue_device_steps(vlcal_nid_ctx* ctx, NmDevice* d_nm, int count) {
  if (ctx->in_flight) {
    set_last_error("an evaluation is in flight on this context");
    return VLCAL_ERR_BUSY;
  }
  if (ctx->mode != VLCAL_NID_MODE_HISTOGRAM) {
    set_last_error("device-resident solver loop needs a histogram-mode context");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  VL_CUDA(cudaSetDevice(ctx->device));
  {
    const int rc = ensure_outputs(ctx, NID_MAX_POSES, false);
    if (rc != VLCAL_OK) return rc;
  }
  if (ctx->max_poses < NID_MAX_POSES) {
    set_last_error("device-resident solver loop needs room for 8 poses per launch (bins too large)");
    return VLCAL_ERR_UNSUPPORTED;
  }
  NidKernel kernel = select_kernel(ctx, /*devloop=*/true);
  NidArgs a;
  fill_common_args(ctx, a);
  a.nm = d_nm;
  a.n_poses = 0;
  a.nid_out = ctx->d_nid;
  for (int k = 0; k < count; k++) {
    const int rc = launch_one(ctx, kernel, a, NID_MAX_POSES, 0);
    if (rc != VLCAL_OK) return rc;
  }
  return VLCAL_OK;
}

int nid_account_device_steps(vlcal_nid_ctx* ctx, int enqueued, int worked, int poses) {
  // sampled events of this enqueue: keep those of launches that did work, drop the ones that found the solver finished
  if (ctx->profiling) {
    const int64_t first_launch = ctx->launch_counter - enqueued;  // index of the first launch of this enqueue
    int sampled = 0;
    for (int k = 0; k < enqueued; k++)
      if (((first_launch + k) % PROFILE_STRIDE) == 0) sampled++;
    const size_t first = ctx->events_used - static_cast<size_t>(sampled);
    int e = 0;
    for (int k = 0; k < enqueued; k++) {
      if (((first_launch + k) % PROFILE_STRIDE) != 0) continue;
      if (k < worked) {
        float ms = 0.f;
        VL_CUDA(cudaEventElapsedTime(&ms, ctx->events[first + e].start, ctx->events[first + e].stop));
        ctx->kernel_ms_accum += ms;
        ctx->timed_launches++;
      }
      e++;
    }
    ctx->events_used = first;
  }
  ctx->launches += worked;
  ctx->passes += worked;
  ctx->poses_total += poses;
  return VLCAL_OK;
}

static int drain_profile(vlcal_nid_ctx* ctx) {
  for (size_t i = 0; i < ctx->events_used; i++) {
    float ms = 0.f;
    VL_CUDA(cudaEventElapsedTime(&ms, ctx->events[i].start, ctx->events[i].stop));
    ctx->kernel_ms_accum += ms;
    ctx->timed_launches++;
  }
  ctx->events_used = 0;
  return VLCAL_OK;
}

int nid_wait(vlcal_nid_ctx* ctx, double* nid_out, int32_t* hist_out) {
  if (!ctx->in_flight) {
    set_last_error("no evaluation in flight on this context");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  VL_CUDA(cudaSetDevice(ctx->device));
  ctx->in_flight = false;
  {
    // the last block of the last launch writes the scores into mapped host memory and then bumps the flag: poll it
    // (a few microseconds) instead of paying a D2H copy + stream synchronisation per Nelder-Mead batch; fall back to
    // the stream (which also surfaces launch / execution errors) if the flag does not arrive promptly.
    volatile unsigned long long* flag = ctx->h_flag;
    bool done = false;
    for (int spin = 0; spin < 4000000; spin++) {
      if (*flag == ctx->seq) {
        done = true;
        break;
      }
      if ((spin & 0x3fff) == 0x3fff && cudaStreamQuery(ctx->stream) != cudaErrorNotReady) break;
      __builtin_ia32_pause();
    }
    if (!done) VL_CUDA(cudaStreamSynchronize(ctx->stream));
    if (*flag != ctx->seq) {
      VL_CUDA(cudaStreamSynchronize(ctx->stream));
      if (*flag != ctx->seq) {
        set_last_error("evaluation finished without publishing its results");
        return VLCAL_ERR_CUDA;
      }
    }
    std::atomic_thread_fence(std::memory_order_acquire);
    if (ctx->p2p && ctx->p2p->h_error && *ctx->p2p->h_error) {
      set_last_error("peer exchange timed out: a rank died or the ranks are not evaluating in lockstep");
      return VLCAL_ERR_CUDA;
    }
  }
  if (ctx->events_used > 256) {
    VL_CUDA(cudaStreamSynchronize(ctx->stream));
    const int rc = drain_profile(ctx);
    if (rc != VLCAL_OK) return rc;
  }
  const int n_poses = ctx->in_flight_poses;
  if (nid_out) std::memcpy(nid_out, ctx->h_nid, sizeof(double) * n_poses);
  if (hist_out) {
    if (!ctx->d_hist_out) {
      set_last_error("histograms were not requested for the evaluation in flight");
      return VLCAL_ERR_INVALID_ARGUMENT;
    }
    VL_CUDA(cudaStreamSynchronize(ctx->stream));  // the flag only orders the scores; histograms come from device memory
    VL_CUDA(cudaMemcpy(hist_out, ctx->d_hist_out, sizeof(int) * static_cast<size_t>(n_poses) * ctx->bins * ctx->bins, cudaMemcpyDeviceToHost));
  }
  return VLCAL_OK;
}

}  // namespace vlcal

// ---------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------

using namespace vlcal;

extern "C" {

const char* vlcal_nid_version(void) {
  return "0.1.0";
}

const char* vlcal_nid_last_error(void) {
  return g_last_error.c_str();
}

int vlcal_nid_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

int vlcal_camera_model_id(const char* camera_model) {
  if (camera_model == nullptr) {
    set_last_error("camera_model is NULL");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  const std::string m(camera_model);  // create_camera.cpp:35-46
  if (m == "plumb_bob") return VLCAL_CAMERA_PLUMB_BOB;
  if (m == "fisheye" || m == "equidistant") return VLCAL_CAMERA_FISHEYE;
  if (m == "atan") return VLCAL_CAMERA_ATAN;
  if (m == "omnidir") return VLCAL_CAMERA_OMNIDIR;
  if (m == "equirectangular") return VLCAL_CAMERA_EQUIRECTANGULAR;
  if (m == "rational_polynomial") return VLCAL_CAMERA_RATIONAL_POLYNOMIAL;
  set_last_error("error: unknown camera model " + m);  // :49
  return VLCAL_ERR_UNKNOWN_CAMERA_MODEL;
}

int vlcal_camera_num_params(int camera_model, int* n_intrinsics, int* n_distortion) {
  int ni = 0, nd = 0;
  if (!camera_num_params(camera_model, &ni, &nd)) {
    set_last_error("unknown camera model id");
    return VLCAL_ERR_UNKNOWN_CAMERA_MODEL;
  }
  if (n_intrinsics) *n_intrinsics = ni;
  if (n_distortion) *n_distortion = nd;
  return VLCAL_OK;
}

int vlcal_camera_project(int camera_model, const double* intrinsics, int n_intrinsics, const double* distortion, int n_distortion, const double point_3d[3], double uv[2]) {
  CameraParams cam;
  const int rc = make_camera(camera_model, intrinsics, n_intrinsics, distortion, n_distortion, &cam);
  if (rc != VLCAL_OK) return rc;
  project_exact_dyn(cam, point_3d[0], point_3d[1], point_3d[2], &uv[0], &uv[1]);
  return VLCAL_OK;
}

int vlcal_se3_expmap_gtsam(const double x[6], double T_colmajor[16]) {
  if (!x || !T_colmajor) {
    set_last_error("NULL argument");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  host::se3_expmap_gtsam(x, T_colmajor);
  return VLCAL_OK;
}

int vlcal_estimate_camera_fov(int camera_model, const double* intrinsics, int n_intrinsics, const double* distortion, int n_distortion, int width, int height, double* max_fov_rad) {
  CameraParams cam;
  const int rc = make_camera(camera_model, intrinsics, n_intrinsics, distortion, n_distortion, &cam);
  if (rc != VLCAL_OK) return rc;
  *max_fov_rad = estimate_camera_fov_host(cam, width, height);
  return VLCAL_OK;
}

int vlcal_nid_create(
  vlcal_nid_ctx** ctx,
  int device,
  int mode,
  int camera_model,
  const double* intrinsics,
  int n_intrinsics,
  const double* distortion,
  int n_distortion,
  const uint8_t* image,
  int width,
  int height,
  int row_stride_bytes,
  const double* points_xyzw,
  const double* intensities,
  int64_t n_points,
  int bins,
  double max_fov_rad) {
  if (!ctx) {
    set_last_error("ctx is NULL");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  *ctx = nullptr;
  if (width <= 0 || height <= 0 || !image || row_stride_bytes < width || n_points < 0 || (n_points > 0 && (!points_xyzw || !intensities))) {
    set_last_error("invalid image / point buffers");
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
  if (max_fov_rad < 0.0) {
    max_fov_rad = estimate_camera_fov_host(cam, width, height);  // cost_calculator_nid.cpp:17
  }
  std::shared_ptr<DeviceCloud> cloud;
  std::shared_ptr<DeviceImage> img;
  rc = upload_cloud(device, points_xyzw, intensities, n_points, /*stream=*/nullptr, &cloud);
  if (rc != VLCAL_OK) return rc;
  rc = upload_image(device, image, width, height, row_stride_bytes, /*stream=*/nullptr, &img);
  if (rc != VLCAL_OK) return rc;
  return nid_ctx_create(device, mode, cam, img, cloud, bins, max_fov_rad, ctx);
}

void vlcal_nid_destroy(vlcal_nid_ctx* ctx) {
  delete ctx;
}

int vlcal_nid_evaluate_async(vlcal_nid_ctx* ctx, const double* T_camera_lidar, int n_poses) {
  if (!ctx || !T_camera_lidar || n_poses <= 0) {
    set_last_error("invalid arguments");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  return nid_evaluate_async(ctx, T_camera_lidar, n_poses, /*want_hist=*/false);
}

int vlcal_nid_wait(vlcal_nid_ctx* ctx, double* nid_out, int32_t* hist_out) {
  if (!ctx) {
    set_last_error("ctx is NULL");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  return nid_wait(ctx, nid_out, hist_out);
}

int vlcal_nid_evaluate(vlcal_nid_ctx* ctx, const double* T_camera_lidar, int n_poses, double* nid_out, int32_t* hist_out) {
  if (!ctx || !T_camera_lidar || n_poses <= 0) {
    set_last_error("invalid arguments");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  // default: the persistent kernel in pose-list mode (one launch for any number of poses); contexts it does not cover
  // (double layout, bins > 32, cameras without the lean classifier, an attached peer exchange) take the round-1 kernels
  if (!ctx->p2p && ctx->variant != 4 && pk_supported(&ctx, 1)) {
    if (!nid_out) {
      set_last_error("nid_out is NULL");
      return VLCAL_ERR_INVALID_ARGUMENT;
    }
    return pk_score_poses(&ctx, 1, T_camera_lidar, n_poses, nid_out, hist_out);
  }
  const int rc = nid_evaluate_async(ctx, T_camera_lidar, n_poses, hist_out != nullptr);
  if (rc != VLCAL_OK) return rc;
  return nid_wait(ctx, nid_out, hist_out);
}

int vlcal_nid_score_poses(vlcal_nid_ctx* const* ctxs, int n_ctxs, const double* T_camera_lidar, int n_poses, double* nid_out) {
  if (!ctxs || n_ctxs <= 0 || !T_camera_lidar || n_poses <= 0 || !nid_out) {
    set_last_error("invalid arguments");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  for (int i = 0; i < n_ctxs; i++) {
    if (!ctxs[i]) {
      set_last_error("NULL context");
      return VLCAL_ERR_INVALID_ARGUMENT;
    }
  }
  if (pk_supported(ctxs, n_ctxs)) return pk_score_poses(ctxs, n_ctxs, T_camera_lidar, n_poses, nid_out, nullptr);
  // contexts the persistent kernel does not cover: one batched evaluation per context, summed in context order
  std::vector<double> part(n_poses);
  for (int p = 0; p < n_poses; p++) nid_out[p] = 0.0;
  for (int i = 0; i < n_ctxs; i++) {
    int rc = nid_evaluate_async(ctxs[i], T_camera_lidar, n_poses, false);
    if (rc == VLCAL_OK) rc = nid_wait(ctxs[i], part.data(), nullptr);
    if (rc != VLCAL_OK) return rc;
    for (int p = 0; p < n_poses; p++) nid_out[p] += part[p];
  }
  return VLCAL_OK;
}

int64_t vlcal_nid_num_points(const vlcal_nid_ctx* ctx) {
  return ctx ? ctx->cloud->n : 0;
}
int vlcal_nid_bins(const vlcal_nid_ctx* ctx) {
  return ctx ? ctx->bins : 0;
}
double vlcal_nid_max_fov(const vlcal_nid_ctx* ctx) {
  return ctx ? ctx->max_fov : 0.0;
}
int vlcal_nid_points_are_f32(const vlcal_nid_ctx* ctx) {
  return ctx && ctx->cloud->f32 ? 1 : 0;
}
int vlcal_nid_max_poses_per_launch(void) {
  return NID_MAX_POSES;
}

int vlcal_nid_set_profiling(vlcal_nid_ctx* ctx, int enable) {
  if (!ctx) return VLCAL_ERR_INVALID_ARGUMENT;
  ctx->profiling = enable != 0;
  return VLCAL_OK;
}

int vlcal_nid_get_profile(vlcal_nid_ctx* ctx, int64_t* kernel_launches, double* kernel_ms_total, int64_t* poses_total) {
  if (!ctx) return VLCAL_ERR_INVALID_ARGUMENT;
  VL_CUDA(cudaSetDevice(ctx->device));
  VL_CUDA(cudaStreamSynchronize(ctx->stream));
  const int rc = drain_profile(ctx);
  if (rc != VLCAL_OK) return rc;
  if (kernel_launches) *kernel_launches = ctx->launches;
  // sampled launches are representative of the rest: report the total scaled to all launches
  if (kernel_ms_total) *kernel_ms_total = ctx->timed_launches > 0 ? ctx->kernel_ms_accum * (static_cast<double>(ctx->launches) / ctx->timed_launches) : 0.0;
  if (poses_total) *poses_total = ctx->poses_total;
  return VLCAL_OK;
}

int vlcal_nid_get_profile_passes(vlcal_nid_ctx* ctx, int64_t* passes) {
  if (!ctx || !passes) return VLCAL_ERR_INVALID_ARGUMENT;
  *passes = ctx->passes;
  return VLCAL_OK;
}

int vlcal_nid_set_poses_per_pass(vlcal_nid_ctx* ctx, int poses_per_pass) {
  if (!ctx || poses_per_pass < 1 || poses_per_pass > PK_MAX_POSES) {
    set_last_error("poses_per_pass must be in [1, 8]");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  ctx->pk_chunk = poses_per_pass;
  return VLCAL_OK;
}

int vlcal_nid_debug_solve_stamps(vlcal_nid_ctx* ctx, int capacity, uint64_t* stamps_out, int* n_out) {
  if (!ctx || capacity < 0) return VLCAL_ERR_INVALID_ARGUMENT;
  if (!stamps_out) {  // arm: the next persistent solve on this context records `capacity` batches
    ctx->pk_stamps_cap = capacity;
    ctx->pk_stamps.clear();
    return VLCAL_OK;
  }
  const int have = static_cast<int>(ctx->pk_stamps.size() / PK_STAMP_SLOTS);
  const int n = std::min(capacity, have);
  for (int i = 0; i < n * PK_STAMP_SLOTS; i++) stamps_out[i] = ctx->pk_stamps[i];
  if (n_out) *n_out = n;
  return VLCAL_OK;
}

int vlcal_nid_debug_tma_stats(vlcal_nid_ctx* ctx, uint64_t stats[2]) {
  if (!ctx || !stats) return VLCAL_ERR_INVALID_ARGUMENT;
  stats[0] = ctx->pk_tma_stats[0], stats[1] = ctx->pk_tma_stats[1];
  return VLCAL_OK;
}

int vlcal_nid_debug_block_times(vlcal_nid_ctx* ctx, int capacity_blocks, uint64_t* times_out, int* n_blocks) {
  if (!ctx || capacity_blocks < 0 || !times_out || !n_blocks) return VLCAL_ERR_INVALID_ARGUMENT;
  const int have = static_cast<int>(ctx->pk_block_times.size() / 4);
  const int n = std::min(capacity_blocks, have);
  for (int i = 0; i < 4 * n; i++) times_out[i] = ctx->pk_block_times[i];
  *n_blocks = n;
  return VLCAL_OK;
}

int vlcal_nid_reset_profile(vlcal_nid_ctx* ctx) {
  if (!ctx) return VLCAL_ERR_INVALID_ARGUMENT;
  VL_CUDA(cudaSetDevice(ctx->device));
  VL_CUDA(cudaStreamSynchronize(ctx->stream));
  ctx->events_used = 0;
  ctx->launches = 0;
  ctx->timed_launches = 0;
  ctx->launch_counter = 0;
  ctx->poses_total = 0;
  ctx->passes = 0;
  ctx->kernel_ms_accum = 0.0;
  return VLCAL_OK;
}

int vlcal_nid_set_kernel_variant(vlcal_nid_ctx* ctx, int variant) {
  if (!ctx || variant < 0 || variant > 4) return VLCAL_ERR_INVALID_ARGUMENT;
  ctx->variant = variant;
  return VLCAL_OK;
}

int vlcal_nid_debug_timeline(vlcal_nid_ctx* ctx, const double* T_camera_lidar, int n_poses, double out_us[12]) {
  if (!ctx || !T_camera_lidar || n_poses <= 0 || n_poses > NID_MAX_POSES || !out_us) {
    set_last_error("invalid arguments (one launch: n_poses <= 8)");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  VL_CUDA(cudaSetDevice(ctx->device));
  if (!ctx->h_timeline) VL_CUDA(MemPool::instance().pinned_alloc(16 * sizeof(unsigned long long), reinterpret_cast<void**>(&ctx->h_timeline)));
  for (int i = 0; i < 16; i++) ctx->h_timeline[i] = 0ull;
  ctx->h_timeline[0] = ~0ull;
  std::vector<double> nid(n_poses);
  timespec ts0, ts1, ts2;
  clock_gettime(CLOCK_MONOTONIC, &ts0);
  int rc = nid_evaluate_async(ctx, T_camera_lidar, n_poses, false);
  clock_gettime(CLOCK_MONOTONIC, &ts1);
  if (rc == VLCAL_OK) rc = nid_wait(ctx, nid.data(), nullptr);
  clock_gettime(CLOCK_MONOTONIC, &ts2);
  VL_CUDA(cudaStreamSynchronize(ctx->stream));
  const unsigned long long* t = ctx->h_timeline;
  const double base = static_cast<double>(t[0]);
  out_us[0] = (static_cast<double>(t[1]) - base) * 1e-3;  // last block: main loop done (since first block start)
  out_us[1] = (static_cast<double>(t[2]) - base) * 1e-3;  // merged + fenced
  out_us[2] = (static_cast<double>(t[3]) - base) * 1e-3;  // ticket known
  out_us[3] = (static_cast<double>(t[4]) - base) * 1e-3;  // finalize math done
  out_us[4] = (static_cast<double>(t[5]) - base) * 1e-3;  // published
  out_us[5] = ((ts1.tv_sec - ts0.tv_sec) * 1e9 + (ts1.tv_nsec - ts0.tv_nsec)) * 1e-3;  // host: launch call
  out_us[6] = ((ts2.tv_sec - ts0.tv_sec) * 1e9 + (ts2.tv_nsec - ts0.tv_nsec)) * 1e-3;  // host: launch -> results visible
  out_us[7] = (static_cast<double>(t[7]) - base) * 1e-3;   // finalize: fence + scratch zeroed
  out_us[8] = (static_cast<double>(t[8]) - base) * 1e-3;   // finalize: marginals + inlier count known
  out_us[9] = (static_cast<double>(t[9]) - base) * 1e-3;   // finalize: entropy terms staged
  out_us[10] = t[10] ? (static_cast<double>(t[10]) - base) * 1e-3 : 0.0;  // peer exchange entered
  out_us[11] = t[11] ? (static_cast<double>(t[11]) - base) * 1e-3 : 0.0;  // all peers' contributions arrived
  MemPool::instance().pinned_free(ctx->h_timeline);
  ctx->h_timeline = nullptr;
  return rc;
}

// layout of the cudaIpc-shared allocation of a rank: [P2PMailbox (round-1 kernels) | pad | PkMailbox (persistent kernel)]
static constexpr size_t P2P_PK_OFFSET = (sizeof(P2PMailbox) + 255) & ~static_cast<size_t>(255);

int vlcal_nid_p2p_create(int device, int rank, int world, vlcal_p2p** out, void* ipc_handle_out) {
  if (!out || !ipc_handle_out || world < 1 || world > P2P_MAX_RANKS || rank < 0 || rank >= world) {
    set_last_error("invalid arguments (1 <= world <= 8)");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  if (vlcal_nid_device_count() == 0) {
    set_last_error("no CUDA device available");
    return VLCAL_ERR_NO_DEVICE;
  }
  if (device < 0) VL_CUDA(cudaGetDevice(&device));
  VL_CUDA(cudaSetDevice(device));
  std::unique_ptr<vlcal_p2p> p(new vlcal_p2p());
  p->device = device, p->rank = rank, p->world = world;
  VL_CUDA(cudaMalloc(reinterpret_cast<void**>(&p->local), P2P_PK_OFFSET + sizeof(PkMailbox)));  // own allocation: cudaIpc shares whole allocations
  VL_CUDA(cudaMemset(p->local, 0, P2P_PK_OFFSET + sizeof(PkMailbox)));
  VL_CUDA(cudaMalloc(reinterpret_cast<void**>(&p->d_counter), sizeof(unsigned long long)));
  VL_CUDA(cudaMemset(p->d_counter, 0, sizeof(unsigned long long)));
  VL_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&p->h_error), sizeof(int), cudaHostAllocDefault));
  *p->h_error = 0;
  cudaIpcMemHandle_t h;
  VL_CUDA(cudaIpcGetMemHandle(&h, p->local));
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
  std::memcpy(ipc_handle_out, &h, sizeof(h));
  p->peers[rank] = p->local;
  p->pk_peers[rank] = reinterpret_cast<PkMailbox*>(reinterpret_cast<char*>(p->local) + P2P_PK_OFFSET);
  *out = p.release();
  return VLCAL_OK;
}

int vlcal_nid_p2p_connect(vlcal_p2p* p, const void* all_handles) {
  if (!p || !all_handles) {
    set_last_error("invalid arguments");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  VL_CUDA(cudaSetDevice(p->device));
  for (int r = 0; r < p->world; r++) {
    if (r == p->rank) continue;
    cudaIpcMemHandle_t h;
    std::memcpy(&h, static_cast<const char*>(all_handles) + 64 * r, sizeof(h));
    void* ptr = nullptr;
    VL_CUDA(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
    p->peers[r] = static_cast<P2PMailbox*>(ptr);
    p->pk_peers[r] = reinterpret_cast<PkMailbox*>(static_cast<char*>(ptr) + P2P_PK_OFFSET);
  }
  p->connected = true;
  return VLCAL_OK;
}

int vlcal_nid_p2p_attach(vlcal_nid_ctx* ctx, vlcal_p2p* p) {
  if (!ctx) {
    set_last_error("ctx is NULL");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  if (p && (!p->connected || p->device != ctx->device)) {
    set_last_error("peer exchange is not connected or lives on another device");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  ctx->p2p = p;
  return VLCAL_OK;
}

void vlcal_nid_p2p_destroy(vlcal_p2p* p) {
  if (!p) return;
  cudaSetDevice(p->device);
  cudaDeviceSynchronize();
  for (int r = 0; r < p->world; r++) {
    if (r != p->rank && p->peers[r]) cudaIpcCloseMemHandle(p->peers[r]);
  }
  if (p->local) cudaFree(p->local);
  if (p->d_counter) cudaFree(p->d_counter);
  if (p->h_error) cudaFreeHost(p->h_error);
  delete p;
}

int vlcal_nid_reorder_for_pose(vlcal_nid_ctx* ctx, const double T_camera_lidar[16]) {
  if (!ctx || !T_camera_lidar) {
    set_last_error("invalid arguments");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  if (ctx->in_flight) {
    set_last_error("an evaluation is in flight on this context");
    return VLCAL_ERR_BUSY;
  }
  VL_CUDA(cudaSetDevice(ctx->device));
  VL_CUDA(cudaStreamSynchronize(ctx->stream));
  std::shared_ptr<DeviceCloud> sorted;
  int64_t kept = 0;
  const int rc = view_cull_device(ctx->cam, ctx->image->width, ctx->image->height, ctx->max_fov, false, *ctx->cloud, T_camera_lidar, nullptr, &sorted, nullptr, &kept, /*keep_all=*/true);
  if (rc != VLCAL_OK) return rc;
  if (kept != ctx->cloud->n) {
    set_last_error("reorder lost points");
    return VLCAL_ERR_CUDA;
  }
  ctx->cloud = sorted;
  return VLCAL_OK;
}

int vlcal_nid_trim_memory(void) {
  MemPool::instance().trim();
  return VLCAL_OK;
}

int vlcal_nid_filter_enabled(const vlcal_nid_ctx* ctx) {
  return ctx && ctx->fast.enabled && ctx->cloud->f32 ? 1 : 0;
}

int vlcal_nid_debug_filter_check(vlcal_nid_ctx* ctx, const double* T_camera_lidar, int n_poses, uint64_t counts[3], double* max_bound_ratio) {
  if (!ctx || !T_camera_lidar || n_poses <= 0 || !counts) {
    set_last_error("invalid arguments");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  if (!vlcal_nid_filter_enabled(ctx) || ctx->mode != VLCAL_NID_MODE_HISTOGRAM) {
    set_last_error("the fp32 filter is not enabled for this context (camera model / FoV / point layout)");
    return VLCAL_ERR_UNSUPPORTED;
  }
  VL_CUDA(cudaSetDevice(ctx->device));
  unsigned long long* d_dbg = nullptr;
  VL_CUDA(MemPool::instance().device_alloc(ctx->device, 4 * sizeof(unsigned long long), reinterpret_cast<void**>(&d_dbg)));
  VL_CUDA(cudaMemsetAsync(d_dbg, 0, 4 * sizeof(unsigned long long), ctx->stream));
  NidKernel kernel = pick_kernel(ctx->cam.model, true, 2);
  // contexts that run the lean classifier (persistent kernel) are checked with it; variant 4 checks the round-1 filter
  const bool lean = ctx->lean.enabled && ctx->variant != 4;
  for (int p0 = 0; p0 < n_poses; p0 += NID_MAX_POSES) {
    const int pc = std::min(NID_MAX_POSES, n_poses - p0);
    NidArgs a;
    std::memset(&a, 0, sizeof(a));
    a.points = ctx->cloud->d_points;
    a.bin_image = ctx->d_bin_image;
    a.n = ctx->cloud->n;
    a.width = ctx->image->width;
    a.height = ctx->image->height;
    a.bins = ctx->bins;
    a.nb = ctx->bins * ctx->bins;
    a.n_poses = pc;
    a.cos_fov = ctx->cos_fov;
    a.cam = ctx->cam;
    for (int p = 0; p < pc; p++) {
      const double* T = T_camera_lidar + 16 * static_cast<size_t>(p0 + p);
      for (int r = 0; r < 3; r++)
        for (int c = 0; c < 4; c++) a.pose[p][4 * r + c] = T[r + 4 * c];
    }
    fill_pose32(a, pc);
    a.fast = ctx->fast;
    a.dbg = d_dbg;
    const long long want_blocks = (a.n + NID_THREADS - 1) / NID_THREADS;
    const int grid = static_cast<int>(std::max<long long>(1, std::min<long long>(want_blocks, static_cast<long long>(ctx->num_sms) * 4)));
    if (lean) {
      switch (ctx->cam.model) {
        case CAM_PLUMB_BOB: nid_lean_verify_kernel<CAM_PLUMB_BOB><<<grid, NID_THREADS, 0, ctx->stream>>>(a, ctx->lean); break;
        case CAM_FISHEYE: nid_lean_verify_kernel<CAM_FISHEYE><<<grid, NID_THREADS, 0, ctx->stream>>>(a, ctx->lean); break;
        case CAM_ATAN: nid_lean_verify_kernel<CAM_ATAN><<<grid, NID_THREADS, 0, ctx->stream>>>(a, ctx->lean); break;
        case CAM_OMNIDIR: nid_lean_verify_kernel<CAM_OMNIDIR><<<grid, NID_THREADS, 0, ctx->stream>>>(a, ctx->lean); break;
        case CAM_EQUIRECTANGULAR: nid_lean_verify_kernel<CAM_EQUIRECTANGULAR><<<grid, NID_THREADS, 0, ctx->stream>>>(a, ctx->lean); break;
        default: nid_lean_verify_kernel<CAM_RATIONAL_POLYNOMIAL><<<grid, NID_THREADS, 0, ctx->stream>>>(a, ctx->lean); break;
      }
    } else {
      kernel<<<grid, NID_THREADS, 0, ctx->stream>>>(a);
    }
    VL_CUDA(cudaGetLastError());
  }
  unsigned long long h[4];
  VL_CUDA(cudaMemcpyAsync(h, d_dbg, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
  VL_CUDA(cudaStreamSynchronize(ctx->stream));
  MemPool::instance().device_free(ctx->device, d_dbg);
  counts[0] = h[0], counts[1] = h[1], counts[2] = h[2];
  if (max_bound_ratio) {
    const unsigned int bits = static_cast<unsigned int>(h[3] & 0xffffffffu);
    float f;
    std::memcpy(&f, &bits, sizeof(f));
    *max_bound_ratio = f;
  }
  return VLCAL_OK;
}


}  // extern "C"
