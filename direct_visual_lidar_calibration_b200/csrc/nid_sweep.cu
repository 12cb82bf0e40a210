// nid_sweep.cu -- host side of K1s (nid_sweep.cuh): scores a long pose list, given on the host or as a search set whose
// poses are generated on the device, on small clouds with one block per group of poses; above SWEEP_MAX_POINTS the entry
// points hand the list to the persistent kernel's pose-list mode (nid_persistent.cu), which wins there.
#include "nid_sweep.cuh"

#include <algorithm>
#include <climits>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "mem_pool.hpp"
#include "nid_context.cuh"

namespace vlcal {

// Cloud size (points of all bags together) above which the pose list goes to the persistent kernel instead.  Measured with
// tools/initial_guess_search_probe.py on an NVIDIA H100 80GB HBM3 (700 W limit): see DESIGN.md section 4e for the table
// this constant is read from.
constexpr long long SWEEP_MAX_POINTS = 262144;

using SweepKernel = void (*)(const SweepArgs);

static SweepKernel sweep_pick(int model) {
  switch (model) {
    case CAM_PLUMB_BOB: return nid_pose_sweep_kernel<CAM_PLUMB_BOB>;
    case CAM_FISHEYE: return nid_pose_sweep_kernel<CAM_FISHEYE>;
    case CAM_ATAN: return nid_pose_sweep_kernel<CAM_ATAN>;
    case CAM_OMNIDIR: return nid_pose_sweep_kernel<CAM_OMNIDIR>;
    case CAM_EQUIRECTANGULAR: return nid_pose_sweep_kernel<CAM_EQUIRECTANGULAR>;
    case CAM_RATIONAL_POLYNOMIAL: return nid_pose_sweep_kernel<CAM_RATIONAL_POLYNOMIAL>;
    default: return nullptr;
  }
}

namespace {

struct DevBuf {
  void* p = nullptr;
  int device = 0;
  ~DevBuf() { MemPool::instance().device_free(device, p); }
};
struct PinBuf {
  void* p = nullptr;
  ~PinBuf() { MemPool::instance().pinned_free(p); }
};
struct EventPair {
  cudaEvent_t start = nullptr, stop = nullptr;
  ~EventPair() {
    if (start) cudaEventDestroy(start);
    if (stop) cudaEventDestroy(stop);
  }
};

std::mutex g_sweep_mu;
std::map<std::pair<int, const void*>, int> g_sweep_occupancy;  // (device, kernel) -> co-resident blocks per SM

thread_local double g_last_kernel_ms = 0.0;
thread_local long long g_last_deferred = -1;  // of vlcal_nid_debug_sweep_kernel; -1 after the other entry points

// the sweep covers what the persistent kernel covers (float4 clouds, bins <= 32, a camera with the lean classifier, one
// camera / image size / device for all bags): everything else is refused, and every accepted list can also take the
// persistent kernel above the size threshold
int sweep_check(vlcal_nid_ctx* const* ctxs, int n_ctxs) {
  if (!ctxs || n_ctxs <= 0) {
    set_last_error("invalid arguments");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  for (int i = 0; i < n_ctxs; i++) {
    if (!ctxs[i]) {
      set_last_error("NULL context");
      return VLCAL_ERR_INVALID_ARGUMENT;
    }
  }
  if (n_ctxs > SW_MAX_BAGS) {
    set_last_error("pose sweep: at most " + std::to_string(SW_MAX_BAGS) + " contexts per call");
    return VLCAL_ERR_UNSUPPORTED;
  }
  for (int i = 0; i < n_ctxs; i++) {
    const vlcal_nid_ctx* c = ctxs[i];
    if (c->mode != VLCAL_NID_MODE_HISTOGRAM) {
      set_last_error("pose sweep: mode-A (histogram) contexts only");
      return VLCAL_ERR_UNSUPPORTED;
    }
    if (c->bins > SW_MAX_BINS) {
      set_last_error("pose sweep: bins = " + std::to_string(c->bins) + " exceeds " + std::to_string(SW_MAX_BINS));
      return VLCAL_ERR_UNSUPPORTED;
    }
    if (!c->cloud->f32) {
      set_last_error("pose sweep: the cloud is stored in the double layout (coordinates or intensities not float32-representable); float4 clouds only");
      return VLCAL_ERR_UNSUPPORTED;
    }
    if (c->in_flight) {
      set_last_error("pose sweep: an asynchronous evaluation is in flight on a context");
      return VLCAL_ERR_BUSY;
    }
  }
  if (!pk_supported(ctxs, n_ctxs)) {
    set_last_error("pose sweep: the contexts must share device, camera, image size, bins and max_fov, and the camera must have the fp32 filter");
    return VLCAL_ERR_UNSUPPORTED;
  }
  return VLCAL_OK;
}

long long total_points(vlcal_nid_ctx* const* ctxs, int n_ctxs) {
  long long n = 0;
  for (int i = 0; i < n_ctxs; i++) n += ctxs[i]->cloud->n;
  return n;
}

int sweep_blocks_per_sm(int device, SweepKernel kernel, int* out) {
  std::lock_guard<std::mutex> lock(g_sweep_mu);
  const auto key = std::make_pair(device, reinterpret_cast<const void*>(kernel));
  auto it = g_sweep_occupancy.find(key);
  if (it == g_sweep_occupancy.end()) {
    int nblk = 0;
    VL_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nblk, kernel, SW_THREADS, 0));
    it = g_sweep_occupancy.emplace(key, std::max(1, nblk)).first;
  }
  *out = it->second;
  return VLCAL_OK;
}

// scores of the device pose list d_poses [n_poses][12] -> nid_out (host), bag 0's histograms -> hist_out (host, optional)
int sweep_launch(vlcal_nid_ctx* const* ctxs, int n_ctxs, const double* d_poses, int64_t n_poses, double* nid_out, int32_t* hist_out, int64_t* inliers_out = nullptr,
                 bool count_deferred = false) {
  vlcal_nid_ctx* c0 = ctxs[0];
  const SweepKernel kernel = sweep_pick(c0->cam.model);
  if (!kernel) {
    set_last_error("pose sweep: unknown camera model");
    return VLCAL_ERR_UNKNOWN_CAMERA_MODEL;
  }
  const int nb = c0->bins * c0->bins;
  int per_sm = 1;
  {
    const int rc = sweep_blocks_per_sm(c0->device, kernel, &per_sm);
    if (rc != VLCAL_OK) return rc;
  }
  const long long groups = (n_poses + SW_POSES - 1) / SW_POSES;
  const int grid = static_cast<int>(std::min<long long>(groups, static_cast<long long>(per_sm) * c0->num_sms));

  DevBuf d_scores, d_hist, d_inl, d_def;
  d_scores.device = d_hist.device = d_inl.device = d_def.device = c0->device;
  static_assert(sizeof(long long) == sizeof(int64_t), "inlier counts are copied out as int64_t");
  if (inliers_out) VL_CUDA(MemPool::instance().device_alloc(c0->device, sizeof(long long) * static_cast<size_t>(n_poses), &d_inl.p));
  VL_CUDA(MemPool::instance().device_alloc(c0->device, sizeof(double) * static_cast<size_t>(n_poses), &d_scores.p));
  if (hist_out) VL_CUDA(MemPool::instance().device_alloc(c0->device, sizeof(int) * static_cast<size_t>(n_poses) * nb, &d_hist.p));
  unsigned long long deferred = 0;
  if (count_deferred) {
    VL_CUDA(MemPool::instance().device_alloc(c0->device, sizeof(unsigned long long), &d_def.p));
    VL_CUDA(cudaMemsetAsync(d_def.p, 0, sizeof(unsigned long long), c0->stream));
  }

  SweepArgs a;
  std::memset(&a, 0, sizeof(a));
  for (int i = 0; i < n_ctxs; i++) {
    a.bag[i].points = static_cast<const float4*>(ctxs[i]->cloud->d_points);
    a.bag[i].bin_image = ctxs[i]->d_bin_image;
    a.bag[i].n = static_cast<unsigned int>(ctxs[i]->cloud->n);
  }
  a.n_bags = n_ctxs;
  a.width = c0->image->width, a.height = c0->image->height;
  a.bins = c0->bins, a.nb = nb;
  a.cos_fov = c0->cos_fov;
  a.cam = c0->cam;
  a.fast = c0->fast;
  a.lean = c0->lean;
  a.poses = d_poses;
  a.n_poses = n_poses;
  a.scores = static_cast<double*>(d_scores.p);
  a.hist_out = static_cast<int*>(d_hist.p);
  a.inliers = static_cast<long long*>(d_inl.p);
  a.deferred = static_cast<unsigned long long*>(d_def.p);

  EventPair ev;
  VL_CUDA(cudaEventCreate(&ev.start));
  VL_CUDA(cudaEventCreate(&ev.stop));
  VL_CUDA(cudaEventRecord(ev.start, c0->stream));
  kernel<<<grid, SW_THREADS, 0, c0->stream>>>(a);
  VL_CUDA(cudaGetLastError());
  VL_CUDA(cudaEventRecord(ev.stop, c0->stream));
  VL_CUDA(cudaMemcpyAsync(nid_out, d_scores.p, sizeof(double) * static_cast<size_t>(n_poses), cudaMemcpyDeviceToHost, c0->stream));
  if (hist_out) VL_CUDA(cudaMemcpyAsync(hist_out, d_hist.p, sizeof(int) * static_cast<size_t>(n_poses) * nb, cudaMemcpyDeviceToHost, c0->stream));
  if (inliers_out) VL_CUDA(cudaMemcpyAsync(inliers_out, d_inl.p, sizeof(int64_t) * static_cast<size_t>(n_poses), cudaMemcpyDeviceToHost, c0->stream));
  if (count_deferred) VL_CUDA(cudaMemcpyAsync(&deferred, d_def.p, sizeof(deferred), cudaMemcpyDeviceToHost, c0->stream));
  VL_CUDA(cudaStreamSynchronize(c0->stream));
  g_last_deferred = count_deferred ? static_cast<long long>(deferred) : -1;
  float ms = 0.f;
  VL_CUDA(cudaEventElapsedTime(&ms, ev.start, ev.stop));
  g_last_kernel_ms = ms;
  c0->launches += 1;
  c0->poses_total += n_poses;
  return VLCAL_OK;
}

// the list through the persistent kernel: P x 16 column-major host poses
int sweep_fallback(vlcal_nid_ctx* const* ctxs, int n_ctxs, const double* T_colmajor, int64_t n_poses, double* nid_out, int32_t* hist_out) {
  if (n_poses > INT_MAX) {
    set_last_error("pose sweep: more than 2^31 - 1 poses on clouds beyond the sweep's size");
    return VLCAL_ERR_UNSUPPORTED;
  }
  g_last_kernel_ms = 0.0;
  g_last_deferred = -1;
  return pk_score_poses(ctxs, n_ctxs, T_colmajor, static_cast<int>(n_poses), nid_out, hist_out);
}

// the same with the inlier counts: they are the sums of the joint histograms, which the persistent kernel delivers for one
// bag per launch, so every bag is scored on its own and the scores are added in bag order as that kernel adds them
int sweep_fallback_inliers(vlcal_nid_ctx* const* ctxs, int n_ctxs, const double* T_colmajor, int64_t n_poses, double* nid_out, int64_t* inliers_out) {
  if (n_poses > INT_MAX) {
    set_last_error("pose sweep: more than 2^31 - 1 poses on clouds beyond the sweep's size");
    return VLCAL_ERR_UNSUPPORTED;
  }
  g_last_kernel_ms = 0.0;
  g_last_deferred = -1;
  const size_t nb = static_cast<size_t>(ctxs[0]->bins) * ctxs[0]->bins;
  std::vector<int32_t> hist(static_cast<size_t>(n_poses) * nb);
  std::vector<double> part(static_cast<size_t>(n_poses));
  for (int64_t p = 0; p < n_poses; p++) inliers_out[p] = 0, nid_out[p] = 0.0;
  for (int b = 0; b < n_ctxs; b++) {
    const int rc = pk_score_poses(ctxs + b, 1, T_colmajor, static_cast<int>(n_poses), part.data(), hist.data());
    if (rc != VLCAL_OK) return rc;
    for (int64_t p = 0; p < n_poses; p++) {
      nid_out[p] = n_ctxs == 1 ? part[p] : nid_out[p] + part[p];
      int64_t s = 0;
      for (size_t k = 0; k < nb; k++) s += hist[static_cast<size_t>(p) * nb + k];
      inliers_out[p] += s;
    }
  }
  return VLCAL_OK;
}

int sweep_host_list(vlcal_nid_ctx* const* ctxs, int n_ctxs, const double* T_colmajor, int64_t n_poses, double* nid_out, int32_t* hist_out, bool may_fall_back) {
  {
    const int rc = sweep_check(ctxs, n_ctxs);
    if (rc != VLCAL_OK) return rc;
  }
  if (!T_colmajor || n_poses <= 0 || !nid_out) {
    set_last_error("invalid arguments");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  if (may_fall_back && total_points(ctxs, n_ctxs) > SWEEP_MAX_POINTS) return sweep_fallback(ctxs, n_ctxs, T_colmajor, n_poses, nid_out, hist_out);
  vlcal_nid_ctx* c0 = ctxs[0];
  VL_CUDA(cudaSetDevice(c0->device));
  const size_t pose_bytes = sizeof(double) * 12 * static_cast<size_t>(n_poses);
  DevBuf d_poses;
  d_poses.device = c0->device;
  PinBuf host;
  VL_CUDA(MemPool::instance().device_alloc(c0->device, pose_bytes, &d_poses.p));
  VL_CUDA(MemPool::instance().pinned_alloc(pose_bytes, &host.p));
  double* hpose = static_cast<double*>(host.p);
  for (int64_t p = 0; p < n_poses; p++) {
    const double* T = T_colmajor + 16 * static_cast<size_t>(p);
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 4; c++) hpose[12 * static_cast<size_t>(p) + 4 * r + c] = T[r + 4 * c];
  }
  VL_CUDA(cudaMemcpyAsync(d_poses.p, hpose, pose_bytes, cudaMemcpyHostToDevice, c0->stream));
  return sweep_launch(ctxs, n_ctxs, static_cast<const double*>(d_poses.p), n_poses, nid_out, hist_out, nullptr, /*count_deferred=*/!may_fall_back);
}

int search_set_check(const vlcal_search_set* s) {
  if (!s || !s->left || !s->base || !s->center || !s->offset || s->n_left <= 0 || s->n_base <= 0 || s->n_offset <= 0 || s->n_poses <= 0) {
    set_last_error("search set: NULL table or non-positive count");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  const long long full = static_cast<long long>(s->n_left) * s->n_base * s->n_offset;
  if (full > INT_MAX) {
    set_last_error("search set: more than 2^31 - 1 combinations");
    return VLCAL_ERR_UNSUPPORTED;
  }
  if (!s->indices && s->n_poses != full) {
    set_last_error("search set: n_poses must equal n_base * n_left * n_offset when no indices are given");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  if (s->indices) {
    for (int64_t j = 0; j < s->n_poses; j++) {
      if (s->indices[j] < 0 || s->indices[j] >= full) {
        set_last_error("search set: index out of range");
        return VLCAL_ERR_INVALID_ARGUMENT;
      }
    }
  }
  return VLCAL_OK;
}

// uploads the tables and generates the [n_poses][12] pose list on `stream`; `tables` keeps the uploads alive
int search_set_generate(int device, const vlcal_search_set* s, cudaStream_t stream, DevBuf* tables, DevBuf* d_poses) {
  const size_t nl = sizeof(double) * 9 * s->n_left, nbs = sizeof(double) * 9 * s->n_base, nc = sizeof(double) * 3 * s->n_base, no = sizeof(double) * 3 * s->n_offset;
  const size_t ni = s->indices ? sizeof(int32_t) * static_cast<size_t>(s->n_poses) : 0;
  tables->device = d_poses->device = device;
  VL_CUDA(MemPool::instance().device_alloc(device, nl + nbs + nc + no + ni, &tables->p));
  VL_CUDA(MemPool::instance().device_alloc(device, sizeof(double) * 12 * static_cast<size_t>(s->n_poses), &d_poses->p));
  char* d = static_cast<char*>(tables->p);
  SearchSetDev dev;
  std::memset(&dev, 0, sizeof(dev));
  // pageable sources: cudaMemcpyAsync stages them before it returns, so the caller's tables may go away afterwards
  VL_CUDA(cudaMemcpyAsync(d, s->left, nl, cudaMemcpyHostToDevice, stream));
  dev.left = reinterpret_cast<const double*>(d);
  d += nl;
  VL_CUDA(cudaMemcpyAsync(d, s->base, nbs, cudaMemcpyHostToDevice, stream));
  dev.base = reinterpret_cast<const double*>(d);
  d += nbs;
  VL_CUDA(cudaMemcpyAsync(d, s->center, nc, cudaMemcpyHostToDevice, stream));
  dev.center = reinterpret_cast<const double*>(d);
  d += nc;
  VL_CUDA(cudaMemcpyAsync(d, s->offset, no, cudaMemcpyHostToDevice, stream));
  dev.offset = reinterpret_cast<const double*>(d);
  d += no;
  if (s->indices) {
    VL_CUDA(cudaMemcpyAsync(d, s->indices, ni, cudaMemcpyHostToDevice, stream));
    dev.indices = reinterpret_cast<const int*>(d);
  }
  dev.n_left = s->n_left, dev.n_base = s->n_base, dev.n_offset = s->n_offset;
  dev.n_poses = s->n_poses;
  const int threads = 128;
  const long long blocks = (s->n_poses + threads - 1) / threads;
  search_set_poses_kernel<<<static_cast<unsigned int>(blocks), threads, 0, stream>>>(dev, static_cast<double*>(d_poses->p));
  VL_CUDA(cudaGetLastError());
  return VLCAL_OK;
}

// device rows [n][12] -> host P x 16 column-major
int poses_to_host_colmajor(const double* d_poses, int64_t n, cudaStream_t stream, std::vector<double>* rows, double* T_out) {
  rows->resize(12 * static_cast<size_t>(n));
  VL_CUDA(cudaMemcpyAsync(rows->data(), d_poses, sizeof(double) * rows->size(), cudaMemcpyDeviceToHost, stream));
  VL_CUDA(cudaStreamSynchronize(stream));
  for (int64_t p = 0; p < n; p++) {
    double* T = T_out + 16 * static_cast<size_t>(p);
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 4; c++) T[r + 4 * c] = (*rows)[12 * static_cast<size_t>(p) + 4 * r + c];
    T[3] = T[7] = T[11] = 0.0;
    T[15] = 1.0;
  }
  return VLCAL_OK;
}

}  // namespace

}  // namespace vlcal

using namespace vlcal;

extern "C" {

int vlcal_nid_sweep_poses(vlcal_nid_ctx* const* ctxs, int n_ctxs, const double* T_camera_lidar, int64_t n_poses, double* nid_out, int32_t* hist_out) {
  return sweep_host_list(ctxs, n_ctxs, T_camera_lidar, n_poses, nid_out, hist_out, /*may_fall_back=*/true);
}

int vlcal_nid_debug_sweep_kernel(vlcal_nid_ctx* const* ctxs, int n_ctxs, const double* T_camera_lidar, int64_t n_poses, double* nid_out, int32_t* hist_out) {
  return sweep_host_list(ctxs, n_ctxs, T_camera_lidar, n_poses, nid_out, hist_out, /*may_fall_back=*/false);
}

int vlcal_nid_sweep_search_set(vlcal_nid_ctx* const* ctxs, int n_ctxs, const vlcal_search_set* set, double* nid_out) {
  return vlcal_nid_sweep_search_set_inliers(ctxs, n_ctxs, set, nid_out, nullptr);
}

int vlcal_nid_sweep_search_set_inliers(vlcal_nid_ctx* const* ctxs, int n_ctxs, const vlcal_search_set* set, double* nid_out, int64_t* inliers_out) {
  {
    int rc = sweep_check(ctxs, n_ctxs);
    if (rc == VLCAL_OK) rc = search_set_check(set);
    if (rc != VLCAL_OK) return rc;
  }
  if (!nid_out) {
    set_last_error("nid_out is NULL");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  vlcal_nid_ctx* c0 = ctxs[0];
  VL_CUDA(cudaSetDevice(c0->device));
  DevBuf tables, d_poses;
  {
    const int rc = search_set_generate(c0->device, set, c0->stream, &tables, &d_poses);
    if (rc != VLCAL_OK) return rc;
  }
  if (total_points(ctxs, n_ctxs) > SWEEP_MAX_POINTS) {
    std::vector<double> rows, T(16 * static_cast<size_t>(set->n_poses));
    const int rc = poses_to_host_colmajor(static_cast<const double*>(d_poses.p), set->n_poses, c0->stream, &rows, T.data());
    if (rc != VLCAL_OK) return rc;
    if (inliers_out) return sweep_fallback_inliers(ctxs, n_ctxs, T.data(), set->n_poses, nid_out, inliers_out);
    return sweep_fallback(ctxs, n_ctxs, T.data(), set->n_poses, nid_out, nullptr);
  }
  return sweep_launch(ctxs, n_ctxs, static_cast<const double*>(d_poses.p), set->n_poses, nid_out, nullptr, inliers_out);
}

int vlcal_search_set_poses(int device, const vlcal_search_set* set, double* T_camera_lidar_out) {
  {
    const int rc = search_set_check(set);
    if (rc != VLCAL_OK) return rc;
  }
  if (!T_camera_lidar_out) {
    set_last_error("T_camera_lidar_out is NULL");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  if (device < 0) VL_CUDA(cudaGetDevice(&device));
  VL_CUDA(cudaSetDevice(device));
  DevBuf tables, d_poses;
  {
    const int rc = search_set_generate(device, set, cudaStreamPerThread, &tables, &d_poses);
    if (rc != VLCAL_OK) return rc;
  }
  std::vector<double> rows;
  return poses_to_host_colmajor(static_cast<const double*>(d_poses.p), set->n_poses, cudaStreamPerThread, &rows, T_camera_lidar_out);
}

int vlcal_nid_sweep_launch_shape(const vlcal_nid_ctx* ctx, int* blocks, int* poses_per_block) {
  if (!ctx || !blocks || !poses_per_block) {
    set_last_error("invalid arguments");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  const SweepKernel kernel = sweep_pick(ctx->cam.model);
  if (!kernel) {
    set_last_error("pose sweep: unknown camera model");
    return VLCAL_ERR_UNKNOWN_CAMERA_MODEL;
  }
  VL_CUDA(cudaSetDevice(ctx->device));
  int per_sm = 1;
  const int rc = sweep_blocks_per_sm(ctx->device, kernel, &per_sm);
  if (rc != VLCAL_OK) return rc;
  *blocks = per_sm * ctx->num_sms;
  *poses_per_block = SW_POSES;
  return VLCAL_OK;
}

int64_t vlcal_nid_sweep_max_points(void) { return SWEEP_MAX_POINTS; }

double vlcal_nid_sweep_last_kernel_ms(void) { return g_last_kernel_ms; }

int64_t vlcal_nid_debug_sweep_last_deferred(void) { return g_last_deferred; }

}  // extern "C"
