// nid_context.cuh -- internal C++ types behind the C ABI (include/vlcal_nid.h).
#pragma once

#include <cuda_runtime.h>

#include <cstdint>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "camera_models.cuh"
#include "lean_filter.cuh"
#include "vlcal_nid.h"

namespace vlcal {

void set_last_error(const std::string& msg);
int cuda_fail(cudaError_t e, const char* what, const char* file, int line);

#define VL_CUDA(expr)                                                   \
  do {                                                                  \
    cudaError_t e__ = (expr);                                           \
    if (e__ != cudaSuccess) return cuda_fail(e__, #expr, __FILE__, __LINE__); \
  } while (0)

// validated camera (create_camera.cpp:17-32 rules)
int make_camera(int model, const double* intr, int n_intr, const double* dist, int n_dist, CameraParams* out);
// estimate_camera_fov (estimate_fov.cpp:36-51)
double estimate_camera_fov_host(const CameraParams& cam, int width, int height);

// a cloud resident in HBM: float4 (x,y,z,intensity) when lossless, double4 otherwise
struct DeviceCloud {
  void* d_points = nullptr;
  int64_t n = 0;
  bool f32 = true;
  int device = 0;
  ~DeviceCloud();
  size_t bytes_per_point() const { return f32 ? 16 : 32; }
};

// a grayscale image resident in HBM (tight rows)
struct DeviceImage {
  uint8_t* d_raw = nullptr;  // H x W u8
  int width = 0, height = 0;
  int device = 0;
  ~DeviceImage();
};

int upload_cloud(int device, const double* points_xyzw, const double* intensities, int64_t n, cudaStream_t stream, std::shared_ptr<DeviceCloud>* out);
int upload_image(int device, const uint8_t* image, int width, int height, int row_stride, cudaStream_t stream, std::shared_ptr<DeviceImage>* out);

// GPU ViewCulling (view_culling.cpp:21-92): returns a compacted cloud and/or the kept indices
int view_cull_device(
  const CameraParams& cam, int width, int height, double max_fov, bool depth_culling, const DeviceCloud& cloud, const double T[16], cudaStream_t stream,
  std::shared_ptr<DeviceCloud>* culled_out, int32_t* indices_host_out, int64_t* n_kept, bool keep_all = false);

struct ProfileEvents {
  cudaEvent_t start, stop;
  int poses;
};

}  // namespace vlcal

namespace vlcal {
struct P2PMailbox;
struct PkMailbox;
}

// one per process: this rank's mailbox + the mapped mailboxes of the peers (vlcal_nid_p2p_*)
struct vlcal_p2p {
  int device = 0, rank = 0, world = 1;
  vlcal::P2PMailbox* local = nullptr;
  vlcal::P2PMailbox* peers[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  // the persistent kernel's mailbox (nid_persistent.cuh) lives in the same cudaIpc-shared allocation, behind the first one
  vlcal::PkMailbox* pk_peers[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  bool connected = false;
  unsigned long long* d_counter = nullptr;  // device word: exchanges done (advanced by the kernels)
  int* h_error = nullptr;  // pinned + mapped
};

struct vlcal_nid_ctx {
  int device = 0;
  int mode = 0;
  int bins = 16;
  int variant = 0;
  double max_fov = 0.0;
  double cos_fov = 0.0;
  vlcal::CameraParams cam{};
  vlcal::FastCam fast{};
  vlcal::LeanCam lean{};  // lean classifier constants (lean_filter.cuh); lean.enabled == 0: round-1 kernels only
  std::shared_ptr<vlcal::DeviceCloud> cloud;
  std::shared_ptr<vlcal::DeviceImage> image;
  uint8_t* d_bin_image = nullptr;
  cudaStream_t stream = nullptr;
  // accumulators / outputs
  int* d_ghist = nullptr;
  unsigned int* d_counter = nullptr;
  double* d_nid = nullptr;
  int d_nid_cap = 0;
  int* d_hist_out = nullptr;
  size_t d_hist_out_cap = 0;
  double* h_nid = nullptr;  // pinned + mapped: the finalize block writes the scores here directly (zero-copy)
  int h_nid_cap = 0;
  unsigned long long* h_flag = nullptr;  // pinned + mapped completion word polled by nid_wait
  unsigned long long seq = 0;
  // launch geometry
  int max_poses = 1;
  int num_sms = 132;  // read from the device at create
  // async state
  bool in_flight = false;
  int in_flight_poses = 0;
  vlcal_p2p* p2p = nullptr;  // attached peer exchange (not owned)
  // debug timeline (vlcal_nid_debug_timeline)
  unsigned long long* h_timeline = nullptr;  // pinned + mapped [16]
  // profiling
  bool profiling = false;
  std::vector<vlcal::ProfileEvents> events;
  size_t events_used = 0;
  int64_t launches = 0;
  int64_t timed_launches = 0;  // launches bracketed by events (profiling samples 1 launch in PROFILE_STRIDE)
  int64_t launch_counter = 0;
  int64_t poses_total = 0;
  int64_t passes = 0;  // passes over the cloud (a persistent launch carries one per Nelder-Mead batch / pose chunk)
  double kernel_ms_accum = 0.0;
  // debug: globaltimer stamps of the persistent kernel's batches (vlcal_nid_debug_solve_stamps)
  int pk_chunk = 8;  // poses per pass of the persistent kernel's pose-list mode (vlcal_nid_set_poses_per_pass)
  int pk_stamps_cap = 0;
  std::vector<unsigned long long> pk_stamps;
  unsigned long long pk_tma_stats[2] = {0, 0};  // TMA variant, last solve: gathers served by the staged window / escaped to global memory
  std::vector<unsigned long long> pk_block_times;  // [grid][4] of one batch (vlcal_nid_debug_block_times)

  ~vlcal_nid_ctx();
};

namespace vlcal {
int nid_ctx_create(
  int device, int mode, const CameraParams& cam, std::shared_ptr<DeviceImage> image, std::shared_ptr<DeviceCloud> cloud, int bins, double max_fov, vlcal_nid_ctx** out);
int nid_evaluate_async(vlcal_nid_ctx* ctx, const double* T_colmajor, int n_poses, bool want_hist);
int nid_wait(vlcal_nid_ctx* ctx, double* nid_out, int32_t* hist_out);
struct NmDevice;
// device-resident solver loop: enqueue `count` launches that read their poses from / advance `d_nm`; no waiting
int nid_enqueue_device_steps(vlcal_nid_ctx* ctx, NmDevice* d_nm, int count);
// after the stream was synchronised: account the first `worked` launches of the last enqueue in the profile
int nid_account_device_steps(vlcal_nid_ctx* ctx, int enqueued, int worked, int poses);

// persistent cooperative kernel (nid_persistent.cu): can these contexts (bags of one camera on one device) run on it?
bool pk_supported(vlcal_nid_ctx* const* ctxs, int n_ctxs);
// a whole Nelder-Mead inner solve (visual_camera_calibration.cpp:103-129) in one launch; sums over the peer exchange
// attached to ctxs[0] when it spans several ranks
int pk_solve(
  vlcal_nid_ctx* const* ctxs, int n_ctxs, const vlcal_calib_params* params, const double init_T[16], vlcal_pose_callback callback, void* user, double T_out[16],
  vlcal_nm_result* nm_result);
// sum over the contexts of calculate(T_p) for a pose list of any length, one launch (hist_out: bag 0's joint histograms)
int pk_score_poses(vlcal_nid_ctx* const* ctxs, int n_ctxs, const double* T_colmajor, int n_poses, double* nid_out, int32_t* hist_out);
}  // namespace vlcal
