// nid_persistent.cu -- host side of K1p (nid_persistent.cuh): the persistent cooperative kernel that runs a whole
// Nelder-Mead inner solve (VisualCameraCalibration::estimate_pose_nelder_mead's optimizer loop,
// src/vlcal/calib/visual_camera_calibration.cpp:103-127) or scores an arbitrarily long pose list
// (CostCalculatorNID::calculate per pose, src/vlcal/calib/cost_calculator_nid.cpp:21-67) in ONE launch.
#include "nid_persistent.cuh"

#include <cuda.h>  // CUtensorMap + cuTensorMapEncodeTiled's signature (resolved through cudaGetDriverEntryPoint: no libcuda link)

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <tuple>
#include <vector>

#include "host_math.hpp"
#include "mem_pool.hpp"
#include "nid_context.cuh"

namespace vlcal {

using PkKernel = void (*)(const PkArgs);

// points per lane and tile: 2 or 4 for the light models, 2 for the ones that carry transcendental calls (more live state
// per point); atom: histogram-increment form (nid_persistent.cuh)
#ifndef PK_K4_ALL
#define PK_K4_ALL 0  // A/B builds: also instantiate 4 points per lane for the models whose classifier is register-heavy
#endif
template <int MODEL>
static PkKernel pk_pick_ka(int k, int atom) {
  constexpr bool heavy = MODEL == CAM_FISHEYE || MODEL == CAM_EQUIRECTANGULAR || MODEL == CAM_ATAN;
  if constexpr (!heavy || PK_K4_ALL) {
    if (k == 4) return atom ? nid_persistent_kernel<MODEL, 4, 1> : nid_persistent_kernel<MODEL, 4, 0>;
  }
  return atom ? nid_persistent_kernel<MODEL, 2, 1> : nid_persistent_kernel<MODEL, 2, 0>;
}

static int pk_tma_requested() {
  static const int v = [] {
    const char* e = std::getenv("VLCAL_PK_TMA");
    return e ? std::atoi(e) : 0;  // A/B: the staged window did not pay for its index arithmetic -> off
  }();
  return v;
}

// TMA variant: instantiated for the C2 shape only (plumb_bob, 2 points per lane, merged increments)
static PkKernel pk_pick_tma(int model, int k) {
  if (model == CAM_PLUMB_BOB && k == 2) return nid_persistent_kernel<CAM_PLUMB_BOB, 2, 0, true>;
  return nullptr;
}

// tensor map of an image-bin plane: u8, W x H, tight rows, box 256 x 1, out-of-bounds bytes read as zero
static int pk_make_tensor_map(const uint8_t* img, int width, int height, PkTensorMap* out) {
  using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static EncodeFn encode = [] {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || qres != cudaDriverEntryPointSuccess) fn = nullptr;
    cudaGetLastError();
    return reinterpret_cast<EncodeFn>(fn);
  }();
  if (!encode) {
    set_last_error("cuTensorMapEncodeTiled is not available from this driver");
    return VLCAL_ERR_UNSUPPORTED;
  }
  static_assert(sizeof(CUtensorMap) == sizeof(PkTensorMap), "CUtensorMap is 128 bytes");
  CUtensorMap m;
  const cuuint64_t gdim[2] = {static_cast<cuuint64_t>(width), static_cast<cuuint64_t>(height)};
  const cuuint64_t gstride[1] = {static_cast<cuuint64_t>(width)};  // bytes between rows (multiple of 16: checked by the caller)
  const cuuint32_t box[2] = {static_cast<cuuint32_t>(PK_TMA_BOX_W), 1u};
  const cuuint32_t estride[2] = {1u, 1u};
  const CUresult r = encode(&m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<uint8_t*>(img), gdim, gstride, box, estride, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                            CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed with code " + std::to_string(static_cast<int>(r)));
    return VLCAL_ERR_CUDA;
  }
  std::memcpy(out, &m, sizeof(m));
  return VLCAL_OK;
}

static PkKernel pk_pick(int model, int k) {
  static const int atom = [] {
    const char* e = std::getenv("VLCAL_PK_ATOM");
    return e ? (std::atoi(e) != 0 ? 1 : 0) : 0;
  }();
  switch (model) {
    case CAM_PLUMB_BOB: return pk_pick_ka<CAM_PLUMB_BOB>(k, atom);
    case CAM_FISHEYE: return pk_pick_ka<CAM_FISHEYE>(k, atom);
    case CAM_ATAN: return pk_pick_ka<CAM_ATAN>(k, atom);
    case CAM_OMNIDIR: return pk_pick_ka<CAM_OMNIDIR>(k, atom);
    case CAM_EQUIRECTANGULAR: return pk_pick_ka<CAM_EQUIRECTANGULAR>(k, atom);
    case CAM_RATIONAL_POLYNOMIAL: return pk_pick_ka<CAM_RATIONAL_POLYNOMIAL>(k, atom);
    default: return nullptr;
  }
}

struct PkGeom {
  int copies;
  size_t smem;
  int max_blocks;  // co-resident blocks of the whole device (cooperative launch limit)
};

static std::mutex g_pk_mu;
static std::map<std::tuple<int, const void*, size_t>, int> g_pk_occupancy;

static int pk_geometry(int device, int num_sms, PkKernel kernel, int nb, PkGeom* g, bool tma = false) {
  // histogram copies for 8 poses (the initial simplex of a 6-D solve is 7) -- two copies while they fit 64 KB
  const size_t per_copy = static_cast<size_t>(PK_MAX_POSES) * nb * sizeof(int);
  g->copies = static_cast<int>(std::max<size_t>(1, std::min<size_t>(PK_WARPS / 4, (64 * 1024) / per_copy)));  // one copy per four warps
  const size_t scratch = static_cast<size_t>(nb) * 8 + 64 * 8 * 2 + 64 * 4 * 2;  // pk_block_nid staging (aliases the copies)
  g->smem = std::max(per_copy * g->copies, scratch);
  if (tma) g->smem = ((g->smem + 127) & ~static_cast<size_t>(127)) + PK_TMA_BYTES;
  std::lock_guard<std::mutex> lock(g_pk_mu);
  const auto key = std::make_tuple(device, reinterpret_cast<const void*>(kernel), g->smem);
  auto it = g_pk_occupancy.find(key);
  if (it == g_pk_occupancy.end()) {
    VL_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(128 * 1024)));
    int nblk = 0;
    VL_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nblk, kernel, PK_THREADS, g->smem));
    it = g_pk_occupancy.emplace(key, std::max(1, nblk)).first;
  }
  g->max_blocks = it->second * num_sms;
  return VLCAL_OK;
}

static unsigned long long pk_timeout_ns() {
  static const unsigned long long v = [] {
    const char* e = std::getenv("VLCAL_SYNC_TIMEOUT_MS");
    const long long ms = e ? std::atoll(e) : 10000;  // a peer rank may enter its solve seconds later (upload / culling skew)
    return static_cast<unsigned long long>(std::max(10LL, ms)) * 1000000ull;
  }();
  return v;
}

// Points per lane and tile (K).  Tiles are dealt to the warps round-robin, so K = 4 (128-point tiles) needs a cloud large
// enough for several tiles per warp to stay balanced -- and there the lighter register footprint of K = 2 (768 threads per
// SM without spills in the pose loop, one packed register pair per coordinate) measured faster anyway.  K = 4 remains as variant 3 / VLCAL_PK_KPT=4 for A/B runs.
static int pk_points_per_lane(const vlcal_nid_ctx* ctx, long long /*total_points*/) {
  if (const char* e = std::getenv("VLCAL_PK_KPT")) return std::atoi(e) == 4 ? 4 : 2;
  return ctx->variant == 3 ? 4 : 2;
}

bool pk_supported(vlcal_nid_ctx* const* ctxs, int n_ctxs) {
  if (n_ctxs < 1 || n_ctxs > PK_MAX_BAGS) return false;
  const vlcal_nid_ctx* c0 = ctxs[0];
  for (int i = 0; i < n_ctxs; i++) {
    const vlcal_nid_ctx* c = ctxs[i];
    if (c->mode != VLCAL_NID_MODE_HISTOGRAM || c->variant == 1 || c->variant == 4 || !c->cloud->f32 || !c->lean.enabled || c->bins > PK_MAX_BINS || c->cloud->n >= 0x7fffffffLL) return false;
    if (c->device != c0->device || c->bins != c0->bins || c->image->width != c0->image->width || c->image->height != c0->image->height || c->max_fov != c0->max_fov) return false;
    if (std::memcmp(&c->cam, &c0->cam, sizeof(CameraParams)) != 0) return false;
    if (c->in_flight) return false;
  }
  return true;
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

// device scratch of one launch, one allocation, zeroed by one memset
struct PkScratchLayout {
  size_t ghist, gmarg, arrive, fin_done, tile_next, abort_flag, seq, tma_stats, box, solve, total;
  PkScratchLayout(int n_bags, int nb) {
    size_t o = 0;
    auto take = [&](size_t bytes) {
      const size_t at = o;
      o = (o + bytes + 255) & ~static_cast<size_t>(255);
      return at;
    };
    ghist = take(sizeof(int) * 3 * n_bags * PK_MAX_POSES * nb);  // three rotating buffers (Nelder-Mead mode), two used by the pose list
    gmarg = take(sizeof(int) * 3 * n_bags * PK_MAX_POSES * PK_MARG_STRIDE);
    arrive = take(sizeof(unsigned int) * 3 * PK_MAX_BAGS);
    fin_done = take(sizeof(unsigned int) * 2);
    tile_next = take(sizeof(unsigned int) * 2 * PK_MAX_BAGS);
    abort_flag = take(sizeof(unsigned int));
    seq = take(sizeof(unsigned long long));
    tma_stats = take(sizeof(unsigned long long) * 2);
    box = take(sizeof(PkMailbox));
    solve = take(sizeof(PkSolve));
    total = o;
  }
};

void pk_fill_common(PkArgs& a, vlcal_nid_ctx* const* ctxs, int n_ctxs, const PkGeom& g, int grid, char* scratch, const PkScratchLayout& L) {
  std::memset(&a, 0, sizeof(a));
  const vlcal_nid_ctx* c0 = ctxs[0];
  a.width = c0->image->width, a.height = c0->image->height;
  a.bins = c0->bins, a.nb = c0->bins * c0->bins;
  a.cos_fov = c0->cos_fov;
  a.cam = c0->cam;
  a.fast = c0->fast;
  a.lean = c0->lean;
  a.n_bags = n_ctxs;
  a.copies = g.copies;
  // blocks per bag in proportion to the point counts, at least one each
  long long total_points = 0;
  for (int i = 0; i < n_ctxs; i++) total_points += std::max<long long>(1, ctxs[i]->cloud->n);
  int assigned = 0;
  for (int i = 0; i < n_ctxs; i++) {
    const long long n = std::max<long long>(1, ctxs[i]->cloud->n);
    int share = i + 1 == n_ctxs ? grid - assigned : static_cast<int>(static_cast<double>(grid) * n / total_points + 0.5);
    share = std::max(1, std::min(share, grid - assigned - (n_ctxs - 1 - i)));
    a.bag[i].points = static_cast<const float4*>(ctxs[i]->cloud->d_points);
    a.bag[i].bin_image = ctxs[i]->d_bin_image;
    a.bag[i].n = static_cast<unsigned int>(ctxs[i]->cloud->n);
    a.bag[i].block_begin = assigned;
    a.bag[i].block_count = share;
    assigned += share;
  }
  a.ghist = reinterpret_cast<int*>(scratch + L.ghist);
  a.gmarg = reinterpret_cast<int*>(scratch + L.gmarg);
  a.arrive = reinterpret_cast<unsigned int*>(scratch + L.arrive);
  a.fin_done = reinterpret_cast<unsigned int*>(scratch + L.fin_done);
  a.abort_flag = reinterpret_cast<unsigned int*>(scratch + L.abort_flag);
  a.seq_counter = reinterpret_cast<unsigned long long*>(scratch + L.seq);
  a.box[0] = reinterpret_cast<PkMailbox*>(scratch + L.box);
  a.world = 1, a.rank = 0;
  a.timeout_ns = pk_timeout_ns();
}

int pk_grid_size(const PkGeom& g, vlcal_nid_ctx* const* ctxs, int n_ctxs) {
  long long total_points = 0;
  for (int i = 0; i < n_ctxs; i++) total_points += ctxs[i]->cloud->n;
  const long long want = std::max<long long>(n_ctxs, (total_points + PK_THREADS - 1) / PK_THREADS);
  return static_cast<int>(std::max<long long>(n_ctxs, std::min<long long>(want, g.max_blocks)));
}


}  // namespace

// ---- Nelder-Mead inner solve ----------------------------------------------------------------------------------------------

int pk_solve(
  vlcal_nid_ctx* const* ctxs, int n_ctxs, const vlcal_calib_params* params, const double init_T[16], vlcal_pose_callback callback, void* user, double T_out[16],
  vlcal_nm_result* nm_result) {
  vlcal_nid_ctx* c0 = ctxs[0];
  VL_CUDA(cudaSetDevice(c0->device));
  long long total_points = 0;
  for (int i = 0; i < n_ctxs; i++) total_points += ctxs[i]->cloud->n;
  const int kpt = pk_points_per_lane(c0, total_points);
  PkKernel kernel = pk_pick(c0->cam.model, kpt);
  // TMA variant (A/B): image windows staged in shared memory; needs 16-byte row pitches and 128-byte aligned histogram copies
  const size_t hist_bytes = static_cast<size_t>(std::max<size_t>(1, std::min<size_t>(PK_WARPS / 4, (64 * 1024) / (static_cast<size_t>(PK_MAX_POSES) * c0->bins * c0->bins * 4)))) * PK_MAX_POSES * c0->bins * c0->bins * 4;
  const bool use_tma = pk_tma_requested() != 0 && pk_pick_tma(c0->cam.model, kpt) != nullptr && c0->image->width % 16 == 0 && hist_bytes % 128 == 0;
  if (use_tma) kernel = pk_pick_tma(c0->cam.model, kpt);
  PkGeom g;
  {
    const int rc = pk_geometry(c0->device, c0->num_sms, kernel, c0->bins * c0->bins, &g, use_tma);
    if (rc != VLCAL_OK) return rc;
  }
  const int grid = pk_grid_size(g, ctxs, n_ctxs);
  const vlcal_p2p* px = c0->p2p && c0->p2p->connected && c0->p2p->world > 1 ? c0->p2p : nullptr;
  if (px && (px->world * n_ctxs * PK_MAX_POSES > PK_MAX_WORDS || !px->pk_peers[px->rank])) {
    set_last_error("peer exchange: world x local bags must be <= 32");
    return VLCAL_ERR_UNSUPPORTED;
  }

  const PkScratchLayout L(n_ctxs, c0->bins * c0->bins);
  DevBuf scratch;
  scratch.device = c0->device;
  VL_CUDA(MemPool::instance().device_alloc(c0->device, L.total, &scratch.p));
  VL_CUDA(cudaMemsetAsync(scratch.p, 0, L.total, c0->stream));

  // host-visible outcome: result + done / error words + evaluation trace, one pinned allocation
  const int trace_cap = 16 + std::max(0, params->max_inner_iterations) * 8;  // <= 7 evaluations per batch, one batch per iteration (+ shrinks)
  const size_t trace_bytes = sizeof(double) * (NM_MAX_N + 1) * static_cast<size_t>(trace_cap);
  const size_t head_bytes = (sizeof(PkResult) + sizeof(PkSolve) + 64 + 255) & ~static_cast<size_t>(255);
  PinBuf host;
  VL_CUDA(MemPool::instance().pinned_alloc(head_bytes + trace_bytes, &host.p));
  char* hp = static_cast<char*>(host.p);
  PkResult* h_result = reinterpret_cast<PkResult*>(hp);
  PkSolve* h_solve = reinterpret_cast<PkSolve*>(hp + sizeof(PkResult));
  unsigned long long* h_done = reinterpret_cast<unsigned long long*>(hp + sizeof(PkResult) + sizeof(PkSolve));
  int* h_error = reinterpret_cast<int*>(h_done + 1);
  double* h_trace = reinterpret_cast<double*>(hp + head_bytes);
  *h_done = 0ull;
  *h_error = 0;
  std::memset(static_cast<void*>(h_result), 0, sizeof(PkResult));

  NmParams nm;  // visual_camera_calibration.cpp:122-125
  nm.init_step = params->nelder_mead_init_step;
  nm.convergence_var_thresh = params->nelder_mead_convergence_criteria;
  nm.max_iterations = params->max_inner_iterations;
  std::memset(static_cast<void*>(h_solve), 0, sizeof(PkSolve));
  const double x0[6] = {0, 0, 0, 0, 0, 0};
  h_solve->nm.begin(6, nm, x0);  // :126 optimize(f, Zero)
  std::memcpy(h_solve->init_T, init_T, sizeof(h_solve->init_T));
  char* sp = static_cast<char*>(scratch.p);
  VL_CUDA(cudaMemcpyAsync(sp + L.solve, h_solve, sizeof(PkSolve), cudaMemcpyHostToDevice, c0->stream));

  PkArgs a;
  pk_fill_common(a, ctxs, n_ctxs, g, grid, sp, L);
  a.solve = reinterpret_cast<const PkSolve*>(sp + L.solve);
  if (use_tma) {
    for (int i = 0; i < n_ctxs; i++) {
      const int rc = pk_make_tensor_map(ctxs[i]->d_bin_image, c0->image->width, c0->image->height, &a.tmap[i]);
      if (rc != VLCAL_OK) return rc;
    }
    a.tma_stats = reinterpret_cast<unsigned long long*>(sp + L.tma_stats);
  }
  a.result_host = h_result;
  a.trace_host = h_trace;
  a.trace_cap = trace_cap;
  a.error_host = h_error;
  a.done_host = h_done;
  a.done_seq = 1ull;
  if (px) {
    for (int r = 0; r < px->world; r++) a.box[r] = px->pk_peers[r];
    a.world = px->world, a.rank = px->rank;
    a.seq_counter = px->d_counter;
  }
  DevBuf stamps;
  stamps.device = c0->device;
  if (c0->pk_stamps_cap > 0) {
    const size_t bytes = sizeof(unsigned long long) * PK_STAMP_SLOTS * static_cast<size_t>(c0->pk_stamps_cap);
    const size_t block_bytes = sizeof(unsigned long long) * 4 * static_cast<size_t>(grid);
    VL_CUDA(MemPool::instance().device_alloc(c0->device, bytes + block_bytes, &stamps.p));
    VL_CUDA(cudaMemsetAsync(stamps.p, 0, bytes + block_bytes, c0->stream));
    a.stamps = static_cast<unsigned long long*>(stamps.p);
    a.stamps_cap = c0->pk_stamps_cap;
    a.block_times = a.stamps + static_cast<size_t>(PK_STAMP_SLOTS) * c0->pk_stamps_cap;
    a.block_times_batch = std::min(8, c0->pk_stamps_cap - 1);
  }

  ProfileEvents ev{};
  const bool timed = c0->profiling;
  if (timed) {
    if (c0->events_used == c0->events.size()) {
      ProfileEvents e;
      VL_CUDA(cudaEventCreate(&e.start));
      VL_CUDA(cudaEventCreate(&e.stop));
      e.poses = 0;
      c0->events.push_back(e);
    }
    ev = c0->events[c0->events_used++];
    VL_CUDA(cudaEventRecord(ev.start, c0->stream));
  }
  void* kargs[] = {&a};
  VL_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<const void*>(kernel), dim3(grid), dim3(PK_THREADS), kargs, g.smem, c0->stream));
  if (timed) VL_CUDA(cudaEventRecord(ev.stop, c0->stream));

  {  // the last block-0 store is the done word: poll it (microseconds) instead of paying a stream synchronise wake-up
    volatile unsigned long long* flag = h_done;
    bool done = false;
    for (long long spin = 0;; spin++) {
      if (*flag == 1ull) {
        done = true;
        break;
      }
      if ((spin & 0xfff) == 0xfff && cudaStreamQuery(c0->stream) != cudaErrorNotReady) break;
      __builtin_ia32_pause();
    }
    std::atomic_thread_fence(std::memory_order_acquire);
    if (!done) {
      VL_CUDA(cudaStreamSynchronize(c0->stream));
      std::atomic_thread_fence(std::memory_order_acquire);
      if (*h_error) {
        set_last_error("persistent solve: a wait timed out (a peer rank died, the ranks are not solving in lockstep, or the grid was not co-resident)");
        return VLCAL_ERR_CUDA;
      }
      if (*flag != 1ull) {
        set_last_error("persistent solve finished without publishing its results");
        return VLCAL_ERR_CUDA;
      }
    }
  }
  if (c0->pk_stamps_cap > 0) {
    VL_CUDA(cudaStreamSynchronize(c0->stream));
    c0->pk_stamps.resize(static_cast<size_t>(PK_STAMP_SLOTS) * c0->pk_stamps_cap);
    VL_CUDA(cudaMemcpy(c0->pk_stamps.data(), stamps.p, sizeof(unsigned long long) * c0->pk_stamps.size(), cudaMemcpyDeviceToHost));
    c0->pk_block_times.resize(static_cast<size_t>(4) * grid);
    VL_CUDA(cudaMemcpy(c0->pk_block_times.data(), a.block_times, sizeof(unsigned long long) * c0->pk_block_times.size(), cudaMemcpyDeviceToHost));
  }
  // scratch goes back to the pool: the kernel has published its last word, nothing else is enqueued on it
  VL_CUDA(cudaStreamSynchronize(c0->stream));
  if (use_tma) VL_CUDA(cudaMemcpy(c0->pk_tma_stats, sp + L.tma_stats, sizeof(c0->pk_tma_stats), cudaMemcpyDeviceToHost));

  const NmMachine& fin = h_result->nm;
  // the objective's side effects in the reference's evaluation order (:112-116)
  if (callback) {
    double best_cost = DBL_MAX;  // :101
    const int count = std::min(h_result->trace_count, trace_cap);
    for (int k = 0; k < count; k++) {
      const double* e = h_trace + static_cast<size_t>(k) * (NM_MAX_N + 1);
      const double y = e[NM_MAX_N];
      if (y < best_cost) {
        best_cost = y;
        double E[16], T[16];
        host::se3_expmap_gtsam(e, E);
        host::isometry_mul(init_T, E, T);
        callback(T, y, user);
      }
    }
  }
  double E[16];
  host::se3_expmap_gtsam(fin.result_x, E);
  host::isometry_mul(init_T, E, T_out);  // :129
  if (nm_result) {
    std::memset(nm_result, 0, sizeof(*nm_result));
    nm_result->converged = fin.converged;
    nm_result->num_iterations = fin.num_iterations;
    for (int d = 0; d < 6; d++) nm_result->x[d] = fin.result_x[d];
    nm_result->y = fin.result_y;
    nm_result->num_evaluations = fin.num_evaluations;
    nm_result->num_batches = fin.num_batches;
    nm_result->num_evaluations_computed = fin.num_evaluations_computed;
  }
  // profile: one launch carried `batches` passes over the cloud(s)
  c0->launches += 1;
  c0->passes += static_cast<int64_t>(h_result->batches);
  c0->poses_total += static_cast<int64_t>(h_result->poses);
  return VLCAL_OK;
}

// ---- pose list ----------------------------------------------------------------------------------------------------------------

int pk_score_poses(vlcal_nid_ctx* const* ctxs, int n_ctxs, const double* T_colmajor, int n_poses, double* nid_out, int32_t* hist_out) {
  vlcal_nid_ctx* c0 = ctxs[0];
  VL_CUDA(cudaSetDevice(c0->device));
  long long total_points = 0;
  for (int i = 0; i < n_ctxs; i++) total_points += ctxs[i]->cloud->n;
  PkKernel kernel = pk_pick(c0->cam.model, pk_points_per_lane(c0, total_points));
  PkGeom g;
  {
    const int rc = pk_geometry(c0->device, c0->num_sms, kernel, c0->bins * c0->bins, &g);
    if (rc != VLCAL_OK) return rc;
  }
  const int grid = pk_grid_size(g, ctxs, n_ctxs);
  const int nb = c0->bins * c0->bins;
  const PkScratchLayout L(n_ctxs, nb);
  DevBuf scratch, d_poses, d_scores, d_hist;
  scratch.device = d_poses.device = d_scores.device = d_hist.device = c0->device;
  VL_CUDA(MemPool::instance().device_alloc(c0->device, L.total, &scratch.p));
  VL_CUDA(cudaMemsetAsync(scratch.p, 0, L.total, c0->stream));
  const int chunk = std::max(1, std::min(PK_MAX_POSES, c0->pk_chunk));
  const int n_chunks = (n_poses + chunk - 1) / chunk;
  const size_t pose_bytes = sizeof(double) * 12 * static_cast<size_t>(n_poses);
  const size_t score_count = static_cast<size_t>(n_chunks) * chunk * n_ctxs;
  VL_CUDA(MemPool::instance().device_alloc(c0->device, pose_bytes, &d_poses.p));
  VL_CUDA(MemPool::instance().device_alloc(c0->device, sizeof(double) * score_count, &d_scores.p));
  if (hist_out) VL_CUDA(MemPool::instance().device_alloc(c0->device, sizeof(int) * static_cast<size_t>(n_chunks) * chunk * nb, &d_hist.p));
  PinBuf host;
  VL_CUDA(MemPool::instance().pinned_alloc(std::max(pose_bytes, sizeof(double) * score_count) + 64, &host.p));
  double* hpose = static_cast<double*>(host.p);
  for (int p = 0; p < n_poses; p++) {
    const double* T = T_colmajor + 16 * static_cast<size_t>(p);
    for (int r = 0; r < 3; r++)
      for (int c = 0; c < 4; c++) hpose[12 * static_cast<size_t>(p) + 4 * r + c] = T[r + 4 * c];
  }
  VL_CUDA(cudaMemcpyAsync(d_poses.p, hpose, pose_bytes, cudaMemcpyHostToDevice, c0->stream));

  PkArgs a;
  pk_fill_common(a, ctxs, n_ctxs, g, grid, static_cast<char*>(scratch.p), L);
  a.poses_in = static_cast<const double*>(d_poses.p);
  a.n_total = n_poses;
  a.chunk = chunk;
  a.scores_out = static_cast<double*>(d_scores.p);
  a.hist_out = hist_out ? static_cast<int*>(d_hist.p) : nullptr;
  int* h_error = reinterpret_cast<int*>(static_cast<char*>(host.p) + std::max(pose_bytes, sizeof(double) * score_count));
  *h_error = 0;
  a.error_host = h_error;

  ProfileEvents ev{};
  const bool timed = c0->profiling;
  if (timed) {
    if (c0->events_used == c0->events.size()) {
      ProfileEvents e;
      VL_CUDA(cudaEventCreate(&e.start));
      VL_CUDA(cudaEventCreate(&e.stop));
      e.poses = 0;
      c0->events.push_back(e);
    }
    ev = c0->events[c0->events_used++];
    VL_CUDA(cudaEventRecord(ev.start, c0->stream));
  }
  void* kargs[] = {&a};
  VL_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<const void*>(kernel), dim3(grid), dim3(PK_THREADS), kargs, g.smem, c0->stream));
  if (timed) VL_CUDA(cudaEventRecord(ev.stop, c0->stream));
  VL_CUDA(cudaStreamSynchronize(c0->stream));  // the pose staging area is reused for the scores below
  double* hscore = static_cast<double*>(host.p);
  VL_CUDA(cudaMemcpyAsync(hscore, d_scores.p, sizeof(double) * score_count, cudaMemcpyDeviceToHost, c0->stream));
  if (hist_out) VL_CUDA(cudaMemcpyAsync(hist_out, d_hist.p, sizeof(int) * static_cast<size_t>(n_poses) * nb, cudaMemcpyDeviceToHost, c0->stream));
  VL_CUDA(cudaStreamSynchronize(c0->stream));
  if (*h_error) {
    set_last_error("persistent evaluation: a wait timed out (grid not co-resident?)");
    return VLCAL_ERR_CUDA;
  }
  for (int p = 0; p < n_poses; p++) {
    if (n_ctxs == 1) {
      nid_out[p] = hscore[p];
    } else {
      double s = 0.0;  // sum_costs over the bags, in bag order (visual_camera_calibration.cpp:105-110)
      for (int b = 0; b < n_ctxs; b++) s += hscore[static_cast<size_t>(p) * n_ctxs + b];
      nid_out[p] = s;
    }
  }
  c0->launches += 1;
  c0->passes += n_chunks;
  c0->poses_total += n_poses;
  return VLCAL_OK;
}

}  // namespace vlcal
