// nid_persistent.cu -- host side of K1p (nid_persistent.cuh): the persistent cooperative kernel that runs a whole
// Nelder-Mead inner solve (VisualCameraCalibration::estimate_pose_nelder_mead's optimizer loop,
// src/vlcal/calib/visual_camera_calibration.cpp:103-127) or scores an arbitrarily long pose list
// (CostCalculatorNID::calculate per pose, src/vlcal/calib/cost_calculator_nid.cpp:21-67) in ONE launch.
#include "nid_persistent.cuh"

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
// per point)
template <int MODEL>
static PkKernel pk_pick_k(int k) {
  constexpr bool heavy = MODEL == CAM_FISHEYE || MODEL == CAM_EQUIRECTANGULAR || MODEL == CAM_ATAN;
  if constexpr (!heavy) {
    if (k == 4) return nid_persistent_kernel<MODEL, 4>;
  }
  return nid_persistent_kernel<MODEL, 2>;
}

// the points per lane of the kernel pk_pick_k returns for a requested k
static int pk_kernel_k(int model, int k) {
  const bool heavy = model == CAM_FISHEYE || model == CAM_EQUIRECTANGULAR || model == CAM_ATAN;
  return k == 4 && !heavy ? 4 : 2;
}

// delta: the launch may carry equirectangular batches of nearby poses (the instance with the delta step, K = 2)
static PkKernel pk_pick(int model, int k, bool delta = false) {
  if (PK_DELTA_POSES && delta && model == CAM_EQUIRECTANGULAR && pk_kernel_k(model, k) == 2) return nid_persistent_kernel<CAM_EQUIRECTANGULAR, 2, true>;
  switch (model) {
    case CAM_PLUMB_BOB: return pk_pick_k<CAM_PLUMB_BOB>(k);
    case CAM_FISHEYE: return pk_pick_k<CAM_FISHEYE>(k);
    case CAM_ATAN: return pk_pick_k<CAM_ATAN>(k);
    case CAM_OMNIDIR: return pk_pick_k<CAM_OMNIDIR>(k);
    case CAM_EQUIRECTANGULAR: return pk_pick_k<CAM_EQUIRECTANGULAR>(k);
    case CAM_RATIONAL_POLYNOMIAL: return pk_pick_k<CAM_RATIONAL_POLYNOMIAL>(k);
    default: return nullptr;
  }
}

struct PkGeom {
  int copies;
  size_t smem;
  unsigned int ring_off;  // byte offset of the tile rings in dynamic shared memory
  int max_blocks;  // co-resident blocks of the whole device (cooperative launch limit)
};

static std::mutex g_pk_mu;
static std::map<std::tuple<int, const void*, size_t>, int> g_pk_occupancy;

// Dynamic shared memory of one block: the histogram copies (whose space the finalizer reuses as staging), then the warps'
// tile rings.  At 16 bins and K = 2: 48 KB of copies + 24 warps x 2 slots x 1 KB of rings = 96 KB, next to ~16 KB of
// static PkShared -- within the 227 KB a block may opt in to on an H100.
static int pk_geometry(int device, int num_sms, const void* kernel, int nb, int kpt, PkGeom* g) {
  // histogram copies for 8 poses (the initial simplex of a 6-D solve is 7) -- two copies while they fit 64 KB
  const size_t per_copy = static_cast<size_t>(PK_MAX_POSES) * nb * sizeof(int);
  g->copies = static_cast<int>(std::max<size_t>(1, std::min<size_t>(PK_WARPS / 4, (64 * 1024) / per_copy)));  // one copy per four warps
  const size_t scratch = static_cast<size_t>(nb) * 8 + 64 * 8 * 2 + 64 * 4 * 2;  // pk_block_nid staging (aliases the copies)
  g->smem = std::max(per_copy * g->copies, scratch);
  const size_t tail = (g->smem + 127) & ~static_cast<size_t>(127);
  g->ring_off = static_cast<unsigned int>(tail);
  g->smem = tail + pk_ring_bytes(kpt);
  std::lock_guard<std::mutex> lock(g_pk_mu);
  const auto key = std::make_tuple(device, kernel, g->smem);
  auto it = g_pk_occupancy.find(key);
  if (it == g_pk_occupancy.end()) {
    int optin = 0;
    VL_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
    cudaFuncAttributes fa;
    VL_CUDA(cudaFuncGetAttributes(&fa, kernel));
    const size_t dyn_max = static_cast<size_t>(optin) - fa.sharedSizeBytes;
    if (g->smem > dyn_max) {
      set_last_error("persistent kernel: " + std::to_string(g->smem) + " bytes of dynamic shared memory exceed the " + std::to_string(dyn_max) + " the device allows");
      return VLCAL_ERR_UNSUPPORTED;
    }
    // the opt-in limit is a property of the kernel: set it to the device's maximum, whatever this launch asks for
    VL_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(dyn_max)));
    int nblk = 0;
    VL_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nblk, kernel, PK_THREADS, g->smem));
    it = g_pk_occupancy.emplace(key, std::max(1, nblk)).first;
  }
  g->max_blocks = it->second * num_sms;
  return VLCAL_OK;
}

// Points per lane and tile (K).  Tiles are dealt to the warps round-robin, so K = 4 (128-point tiles) needs a cloud large
// enough for several tiles per warp to stay balanced -- and there the lighter register footprint of K = 2 (768 threads per
// SM without spills in the pose loop, one packed register pair per coordinate) measured faster anyway.  K = 4 remains as
// variant 3.
static int pk_points_per_lane(const vlcal_nid_ctx* ctx) { return ctx->variant == 3 ? 4 : 2; }

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
  size_t ghist, gmarg, arrive, fin_done, tile_next, abort_flag, seq, delta_stats, box, solve, total;
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
    delta_stats = take(sizeof(unsigned long long) * 4);
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
  a.ring_off = g.ring_off;
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
  a.delta_stats = reinterpret_cast<unsigned long long*>(scratch + L.delta_stats);
  a.world = 1, a.rank = 0;
  a.timeout_ns = sync_timeout_ns();
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
  vlcal_nm_result* nm_result, bool score_centroid) {
  vlcal_nid_ctx* c0 = ctxs[0];
  VL_CUDA(cudaSetDevice(c0->device));
  const int kpt = pk_points_per_lane(c0);
  const PkKernel kernel = pk_pick(c0->cam.model, kpt, true);  // Nelder-Mead batches close in as the simplex shrinks
  PkGeom g;
  {
    const int rc = pk_geometry(c0->device, c0->num_sms, reinterpret_cast<const void*>(kernel), c0->bins * c0->bins, pk_kernel_k(c0->cam.model, kpt), &g);
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
  // n + 1 evaluations of the initial simplex, then at most n + 3 per iteration: xo, xr, xc and the n shrunk vertices.
  // Without the centroid nothing replays the trace (run_inner_solve), so block 0 writes none.
  const int trace_cap = score_centroid ? 7 + std::max(0, params->max_inner_iterations) * 9 : 0;
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
  h_solve->nm.begin(6, nm, x0, score_centroid);  // :126 optimize(f, Zero)
  std::memcpy(h_solve->init_T, init_T, sizeof(h_solve->init_T));
  char* sp = static_cast<char*>(scratch.p);
  VL_CUDA(cudaMemcpyAsync(sp + L.solve, h_solve, sizeof(PkSolve), cudaMemcpyHostToDevice, c0->stream));

  PkArgs a;
  pk_fill_common(a, ctxs, n_ctxs, g, grid, sp, L);
  a.solve = reinterpret_cast<const PkSolve*>(sp + L.solve);
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
  unsigned long long delta_stats[4];
  VL_CUDA(cudaMemcpy(delta_stats, sp + L.delta_stats, sizeof(delta_stats), cudaMemcpyDeviceToHost));

  const NmMachine& fin = h_result->nm;
  // the objective's side effects in the reference's evaluation order (:112-116)
  {
    double best_cost = DBL_MAX;  // :101
    const int count = std::min(h_result->trace_count, trace_cap);
    for (int k = 0; k < count; k++) {
      const double* e = h_trace + static_cast<size_t>(k) * (NM_MAX_N + 1);
      const double y = e[NM_MAX_N];
      solve_trace_push(e, y);
      if (y < best_cost && callback) {
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
  for (int i = 0; i < n_ctxs; i++) ctxs[i]->pk_last_kpt = pk_kernel_k(c0->cam.model, kpt);
  c0->launches += 1;
  c0->passes += static_cast<int64_t>(h_result->batches);
  for (int i = 0; i < 4; i++) c0->delta_stats[i] += static_cast<int64_t>(delta_stats[i]);
  c0->poses_total += static_cast<int64_t>(h_result->poses);
  return VLCAL_OK;
}

// ---- S independent Nelder-Mead solves in one launch (the solve axis) ----------------------------------------------------------

static const void* pk_pick_solves(int model) {
  switch (model) {
    case CAM_PLUMB_BOB: return reinterpret_cast<const void*>(nid_persistent_solves_kernel<CAM_PLUMB_BOB>);
    case CAM_FISHEYE: return reinterpret_cast<const void*>(nid_persistent_solves_kernel<CAM_FISHEYE>);
    case CAM_ATAN: return reinterpret_cast<const void*>(nid_persistent_solves_kernel<CAM_ATAN>);
    case CAM_OMNIDIR: return reinterpret_cast<const void*>(nid_persistent_solves_kernel<CAM_OMNIDIR>);
    case CAM_EQUIRECTANGULAR: return reinterpret_cast<const void*>(nid_persistent_solves_kernel<CAM_EQUIRECTANGULAR, PK_DELTA_POSES != 0>);
    case CAM_RATIONAL_POLYNOMIAL: return reinterpret_cast<const void*>(nid_persistent_solves_kernel<CAM_RATIONAL_POLYNOMIAL>);
    default: return nullptr;
  }
}

int pk_solve_many(
  vlcal_nid_ctx* const* ctxs, int n_ctxs, const vlcal_calib_params* params, int n_solves, const double* init_T, const uint8_t* bag_mask, double* T_out, vlcal_nm_result* results) {
  vlcal_nid_ctx* c0 = ctxs[0];
  VL_CUDA(cudaSetDevice(c0->device));
  if (n_solves > PK_MAX_SOLVES) {
    set_last_error("solve axis: at most " + std::to_string(PK_MAX_SOLVES) + " solves per launch");
    return VLCAL_ERR_UNSUPPORTED;
  }
  const void* kernel = pk_pick_solves(c0->cam.model);
  const int nb = c0->bins * c0->bins;
  PkGeom g;
  {
    const int rc = pk_geometry(c0->device, c0->num_sms, kernel, nb, 2, &g);
    if (rc != VLCAL_OK) return rc;
  }
  // the bags of every solve, in context order (the order its scores are summed in)
  std::vector<std::vector<vlcal_nid_ctx*>> bags(n_solves);
  long long need = 0, want_sum = 0;
  std::vector<long long> want(n_solves);
  for (int s = 0; s < n_solves; s++) {
    for (int b = 0; b < n_ctxs; b++)
      if (bag_mask[static_cast<size_t>(s) * n_ctxs + b]) bags[s].push_back(ctxs[b]);
    if (bags[s].empty()) {
      set_last_error("solve " + std::to_string(s) + " includes no bag");
      return VLCAL_ERR_INVALID_ARGUMENT;
    }
    want[s] = pk_grid_size(g, bags[s].data(), static_cast<int>(bags[s].size()));  // what a single solve of these bags takes
    want_sum += want[s];
    need += static_cast<long long>(bags[s].size());
  }
  // blocks: every solve what it would take alone while the device holds them all, otherwise in proportion to that, and at
  // least one per bag of the solve
  const long long total = std::min<long long>(want_sum, g.max_blocks);
  if (need > total) {
    set_last_error("solve axis: " + std::to_string(n_solves) + " solves need " + std::to_string(need) + " blocks (one per bag of each), the device runs " + std::to_string(g.max_blocks) +
                   " co-resident blocks");
    return VLCAL_ERR_UNSUPPORTED;
  }
  std::vector<int> share(n_solves);
  long long assigned = 0;
  for (int s = 0; s < n_solves; s++) {
    share[s] = static_cast<int>(std::max<long long>(static_cast<long long>(bags[s].size()), want[s] * total / want_sum));
    assigned += share[s];
  }
  while (assigned > total) {  // rounding up to the per-bag minimum can overshoot: take the excess from the largest shares
    int k = -1;
    for (int s = 0; s < n_solves; s++)
      if (share[s] > static_cast<int>(bags[s].size()) && (k < 0 || share[s] > share[k])) k = s;
    share[k]--, assigned--;
  }
  PkSolvesArgs m;
  std::memset(&m, 0, sizeof(m));
  m.n_groups = n_solves;
  for (int s = 0; s < n_solves; s++) m.block_begin[s + 1] = m.block_begin[s] + share[s];
  const int grid = m.block_begin[n_solves];

  // device scratch: every solve's accumulators and counters (PkScratchLayout), then the group arguments; one memset
  std::vector<size_t> off(n_solves + 1, 0);
  for (int s = 0; s < n_solves; s++) off[s + 1] = off[s] + PkScratchLayout(static_cast<int>(bags[s].size()), nb).total;
  const size_t args_off = off[n_solves];
  DevBuf scratch;
  scratch.device = c0->device;
  VL_CUDA(MemPool::instance().device_alloc(c0->device, args_off + sizeof(PkArgs) * n_solves, &scratch.p));
  char* sp = static_cast<char*>(scratch.p);
  VL_CUDA(cudaMemsetAsync(sp, 0, args_off, c0->stream));

  // host side: the outcomes (mapped pinned memory, written by each group's block 0), the error word, and the staging of
  // the solves' initial states and the group arguments
  const size_t res_bytes = (sizeof(PkResult) * n_solves + 64 + 255) & ~static_cast<size_t>(255);
  const size_t stage_bytes = sizeof(PkSolve) * n_solves + sizeof(PkArgs) * n_solves + 64;
  PinBuf host;
  VL_CUDA(MemPool::instance().pinned_alloc(res_bytes + stage_bytes, &host.p));
  char* hp = static_cast<char*>(host.p);
  PkResult* h_results = reinterpret_cast<PkResult*>(hp);
  int* h_error = reinterpret_cast<int*>(hp + sizeof(PkResult) * n_solves);
  std::memset(hp, 0, res_bytes);
  PkSolve* h_solves = reinterpret_cast<PkSolve*>(hp + res_bytes);
  PkArgs* h_args = reinterpret_cast<PkArgs*>((reinterpret_cast<uintptr_t>(h_solves + n_solves) + 63) & ~static_cast<uintptr_t>(63));

  NmParams nm;  // visual_camera_calibration.cpp:122-125, as pk_solve
  nm.init_step = params->nelder_mead_init_step;
  nm.convergence_var_thresh = params->nelder_mead_convergence_criteria;
  nm.max_iterations = params->max_inner_iterations;
  const double x0[6] = {0, 0, 0, 0, 0, 0};
  for (int s = 0; s < n_solves; s++) {
    const PkScratchLayout L(static_cast<int>(bags[s].size()), nb);
    char* gs = sp + off[s];
    std::memset(static_cast<void*>(&h_solves[s]), 0, sizeof(PkSolve));
    h_solves[s].nm.begin(6, nm, x0, /*score_centroid=*/false);  // nobody observes the evaluations: as pk_solve without a callback
    std::memcpy(h_solves[s].init_T, init_T + 16 * static_cast<size_t>(s), sizeof(h_solves[s].init_T));
    VL_CUDA(cudaMemcpyAsync(gs + L.solve, &h_solves[s], sizeof(PkSolve), cudaMemcpyHostToDevice, c0->stream));
    PkArgs& a = h_args[s];
    pk_fill_common(a, bags[s].data(), static_cast<int>(bags[s].size()), g, share[s], gs, L);
    a.solve = reinterpret_cast<const PkSolve*>(gs + L.solve);
    a.result_host = &h_results[s];
    a.error_host = h_error;
    a.abort_flag = reinterpret_cast<unsigned int*>(sp + PkScratchLayout(static_cast<int>(bags[0].size()), nb).abort_flag);  // one for the launch
  }
  VL_CUDA(cudaMemcpyAsync(sp + args_off, h_args, sizeof(PkArgs) * n_solves, cudaMemcpyHostToDevice, c0->stream));
  m.group = reinterpret_cast<const PkArgs*>(sp + args_off);
  m.common = h_args[0];  // pk_supported: one camera, image size and bin count for every context

  void* kargs[] = {&m};
  VL_CUDA(cudaLaunchCooperativeKernel(kernel, dim3(grid), dim3(PK_THREADS), kargs, g.smem, c0->stream));
  VL_CUDA(cudaStreamSynchronize(c0->stream));
  std::atomic_thread_fence(std::memory_order_acquire);
  if (*h_error) {
    set_last_error("persistent solves: a wait timed out (the grid was not co-resident)");
    return VLCAL_ERR_CUDA;
  }
  for (int s = 0; s < n_solves; s++) {
    const NmMachine& fin = h_results[s].nm;
    double E[16];
    host::se3_expmap_gtsam(fin.result_x, E);
    host::isometry_mul(init_T + 16 * static_cast<size_t>(s), E, T_out + 16 * static_cast<size_t>(s));  // :129
    vlcal_nm_result& r = results[s];
    std::memset(&r, 0, sizeof(r));
    r.converged = fin.converged;
    r.num_iterations = fin.num_iterations;
    for (int d = 0; d < 6; d++) r.x[d] = fin.result_x[d];
    r.y = fin.result_y;
    r.num_evaluations = fin.num_evaluations;
    r.num_batches = fin.num_batches;
    r.num_evaluations_computed = fin.num_evaluations_computed;
    c0->passes += static_cast<int64_t>(h_results[s].batches);
    c0->poses_total += static_cast<int64_t>(h_results[s].poses);
  }
  for (int i = 0; i < n_ctxs; i++) ctxs[i]->pk_last_kpt = 2;
  c0->launches += 1;
  return VLCAL_OK;
}

// ---- pose list ----------------------------------------------------------------------------------------------------------------

int pk_score_poses(vlcal_nid_ctx* const* ctxs, int n_ctxs, const double* T_colmajor, int n_poses, double* nid_out, int32_t* hist_out) {
  vlcal_nid_ctx* c0 = ctxs[0];
  VL_CUDA(cudaSetDevice(c0->device));
  const int kpt = pk_points_per_lane(c0);
  // the instance with the delta step only when some chunk of the list lies within its gate (the kernel checks every
  // chunk again); widely spread lists and one-pose chunks keep the plain instance
  bool delta = false;
  if (c0->cam.model == CAM_EQUIRECTANGULAR) {
    const int ch = std::max(1, std::min(PK_MAX_POSES, c0->pk_chunk));
    for (int b = 0; b < n_poses && !delta; b += ch) {
      const int cnt = std::min(ch, n_poses - b);
      double R[PK_MAX_POSES][12];
      for (int k = 0; k < cnt; k++)
        for (int r = 0; r < 3; r++)
          for (int c = 0; c < 4; c++) R[k][4 * r + c] = T_colmajor[16 * static_cast<size_t>(b + k) + r + 4 * c];
      const int anc = lean_delta_anchor(R, cnt);  // the kernel's anchor (pk_delta_rows)
      float Q[16];
      bool close = cnt >= 2;
      for (int k = 0; k < cnt && close; k++)
        if (k != anc) close = lean_delta_pose(R[k], R[anc], Q);
      delta = close;
    }
  }
  PkKernel kernel = pk_pick(c0->cam.model, kpt, delta);
  PkGeom g;
  {
    const int rc = pk_geometry(c0->device, c0->num_sms, reinterpret_cast<const void*>(kernel), c0->bins * c0->bins, pk_kernel_k(c0->cam.model, kpt), &g);
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
  unsigned long long delta_stats[4];
  VL_CUDA(cudaMemcpyAsync(delta_stats, static_cast<char*>(scratch.p) + L.delta_stats, sizeof(delta_stats), cudaMemcpyDeviceToHost, c0->stream));
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
  for (int i = 0; i < n_ctxs; i++) ctxs[i]->pk_last_kpt = pk_kernel_k(c0->cam.model, kpt);
  c0->launches += 1;
  c0->passes += n_chunks;
  for (int i = 0; i < 4; i++) c0->delta_stats[i] += static_cast<int64_t>(delta_stats[i]);
  c0->poses_total += n_poses;
  return VLCAL_OK;
}

}  // namespace vlcal
