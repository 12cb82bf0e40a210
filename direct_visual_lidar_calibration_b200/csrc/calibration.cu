// calibration.cu -- the caller of the hot path: VisualCameraCalibration, NID_NELDER_MEAD branch
// (reference: src/vlcal/calib/visual_camera_calibration.cpp:35-139, include/vlcal/calib/visual_camera_calibration.hpp).
//
// Same decisions as the reference (outer loop, culling at the start pose of every inner solve, one cost object per
// bag, dfo::NelderMead<6> with the calibration parameters), but every Nelder-Mead iteration scores its candidate
// poses {xr, xe, xc} (plus the centroid xo when its value can be observed, run_inner_solve) in ONE batched kernel launch
// per bag, and bags run concurrently on their own streams.
#include <chrono>
#include <cstring>
#include <vector>

#include "host_math.hpp"
#include "mem_pool.hpp"
#include "nid_context.cuh"
#include "nid_kernels.cuh"

using namespace vlcal;

namespace {

double now_ms() {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

vlcal_p2p* g_default_p2p = nullptr;  // vlcal_nid_p2p_set_default
int g_solver_mode = 0;                // vlcal_nid_set_solver_mode: 0 auto, 1 host loop, 3 persistent kernel
thread_local bool g_record_solve_trace = false;  // vlcal_nid_debug_record_solve_trace
thread_local std::vector<double> g_solve_trace;  // [k][7]: solve_trace_push

// the kernel sums over ranks only when a CONNECTED exchange spanning more than one rank is attached (fill_common_args)
inline bool ctx_exchange_is_fused(const vlcal_nid_ctx* c) {
  return c->p2p != nullptr && c->p2p->connected && c->p2p->world > 1;
}

struct PoseObjective {
  vlcal_nid_ctx* const* ctxs;
  int n_ctxs;
  const double* init_T;
  vlcal_pose_callback callback;
  vlcal_allreduce_fn allreduce;
  void* user;
  double best_cost = DBL_MAX;  // visual_camera_calibration.cpp:101
  int status = VLCAL_OK;
  std::vector<double> Ts, partial, vals;

  // f(x) for a batch: T = init_T * Expmap(x)  (:104), sum over bags of calculate(T)  (:105-110)
  void evaluate(const double* xs, int count, double* ys) {
    Ts.resize(static_cast<size_t>(count) * 16);
    partial.assign(count, 0.0);
    vals.resize(count);
    for (int i = 0; i < count; i++) {
      double E[16];
      host::se3_expmap_gtsam(xs + 6 * i, E);
      host::isometry_mul(init_T, E, &Ts[16 * static_cast<size_t>(i)]);
    }
    if (status == VLCAL_OK) {
      int launched = 0;
      for (; launched < n_ctxs; launched++) {
        const int rc = nid_evaluate_async(ctxs[launched], Ts.data(), count, false);
        if (rc != VLCAL_OK) {
          status = rc;
          break;
        }
      }
      for (int b = 0; b < launched; b++) {
        const int rc = nid_wait(ctxs[b], vals.data(), nullptr);
        if (rc != VLCAL_OK) {
          status = rc;
          continue;
        }
        for (int i = 0; i < count; i++) partial[i] += vals[i];  // sum_costs += costs[i]->calculate(T)
      }
    }
    // with a peer exchange attached (one bag per rank) the kernel already returned the sum over ranks
    const bool fused = n_ctxs == 1 && ctx_exchange_is_fused(ctxs[0]);
    if (allreduce && !fused) allreduce(partial.data(), count, user);
    for (int i = 0; i < count; i++) ys[i] = status == VLCAL_OK ? partial[i] : NAN;
  }

  // the objective's side effects, in the reference's evaluation order (:112-116)
  void observe(const double* x, double y) {
    solve_trace_push(x, y);
    if (y < best_cost) {
      best_cost = y;
      if (callback) {
        double E[16], T[16];
        host::se3_expmap_gtsam(x, E);
        host::isometry_mul(init_T, E, T);
        callback(T, y, user);
      }
    }
  }
};

// What a rank of a peer exchange would do on its own: whether its contexts can take the persistent kernel, its solver
// mode, its number of local bags and its bins.  Packed into one word for p2p_gather.
struct SolvePlan {
  bool pk;
  int mode, n_bags, bins;
  unsigned long long word() const {
    return static_cast<unsigned long long>(pk ? 1 : 0) | static_cast<unsigned long long>(mode & 0xff) << 8 | static_cast<unsigned long long>(n_bags & 0xffff) << 16 |
           static_cast<unsigned long long>(bins & 0xffff) << 32;
  }
  static SolvePlan of(unsigned long long w) {
    return SolvePlan{(w & 1ull) != 0, static_cast<int>((w >> 8) & 0xff), static_cast<int>((w >> 16) & 0xffff), static_cast<int>((w >> 32) & 0xffff)};
  }
  std::string describe() const {
    return std::string(pk ? "persistent-capable" : "host loop only") + ", solver mode " + std::to_string(mode) + ", " + std::to_string(n_bags) + " bag(s), " +
           std::to_string(bins) + " bins";
  }
};

// The solve-path agreement.  Each rank picks its path from its own bags, but the round-1 exchange (host loop, one bag per
// rank) and the persistent kernel's exchange ((rank, bag) words, the same number of bags on every rank) only meet their
// own kind: ranks that chose differently would each wait for words that never come.  So before a solve every rank
// publishes its plan in one exchange and reads all of them; every rank then decides the same way:
//   * plans equal: the path each rank would take alone (it is the same everywhere);
//   * plans differ and every rank holds one bag, with no rank in solver mode 3: all ranks take the host loop (the
//     round-1 exchange sums one bag per rank whatever the layout, camera or bins);
//   * otherwise every rank refuses with VLCAL_ERR_UNSUPPORTED, naming the ranks whose plan differs from rank 0's.
int agree_solve_path(vlcal_p2p* px, cudaStream_t stream, const SolvePlan& mine, bool* host_loop) {
  *host_loop = false;
  unsigned long long words[P2P_MAX_RANKS];
  const int rc = p2p_gather(px, stream, mine.word(), words);
  if (rc != VLCAL_OK) return rc;
  bool equal = true, one_bag_each = true, mode3 = false;
  for (int r = 0; r < px->world; r++) {
    const SolvePlan p = SolvePlan::of(words[r]);
    equal = equal && words[r] == words[0];
    one_bag_each = one_bag_each && p.n_bags == 1;
    mode3 = mode3 || p.mode == 3;
  }
  if (equal) return VLCAL_OK;
  if (one_bag_each && !mode3) {
    *host_loop = true;
    return VLCAL_OK;
  }
  std::string differ, plans;
  for (int r = 0; r < px->world; r++) {
    if (words[r] != words[0]) differ += (differ.empty() ? "" : ", ") + std::to_string(r);
    plans += "; rank " + std::to_string(r) + ": " + SolvePlan::of(words[r]).describe();
  }
  set_last_error("peer exchange: the ranks' solve plans differ (rank(s) " + differ + " against rank 0" + plans +
                 "): with several bags per rank, or solver mode 3, every rank needs the same number of bags, bins, layout and mode");
  return VLCAL_ERR_UNSUPPORTED;
}

int run_inner_solve(
  vlcal_nid_ctx* const* ctxs, int n_ctxs, const vlcal_calib_params* params, const double init_T[16], vlcal_pose_callback callback, vlcal_allreduce_fn allreduce, void* user,
  double T_out[16], vlcal_nm_result* nm_result) {
  // Persistent cooperative kernel (nid_persistent.cuh; default): the whole solve is ONE launch -- candidates scored,
  // summed over bags and ranks, and the Nelder-Mead machine stepped inside the kernel.  Needs what pk_supported checks
  // (float4 clouds, lean classifier, bins <= 32, one camera / image size / device) and no host-side all-reduce callback
  // (a connected peer exchange is summed in-kernel instead).
  solve_trace_clear();
  bool same_px = true;
  for (int i = 1; i < n_ctxs; i++) same_px = same_px && ctxs[i]->p2p == ctxs[0]->p2p;
  const bool px_fused = n_ctxs >= 1 && ctx_exchange_is_fused(ctxs[0]);
  bool pk_ok = n_ctxs >= 1 && params->max_inner_iterations >= 0 && same_px && (allreduce == nullptr || px_fused) && pk_supported(ctxs, n_ctxs);
  if (px_fused) {
    bool host_loop = false;
    const int rc = agree_solve_path(ctxs[0]->p2p, ctxs[0]->stream, SolvePlan{pk_ok, g_solver_mode, n_ctxs, ctxs[0]->bins}, &host_loop);
    if (rc != VLCAL_OK) return rc;
    pk_ok = pk_ok && !host_loop;
  }
  // The centroid xo of an iteration (nelder_mead.hpp:58) never feeds a decision; its value reaches a user only as a side
  // effect of the objective: the best-cost callback or the recorded solve trace.  Without either, the iteration batches
  // score {xr, xe, xc} only.  Several ranks (a host all-reduce or an attached peer exchange) keep scoring it: every rank
  // must issue batches of the same size, and a rank with a callback would otherwise wait for words the others never send.
  bool px_any = false;
  for (int i = 0; i < n_ctxs; i++) px_any = px_any || ctx_exchange_is_fused(ctxs[i]);
  const bool score_centroid = callback != nullptr || g_record_solve_trace || allreduce != nullptr || px_any;
  if (g_solver_mode == 3 && !pk_ok) {
    set_last_error("persistent solve requested but these contexts need the host loop (double-layout cloud / bins > 32 / camera without the lean classifier / host all-reduce / mixed image sizes)");
    return VLCAL_ERR_UNSUPPORTED;
  }
  if (pk_ok && (g_solver_mode == 0 || g_solver_mode == 3)) {
    return pk_solve(ctxs, n_ctxs, params, init_T, callback, user, T_out, nm_result, score_centroid);
  }
  // the round-1 kernels exchange one bag per rank; with several local bags only the persistent kernel sums in-kernel, or
  // a host all-reduce callback sums the host loop's partial sums (the contexts then run without their exchange)
  std::vector<vlcal_p2p*> detached;
  if (n_ctxs > 1 && px_fused) {
    if (!allreduce) {
      set_last_error("several local bags with an attached peer exchange need the persistent solve (solver mode 0 / 3) or a host all-reduce");
      return VLCAL_ERR_UNSUPPORTED;
    }
    for (int i = 0; i < n_ctxs; i++) detached.push_back(ctxs[i]->p2p), ctxs[i]->p2p = nullptr;
  }
  struct Reattach {
    vlcal_nid_ctx* const* ctxs;
    const std::vector<vlcal_p2p*>& px;
    ~Reattach() {
      for (size_t i = 0; i < px.size(); i++) ctxs[i]->p2p = px[i];
    }
  } reattach{ctxs, detached};
  PoseObjective obj;
  obj.ctxs = ctxs, obj.n_ctxs = n_ctxs, obj.init_T = init_T, obj.callback = callback, obj.allreduce = allreduce, obj.user = user;

  host::NelderMeadParams nm;  // :122-125
  nm.init_step = params->nelder_mead_init_step;
  nm.convergence_var_thresh = params->nelder_mead_convergence_criteria;
  nm.max_iterations = params->max_inner_iterations;
  const double x0[6] = {0, 0, 0, 0, 0, 0};
  auto f = [&](const double* xs, int count, double* ys) { obj.evaluate(xs, count, ys); };
  auto ob = [&](const double* x, double y) { obj.observe(x, y); };
  const host::NelderMeadResult r = host::nelder_mead(6, f, ob, x0, nm, /*speculate=*/true, score_centroid);  // :126-127
  if (obj.status != VLCAL_OK) return obj.status;

  double E[16];
  host::se3_expmap_gtsam(r.x.data(), E);
  host::isometry_mul(init_T, E, T_out);  // :129
  if (nm_result) {
    std::memset(nm_result, 0, sizeof(*nm_result));
    nm_result->converged = r.converged ? 1 : 0;
    nm_result->num_iterations = r.num_iterations;
    for (int d = 0; d < 6; d++) nm_result->x[d] = r.x[d];
    nm_result->y = r.y;
    nm_result->num_evaluations = r.num_evaluations;
    nm_result->num_batches = r.num_batches;
    nm_result->num_evaluations_computed = r.num_evaluations_computed;
  }
  return VLCAL_OK;
}

// a bag resident in HBM for the whole calibration (uploaded once, culled per outer iteration)
struct ResidentBag {
  std::shared_ptr<DeviceCloud> cloud;
  std::shared_ptr<DeviceImage> image;
  double max_fov = 0.0;  // estimate_camera_fov(proj, this bag's image size)  (cost_calculator_nid.cpp:17)
};

int upload_bags(int device, const CameraParams& cam, const vlcal_bag* bags, int n_bags, std::vector<ResidentBag>* out) {
  out->resize(n_bags);
  for (int b = 0; b < n_bags; b++) {
    const vlcal_bag& bag = bags[b];
    if (!bag.image || bag.width <= 0 || bag.height <= 0 || bag.row_stride_bytes < bag.width || bag.n_points < 0 || (bag.n_points > 0 && (!bag.points_xyzw || !bag.intensities))) {
      set_last_error("invalid bag " + std::to_string(b));
      return VLCAL_ERR_INVALID_ARGUMENT;
    }
    int rc = upload_cloud(device, bag.points_xyzw, bag.intensities, bag.n_points, nullptr, &(*out)[b].cloud);
    if (rc != VLCAL_OK) return rc;
    rc = upload_image(device, bag.image, bag.width, bag.height, bag.row_stride_bytes, nullptr, &(*out)[b].image);
    if (rc != VLCAL_OK) return rc;
    // identical for bags that share an image size; cheap (three 2-D Nelder-Mead solves on the host)
    (*out)[b].max_fov = (b > 0 && bag.width == bags[0].width && bag.height == bags[0].height) ? (*out)[0].max_fov : estimate_camera_fov_host(cam, bag.width, bag.height);
  }
  return VLCAL_OK;
}

struct CtxList {
  std::vector<vlcal_nid_ctx*> v;
  ~CtxList() {
    for (auto* c : v) delete c;
  }
};

// estimate_pose_nelder_mead (:70-139) on resident bags
int inner_solve_resident(
  int device, const CameraParams& cam, const std::vector<ResidentBag>& bags, const vlcal_calib_params* params, const double init_T[16], vlcal_pose_callback callback,
  vlcal_allreduce_fn allreduce, void* user, int profiling, double T_out[16], vlcal_nm_result* nm_result, vlcal_calib_stats* stats, int outer_index) {
  // :71-73 one ViewCulling object, built on dataset.front()'s image size
  const double cull_fov = bags.empty() ? 0.0 : bags[0].max_fov;
  const double t_cull0 = now_ms();
  CtxList ctxs;
  for (size_t b = 0; b < bags.size(); b++) {
    std::shared_ptr<DeviceCloud> culled;
    int64_t kept = 0;
    int rc = view_cull_device(cam, bags[0].image->width, bags[0].image->height, cull_fov, !params->disable_z_buffer_culling, *bags[b].cloud, init_T, nullptr, &culled, nullptr, &kept);  // :78
    if (rc != VLCAL_OK) return rc;
    if (stats && b == 0 && outer_index < 16) stats->culled_points[outer_index] = kept;
    vlcal_nid_ctx* ctx = nullptr;
    rc = nid_ctx_create(device, VLCAL_NID_MODE_HISTOGRAM, cam, bags[b].image, culled, params->nid_bins, bags[b].max_fov, &ctx);  // :82-84
    if (rc != VLCAL_OK) return rc;
    ctx->profiling = profiling != 0;
    ctxs.v.push_back(ctx);
  }
  // every context takes the default exchange, whatever this rank's bags: run_inner_solve then agrees on the path with the
  // other ranks (agree_solve_path), which a rank deciding alone to solve without the exchange would leave waiting
  if (g_default_p2p && g_default_p2p->device == device)
    for (auto* c : ctxs.v) c->p2p = g_default_p2p;
  const double t_solve0 = now_ms();
  if (stats) stats->cull_ms += t_solve0 - t_cull0;
  vlcal_nm_result local;
  const int rc = run_inner_solve(ctxs.v.data(), static_cast<int>(ctxs.v.size()), params, init_T, callback, allreduce, user, T_out, &local);
  if (rc != VLCAL_OK) return rc;
  if (nm_result) *nm_result = local;
  if (stats) {
    stats->solve_ms += now_ms() - t_solve0;
    stats->total_evaluations += local.num_evaluations;
    stats->total_evaluations_computed += local.num_evaluations_computed;
    stats->total_batches += local.num_batches;
    if (outer_index < 16) {
      stats->inner_iterations[outer_index] = local.num_iterations;
      stats->inner_final_cost[outer_index] = local.y;
    }
    for (auto* c : ctxs.v) {
      int64_t launches = 0, poses = 0;
      double ms = 0.0;
      if (vlcal_nid_get_profile(c, &launches, &ms, &poses) == VLCAL_OK) {
        stats->kernel_launches += launches;
        stats->kernel_ms_total += ms;
      }
    }
  }
  return VLCAL_OK;
}

int check_common(const vlcal_calib_params* params, const double* init_T, double* T_out, int n_bags) {
  if (!params || !init_T || !T_out || n_bags <= 0) {
    set_last_error("invalid arguments");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  if (vlcal_nid_device_count() == 0) {
    set_last_error("no CUDA device available: this library has no CPU fallback");
    return VLCAL_ERR_NO_DEVICE;
  }
  return VLCAL_OK;
}

// visual_camera_calibration.cpp:50-54: delta = new_T^-1 * T, its translation norm and its rotation angle
void outer_step_delta(const double T[16], const double new_T[16], double* delta_t, double* delta_r) {
  double inv[16], delta[16];
  host::isometry_inverse(new_T, inv);
  host::isometry_mul(inv, T, delta);  // :50
  const double tx = host::m4(delta, 0, 3), ty = host::m4(delta, 1, 3), tz = host::m4(delta, 2, 3);
  *delta_t = std::sqrt((tx * tx + ty * ty) + tz * tz);  // :53
  *delta_r = host::rotation_angle(delta);               // :54
}

}  // namespace

void vlcal::solve_trace_clear() {
  g_solve_trace.clear();
}

void vlcal::solve_trace_push(const double* x, double y) {
  if (!g_record_solve_trace) return;
  g_solve_trace.insert(g_solve_trace.end(), x, x + 6);
  g_solve_trace.push_back(y);
}

extern "C" {

int vlcal_nid_debug_record_solve_trace(int enable) {
  g_record_solve_trace = enable != 0;
  g_solve_trace.clear();
  return VLCAL_OK;
}

int vlcal_nid_debug_last_solve_trace(int capacity, double* rows_out, int* n_out) {
  if (capacity < 0 || (capacity > 0 && !rows_out) || !n_out) return VLCAL_ERR_INVALID_ARGUMENT;
  const int have = static_cast<int>(g_solve_trace.size() / 7);
  if (capacity > 0) std::memcpy(rows_out, g_solve_trace.data(), sizeof(double) * 7 * static_cast<size_t>(std::min(capacity, have)));
  *n_out = have;
  return VLCAL_OK;
}

int vlcal_nid_set_solver_mode(int mode) {
  if (mode == 2) {
    set_last_error("solver mode 2: the round-1 device-resident loop was removed; use 0 (auto), 1 (host loop) or 3 (persistent kernel)");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  if (mode < 0 || mode > 3) {
    set_last_error("solver mode must be 0 (auto), 1 (host loop) or 3 (persistent kernel)");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  g_solver_mode = mode;
  return VLCAL_OK;
}

int vlcal_nid_p2p_set_default(vlcal_p2p* px) {
  if (px && !px->connected) {
    set_last_error("peer exchange is not connected");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  g_default_p2p = px;
  return VLCAL_OK;
}

void vlcal_nm_default_params(vlcal_nm_params* p) {  // nelder_mead.hpp:12
  const host::NelderMeadParams d;
  p->init_step = d.init_step;
  p->alpha = d.alpha;
  p->gamma = d.gamma;
  p->rho = d.rho;
  p->sigma = d.sigma;
  p->max_iterations = d.max_iterations;
  p->convergence_var_thresh = d.convergence_var_thresh;
}

int vlcal_nelder_mead_batched(int n, vlcal_nm_batch_fn f, vlcal_nm_observe_fn observe, void* user, const double* x0, const vlcal_nm_params* params, vlcal_nm_result* result) {
  if (n < 1 || n > NM_MAX_N || !f || !x0 || !params || !result) {
    set_last_error("invalid arguments (1 <= n <= 8)");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  host::NelderMeadParams p;
  p.init_step = params->init_step;
  p.alpha = params->alpha;
  p.gamma = params->gamma;
  p.rho = params->rho;
  p.sigma = params->sigma;
  p.max_iterations = params->max_iterations;
  p.convergence_var_thresh = params->convergence_var_thresh;
  auto bf = [&](const double* xs, int count, double* ys) { f(xs, count, n, ys, user); };
  auto ob = [&](const double* x, double y) {
    if (observe) observe(x, n, y, user);
  };
  const host::NelderMeadResult r = host::nelder_mead(n, bf, ob, x0, p, /*speculate=*/true);
  std::memset(result, 0, sizeof(*result));
  result->converged = r.converged ? 1 : 0;
  result->num_iterations = r.num_iterations;
  for (int d = 0; d < n; d++) result->x[d] = r.x[d];
  result->y = r.y;
  result->num_evaluations = r.num_evaluations;
  result->num_batches = r.num_batches;
  result->num_evaluations_computed = r.num_evaluations_computed;
  return VLCAL_OK;
}

void vlcal_calib_default_params(vlcal_calib_params* p) {  // visual_camera_calibration.hpp:12-26
  p->max_outer_iterations = 10;
  p->max_inner_iterations = 256;
  p->delta_trans_thresh = 0.1;
  p->delta_rot_thresh = 0.5 * M_PI / 180.0;
  p->disable_z_buffer_culling = 0;
  p->nid_bins = 16;
  p->nelder_mead_init_step = 1e-3;
  p->nelder_mead_convergence_criteria = 1e-8;
}

int vlcal_estimate_pose_nelder_mead_ctx(
  vlcal_nid_ctx* const* ctxs,
  int n_ctxs,
  const vlcal_calib_params* params,
  const double init_T_camera_lidar[16],
  vlcal_pose_callback callback,
  vlcal_allreduce_fn allreduce,
  void* user,
  double T_out[16],
  vlcal_nm_result* nm_result) {
  if (!ctxs || n_ctxs < 0 || !params || !init_T_camera_lidar || !T_out) {
    set_last_error("invalid arguments");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  for (int i = 0; i < n_ctxs; i++) {
    if (!ctxs[i]) {
      set_last_error("NULL context");
      return VLCAL_ERR_INVALID_ARGUMENT;
    }
  }
  return run_inner_solve(ctxs, n_ctxs, params, init_T_camera_lidar, callback, allreduce, user, T_out, nm_result);
}

int vlcal_estimate_poses_nelder_mead_ctx(
  vlcal_nid_ctx* const* ctxs,
  int n_ctxs,
  const vlcal_calib_params* params,
  int n_solves,
  const double* init_T_camera_lidar,
  const uint8_t* bag_mask,
  double* T_out,
  vlcal_nm_result* nm_results) {
  if (!ctxs || n_ctxs < 1 || !params || n_solves < 1 || !init_T_camera_lidar || !bag_mask || !T_out || !nm_results || params->max_inner_iterations < 0) {
    set_last_error("invalid arguments");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  for (int i = 0; i < n_ctxs; i++) {
    if (!ctxs[i]) {
      set_last_error("NULL context");
      return VLCAL_ERR_INVALID_ARGUMENT;
    }
    if (ctx_exchange_is_fused(ctxs[i])) {
      set_last_error("the solve axis is single-process: detach the peer exchange of every context");
      return VLCAL_ERR_UNSUPPORTED;
    }
  }
  if (!pk_supported(ctxs, n_ctxs)) {
    set_last_error("several solves per launch need the persistent kernel (float clouds, lean classifier, bins <= 32, one camera, image size and device)");
    return VLCAL_ERR_UNSUPPORTED;
  }
  return pk_solve_many(ctxs, n_ctxs, params, n_solves, init_T_camera_lidar, bag_mask, T_out, nm_results);
}

int vlcal_estimate_pose_nelder_mead(
  int device,
  int camera_model,
  const double* intrinsics,
  int n_intrinsics,
  const double* distortion,
  int n_distortion,
  const vlcal_bag* bags,
  int n_bags,
  const vlcal_calib_params* params,
  const double init_T_camera_lidar[16],
  vlcal_pose_callback callback,
  vlcal_allreduce_fn allreduce,
  void* user,
  int profiling,
  double T_out[16],
  vlcal_nm_result* nm_result,
  vlcal_calib_stats* stats) {
  int rc = check_common(params, init_T_camera_lidar, T_out, n_bags);
  if (rc != VLCAL_OK) return rc;
  CameraParams cam;
  rc = make_camera(camera_model, intrinsics, n_intrinsics, distortion, n_distortion, &cam);
  if (rc != VLCAL_OK) return rc;
  if (device < 0) VL_CUDA(cudaGetDevice(&device));
  VL_CUDA(cudaSetDevice(device));
  std::vector<ResidentBag> resident;
  const double t_up0 = now_ms();
  rc = upload_bags(device, cam, bags, n_bags, &resident);
  if (rc != VLCAL_OK) return rc;
  if (stats) {
    std::memset(stats, 0, sizeof(*stats));
    stats->upload_ms = now_ms() - t_up0;
  }
  rc = inner_solve_resident(device, cam, resident, params, init_T_camera_lidar, callback, allreduce, user, profiling, T_out, nm_result, stats, 0);
  if (rc == VLCAL_OK && stats) stats->outer_iterations = 1;
  return rc;
}

int vlcal_calibrate_nelder_mead(
  int device,
  int camera_model,
  const double* intrinsics,
  int n_intrinsics,
  const double* distortion,
  int n_distortion,
  const vlcal_bag* bags,
  int n_bags,
  const vlcal_calib_params* params,
  const double init_T_camera_lidar[16],
  vlcal_pose_callback callback,
  vlcal_allreduce_fn allreduce,
  void* user,
  int profiling,
  double T_out[16],
  vlcal_calib_stats* stats) {
  int rc = check_common(params, init_T_camera_lidar, T_out, n_bags);
  if (rc != VLCAL_OK) return rc;
  CameraParams cam;
  rc = make_camera(camera_model, intrinsics, n_intrinsics, distortion, n_distortion, &cam);
  if (rc != VLCAL_OK) return rc;
  if (device < 0) VL_CUDA(cudaGetDevice(&device));
  VL_CUDA(cudaSetDevice(device));
  std::vector<ResidentBag> resident;
  const double t_up0 = now_ms();
  rc = upload_bags(device, cam, bags, n_bags, &resident);
  if (rc != VLCAL_OK) return rc;
  if (stats) {
    std::memset(stats, 0, sizeof(*stats));
    stats->upload_ms = now_ms() - t_up0;
  }

  double T[16];
  std::memcpy(T, init_T_camera_lidar, sizeof(T));
  for (int i = 0; i < params->max_outer_iterations; i++) {  // visual_camera_calibration.cpp:39
    double new_T[16];
    rc = inner_solve_resident(device, cam, resident, params, T, callback, allreduce, user, profiling, new_T, nullptr, stats, i);  // :46
    if (rc != VLCAL_OK) return rc;
    double delta_t, delta_r;
    outer_step_delta(T, new_T, &delta_t, &delta_r);
    std::memcpy(T, new_T, sizeof(T));  // :51
    const bool converged = delta_t < params->delta_trans_thresh && delta_r < params->delta_rot_thresh;  // :55
    if (stats) stats->outer_iterations = i + 1;
    if (converged) break;  // :62-64
  }
  std::memcpy(T_out, T, sizeof(T));
  return VLCAL_OK;
}

int vlcal_outer_step_delta(const double T_colmajor[16], const double new_T_colmajor[16], double* delta_t, double* delta_r) {
  if (!T_colmajor || !new_T_colmajor || !delta_t || !delta_r) {
    set_last_error("NULL argument");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  outer_step_delta(T_colmajor, new_T_colmajor, delta_t, delta_r);
  return VLCAL_OK;
}

}  // extern "C"
