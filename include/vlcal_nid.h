/*
 * vlcal_nid.h -- C ABI of the GPU-native (H100) NID registration engine (libvlcal_nid.so).
 *
 * This is the drop-in boundary for ONE hot path of koide3/direct_visual_lidar_calibration:
 * the per-evaluation NID cost and the Nelder-Mead solve that drives it.  Every entry point
 * names the reference interface it replaces (paths relative to the reference repo root).
 * Plain pointers and sizes only; no C++/torch types.  All matrices are 4x4 double,
 * COLUMN-MAJOR (the memory of Eigen::Isometry3d::matrix().data()).
 *
 * Error convention (reference: I/O failure -> abort(), src/calibrate.cpp:31-34; unknown camera
 * model -> nullptr, src/camera/create_camera.cpp:49-50): every function returns an int status,
 * 0 = OK, < 0 = error; nothing throws or aborts across this boundary.  vlcal_nid_last_error()
 * returns a thread-local message for the last failure.  There is NO CPU fallback: without a
 * usable CUDA device the create/evaluate functions fail with VLCAL_ERR_CUDA / VLCAL_ERR_NO_DEVICE.
 *
 * Threading (reference: calculate() is called from OpenMP workers, one cost object per bag,
 * never re-entered; src/vlcal/calib/visual_camera_calibration.cpp:107-110): contexts may be
 * created / used from any host thread; different contexts may be used concurrently; one context
 * must not be used from two threads at once.
 */
#ifndef VLCAL_NID_H
#define VLCAL_NID_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VLCAL_OK 0
#define VLCAL_ERR_INVALID_ARGUMENT (-1)
#define VLCAL_ERR_UNKNOWN_CAMERA_MODEL (-2) /* create_camera.cpp:49-50 (nullptr) */
#define VLCAL_ERR_INTRINSIC_COUNT (-3)      /* create_camera.cpp:19-22 (nullptr) */
#define VLCAL_ERR_CUDA (-4)
#define VLCAL_ERR_NO_DEVICE (-5)
#define VLCAL_ERR_UNSUPPORTED (-6)
#define VLCAL_ERR_BUSY (-7)

/* camera model ids, in the order of the string switch at src/camera/create_camera.cpp:35-46 */
#define VLCAL_CAMERA_PLUMB_BOB 0           /* "plumb_bob"            include/camera/pinhole.hpp */
#define VLCAL_CAMERA_FISHEYE 1             /* "fisheye"|"equidistant" include/camera/fisheye.hpp */
#define VLCAL_CAMERA_ATAN 2                /* "atan"                 include/camera/atan.hpp */
#define VLCAL_CAMERA_OMNIDIR 3             /* "omnidir"              include/camera/omnidir.hpp */
#define VLCAL_CAMERA_EQUIRECTANGULAR 4     /* "equirectangular"      include/camera/equirectangular.hpp */
#define VLCAL_CAMERA_RATIONAL_POLYNOMIAL 5 /* "rational_polynomial"  include/camera/rational_polynomial.hpp */

/* cost modes */
#define VLCAL_NID_MODE_HISTOGRAM 0 /* "mode A": CostCalculatorNID::calculate, integer joint histogram, nearest pixel
                                      src/vlcal/calib/cost_calculator_nid.cpp:21-67 (what dfo::NelderMead scores) */
#define VLCAL_NID_MODE_BSPLINE 1   /* "mode B": NIDCost::operator()<double>, 4x4 cubic-B-spline soft histogram (value only)
                                      include/vlcal/costs/nid_cost.hpp:36-107 */

typedef struct vlcal_nid_ctx vlcal_nid_ctx;

/* ---- library / errors ------------------------------------------------------------------ */

/* "major.minor.patch" of this library */
const char* vlcal_nid_version(void);
/* message of the last error on the calling thread ("" if none) */
const char* vlcal_nid_last_error(void);
/* number of visible CUDA devices (0 if none / no driver); never fails */
int vlcal_nid_device_count(void);

/* ---- camera factory facts (src/camera/create_camera.cpp:17-50) ----------------------- */

/* model string -> id; VLCAL_ERR_UNKNOWN_CAMERA_MODEL where the reference returns nullptr */
int vlcal_camera_model_id(const char* camera_model);
/* CameraModelTraits<>::num_intrinsic_params / num_distortion_params of a model id */
int vlcal_camera_num_params(int camera_model, int* n_intrinsics, int* n_distortion);
/* GenericCameraBase::project(point_3d) for one point (host, double) -- include/camera/generic_camera.hpp:21-28.
 * Intrinsic count must match the model (else VLCAL_ERR_INTRINSIC_COUNT); distortion is zero-padded/truncated. */
int vlcal_camera_project(int camera_model, const double* intrinsics, int n_intrinsics, const double* distortion, int n_distortion, const double point_3d[3], double uv[2]);

/* ---- host math shared by callers ----------------------------------------------------- */

/* gtsam::Pose3::Expmap(x).matrix(), x = (wx,wy,wz,vx,vy,vz) -- call sites visual_camera_calibration.cpp:104,129 */
int vlcal_se3_expmap_gtsam(const double x[6], double T_colmajor[16]);
/* vlcal::estimate_camera_fov(proj, image_size) -- src/vlcal/common/estimate_fov.cpp:36-51 */
int vlcal_estimate_camera_fov(int camera_model, const double* intrinsics, int n_intrinsics, const double* distortion, int n_distortion, int width, int height, double* max_fov_rad);

/* ---- the cost object: CostCalculatorNID(proj, data, NIDCostParams{bins}) ---------------
 * replaces the constructor at src/vlcal/calib/cost_calculator_nid.cpp:13-17 (one per bag per outer
 * iteration, visual_camera_calibration.cpp:82-84).  Copies image and points host -> device (caller keeps
 * ownership).  points_xyzw = Eigen::Vector4d[n] (x,y,z,1), intensities = double[n]
 * (include/vlcal/common/frame.hpp:66,69).  max_fov_rad: pass a negative value to have the library compute
 * estimate_camera_fov(camera, {width,height}) exactly as the reference constructor does (:17).
 * device: CUDA ordinal, or -1 for the current device. */
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
  double max_fov_rad);

/* CostCalculatorNID::~CostCalculatorNID; frees device memory; NULL is a no-op */
void vlcal_nid_destroy(vlcal_nid_ctx* ctx);

/* CostCalculator::calculate(T_camera_lidar) for P poses in ONE pass over the cloud
 * (include/vlcal/calib/cost_calculator.hpp:17; src/vlcal/calib/cost_calculator_nid.cpp:21-67).
 * T_camera_lidar: P x 16 doubles (column-major 4x4 each).  nid_out: P doubles (NaN where the reference returns
 * NaN, i.e. no inliers).  hist_out: optional P x bins x bins int32, index = image_bin + lidar_bin*bins
 * (the storage of Eigen::MatrixXi hist(image_bin, lidar_bin)); pass NULL to skip.  Synchronous. */
int vlcal_nid_evaluate(vlcal_nid_ctx* ctx, const double* T_camera_lidar, int n_poses, double* nid_out, int32_t* hist_out);

/* same, split so that several contexts (bags) overlap on the GPU: _async enqueues on the context's stream and
 * returns; _wait blocks until that evaluation is done and delivers the results. One evaluation in flight per
 * context (VLCAL_ERR_BUSY otherwise).  _async computes no histograms: after it, _wait's hist_out must be NULL
 * (VLCAL_ERR_INVALID_ARGUMENT otherwise; the scores are still delivered and the evaluation is no longer in flight). */
int vlcal_nid_evaluate_async(vlcal_nid_ctx* ctx, const double* T_camera_lidar, int n_poses);
int vlcal_nid_wait(vlcal_nid_ctx* ctx, double* nid_out, int32_t* hist_out);

/* the objective of visual_camera_calibration.cpp:105-110 for a pose LIST of any length: nid_out[p] = sum over the contexts
 * (bags, in the order given) of CostCalculatorNID::calculate(T_p).  One persistent launch scores every pose on every bag
 * (pose-grid search, BASELINE config 5: 16 384 poses x 5 M points); contexts must share camera, image size, bins and
 * device for that -- otherwise it falls back to one batched evaluation per context.  Every score equals the one
 * vlcal_nid_evaluate returns for that pose, bit for bit. */
int vlcal_nid_score_poses(vlcal_nid_ctx* const* ctxs, int n_ctxs, const double* T_camera_lidar, int n_poses, double* nid_out);

/* ---- pose sweep: very long pose lists on small clouds (the global initial-guess search) -----------------------------
 * Same scores as vlcal_nid_score_poses -- nid_out[p] = sum over the contexts, in the order given, of
 * CostCalculatorNID::calculate(T_p), bit for bit -- computed pose-parallel: one thread block owns a few poses from the
 * first point to the finished NID, so 10^5-10^6 poses on 10^4-10^5 points fill the GPU, where the persistent kernel's
 * pose-list mode (8 poses per pass, one block per 768 points) leaves most of it idle.  When the contexts hold more than
 * vlcal_nid_sweep_max_points() points together the list is handed to that kernel instead (same results).
 * Contexts: mode A, float4 clouds, bins <= 32, one camera / image size / bins / device, at most 8 of them; anything else
 * is VLCAL_ERR_UNSUPPORTED.  hist_out: optional P x bins x bins int32 joint histograms of ctxs[0], laid out as in
 * vlcal_nid_evaluate.  Synchronous. */
int vlcal_nid_sweep_poses(vlcal_nid_ctx* const* ctxs, int n_ctxs, const double* T_camera_lidar, int64_t n_poses, double* nid_out, int32_t* hist_out);

/* A pose list described by small tables instead of P matrices; the poses are generated on the device.  Pose i, with
 * i = (ib * n_left + il) * n_offset + io:
 *     R = left[il] * base[ib],   t = R * (center[ib] + offset[io]),   T_camera_lidar = [R | t]
 * so with center = -(camera position in the LiDAR frame) the offsets move the camera position and leave the rotation
 * alone.  Every product and sum is one IEEE round-to-nearest operation, row by row, ((a0*b0 + a1*b1) + a2*b2): a host that
 * does the same operations gets the same bits.  indices: optional n_poses flat indices i (a subset, in any order); NULL
 * means all n_base * n_left * n_offset poses in order, and n_poses must be that product. */
typedef struct vlcal_search_set {
  const double* left;   /* n_left x 9, row-major 3x3 */
  const double* base;   /* n_base x 9 */
  const double* center; /* n_base x 3 */
  const double* offset; /* n_offset x 3 */
  const int32_t* indices;
  int32_t n_left, n_base, n_offset;
  int64_t n_poses;
} vlcal_search_set;

/* vlcal_nid_sweep_poses for the poses of a search set (no upload of the matrices) */
int vlcal_nid_sweep_search_set(vlcal_nid_ctx* const* ctxs, int n_ctxs, const vlcal_search_set* set, double* nid_out);
/* the same, and per pose the number of points the reference counts (hist_image.sum(), cost_calculator_nid.cpp:54) summed
 * over the contexts: a search uses it to set aside poses that see next to nothing, whose NID is meaninglessly low */
int vlcal_nid_sweep_search_set_inliers(vlcal_nid_ctx* const* ctxs, int n_ctxs, const vlcal_search_set* set, double* nid_out, int64_t* inliers_out);
/* the poses of a search set as the device generates them: n_poses x 16 doubles, column-major (device -1: the current one) */
int vlcal_search_set_poses(int device, const vlcal_search_set* set, double* T_camera_lidar_out);
/* cloud size (points of all contexts together) up to which the sweep kernel runs */
int64_t vlcal_nid_sweep_max_points(void);
/* launch geometry of the sweep kernel for this context's camera model: blocks that are resident at once on its device,
 * and the poses one block scores together */
int vlcal_nid_sweep_launch_shape(const vlcal_nid_ctx* ctx, int* blocks, int* poses_per_block);
/* measurement hooks: the sweep kernel whatever the cloud size (the crossover measurement), and the kernel time of the
 * calling thread's last sweep in milliseconds (CUDA events around the kernel; 0 when the persistent kernel ran instead) */
int vlcal_nid_debug_sweep_kernel(vlcal_nid_ctx* const* ctxs, int n_ctxs, const double* T_camera_lidar, int64_t n_poses, double* nid_out, int32_t* hist_out);
double vlcal_nid_sweep_last_kernel_ms(void);
/* debug count of the calling thread's last vlcal_nid_debug_sweep_kernel call: (point, pose) pairs, summed over the
 * contexts, that the sweep kernel's fp32 filter deferred to the exact path; -1 after any other sweep entry point */
int64_t vlcal_nid_debug_sweep_last_deferred(void);

/* mode B evaluation with the reference's parameterisation: T_params = P x 7 doubles [qx qy qz qw tx ty tz]
 * (Sophus::SE3d storage, include/vlcal/costs/nid_cost.hpp:38).  ok_out[p] = 0 where the reference functor returns
 * false (non-finite NID, :98-102).  hist_out: optional P x bins x bins doubles (un-normalised). */
int vlcal_nid_evaluate_bspline(vlcal_nid_ctx* ctx, const double* T_params, int n_poses, double* nid_out, int32_t* ok_out, double* hist_out);

/* mode B value AND gradient: what ceres::AutoDiffFirstOrderFunction<MultiNIDCost, 7> evaluates per bag in the
 * reference's BFGS branch (NIDCost::operator()<ceres::Jet<double, 7>>, nid_cost.hpp:36-107 called from
 * visual_camera_calibration.cpp:141-173,211).  grad_out = P x 7 doubles, d NID / d [qx qy qz qw tx ty tz] (ambient
 * parameters; the reference's Sophus::Manifold<SE3> projects them onto the 6-D tangent space afterwards).
 * ok_out as above.  One kernel launch per pose. */
int vlcal_nid_evaluate_bspline_grad(vlcal_nid_ctx* ctx, const double* T_params, int n_poses, double* nid_out, double* grad_out, int32_t* ok_out);

/* introspection */
int64_t vlcal_nid_num_points(const vlcal_nid_ctx* ctx);
int vlcal_nid_bins(const vlcal_nid_ctx* ctx);
double vlcal_nid_max_fov(const vlcal_nid_ctx* ctx);
/* 1 if the cloud is stored as float4 (x,y,z,intensity) = 16 B/point (lossless: inputs were float32-representable,
 * SURVEY D9), 0 if the 32 B/point double layout had to be used */
int vlcal_nid_points_are_f32(const vlcal_nid_ctx* ctx);
/* max poses one kernel launch carries (larger batches are split into several launches) */
int vlcal_nid_max_poses_per_launch(void);

/* measurement hooks (bench.py): with profiling on, every histogram-kernel launch is bracketed by CUDA events on the
 * context's stream. get_profile returns totals since the last reset. */
int vlcal_nid_set_profiling(vlcal_nid_ctx* ctx, int enable);
int vlcal_nid_get_profile(vlcal_nid_ctx* ctx, int64_t* kernel_launches, double* kernel_ms_total, int64_t* poses_total);
int vlcal_nid_reset_profile(vlcal_nid_ctx* ctx);
/* passes over the cloud since the last reset: a persistent launch (one per inner solve / pose list) carries one pass per
 * Nelder-Mead batch / chunk of 8 poses, a round-1 launch is one pass.  Algorithmic bytes = passes x (16 N + W H). */
int vlcal_nid_get_profile_passes(vlcal_nid_ctx* ctx, int64_t* passes);
/* persistent kernel, since the last reset: stats[0] passes whose poses were classified as first-order updates from the
 * batch's anchor (equirectangular batches of nearby poses), stats[1] the poses of those passes, stats[2] point-poses
 * deferred to the exact fp64 path in the other passes, stats[3] point-poses deferred in the delta passes */
int vlcal_nid_get_profile_delta(vlcal_nid_ctx* ctx, int64_t stats[4]);
/* measurement hook: poses carried by one pass over the cloud in pose-list evaluations (vlcal_nid_evaluate /
 * vlcal_nid_score_poses) of this context, 1..8 (default 8).  Results do not depend on it; bench.py uses 1 to measure the
 * P = 1 roofline point (one pose per 16 N + W H algorithmic bytes). */
int vlcal_nid_set_poses_per_pass(vlcal_nid_ctx* ctx, int poses_per_pass);
/* measurement hook for the persistent solve: call with stamps_out == NULL to arm (the next persistent solve on this
 * context records %globaltimer stamps for its first `capacity` batches), then again with a buffer of capacity x 8 words:
 * per batch {block 0 enters, main loop done, merged + arrived, finalizer: all blocks arrived, score published,
 * block 0: all scores seen, next poses ready, unused}. */
int vlcal_nid_debug_solve_stamps(vlcal_nid_ctx* ctx, int capacity, uint64_t* stamps_out, int* n_out);
/* with the stamps armed, every block of the persistent solve also records {enters the batch, histogram copies zeroed, main
 * loop done, arrived} for one batch (the 9th): capacity_blocks x 4 words out, *n_blocks = blocks of that launch */
int vlcal_nid_debug_block_times(vlcal_nid_ctx* ctx, int capacity_blocks, uint64_t* times_out, int* n_blocks);
/* kernel selection for A/B measurements: 0 = default (fp32 filter + exact fp64 recheck; the persistent kernel at 2 points
 * per lane and tile, the round-1 kernels, where they run, at 2 or 4 chosen from the camera model and the cloud size),
 * 1 = exact fp64 only, 2 = filter forced to 2 points, 3 = filter forced to 4 points (in the persistent kernel for
 * plumb_bob, omnidir and rational_polynomial only; the other models keep 2), 4 = round-1 kernels (one launch per batch;
 * the persistent kernel is not used) */
int vlcal_nid_set_kernel_variant(vlcal_nid_ctx* ctx, int variant);

/* measurement hook: one launch (n_poses <= 8) with %globaltimer stamps; out_us = {main loop done, merged, ticket, finalize done,
 * published} in microseconds since the first block started, host-side {launch call, launch->results visible}, then inside the
 * finalize {scratch zeroed, marginals known, entropy terms staged}; 12 doubles */
int vlcal_nid_debug_timeline(vlcal_nid_ctx* ctx, const double* T_camera_lidar, int n_poses, double out_us[12]);
/* permutes the context's cloud so that points projecting to the same 32x8-pixel image tile at pose T are adjacent (GPU
 * counting sort).  The integer histogram -- hence every NID value -- is invariant under this permutation; it only makes
 * the per-point image gathers of later evaluations near T coalesce.  Contexts built by vlcal_estimate_pose_nelder_mead /
 * vlcal_calibrate_nelder_mead are ordered this way by their culling pass already. */
int vlcal_nid_reorder_for_pose(vlcal_nid_ctx* ctx, const double T_camera_lidar[16]);
/* device / pinned buffers of destroyed contexts are cached for reuse (contexts are rebuilt every outer iteration);
 * this releases the cache back to the CUDA driver */
int vlcal_nid_trim_memory(void);
/* 1 if evaluations of this context run the fp32-filter kernel (camera model / FoV / float32-representable cloud) */
int vlcal_nid_filter_enabled(const vlcal_nid_ctx* ctx);
/* test hook: runs the fp32 filter AND the exact path on every (point, pose) and reports counts[0] = point-poses,
 * counts[1] = verdicts the filter deferred to the exact path, counts[2] = filter verdicts it kept that disagree with the
 * exact path (MUST be 0), *max_bound_ratio = max |uv_fp32 - uv_exact| / error-bound over kept in-image verdicts (< 1). */
int vlcal_nid_debug_filter_check(vlcal_nid_ctx* ctx, const double* T_camera_lidar, int n_poses, uint64_t counts[3], double* max_bound_ratio);
/* the same for the equirectangular delta step of the persistent kernel: in every group of 8 poses the kernel's anchor
 * (the most central pose) is classified as the anchor and the others as first-order updates from it (whatever their
 * spread) */
int vlcal_nid_debug_filter_check_delta(vlcal_nid_ctx* ctx, const double* T_camera_lidar, int n_poses, uint64_t counts[3], double* max_bound_ratio);

/* ---- multi-GPU: fused bag all-reduce over NVLink peer memory ---------------------------------------------------------
 * One process per GPU, the same number of bags (cost objects) per process.  The joint objective is sum_bags NID
 * (visual_camera_calibration.cpp:105-110).  With an exchange attached, an inner solve (vlcal_estimate_pose_* on the
 * attached contexts) is one persistent launch per rank: per Nelder-Mead batch one block per (bag, pose) stores the score into
 * every other rank's mailbox (P2P stores, cudaIpc-shared buffers, tagged words) and every block of every rank adds the
 * contributions in (rank, bag) order -- identical bits on every rank, no separate collective, no host in the loop.
 * vlcal_nid_evaluate / _wait on an attached context (one bag per process) run the round-1 kernels, whose finalizing block
 * performs the same exchange and returns the SUM OVER RANKS.  All ranks must evaluate the same number of poses in the same
 * order (Nelder-Mead does).
 *   1. every rank: vlcal_nid_p2p_create(device, rank, world, &px, handle)   (handle: 64 bytes out)
 *   2. exchange the 64-byte handles between the ranks (e.g. torch.distributed.all_gather), concatenate in rank order
 *   3. every rank: vlcal_nid_p2p_connect(px, all_handles);   4. vlcal_nid_p2p_attach(ctx, px) on each new context */
typedef struct vlcal_p2p vlcal_p2p;
int vlcal_nid_p2p_create(int device, int rank, int world, vlcal_p2p** out, void* ipc_handle_out);
int vlcal_nid_p2p_connect(vlcal_p2p* px, const void* all_handles);
int vlcal_nid_p2p_attach(vlcal_nid_ctx* ctx, vlcal_p2p* px); /* px == NULL detaches */
void vlcal_nid_p2p_destroy(vlcal_p2p* px);
/* contexts that vlcal_estimate_pose_nelder_mead / vlcal_calibrate_nelder_mead build internally attach this exchange; NULL
 * clears it.  Before every solve on a connected exchange the ranks agree on the solve path (DESIGN.md section 7): ranks
 * whose plans differ take the host loop together when each holds one bag, and otherwise all return
 * VLCAL_ERR_UNSUPPORTED.  With several local bags and no persistent solve, an allreduce callback sums the host loop. */
int vlcal_nid_p2p_set_default(vlcal_p2p* px);

/* ---- view culling: ViewCulling::cull (src/vlcal/calib/view_culling.cpp:21-92) ------------
 * GPU z-buffer hidden-point removal at pose T.  indices_out: capacity n_points int32, receives the kept
 * original indices in ascending order; *n_kept their count.  max_fov_rad < 0 -> estimate_camera_fov. */
int vlcal_view_cull(
  int device,
  int camera_model,
  const double* intrinsics,
  int n_intrinsics,
  const double* distortion,
  int n_distortion,
  int width,
  int height,
  double max_fov_rad,
  int enable_depth_buffer_culling,
  const double* points_xyzw,
  int64_t n_points,
  const double T_camera_lidar[16],
  int32_t* indices_out,
  int64_t* n_kept);
/* test hook: view culling as the cost objects of the solver run it, with the culled cloud kept on the device and no index
 * list.  keep_all == 0: the kept points grouped by 32 x 8-pixel image tile at T (the cloud vlcal_calibrate_nelder_mead
 * scores); keep_all != 0: every point, grouped the same way, the ones out of view last (vlcal_nid_reorder_for_pose).
 * points_out: capacity n_points x 4 doubles, receives (x, y, z, intensity) of the culled cloud in its device order;
 * *n_kept its count; *points_are_f32 (may be NULL): 1 if the cloud went to the device in the float4 layout. */
int vlcal_debug_view_cull_points(
  int device,
  int camera_model,
  const double* intrinsics,
  int n_intrinsics,
  const double* distortion,
  int n_distortion,
  int width,
  int height,
  double max_fov_rad,
  int enable_depth_buffer_culling,
  int keep_all,
  const double* points_xyzw,
  const double* intensities,
  int64_t n_points,
  const double T_camera_lidar[16],
  double* points_out,
  int64_t* n_kept,
  int* points_are_f32);

/* ---- LiDAR intensity image: vlcal::generate_lidar_image (src/vlcal/preprocess/generate_lidar_image.cpp:8-41) ----------
 * The rendering `preprocess` / `initial_guess_*` use: per pixel the projected point with the smallest squared range (of
 * equal ones the last), same FoV / projection / truncation rules as the NID cost, FoV from estimate_camera_fov(camera,
 * {width, height}).  intensity_image_out: H x W doubles (CV_64FC1; 0 where no point lands), index_image_out: H x W int32
 * (CV_32SC1; -1 where no point lands).  Exact: both images equal the reference's bit for bit.  At most 2^31-1 points and
 * 2^31-1 pixels (width * height); larger inputs are refused with VLCAL_ERR_INVALID_ARGUMENT before anything is allocated. */
int vlcal_generate_lidar_image(
  int device,
  int camera_model,
  const double* intrinsics,
  int n_intrinsics,
  const double* distortion,
  int n_distortion,
  int width,
  int height,
  const double T_camera_lidar[16],
  const double* points_xyzw,
  const double* intensities,
  int64_t n_points,
  double* intensity_image_out,
  int32_t* index_image_out);

/* ---- headless viewer: looking at a calibration (src/viewer.cpp, src/vlcal/common/points_color_updater.cpp) -------------
 * Both entry points take the camera, the uint8 grayscale image (row_stride bytes per row), the pose and the cloud as
 * vlcal_generate_lidar_image does, and follow its argument rules (at most 2^31-1 points and pixels; an empty cloud is
 * legal).  blend_weight in [0, 1] is the weight w of the camera image; a colour is
 *     gray * w + turbo(intensity) * (1 - w)          gray = pixel / 255.0f, all in float32, 1 - w rounded from double
 * with turbo(x) = entry clamp(int(float(x) * 255.0), 0, 255) (NaN: 0) of the 256-entry Turbo table / 255.0f.
 * kernel_ms_out (may be NULL): time of the kernels alone between CUDA events, without uploads and read-back. */

/* the 256 RGB byte triples of the Turbo table the viewer colours intensities with (host data; needs no device) */
int vlcal_turbo_colormap(uint8_t rgb_out[768]);

/* PointsColorUpdater::update (points_color_updater.cpp:37-61): rgba_out[4 i ..] = colour of point i with alpha 1, or
 * (0, 0, 0, 0) where the reference skips the point: outside cos(estimate_camera_fov(camera, {width, height}) + 0.5 deg)
 * -- the viewer's own threshold, looser than the cost's -- or projected outside the image.  Projection, truncation and
 * bounds test are the NID cost's, decision for decision. */
int vlcal_colorize_points(
  int device,
  int camera_model,
  const double* intrinsics,
  int n_intrinsics,
  const double* distortion,
  int n_distortion,
  int width,
  int height,
  const uint8_t* image,
  int row_stride,
  const double T_camera_lidar[16],
  const double* points_xyzw,
  const double* intensities,
  int64_t n_points,
  float blend_weight,
  float* rgba_out, /* n_points x 4 */
  double* kernel_ms_out);

/* The cloud drawn into the camera image with hidden points removed: per pixel the point with the smallest squared range
 * wins (of equal ones the last), by the rules and FoV of vlcal_generate_lidar_image, where every point covers the
 * (2 point_radius + 1)^2 square of pixels around its own, clipped to the image; point_radius in [0, 8], and 0 gives the
 * index map of vlcal_generate_lidar_image.  bgr_out: H x W x 3 bytes (CV_8UC3), a covered pixel the colour above of its
 * winner and its own gray value, rounded to nearest, an uncovered pixel its gray value.  index_image_out (may be NULL):
 * H x W int32, the winner per pixel, -1 where none. */
int vlcal_render_overlay(
  int device,
  int camera_model,
  const double* intrinsics,
  int n_intrinsics,
  const double* distortion,
  int n_distortion,
  int width,
  int height,
  const uint8_t* image,
  int row_stride,
  const double T_camera_lidar[16],
  const double* points_xyzw,
  const double* intensities,
  int64_t n_points,
  int point_radius,
  float blend_weight,
  uint8_t* bgr_out,
  int32_t* index_image_out,
  double* kernel_ms_out);

/* Agreement map at T_camera_lidar: per point, the pointwise mutual information log(p(a,b) / (p(a) p(b))) of its joint bin
 * (image bin a, LiDAR bin b) in the NID histogram of the pose, computed as log(c_ab * N / (c_a * c_b)) from the integer
 * counts; the histogram is calculate's (same decision per point, same bins, same FoV).  pmi_out: [n_points], NaN for a
 * point the histogram does not count.  hist_out (may be NULL): [bins * bins] at image_bin + lidar_bin * bins, as
 * vlcal_nid_evaluate's hist_out.  bgr_out / index_image_out: as vlcal_render_overlay, with the winner's colour
 * turbo(0.5 + PMI / (2 * VLCAL_AGREEMENT_PMI_RANGE)) in place of turbo(intensity): red where the point's bin pair is more
 * frequent than chance (the LiDAR and the camera agree), blue where it is rarer.  bins in [1, 32]. */
#define VLCAL_AGREEMENT_PMI_RANGE 2.0
int vlcal_agreement_map(
  int device,
  int camera_model,
  const double* intrinsics,
  int n_intrinsics,
  const double* distortion,
  int n_distortion,
  int width,
  int height,
  const uint8_t* image,
  int row_stride,
  const double T_camera_lidar[16],
  const double* points_xyzw,
  const double* intensities,
  int64_t n_points,
  int bins,
  int point_radius,
  float blend_weight,
  double* pmi_out,
  int32_t* hist_out,
  uint8_t* bgr_out,
  int32_t* index_image_out);

/* ---- solver surface ------------------------------------------------------------------ */

/* how vlcal_estimate_pose_nelder_mead* / vlcal_calibrate_nelder_mead iterate (process-wide):
 *   0 auto (default): 3 where possible, else 1.
 *   3 persistent kernel: the whole inner solve is ONE cooperative launch -- candidates scored on every local bag, summed
 *     over bags and (peer exchange) ranks, Nelder-Mead machine stepped redundantly by every block in shared memory.
 *     Needs float4 clouds, bins <= 32, one camera / image size / device, no host all-reduce callback; VLCAL_ERR_UNSUPPORTED
 *     otherwise.  params.callback is delivered after the solve from the evaluation trace, in the reference's order.
 *   1 host loop: one launch per Nelder-Mead batch, scores published to mapped host memory, host polls.
 * Both loops walk the same Nelder-Mead trajectory, bit for bit (tests/test_gpu_parity.py).  Any other mode, 2 included,
 * is VLCAL_ERR_INVALID_ARGUMENT. */
int vlcal_nid_set_solver_mode(int mode);
/* test hook: with recording armed on the calling thread (enable != 0; off by default, 0 turns it off again), every inner
 * solve (vlcal_estimate_pose_nelder_mead*, any solver mode) run on that thread keeps its evaluations as the best-cost
 * callback logic saw them, in the reference's order; vlcal_nid_debug_last_solve_trace returns those of the last solve --
 * capacity x 7 doubles {x[6], y} out, *n_out = the solve's count (may exceed capacity) */
int vlcal_nid_debug_record_solve_trace(int enable);
int vlcal_nid_debug_last_solve_trace(int capacity, double* rows_out, int* n_out);
/* test hook: points per lane (2 or 4) of the kernel instance the last persistent launch on this context ran (0: none yet) */
int vlcal_nid_debug_last_points_per_lane(const vlcal_nid_ctx* ctx, int* k_out);

/* dfo::NelderMead<N>::Params (include/dfo/nelder_mead.hpp:11-22) */
typedef struct {
  double init_step;              /* 0.1  */
  double alpha;                  /* 1.0  */
  double gamma;                  /* 2.0  */
  double rho;                    /* 0.5  */
  double sigma;                  /* 0.5 (unused by the reference) */
  int max_iterations;            /* 1024 */
  double convergence_var_thresh; /* 1e-5 */
} vlcal_nm_params;

/* dfo::OptimizationResult<N> (include/dfo/optimizer.hpp:8-20) + evaluation counters */
typedef struct {
  int converged;
  int num_iterations;
  double x[8];
  double y;
  int num_evaluations;           /* evaluations the reference's serial NelderMead would have requested */
  int num_batches;               /* batched objective calls issued */
  int num_evaluations_computed;  /* poses actually scored (incl. speculative ones) */
} vlcal_nm_result;

void vlcal_nm_default_params(vlcal_nm_params* p);

/* batch objective: ys[i] = f(xs + i*n) for i < count */
typedef void (*vlcal_nm_batch_fn)(const double* xs, int count, int n, double* ys, void* user);
/* observer called once per evaluation THE REFERENCE WOULD HAVE MADE, in the reference's order (this is where the
 * objective's side effects -- best-cost bookkeeping / params.callback, visual_camera_calibration.cpp:112-116 -- go) */
typedef void (*vlcal_nm_observe_fn)(const double* x, int n, double y, void* user);

/* dfo::NelderMead<N>::optimize with the exact trajectory of the serial reference (include/dfo/nelder_mead.hpp:32-101),
 * but asking for all candidates of an iteration {xo, xr, xe, xc} (or the shrink set) in one batch call. n <= 8. */
int vlcal_nelder_mead_batched(int n, vlcal_nm_batch_fn f, vlcal_nm_observe_fn observe, void* user, const double* x0, const vlcal_nm_params* params, vlcal_nm_result* result);

/* VisualCameraCalibrationParams (include/vlcal/calib/visual_camera_calibration.hpp:10-40) -- Nelder-Mead branch */
typedef struct {
  int max_outer_iterations;                /* 10 */
  int max_inner_iterations;                /* 256 */
  double delta_trans_thresh;               /* 0.1 [m] */
  double delta_rot_thresh;                 /* 0.5 deg in rad */
  int disable_z_buffer_culling;            /* 0 */
  int nid_bins;                            /* 16 */
  double nelder_mead_init_step;            /* 1e-3 */
  double nelder_mead_convergence_criteria; /* 1e-8 */
} vlcal_calib_params;
void vlcal_calib_default_params(vlcal_calib_params* p);

/* params.callback(T_camera_lidar) (visual_camera_calibration.hpp:38) -- fired on each best-cost improvement */
typedef void (*vlcal_pose_callback)(const double T_camera_lidar[16], double cost, void* user);
/* optional cross-process reduction of the per-pose partial sums over LOCAL bags (multi-GPU bag sharding):
 * must replace vals[0..count) by the sum over all ranks, identically on every rank. NULL = single process. */
typedef void (*vlcal_allreduce_fn)(double* vals, int count, void* user);

/* one bag as the reference's VisualLiDARData (include/vlcal/common/visual_lidar_data.hpp:10-23): host buffers */
typedef struct {
  const uint8_t* image; /* CV_8UC1 */
  int width, height, row_stride_bytes;
  const double* points_xyzw; /* Eigen::Vector4d[n] */
  const double* intensities; /* double[n] */
  int64_t n_points;
} vlcal_bag;

typedef struct {
  int outer_iterations;
  int total_evaluations;          /* reference-equivalent objective evaluations */
  int total_evaluations_computed; /* poses actually scored per bag */
  int total_batches;
  int inner_iterations[16];
  double inner_final_cost[16];
  int64_t culled_points[16]; /* points kept by view culling in bag 0 per outer iteration */
  int64_t kernel_launches;
  double kernel_ms_total; /* only if profiling != 0 */
  /* host wall-clock breakdown of the call, milliseconds (summed over outer iterations) */
  double upload_ms;  /* host double -> float4 conversion + H2D of clouds and images */
  double cull_ms;    /* GPU view culling + cost-object construction */
  double solve_ms;   /* Nelder-Mead inner solves */
} vlcal_calib_stats;

/* the objective of estimate_pose_nelder_mead (visual_camera_calibration.cpp:103-119) over already-built cost
 * objects: T = init_T * Expmap(x), sum over ctxs of calculate(T), Nelder-Mead with the calibration parameters
 * (:122-127), result pose init_T * Expmap(result.x) (:129).  The contexts play the role of `costs` (:75-84). */
int vlcal_estimate_pose_nelder_mead_ctx(
  vlcal_nid_ctx* const* ctxs,
  int n_ctxs,
  const vlcal_calib_params* params,
  const double init_T_camera_lidar[16],
  vlcal_pose_callback callback,
  vlcal_allreduce_fn allreduce,
  void* user,
  double T_out[16],
  vlcal_nm_result* nm_result);

/* n_solves independent inner solves of vlcal_estimate_pose_nelder_mead_ctx (no callback, no all-reduce) in ONE launch of
 * the persistent kernel: solve s starts from init_T_camera_lidar[16 s .. 16 s + 15] (T = init_T_s * Expmap(x), x0 = 0)
 * and sums the contexts b with bag_mask[s * n_ctxs + b] != 0, in context order.  Each solve takes exactly the
 * trajectory a single-solve call from the same start over the same contexts takes (same simplex, iterations, result,
 * bit for bit).  T_out: [n_solves][16]; nm_results: [n_solves].
 * VLCAL_ERR_UNSUPPORTED: the contexts cannot run on the persistent kernel (double-layout cloud, bins > 32, ...), one of
 * them has a multi-rank peer exchange attached (the solve axis is single-process), n_solves > 64, or the device cannot
 * hold one block per included bag of every solve at once.  The solves always run on the persistent kernel, whatever
 * vlcal_nid_set_solver_mode selects for single solves, and record no profiling events (vlcal_nid_get_profile counts the
 * launch, its passes and poses, not its time). */
int vlcal_estimate_poses_nelder_mead_ctx(
  vlcal_nid_ctx* const* ctxs,
  int n_ctxs,
  const vlcal_calib_params* params,
  int n_solves,
  const double* init_T_camera_lidar,
  const uint8_t* bag_mask,
  double* T_out,
  vlcal_nm_result* nm_results);

/* VisualCameraCalibration::estimate_pose_nelder_mead (visual_camera_calibration.cpp:70-139) from host data:
 * view culling at init_T (GPU), one cost context per bag, Nelder-Mead, pose out. */
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
  vlcal_calib_stats* stats);

/* VisualCameraCalibration::calibrate, NID_NELDER_MEAD branch (visual_camera_calibration.cpp:35-68) */
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
  vlcal_calib_stats* stats);

/* the outer loop's step size (visual_camera_calibration.cpp:50-54): delta = new_T^-1 * T as isometries,
 * delta_t = |delta.translation()|, delta_r = AngleAxisd(delta.linear()).angle().  Both branches' outer loops stop on
 * delta_t < delta_trans_thresh && delta_r < delta_rot_thresh with these values. */
int vlcal_outer_step_delta(const double T_colmajor[16], const double new_T_colmajor[16], double* delta_t, double* delta_r);

/* ---- NID_BFGS branch (VisualCameraCalibration::estimate_pose_bfgs, visual_camera_calibration.cpp:187-238) -------------
 * The reference solves min_T sum_bags NIDCost(T) with ceres::GradientProblemSolver (line-search BFGS) on the
 * Sophus::Manifold<SE3>.  Ceres is not available to this build, so this is a Ceres-free BFGS with the same problem
 * structure and Ceres' documented defaults (csrc/bfgs.cu); its iterates are not claimed to coincide with Ceres'. */
typedef struct vlcal_bfgs_params {
  int max_num_iterations;               /* 50   */
  double function_tolerance;            /* 1e-6  |d cost| <= tol * cost */
  double gradient_tolerance;            /* 1e-10 max norm of the tangent-space gradient */
  double parameter_tolerance;           /* 1e-8  */
  double sufficient_decrease;           /* 1e-4  (Armijo) */
  double sufficient_curvature_decrease; /* 0.9   (strong Wolfe) */
  double max_step_expansion;            /* 10    */
  int max_line_search_steps;            /* 20    */
  double max_translation_from_init;     /* 0.2 m   MultiNIDCost returns false beyond it (:154) */
  double max_rotation_from_init;        /* 2 deg in rad (:154) */
} vlcal_bfgs_params;

enum {
  VLCAL_BFGS_NO_CONVERGENCE = 0, /* max_num_iterations reached */
  VLCAL_BFGS_CONVERGED_GRADIENT = 1,
  VLCAL_BFGS_CONVERGED_FUNCTION = 2,
  VLCAL_BFGS_CONVERGED_PARAMETER = 3,
  VLCAL_BFGS_LINE_SEARCH_FAILED = 4,
  VLCAL_BFGS_FAILURE = 5 /* objective invalid at the initial pose */
};

typedef struct vlcal_bfgs_result {
  int iterations;
  int evaluations; /* value + gradient evaluations requested (each = one pose over all bags) */
  int termination;
  int line_search_restarts;
  double initial_cost, final_cost;
  double gradient_max_norm;
} vlcal_bfgs_result;

void vlcal_bfgs_default_params(vlcal_bfgs_params* p);

/* value and AMBIENT gradient (d/d[qx qy qz qw tx ty tz]) of an objective on SE(3); return 0 for "invalid here" */
typedef int (*vlcal_se3_objective)(const double x[7], double* cost, double grad7[7], void* user);

/* the solver on a caller-supplied objective (host only; used by the CPU tests and for custom costs) */
int vlcal_bfgs_minimize_se3(
  vlcal_se3_objective objective,
  void* user,
  const vlcal_bfgs_params* params,
  const double init_T[16],
  vlcal_pose_callback callback, /* once per accepted iteration (IterationCallback, :222-226) */
  void* callback_user,
  double T_out[16],
  vlcal_bfgs_result* result);

/* the inner BFGS solve over mode-B contexts (one per bag, already culled at init_T like :196-206).
 * allreduce (optional): bags sharded over ranks -- called once per evaluation with 9 doubles (cost, 7 partials, number of
 * failed bags) to be summed in place over all ranks; every rank then takes identical steps. */
int vlcal_estimate_pose_bfgs_ctx(
  vlcal_nid_ctx* const* ctxs,
  int n_ctx,
  const vlcal_bfgs_params* params,
  const double init_T_camera_lidar[16],
  vlcal_pose_callback callback,
  vlcal_allreduce_fn allreduce,
  void* user,
  double T_out[16],
  vlcal_bfgs_result* result);

/* ---- initial guess from 2D-3D correspondences: PoseEstimation (src/vlcal/common/estimate_pose.cpp) ------------------
 * initial_guess_auto's solver.  1. bearings: camera side estimate_direction(kp0) (host NelderMead<2>, as
 * estimate_camera_fov), LiDAR side the normalised point.  2. rotation RANSAC: hypotheses drawn on the host exactly as a
 * one-thread reference run draws them (std::mt19937 seeded with mt19937()(), two uniform_int_distribution(0, M-1) draws per
 * iteration); ONE kernel launch computes every hypothesis's rotation (Umeyama on its two bearing pairs) and counts the
 * correspondences with |kp0 - project(R d_lidar)|^2 < ransac_error_thresh^2 (project_exact, never-contracted doubles).
 * The winner is the largest count, ties to the lowest index; a second launch writes its inlier mask.  Hypotheses whose
 * rotation is not unique (the same index twice, or bearings within 1e-9 of parallel / antiparallel on either side) score
 * 0 and are counted in stats->degenerate.  3. refinement: Levenberg-Marquardt on SE(3) of
 * 1/2 sum_i rho(|project(T p_i) - kp0_i|^2) over ALL correspondences, rho = Cauchy with b = robust_kernel_width^2, from
 * [R_ransac | 0], with Ceres' default stopping rules (host; M is small).
 * Errors: M < 2 (VLCAL_ERR_INVALID_ARGUMENT), no hypothesis with an inlier (VLCAL_ERR_INVALID_ARGUMENT). */
typedef struct {
  int ransac_iterations;      /* 8192 */
  double ransac_error_thresh; /* 5.0 px */
  double robust_kernel_width; /* 10.0 px */
} vlcal_pose_estimation_params;

typedef struct {
  int hypotheses;   /* = ransac_iterations */
  int degenerate;   /* hypotheses without a unique rotation (scored 0) */
  int best_index;   /* winning hypothesis */
  int best_inliers; /* its count */
  int lm_iterations;
  double final_cost; /* 1/2 sum rho(s_i) at T_camera_lidar_out */
} vlcal_pose_estimation_stats;

void vlcal_pose_estimation_default_params(vlcal_pose_estimation_params* p);

/* kp0: M x 2 pixels, points: M x 3 (LiDAR frame).  T_camera_lidar_out: 4x4 column-major.  inlier_mask_out (optional):
 * M bytes, 1 where the RANSAC winner's rotation reprojects the correspondence within the threshold.  device = -1: the
 * current device. */
int vlcal_estimate_pose_from_correspondences(
  int device,
  int camera_model,
  const double* intrinsics,
  int n_intrinsics,
  const double* distortion,
  int n_distortion,
  const double* kp0,
  const double* points,
  int64_t n_correspondences,
  const vlcal_pose_estimation_params* params,
  double T_camera_lidar_out[16],
  uint8_t* inlier_mask_out,
  vlcal_pose_estimation_stats* stats_out);

/* estimate_direction for n pixels (n x 2) -> n x 3 unit bearings (host) */
int vlcal_estimate_directions(
  int camera_model, const double* intrinsics, int n_intrinsics, const double* distortion, int n_distortion, const double* pixels, int64_t n, double* dirs_out);

/* test hook: the RANSAC scoring launch on caller-given index pairs (n_pairs x 2, each in [0, M)).  counts_out: n_pairs
 * int32 inlier counts; degenerate_out (optional): n_pairs bytes, 1 for a hypothesis without a unique rotation;
 * kernel_ms_out (optional): the scoring launch's time between CUDA events. */
int vlcal_pose_debug_score_pairs(
  int device,
  int camera_model,
  const double* intrinsics,
  int n_intrinsics,
  const double* distortion,
  int n_distortion,
  const double* kp0,
  const double* points,
  int64_t n_correspondences,
  const int32_t* pairs,
  int n_pairs,
  double ransac_error_thresh,
  int32_t* counts_out,
  uint8_t* degenerate_out,
  double* kernel_ms_out);

/* test hook: the index pairs the RANSAC draws for M correspondences (n_iterations x 2) */
int vlcal_pose_debug_sample_pairs(int64_t n_correspondences, int n_iterations, int32_t* pairs_out);

/* test hook: the Levenberg-Marquardt refinement alone from init_T_camera_lidar (column-major) */
int vlcal_pose_debug_refine(
  int camera_model,
  const double* intrinsics,
  int n_intrinsics,
  const double* distortion,
  int n_distortion,
  const double* kp0,
  const double* points,
  int64_t n_correspondences,
  double robust_kernel_width,
  const double init_T_camera_lidar[16],
  double T_camera_lidar_out[16],
  int* iterations_out,
  double* final_cost_out);

/* ---- preprocess_map (src/preprocess_map.cpp:34-214, src/vlcal/common/estimate_fov.cpp:53-91) ----------------------------
 * The GPU stages of building a calibration dataset from a point-cloud map.  Each gives the reference's bits except where
 * noted; DESIGN §4 "preprocess_map" has the decomposition.  Invalid input (null buffers, negative or too large counts,
 * non-finite values) gives VLCAL_ERR_INVALID_ARGUMENT with a message.  device = -1: the current device. */

/* pcl::ApproximateVoxelGrid<PointXYZI> with leaf float(leaf_size) (histsize_ 512, downsample_all_data_ true), as
 * load_lidar_points runs it (preprocess_map.cpp:140-147): sequential over the points in input order, a 512-slot hash of
 * the voxel index (ix * 7171 + iy * 3079 + iz * 4231) & 511, a slot flushed (centroid / float(count) emitted) when a
 * point of another voxel arrives, the occupied slots flushed in slot order at the end.  points_xyzi: n x 4 floats
 * (x, y, z, intensity); points_out: room for n x 4 floats, the centroids in flush order; *n_out their count.
 * Voxel indices outside int range become INT_MIN as x86-64's float->int conversion gives them (the reference then merges
 * voxels along that axis); out_of_range_points (optional) counts the points where that happened.  stage_ms_out
 * (optional, 4 doubles): keys, sort, runs, emission order, between CUDA events.  At most 2^31 - 513 points. */
int vlcal_approximate_voxel_grid(
  int device,
  const float* points_xyzi,
  int64_t n_points,
  double leaf_size,
  float* points_out,
  int64_t* n_out,
  int64_t* out_of_range_points,
  double* stage_ms_out);

/* The rank equalisation of load_lidar_points (preprocess_map.cpp:158-167): with idx sorted by intensity,
 * intensities_out[idx[i]] = floor(256 * double(i) / n) / 256.  Ties are broken by point index (std::sort leaves them
 * unspecified; the multiset of outputs is the same).  kernel_ms_out (optional): the GPU time between CUDA events. */
int vlcal_equalize_intensities(int device, const float* intensities, int64_t n_points, double* intensities_out, double* kernel_ms_out);

/* estimate_lidar_fov's point set before the hull (estimate_fov.cpp:53-66): pcl::VoxelGrid<PointXYZ> at 0.2 m (voxels in
 * ascending grid index, each the float mean of its points summed in point-index order), or the input itself where the
 * grid's dx * dy * dz exceeds INT32_MAX (*unfiltered_out = 1, PCL's fallback); then the points with float norm < 1.0
 * removed, order kept.  points_xyz: n x 3 floats; candidates_out: room for n x 3 floats.  kernel_ms_out optional. */
int vlcal_lidar_fov_candidates(
  int device, const float* points_xyz, int64_t n_points, float* candidates_out, int64_t* n_out, int* unfiltered_out, double* kernel_ms_out);

/* min over vertex pairs i < j of dot(dirs_i, dirs_j), dirs = double(vertex).normalized(), starting from M_PI
 * (estimate_fov.cpp:78-89); never-contracted double, Eigen's left-to-right term order.  Fewer than 2 vertices: M_PI. */
int vlcal_min_bearing_cosine(int device, const float* vertices_xyz, int64_t n_vertices, double* min_cosine_out);

/* ---- preprocess from bags (src/vlcal/preprocess/preprocess.cpp:406-476) -------------------------------------------------
 * One accepted sensor_msgs/PointCloud2 scan of a bag: its little-endian `data` starts at byte_offset of the concatenated
 * blob and holds n_points = width * height points of point_step bytes.  Datatypes are PointField's: xyz_type 7 (FLOAT32)
 * or 8 (FLOAT64) -- x's datatype, with which y and z are read as the reference reads them; intensity_type 2, 4, 6, 7
 * or 8 (UINT8, UINT16, UINT32, FLOAT32, FLOAT64).  Offsets need not be aligned. */
typedef struct {
  int64_t byte_offset;
  int64_t n_points;
  int32_t point_step;
  int32_t x_offset;
  int32_t y_offset;
  int32_t z_offset;
  int32_t xyz_type;
  int32_t intensity_offset;
  int32_t intensity_type;
  int32_t reserved;
} vlcal_scan_desc;

/* extract_raw_points, the finiteness filter and StaticPointCloudIntegrator::insert_points / get_points over every point
 * of the scans in order (DESIGN §4c): points with a non-finite coordinate or a norm below min_distance are dropped, the
 * rest written to the voxel floor(p / voxel_resolution) (double, cast to int; out of int range gives INT_MIN as on
 * x86-64, counted in out_of_range_points), the last point written to a voxel wins.  points_out: room for 4 floats per
 * input point; receives (float(x), float(y), float(z), float(intensity)) of the winners in first-write order (the order
 * in which their voxels were first written; the reference's is its hash table's), *n_out of them.  stage_ms_out
 * (optional, 3 doubles): decode, sort, runs + emission, between CUDA events.  At most 2^31 - 1 points. */
int vlcal_bag_integrate(
  int device,
  const uint8_t* data,
  int64_t data_bytes,
  const vlcal_scan_desc* scans,
  int64_t n_scans,
  double voxel_resolution,
  double min_distance,
  float* points_out,
  int64_t* n_out,
  int64_t* out_of_range_points,
  double* stage_ms_out);

/* ---- compressed bag chunks (DESIGN §4f) ---------------------------------------------------------------------------
 * A batch of independent frames decoded on the GPU: MCAP chunks (zstd, lz4), ROS 1 lz4 chunks, rosbag2 zstd messages.
 * A frame's src range holds one or more concatenated frames of its codec, skippable frames among them:
 *   VLCAL_CODEC_ZSTD        zstd (RFC 8878) without dictionaries; the content checksum is verified when present.
 *   VLCAL_CODEC_LZ4_FRAME   the LZ4 frame format (magic 0x184D2204), linked or independent blocks, uncompressed blocks;
 *                           the header, block and content checksums are verified when present.
 * It must decode to exactly dst_size bytes, written to dst[dst_offset, dst_offset + dst_size).  has_crc32: crc32 is the
 * CRC-32 (zlib polynomial) of those bytes and is verified (MCAP's uncompressed_crc when it is not 0). */
#define VLCAL_CODEC_ZSTD 1
#define VLCAL_CODEC_LZ4_FRAME 2
typedef struct {
  int64_t src_offset;
  int64_t src_size;
  int64_t dst_offset;
  int64_t dst_size;
  int32_t codec;
  int32_t has_crc32;
  uint32_t crc32;
  int32_t reserved;
} vlcal_frame;

/* per-frame status_out */
#define VLCAL_FRAME_OK 0
#define VLCAL_FRAME_CORRUPT 1          /* malformed, truncated, or a match reaching before the start of its output */
#define VLCAL_FRAME_CHECKSUM 2         /* a checksum of the format, or crc32, does not match */
#define VLCAL_FRAME_SIZE 3             /* the frame decodes to a size other than dst_size */
#define VLCAL_FRAME_UNSUPPORTED 4      /* a zstd or LZ4 dictionary id, the legacy LZ4 format, a window above 2 GiB */

/* Decodes frames[0, n_frames) from host src[0, src_bytes) into host dst[0, dst_bytes); status_out[i] is frame i's
 * status.  The dst bytes of a frame whose status is not 0 are unspecified; bytes of dst outside every frame's range are
 * not touched.  Checked on the host before any GPU work (VLCAL_ERR_INVALID_ARGUMENT): a known codec, has_crc32 0 or 1,
 * every range inside its buffer, no two non-empty dst ranges overlapping.  Malformed frame data never reads or writes
 * outside the frame's own ranges.  ms_out (optional, 3 doubles): copy in, kernel, copy out, between CUDA events. */
int vlcal_decode_frames(
  int device,
  const uint8_t* src,
  int64_t src_bytes,
  const vlcal_frame* frames,
  int n_frames,
  uint8_t* dst,
  int64_t dst_bytes,
  int32_t* status_out,
  double* ms_out);

#ifdef __cplusplus
}
#endif
#endif /* VLCAL_NID_H */
