/*
 * vlcal_oracle.h -- CPU ORACLE (test infrastructure, NOT product code).
 *
 * A dependency-free, plain-C restatement of the NID hot path of
 * koide3/direct_visual_lidar_calibration (commit d3c2474).  Every function cites the
 * reference file:line it follows.  Only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs may link or call this.  The product library
 * (direct_visual_lidar_calibration_b200/csrc) never includes or links it.
 *
 * PARITY STATUS: pinned against the reference's OWN sources of the path (camera models,
 * dfo::NelderMead, estimate_camera_fov, CostCalculatorNID::calculate, ViewCulling::cull, NIDCost<double>,
 * VisualCameraCalibration::calibrate / estimate_pose_nelder_mead), compiled
 * from /root/reference against stand-in third-party headers -- oracle/ref_shim.cpp,
 * oracle/ref_standin/, tests/test_reference_pin.py: bit-exact on every comparison.  The reference
 * cannot be built as it ships (no Eigen/OpenCV/Ceres/GTSAM/Boost/Iridescence/PCL in this image) and
 * has no tests or golden vectors (SURVEY.md section 4, 8c), so what stays "parity unpinned" is the
 * third-party arithmetic itself, restated from published semantics here and in the stand-ins alike:
 *   - GTSAM 4.2a9 Pose3::Expmap / SO3::Expmap (docs/installation.md:27)
 *   - Eigen 3.4 Isometry3d*Vector4d, normalized(), reduction orders, cast<int>(), AngleAxisd(Matrix3d)
 *   - libstdc++ std::sort insertion-sort branch for n <= 16 (pinned: the reference build uses the real std::sort)
 *   - Sophus SO3/SE3 point action (thirdparty/Sophus/sophus/so3.hpp:408-417, se3.hpp:319-322)
 * Further pins of ours: hand-derived known answers (tests/golden/), OpenCV cross-checks of the
 * camera models the reference declares OpenCV-compatible, property tests.
 *
 * Build: see oracle/Makefile (gcc -O2 -g -ffp-contract=off, the reference's RelWithDebInfo
 * without -march, CMakeLists.txt:7-10).
 */
#ifndef VLCAL_ORACLE_H
#define VLCAL_ORACLE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* camera model ids; order follows src/camera/create_camera.cpp:35-46 */
enum {
  ORC_CAM_PLUMB_BOB = 0,          /* PinholeProjection,  4 intr, 5 dist  include/camera/pinhole.hpp */
  ORC_CAM_FISHEYE = 1,            /* FisheyeProjection,  4 intr, 4 dist  include/camera/fisheye.hpp ("fisheye"/"equidistant") */
  ORC_CAM_ATAN = 2,               /* ATANProjection,     4 intr, 1 dist  include/camera/atan.hpp */
  ORC_CAM_OMNIDIR = 3,            /* Omnidirectional,    5 intr, 4 dist  include/camera/omnidir.hpp */
  ORC_CAM_EQUIRECTANGULAR = 4,    /* Equirectangular,    2 intr, 0 dist  include/camera/equirectangular.hpp */
  ORC_CAM_RATIONAL_POLYNOMIAL = 5 /* RationalPolynomial, 4 intr, 8 dist  include/camera/rational_polynomial.hpp */
};

typedef struct {
  int model;
  int n_intr;
  int n_dist;
  double intr[5];
  double dist[8];
} orc_camera;

/* create_camera(model_string, intrinsics, distortion)  src/camera/create_camera.cpp:17-50.
 * Returns 0 on success; -1 = unknown model (nullptr), -2 = intrinsic count mismatch (nullptr). */
int orc_create_camera(const char* camera_model, const double* intrinsics, int n_intr, const double* distortion, int n_dist, orc_camera* out);

/* GenericCamera<Projection>::project  include/camera/generic_camera.hpp:21-28 */
void orc_project(const orc_camera* cam, const double p[3], double uv[2]);
/* orc_project over n points: p[3n] -> uv[2n] */
void orc_project_n(const orc_camera* cam, const double* p, int64_t n, double* uv);

/* gtsam::Pose3::Expmap(x).matrix(), x = (wx,wy,wz,vx,vy,vz); 4x4 column-major out.
 * call sites: src/vlcal/calib/visual_camera_calibration.cpp:104,129 */
void orc_se3_expmap_gtsam(const double x[6], double T_colmajor[16]);

/* 4x4 column-major affine composition C = A*B (Eigen Isometry3d * Isometry3d) */
void orc_isometry_mul(const double A[16], const double B[16], double C[16]);
/* Isometry3d::inverse() */
void orc_isometry_inverse(const double A[16], double Ainv[16]);
/* Eigen::AngleAxisd(R).angle() for the linear part of a 4x4 column-major transform */
double orc_rotation_angle(const double T[16]);

/* estimate_camera_fov  src/vlcal/common/estimate_fov.cpp:17-51 */
double orc_estimate_camera_fov(const orc_camera* cam, int width, int height);

/* dfo::NelderMead<N>  include/dfo/nelder_mead.hpp:10-116 */
typedef struct {
  double init_step, alpha, gamma, rho, sigma;
  int max_iterations;
  double convergence_var_thresh;
} orc_nm_params;
typedef struct {
  int converged;
  int num_iterations;
  double x[8];
  double y;
  int num_evaluations; /* extra bookkeeping (not in the reference) */
} orc_nm_result;
typedef double (*orc_nm_function)(const double* x, void* user);
void orc_nm_default_params(orc_nm_params* p); /* nelder_mead.hpp:12 */
void orc_nelder_mead(int n, orc_nm_function f, void* user, const double* x0, const orc_nm_params* params, orc_nm_result* result);

/* CostCalculatorNID::calculate  src/vlcal/calib/cost_calculator_nid.cpp:21-67  (mode A).
 * points_xyzw: N x 4 doubles (Eigen::Vector4d layout, w ignored = 1), intensities: N doubles.
 * image: uint8, row stride in bytes.  hist_out (optional): bins*bins int32, index = image_bin + lidar_bin*bins
 * (Eigen column-major MatrixXi(image_bin, lidar_bin)).  Returns NID (NaN if no inliers). */
double orc_nid_calculate(
  const orc_camera* cam,
  const uint8_t* image,
  int width,
  int height,
  int row_stride,
  const double* points_xyzw,
  const double* intensities,
  int64_t n,
  int bins,
  double max_fov,
  const double T_camera_lidar[16],
  int32_t* hist_out);

/* same arithmetic, OpenMP over points with thread-private histograms.
 * NOT what the reference does (it is serial over points); used only as a "best-effort CPU" timing. */
double orc_nid_calculate_omp(
  const orc_camera* cam,
  const uint8_t* image,
  int width,
  int height,
  int row_stride,
  const double* points_xyzw,
  const double* intensities,
  int64_t n,
  int bins,
  double max_fov,
  const double T_camera_lidar[16],
  int32_t* hist_out);

/* entropy / NID finalize alone  cost_calculator_nid.cpp:54-64 ; hist index = image_bin + lidar_bin*bins */
double orc_nid_from_hist(const int32_t* hist, int bins, double* Hr, double* Hs, double* Hrs, double* MI);

/* ViewCulling::cull  src/vlcal/calib/view_culling.cpp:21-92.
 * indices_out must hold n ints; returns the number kept (ascending original index). */
int64_t orc_view_cull(
  const orc_camera* cam,
  int width,
  int height,
  double max_fov, /* estimate_camera_fov(cam, size); min_z = cos(max_fov)  view_culling.cpp:17 */
  int enable_depth_buffer_culling,
  const double* points_xyzw,
  int64_t n,
  const double T_camera_lidar[16],
  int32_t* indices_out);

/* NIDCost::operator()<double>  include/vlcal/costs/nid_cost.hpp:36-107  (mode B, value only).
 * T_params = [qx qy qz qw tx ty tz] (Sophus SE3 storage).  image64: H x W doubles (u8/255.0).
 * Returns 1 (true) and writes *nid, or 0 (false) if NID is not finite.  hist_out optional bins*bins doubles
 * (index = bin_image + bin_points*bins, un-normalised). */
int orc_nid_cost_bspline(
  const orc_camera* cam,
  const double* image64,
  int width,
  int height,
  const double* points_xyzw,
  const double* intensities,
  int64_t n,
  int bins,
  const double T_params[7],
  double* nid,
  double* hist_out);

/* VisualCameraCalibration::estimate_pose_nelder_mead  src/vlcal/calib/visual_camera_calibration.cpp:70-139
 * and ::calibrate :35-68 (NID_NELDER_MEAD branch) over n_bags bags sharing one camera. */
typedef struct {
  const uint8_t* image;
  int width, height, row_stride;
  const double* points_xyzw;
  const double* intensities;
  int64_t n;
} orc_bag;

typedef struct {
  int max_outer_iterations;  /* 10     visual_camera_calibration.hpp:13 */
  int max_inner_iterations;  /* 256    :14 */
  double delta_trans_thresh; /* 0.1    :16 */
  double delta_rot_thresh;   /* 0.5deg :17 */
  int disable_z_buffer_culling;
  int nid_bins;                            /* 16   :21 */
  double nelder_mead_init_step;            /* 1e-3 :24 */
  double nelder_mead_convergence_criteria; /* 1e-8 :25 */
} orc_calib_params;
void orc_calib_default_params(orc_calib_params* p);

typedef struct {
  int outer_iterations;
  int total_evaluations; /* objective evaluations (each = one pose over all bags) */
  int inner_iterations[16];
  double inner_final_cost[16];
  double best_cost_last; /* best_cost of the last inner solve */
} orc_calib_stats;

/* trace (optional): records every objective evaluation as 7 doubles [x0..x5, cost]; capacity in evals */
typedef struct {
  double* evals;
  int capacity;
  int count;
} orc_trace;

void orc_estimate_pose_nelder_mead(
  const orc_camera* cam,
  const orc_bag* bags,
  int n_bags,
  const orc_calib_params* params,
  const double init_T_camera_lidar[16],
  double T_out[16],
  orc_nm_result* nm_result,
  orc_trace* trace);

void orc_calibrate(
  const orc_camera* cam,
  const orc_bag* bags,
  int n_bags,
  const orc_calib_params* params,
  const double init_T_camera_lidar[16],
  double T_out[16],
  orc_calib_stats* stats,
  orc_trace* trace);

/* NIDCost::operator()<ceres::Jet<double, 7>> (nid_cost.hpp:36-107): value + d/d(qx qy qz qw tx ty tz); vlcal_oracle_grad.c */
int orc_nid_cost_bspline_grad(
  const orc_camera* cam,
  const double* image64,
  int width,
  int height,
  const double* points_xyzw,
  const double* intensities,
  int64_t n,
  int bins,
  const double T_params[7],
  double* nid_out,
  double* grad_out,
  double* hist_out);

/* generate_lidar_image (src/vlcal/preprocess/generate_lidar_image.cpp:8-41): intensity_image[H*W] doubles, index_image[H*W] */
void orc_generate_lidar_image(
  const orc_camera* cam, int width, int height, const double T[16], const double* points_xyzw, const double* intensities, int64_t n, double* intensity_image, int32_t* index_image);

/* team size of the objective's OpenMP loop over bags (visual_camera_calibration.cpp:107): 0 = one thread per bag
 * (the reference's behaviour on a host with enough cores), 1 = serial.  Results do not depend on it. */
void orc_set_bag_threads(int n);

#ifdef __cplusplus
}
#endif
#endif
