// host_math.hpp -- host-side SE(3) helpers and the Nelder-Mead solver of the product library.
//
// These mirror the third-party / header-only pieces the reference's caller uses around the hot path:
//   gtsam::Pose3::Expmap            (call sites src/vlcal/calib/visual_camera_calibration.cpp:104,129; GTSAM 4.2a9)
//   Eigen::Isometry3d product / inverse / AngleAxisd(R).angle()   (visual_camera_calibration.cpp:50-54)
//   dfo::NelderMead<N>              (include/dfo/nelder_mead.hpp:32-113)
// Compiled with -ffp-contract=off so results do not depend on FMA availability.
#pragma once

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <vector>

#include "nm_machine.cuh"
#include "se3_math.cuh"

namespace vlcal {
namespace host {

// 4x4 column-major accessors (Eigen::Isometry3d::matrix().data())
inline double& m4(double* T, int r, int c) { return T[r + 4 * c]; }
inline double m4(const double* T, int r, int c) { return T[r + 4 * c]; }

// gtsam::Pose3::Expmap(xi).matrix(), xi = (omega, v)  [GTSAM 4.2a9: so3::ExpmapFunctor + Pose3::Expmap]
inline void se3_expmap_gtsam(const double xi[6], double T[16]) {
  se3_expmap_gtsam_hd(xi, T);
}

// Isometry3d * Isometry3d
inline void isometry_mul(const double A[16], const double B[16], double C[16]) {
  isometry_mul_hd(A, B, C);
}

// Isometry3d::inverse()
inline void isometry_inverse(const double A[16], double Ainv[16]) {
  double R[16];
  std::memset(R, 0, sizeof(R));
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) m4(R, i, j) = m4(A, j, i);
  for (int i = 0; i < 3; i++) m4(R, i, 3) = -(m4(R, i, 0) * m4(A, 0, 3) + m4(R, i, 1) * m4(A, 1, 3) + m4(R, i, 2) * m4(A, 2, 3));
  m4(R, 3, 3) = 1.0;
  std::memcpy(Ainv, R, sizeof(R));
}

// Eigen::AngleAxisd(T.linear()).angle(): rotation matrix -> quaternion -> 2*atan2(|vec|, |w|)
inline double rotation_angle(const double T[16]) {
  double q[4];  // x y z w
  double t = m4(T, 0, 0) + m4(T, 1, 1) + m4(T, 2, 2);
  if (t > 0.0) {
    t = std::sqrt(t + 1.0);
    q[3] = 0.5 * t;
    t = 0.5 / t;
    q[0] = (m4(T, 2, 1) - m4(T, 1, 2)) * t;
    q[1] = (m4(T, 0, 2) - m4(T, 2, 0)) * t;
    q[2] = (m4(T, 1, 0) - m4(T, 0, 1)) * t;
  } else {
    int i = 0;
    if (m4(T, 1, 1) > m4(T, 0, 0)) i = 1;
    if (m4(T, 2, 2) > m4(T, i, i)) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    t = std::sqrt(m4(T, i, i) - m4(T, j, j) - m4(T, k, k) + 1.0);
    q[i] = 0.5 * t;
    t = 0.5 / t;
    q[3] = (m4(T, k, j) - m4(T, j, k)) * t;
    q[j] = (m4(T, j, i) + m4(T, i, j)) * t;
    q[k] = (m4(T, k, i) + m4(T, i, k)) * t;
  }
  const double n = std::sqrt((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]);
  return n != 0.0 ? 2.0 * std::atan2(n, std::fabs(q[3])) : 0.0;
}

// ---------------------------------------------------------------------------------------------
// Nelder-Mead with the reference's exact decision sequence (include/dfo/nelder_mead.hpp:32-113): host driver of the
// shared state machine (nm_machine.cuh)
// ---------------------------------------------------------------------------------------------

using NelderMeadParams = NmParams;

struct NelderMeadResult {  // optimizer.hpp:8-20
  bool converged = false;
  int num_iterations = 0;
  std::vector<double> x;
  double y = 0.0;
  int num_evaluations = 0;           // what the serial reference would have requested
  int num_batches = 0;               // objective batches issued
  int num_evaluations_computed = 0;  // poses actually scored (speculation included)
};

// BatchF:   void(const double* xs /*count x n*/, int count, double* ys)
// ObserveF: void(const double* x, double y)   -- called once per reference evaluation, in reference order
// (`speculate` is kept for call-site readability: candidates are always scored one batch per iteration; only the
// values the reference would have requested are consumed.)  score_centroid = false: iteration batches leave out the
// centroid, whose value then never reaches `observe` (NmMachine::begin); for callers that read no side effects.
template <typename BatchF, typename ObserveF>
NelderMeadResult nelder_mead(int n, BatchF&& f, ObserveF&& observe, const double* x0, const NelderMeadParams& params, bool /*speculate*/, bool score_centroid = true) {
  NmMachine nm;
  nm.begin(n, params, x0, score_centroid);
  std::vector<double> xs(static_cast<size_t>(NM_MAX_N + 1) * n), ys(NM_MAX_N + 1);
  while (nm.phase != 3) {
    for (int k = 0; k < nm.n_cand; k++) std::memcpy(&xs[static_cast<size_t>(k) * n], &nm.cand[k][1], sizeof(double) * n);
    f(xs.data(), nm.n_cand, ys.data());
    nm.step(ys.data());
    for (int k = 0; k < nm.n_obs; k++) observe(nm.obs_x[k], nm.obs_y[k]);
  }
  NelderMeadResult result;
  result.converged = nm.converged != 0;
  result.num_iterations = nm.num_iterations;
  result.x.assign(nm.result_x, nm.result_x + n);
  result.y = nm.result_y;
  result.num_evaluations = nm.num_evaluations;
  result.num_batches = nm.num_batches;
  result.num_evaluations_computed = nm.num_evaluations_computed;
  return result;
}

}  // namespace host
}  // namespace vlcal
