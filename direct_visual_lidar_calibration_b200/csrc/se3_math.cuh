// se3_math.cuh -- __host__ __device__ SE(3) helpers of the host solver (the persistent kernel repeats their operations):
//   gtsam::Pose3::Expmap            (call sites src/vlcal/calib/visual_camera_calibration.cpp:104,129; GTSAM 4.2a9)
//   Eigen::Isometry3d * Isometry3d  (visual_camera_calibration.cpp:104)
// 4x4 matrices are column-major (Eigen::Isometry3d::matrix().data()).  Arithmetic goes through exact_math.cuh, so the
// operation order and rounding are the same on both sides; sin() is libm on the host and the CUDA math library on the
// device (both within 1-2 ulp of the true value; the host path is the one compared bit-for-bit with the oracle).
#pragma once

#include <cfloat>

#include "exact_math.cuh"

namespace vlcal {

VL_HD double m4get(const double* T, int r, int c) {
  return T[r + 4 * c];
}

// gtsam::Pose3::Expmap(xi).matrix(), xi = (omega, v)  [so3::ExpmapFunctor + Pose3::Expmap]
VL_HD void se3_expmap_gtsam_hd(const double xi[6], double T[16]) {
  const xd wx(xi[0]), wy(xi[1]), wz(xi[2]);
  const xd v[3] = {xd(xi[3]), xd(xi[4]), xd(xi[5])};
  const xd theta2 = (wx * wx + wy * wy) + wz * wz;
  const xd zero(0.0);
  const xd W[3][3] = {{zero, -wz, wy}, {wz, zero, -wx}, {-wy, wx, zero}};
  xd R[3][3];
  if (theta2.v <= DBL_EPSILON) {  // nearZero: I + W
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) R[i][j] = W[i][j] + xd(i == j ? 1.0 : 0.0);
  } else {
    const xd theta = xsqrt(theta2);
    const xd sin_theta(sin(theta.v));
    const xd s2(sin((theta / xd(2.0)).v));
    const xd one_minus_cos = xd(2.0) * s2 * s2;
    xd K[3][3], KK[3][3];
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) K[i][j] = W[i][j] / theta;
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) KK[i][j] = K[i][0] * K[0][j] + K[i][1] * K[1][j] + K[i][2] * K[2][j];
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) R[i][j] = xd(i == j ? 1.0 : 0.0) + sin_theta * K[i][j] + one_minus_cos * KK[i][j];
  }
  xd t[3];
  if (theta2.v > DBL_EPSILON) {
    const xd w[3] = {wx, wy, wz};
    const xd wv = (w[0] * v[0] + w[1] * v[1]) + w[2] * v[2];
    const xd c[3] = {w[1] * v[2] - w[2] * v[1], w[2] * v[0] - w[0] * v[2], w[0] * v[1] - w[1] * v[0]};
    for (int i = 0; i < 3; i++) {
      const xd Rc = R[i][0] * c[0] + R[i][1] * c[1] + R[i][2] * c[2];
      t[i] = (c[i] - Rc + w[i] * wv) / theta2;
    }
  } else {
    t[0] = v[0], t[1] = v[1], t[2] = v[2];
  }
  for (int k = 0; k < 16; k++) T[k] = 0.0;
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) T[i + 4 * j] = R[i][j].v;
    T[i + 12] = t[i].v;
  }
  T[15] = 1.0;
}

// Isometry3d * Isometry3d: linear = Ra Rb, translation = Ra tb + ta
VL_HD void isometry_mul_hd(const double A[16], const double B[16], double C[16]) {
  double R[16];
  for (int k = 0; k < 16; k++) R[k] = 0.0;
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) {
      R[i + 4 * j] = (xd(m4get(A, i, 0)) * xd(m4get(B, 0, j)) + xd(m4get(A, i, 1)) * xd(m4get(B, 1, j)) + xd(m4get(A, i, 2)) * xd(m4get(B, 2, j))).v;
    }
    R[i + 12] = ((xd(m4get(A, i, 0)) * xd(m4get(B, 0, 3)) + xd(m4get(A, i, 1)) * xd(m4get(B, 1, 3)) + xd(m4get(A, i, 2)) * xd(m4get(B, 2, 3))) + xd(m4get(A, i, 3))).v;
  }
  R[15] = 1.0;
  for (int k = 0; k < 16; k++) C[k] = R[k];
}

}  // namespace vlcal
