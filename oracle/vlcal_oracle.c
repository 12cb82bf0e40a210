/*
 * vlcal_oracle.c -- CPU ORACLE (test infrastructure, NOT product code).  See vlcal_oracle.h.
 *
 * All arithmetic is IEEE double, written operation-by-operation in the order of the reference
 * expressions; build with -ffp-contract=off so no FMA contraction happens (the reference's
 * default x86-64 build has no FMA either: CMakeLists.txt:7-10, no -march).
 * Reference paths are relative to /root/reference.
 */
#include "vlcal_oracle.h"

#include <float.h>
#include <limits.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#ifndef M_PI
#define M_PI 3.14159265358979323846
#endif

/* static_cast<int>(double) as x86-64 cvttsd2si does it: truncation toward zero,
 * NaN / out-of-range -> INT_MIN ("integer indefinite").  Used for Eigen cast<int>()
 * (cost_calculator_nid.cpp:37) and the implicit double->int conversions at :46-47. */
static int orc_cast_int(double v) {
  if (!(v > -2147483649.0 && v < 2147483648.0)) {
    return INT_MIN;
  }
  return (int)v;
}

/* ------------------------------------------------------------------------------------------
 * camera models
 * ---------------------------------------------------------------------------------------- */

/* src/camera/create_camera.cpp:17-50 */
int orc_create_camera(const char* camera_model, const double* intrinsics, int n_intr, const double* distortion, int n_dist, orc_camera* out) {
  int model, ni, nd;
  if (strcmp(camera_model, "plumb_bob") == 0) { /* :35 */
    model = ORC_CAM_PLUMB_BOB, ni = 4, nd = 5;  /* pinhole.hpp:57-58 */
  } else if (strcmp(camera_model, "fisheye") == 0 || strcmp(camera_model, "equidistant") == 0) { /* :37 */
    model = ORC_CAM_FISHEYE, ni = 4, nd = 4; /* fisheye.hpp:42-43 */
  } else if (strcmp(camera_model, "atan") == 0) { /* :39 */
    model = ORC_CAM_ATAN, ni = 4, nd = 1; /* atan.hpp:45-46 */
  } else if (strcmp(camera_model, "omnidir") == 0) { /* :41 */
    model = ORC_CAM_OMNIDIR, ni = 5, nd = 4; /* omnidir.hpp:47-48 */
  } else if (strcmp(camera_model, "equirectangular") == 0) { /* :43 */
    model = ORC_CAM_EQUIRECTANGULAR, ni = 2, nd = 0; /* equirectangular.hpp:34-35 */
  } else if (strcmp(camera_model, "rational_polynomial") == 0) { /* :45 */
    model = ORC_CAM_RATIONAL_POLYNOMIAL, ni = 4, nd = 8; /* rational_polynomial.hpp:64-65 */
  } else {
    return -1; /* :49-50 unknown camera model -> nullptr */
  }
  if (n_intr != ni) {
    return -2; /* :19-22 num of intrinsic parameters mismatch -> nullptr */
  }
  memset(out, 0, sizeof(*out));
  out->model = model;
  out->n_intr = ni;
  out->n_dist = nd;
  for (int i = 0; i < ni; i++) {
    out->intr[i] = intrinsics[i];
  }
  /* :24-27 zero-padded / truncated distortion */
  for (int i = 0; i < nd && i < n_dist; i++) {
    out->dist[i] = distortion[i];
  }
  return 0;
}

/* Eigen 3.4 squaredNorm of a 3-vector with 2-wide packets: (x*x + y*y) + z*z  (ULP-level, unpinned) */
static double sqnorm3(const double p[3]) {
  return (p[0] * p[0] + p[1] * p[1]) + p[2] * p[2];
}

/* Eigen normalized(): v / sqrt(|v|^2) if |v|^2 > 0 else v */
static void normalized3(const double p[3], double out[3]) {
  const double z = sqnorm3(p);
  if (z > 0.0) {
    const double n = sqrt(z);
    out[0] = p[0] / n;
    out[1] = p[1] / n;
    out[2] = p[2] / n;
  } else {
    out[0] = p[0], out[1] = p[1], out[2] = p[2];
  }
}

/* include/camera/pinhole.hpp:13-38 distort */
static void plumb_bob_distort(const double* d, double x, double y, double* xo, double* yo) {
  const double k1 = d[0], k2 = d[1], k3 = d[4];
  const double p1 = d[2], p2 = d[3];
  const double x2 = x * x;
  const double y2 = y * y;
  const double r2 = x2 + y2;
  const double r4 = r2 * r2;
  const double r6 = r2 * r4;
  const double r_coeff = 1.0 + k1 * r2 + k2 * r4 + k3 * r6;
  const double t_coeff1 = 2.0 * x * y;
  const double t_coeff2 = r2 + 2.0 * x2;
  const double t_coeff3 = r2 + 2.0 * y2;
  *xo = r_coeff * x + p1 * t_coeff1 + p2 * t_coeff2;
  *yo = r_coeff * y + p1 * t_coeff3 + p2 * t_coeff1;
}

/* include/camera/rational_polynomial.hpp:11-44 distort */
static void rational_distort(const double* d, double x, double y, double* xo, double* yo) {
  const double k1 = d[0], k2 = d[1], p1 = d[2], p2 = d[3], k3 = d[4], k4 = d[5], k5 = d[6], k6 = d[7];
  const double x2 = x * x;
  const double y2 = y * y;
  const double r2 = x2 + y2;
  const double r4 = r2 * r2;
  const double r6 = r2 * r4;
  const double numerator = 1.0 + k1 * r2 + k2 * r4 + k3 * r6;
  const double denominator = 1.0 + k4 * r2 + k5 * r4 + k6 * r6;
  const double r_coeff = denominator > 1e-8 ? numerator / denominator : numerator; /* :33 */
  const double t_coeff1 = 2.0 * x * y;
  const double t_coeff2 = r2 + 2.0 * x2;
  const double t_coeff3 = r2 + 2.0 * y2;
  *xo = r_coeff * x + p1 * t_coeff1 + p2 * t_coeff2;
  *yo = r_coeff * y + p1 * t_coeff3 + p2 * t_coeff1;
}

void orc_project(const orc_camera* cam, const double p[3], double uv[2]) {
  const double* in = cam->intr;
  const double* d = cam->dist;
  switch (cam->model) {
    case ORC_CAM_PLUMB_BOB: { /* pinhole.hpp:40-51 */
      const double x = p[0] / p[2];
      const double y = p[1] / p[2];
      double xd, yd;
      plumb_bob_distort(d, x, y, &xd, &yd);
      uv[0] = in[0] * xd + in[2];
      uv[1] = in[1] * yd + in[3];
      return;
    }
    case ORC_CAM_FISHEYE: { /* fisheye.hpp:13-36 */
      const double r = sqrt(p[0] * p[0] + p[1] * p[1]);
      const double theta = atan2(r, fabs(p[2])); /* :16 abs(z) */
      const double theta2 = pow(theta, 2);
      const double theta4 = pow(theta, 4);
      const double theta6 = pow(theta, 6);
      const double theta8 = pow(theta, 8);
      const double k1 = d[0], k2 = d[1], k3 = d[2], k4 = d[3];
      const double theta_d = theta * (1.0 + k1 * theta2 + k2 * theta4 + k3 * theta6 + k4 * theta8);
      const double s = theta_d / r; /* r == 0 -> NaN, kept */
      const double xd = s * p[0];
      const double yd = s * p[1];
      uv[0] = in[0] * xd + in[2];
      uv[1] = in[1] * yd + in[3];
      return;
    }
    case ORC_CAM_ATAN: { /* atan.hpp:13-39 */
      const double x = p[0] / p[2];
      const double y = p[1] / p[2];
      double xd = x, yd = y;
      const double d0 = d[0];
      const double r = sqrt(x * x + y * y);
      if (!(r < 1e-3 || d0 < 1e-7)) { /* :17 */
        const double d1 = 1.0 / d0;
        const double d2 = 2.0 * tan(d0 / 2.0);
        const double factor = d1 * atan(r * d2) / r;
        xd = factor * x;
        yd = factor * y;
      }
      uv[0] = in[0] * xd + in[2];
      uv[1] = in[1] * yd + in[3];
      return;
    }
    case ORC_CAM_OMNIDIR: { /* omnidir.hpp:13-41 */
      const double fx = in[0], fy = in[1], cx = in[2], cy = in[3], xi = in[4];
      const double k1 = d[0], k2 = d[1], p1 = d[2], p2 = d[3];
      double s[3];
      normalized3(p, s);
      const double ux = s[0] / (s[2] + xi);
      const double uy = s[1] / (s[2] + xi);
      const double r2 = ux * ux + uy * uy;
      const double r4 = r2 * r2;
      const double dr = (1.0 + k1 * r2 + k2 * r4);
      const double x2 = ux * ux;
      const double y2 = uy * uy;
      const double xy = ux * uy;
      const double nx = ux * dr + 2.0 * p1 * xy + p2 * (r2 + 2.0 * x2);
      const double ny = uy * dr + p1 * (r2 + 2.0 * y2) + 2.0 * p2 * xy;
      uv[0] = fx * nx + cx;
      uv[1] = fy * ny + cy;
      return;
    }
    case ORC_CAM_EQUIRECTANGULAR: { /* equirectangular.hpp:13-28 */
      if (sqnorm3(p) < 1e-3) {
        uv[0] = in[0] / 2;
        uv[1] = in[1] / 2;
        return;
      }
      double b[3];
      normalized3(p, b);
      const double lat = -asin(b[1]);
      const double lon = atan2(b[0], b[2]);
      uv[0] = in[0] * (0.5 + lon / (2.0 * M_PI));
      uv[1] = in[1] * (0.5 - lat / M_PI);
      return;
    }
    case ORC_CAM_RATIONAL_POLYNOMIAL: { /* rational_polynomial.hpp:46-58 */
      const double x = p[0] / p[2];
      const double y = p[1] / p[2];
      double xd, yd;
      rational_distort(d, x, y, &xd, &yd);
      uv[0] = in[0] * xd + in[2];
      uv[1] = in[1] * yd + in[3];
      return;
    }
    default:
      uv[0] = uv[1] = NAN;
  }
}

/* ------------------------------------------------------------------------------------------
 * SE3 helpers (third-party semantics restated; ULP-level details unpinned)
 * ---------------------------------------------------------------------------------------- */

#define M4(T, r, c) ((T)[(r) + 4 * (c)])

static void mat3_mul(const double A[9], const double B[9], double C[9]) { /* row-major 3x3 */
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) {
      C[3 * i + j] = A[3 * i + 0] * B[0 + j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
    }
  }
}

/* GTSAM 4.2a9  so3::ExpmapFunctor + Pose3::Expmap (gtsam/geometry/SO3.cpp, Pose3.cpp) */
void orc_se3_expmap_gtsam(const double x[6], double T[16]) {
  const double wx = x[0], wy = x[1], wz = x[2];
  const double v[3] = {x[3], x[4], x[5]};
  const double theta2 = (wx * wx + wy * wy) + wz * wz;
  const double theta = sqrt(theta2);
  const double W[9] = {0.0, -wz, +wy, +wz, 0.0, -wx, -wy, +wx, 0.0};
  double R[9];
  const int near_zero = theta2 <= DBL_EPSILON;
  if (near_zero) {
    for (int i = 0; i < 9; i++) R[i] = W[i];
    R[0] += 1.0, R[4] += 1.0, R[8] += 1.0; /* I + W */
  } else {
    const double sin_theta = sin(theta);
    const double s2 = sin(theta / 2.0);
    const double one_minus_cos = 2.0 * s2 * s2;
    double K[9], KK[9];
    for (int i = 0; i < 9; i++) K[i] = W[i] / theta;
    mat3_mul(K, K, KK);
    for (int i = 0; i < 9; i++) {
      const double I = (i == 0 || i == 4 || i == 8) ? 1.0 : 0.0;
      R[i] = I + sin_theta * K[i] + one_minus_cos * KK[i];
    }
  }
  double t[3];
  if (theta2 > DBL_EPSILON) {
    const double w[3] = {wx, wy, wz};
    const double wv = (w[0] * v[0] + w[1] * v[1]) + w[2] * v[2];
    const double t_parallel[3] = {w[0] * wv, w[1] * wv, w[2] * wv};
    const double c[3] = {w[1] * v[2] - w[2] * v[1], w[2] * v[0] - w[0] * v[2], w[0] * v[1] - w[1] * v[0]};
    for (int i = 0; i < 3; i++) {
      const double Rc = R[3 * i + 0] * c[0] + R[3 * i + 1] * c[1] + R[3 * i + 2] * c[2];
      t[i] = (c[i] - Rc + t_parallel[i]) / theta2;
    }
  } else {
    t[0] = v[0], t[1] = v[1], t[2] = v[2];
  }
  memset(T, 0, 16 * sizeof(double));
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) {
      M4(T, i, j) = R[3 * i + j];
    }
    M4(T, i, 3) = t[i];
  }
  M4(T, 3, 3) = 1.0;
}

/* Eigen Transform<double,3,Isometry> * Transform: linear = Ra*Rb, translation = Ra*tb + ta */
void orc_isometry_mul(const double A[16], const double B[16], double C[16]) {
  double R[16];
  memset(R, 0, sizeof(R));
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) {
      M4(R, i, j) = M4(A, i, 0) * M4(B, 0, j) + M4(A, i, 1) * M4(B, 1, j) + M4(A, i, 2) * M4(B, 2, j);
    }
    M4(R, i, 3) = (M4(A, i, 0) * M4(B, 0, 3) + M4(A, i, 1) * M4(B, 1, 3) + M4(A, i, 2) * M4(B, 2, 3)) + M4(A, i, 3);
  }
  M4(R, 3, 3) = 1.0;
  memcpy(C, R, sizeof(R));
}

/* Eigen Transform::inverse(Isometry): R^T, -(R^T t) */
void orc_isometry_inverse(const double A[16], double Ainv[16]) {
  double R[16];
  memset(R, 0, sizeof(R));
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) {
      M4(R, i, j) = M4(A, j, i);
    }
  }
  for (int i = 0; i < 3; i++) {
    M4(R, i, 3) = -(M4(R, i, 0) * M4(A, 0, 3) + M4(R, i, 1) * M4(A, 1, 3) + M4(R, i, 2) * M4(A, 2, 3));
  }
  M4(R, 3, 3) = 1.0;
  memcpy(Ainv, R, sizeof(R));
}

/* Eigen::AngleAxisd(Matrix3d).angle(): matrix -> quaternion -> 2*atan2(|vec|, |w|) */
double orc_rotation_angle(const double T[16]) {
  double q[4]; /* x y z w */
  double t = M4(T, 0, 0) + M4(T, 1, 1) + M4(T, 2, 2);
  if (t > 0.0) {
    t = sqrt(t + 1.0);
    q[3] = 0.5 * t;
    t = 0.5 / t;
    q[0] = (M4(T, 2, 1) - M4(T, 1, 2)) * t;
    q[1] = (M4(T, 0, 2) - M4(T, 2, 0)) * t;
    q[2] = (M4(T, 1, 0) - M4(T, 0, 1)) * t;
  } else {
    int i = 0;
    if (M4(T, 1, 1) > M4(T, 0, 0)) i = 1;
    if (M4(T, 2, 2) > M4(T, i, i)) i = 2;
    const int j = (i + 1) % 3;
    const int k = (j + 1) % 3;
    t = sqrt(M4(T, i, i) - M4(T, j, j) - M4(T, k, k) + 1.0);
    q[i] = 0.5 * t;
    t = 0.5 / t;
    q[3] = (M4(T, k, j) - M4(T, j, k)) * t;
    q[j] = (M4(T, j, i) + M4(T, i, j)) * t;
    q[k] = (M4(T, k, i) + M4(T, i, k)) * t;
  }
  const double n = sqrt((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]);
  if (n != 0.0) {
    return 2.0 * atan2(n, fabs(q[3]));
  }
  return 0.0;
}

/* ------------------------------------------------------------------------------------------
 * dfo::NelderMead<N>   include/dfo/nelder_mead.hpp:32-113
 * ---------------------------------------------------------------------------------------- */

void orc_nm_default_params(orc_nm_params* p) { /* nelder_mead.hpp:12 */
  p->init_step = 0.1;
  p->alpha = 1.0;
  p->gamma = 2.0;
  p->rho = 0.5;
  p->sigma = 0.5;
  p->max_iterations = 1024;
  p->convergence_var_thresh = 1e-5;
}

#define NM_MAXN 8
typedef struct {
  double v[NM_MAXN + 1]; /* VectorM: [0] = value, [1..N] = sample  (nelder_mead.hpp:27) */
} nm_vec;

/* std::sort(x.begin(), x.end(), lhs[0] < rhs[0]) for n <= 16: libstdc++ __insertion_sort */
static void nm_sort(nm_vec* x, int count) {
  for (int i = 1; i < count; i++) {
    nm_vec val = x[i];
    if (val.v[0] < x[0].v[0]) {
      memmove(&x[1], &x[0], sizeof(nm_vec) * (size_t)i);
      x[0] = val;
    } else {
      int j = i;
      while (val.v[0] < x[j - 1].v[0]) { /* __unguarded_linear_insert */
        x[j] = x[j - 1];
        j--;
      }
      x[j] = val;
    }
  }
}

/* nelder_mead.hpp:105-113 */
static int nm_is_converged(const nm_vec* x, int n, double thresh) {
  const int m = n + 1;
  double mean[NM_MAXN + 1], var[NM_MAXN + 1];
  for (int d = 0; d < m; d++) {
    double s = 0.0;
    for (int k = 0; k < m; k++) s = s + x[k].v[d];
    mean[d] = s / (double)m;
    var[d] = 0.0;
  }
  for (int k = 0; k < m; k++) {
    for (int d = 0; d < m; d++) {
      const double e = x[k].v[d] - mean[d];
      var[d] = var[d] + e * e;
    }
  }
  double sum = 0.0;
  for (int d = 1; d < m; d++) sum = sum + var[d];
  return sum < thresh;
}

void orc_nelder_mead(int n, orc_nm_function f, void* user, const double* x0, const orc_nm_params* params, orc_nm_result* result) {
  const int m = n + 1;
  nm_vec x[NM_MAXN + 1];
  int evals = 0;
  memset(result, 0, sizeof(*result));
  memset(x, 0, sizeof(x));

  /* :35-37 */
  x[0].v[0] = f(x0, user), evals++;
  for (int d = 0; d < n; d++) x[0].v[1 + d] = x0[d];
  /* :39-46 */
  for (int i = 0; i < n; i++) {
    nm_vec xi;
    memset(&xi, 0, sizeof(xi));
    for (int d = 0; d < n; d++) xi.v[1 + d] = x0[d];
    xi.v[1 + i] += params->init_step;
    xi.v[0] = f(&xi.v[1], user), evals++;
    x[1 + i] = xi;
  }

  for (int it = 0; it < params->max_iterations; it++) { /* :49 */
    result->num_iterations = it;                          /* :50 */
    nm_sort(x, m);                                        /* :51 */
    if (nm_is_converged(x, n, params->convergence_var_thresh)) { /* :52-55 */
      result->converged = 1;
      break;
    }

    nm_vec xo, xr; /* :57-61 */
    for (int d = 0; d < m; d++) {
      double s = 0.0;
      for (int k = 0; k < n; k++) s = s + x[k].v[d];
      xo.v[d] = s / (double)n;
    }
    xo.v[0] = f(&xo.v[1], user), evals++; /* value never used */
    for (int d = 0; d < m; d++) xr.v[d] = xo.v[d] + params->alpha * (xo.v[d] - x[n].v[d]);
    xr.v[0] = f(&xr.v[1], user), evals++;

    if (x[0].v[0] <= xr.v[0] && xr.v[0] < x[n - 1].v[0]) { /* :63-64 */
      x[n] = xr;
    } else if (xr.v[0] < x[0].v[0]) { /* :65-73 */
      nm_vec xe;
      for (int d = 0; d < m; d++) xe.v[d] = xo.v[d] + params->gamma * (xo.v[d] - x[n].v[d]);
      xe.v[0] = f(&xe.v[1], user), evals++;
      x[n] = (xe.v[0] < xr.v[0]) ? xe : xr;
    } else { /* :74-86 */
      nm_vec xc;
      for (int d = 0; d < m; d++) xc.v[d] = xo.v[d] + params->rho * (xo.v[d] - x[n].v[d]);
      xc.v[0] = f(&xc.v[1], user), evals++;
      if (xc.v[0] < x[n].v[0]) {
        x[n] = xc;
      } else {
        for (int j = 1; j < m; j++) {
          for (int d = 0; d < m; d++) x[j].v[d] = x[0].v[d] + params->rho * (x[j].v[d] - x[0].v[d]);
          x[j].v[0] = f(&x[j].v[1], user), evals++;
        }
      }
    }
    /* :88-96 callbacks are unset by VisualCameraCalibration and estimate_direction */
  }

  for (int d = 0; d < n; d++) result->x[d] = x[0].v[1 + d]; /* :99 */
  result->y = x[0].v[0];                                    /* :100 */
  result->num_evaluations = evals;
}

/* ------------------------------------------------------------------------------------------
 * estimate_camera_fov   src/vlcal/common/estimate_fov.cpp:17-51
 * ---------------------------------------------------------------------------------------- */

/* to_dir: AngleAxisd(x0, UnitX) * AngleAxisd(x1, UnitY) * UnitZ   (:18-20)
 * Eigen: AngleAxis*AngleAxis -> Quaternion product; Quaternion*Vector3 -> _transformVector */
static void fov_to_dir(const double x[2], double dir[3]) {
  const double ha = 0.5 * x[0], hb = 0.5 * x[1];
  const double aw = cos(ha), ax = sin(ha); /* (w, x,0,0) */
  const double bw = cos(hb), by = sin(hb); /* (w, 0,y,0) */
  /* quaternion product a*b (Eigen quat_product) with a.y=a.z=b.x=b.z=0 */
  const double qw = aw * bw - ax * 0.0 - 0.0 * by - 0.0 * 0.0;
  const double qx = aw * 0.0 + ax * bw + 0.0 * 0.0 - 0.0 * by;
  const double qy = aw * by + 0.0 * bw + 0.0 * 0.0 - ax * 0.0;
  const double qz = aw * 0.0 + 0.0 * bw + ax * by - 0.0 * 0.0;
  /* _transformVector(v = ez): uv = 2 * vec x v ; v + w*uv + vec x uv */
  const double v[3] = {0.0, 0.0, 1.0};
  double uv[3] = {qy * v[2] - qz * v[1], qz * v[0] - qx * v[2], qx * v[1] - qy * v[0]};
  uv[0] += uv[0], uv[1] += uv[1], uv[2] += uv[2];
  const double c[3] = {qy * uv[2] - qz * uv[1], qz * uv[0] - qx * uv[2], qx * uv[1] - qy * uv[0]};
  dir[0] = v[0] + qw * uv[0] + c[0];
  dir[1] = v[1] + qw * uv[1] + c[1];
  dir[2] = v[2] + qw * uv[2] + c[2];
}

typedef struct {
  const orc_camera* cam;
  double pt_2d[2];
} fov_ctx;

static double fov_objective(const double* x, void* user) { /* :22-26 */
  const fov_ctx* c = (const fov_ctx*)user;
  double dir[3], uv[2];
  fov_to_dir(x, dir);
  orc_project(c->cam, dir, uv);
  const double ex = c->pt_2d[0] - uv[0];
  const double ey = c->pt_2d[1] - uv[1];
  const double err = ex * ex + ey * ey;
  return isfinite(err) ? err : DBL_MAX;
}

double orc_estimate_camera_fov(const orc_camera* cam, int width, int height) {
  /* :37 -- note the integer divisions image_size[0] / 2 */
  const double corners[3][2] = {{0.0, 0.0}, {(double)(width / 2), 0.0}, {0.0, (double)(height / 2)}};
  double max_fov = 0.0;
  for (int k = 0; k < 3; k++) {
    fov_ctx ctx;
    ctx.cam = cam;
    ctx.pt_2d[0] = corners[k][0], ctx.pt_2d[1] = corners[k][1];
    orc_nm_params p;
    orc_nm_default_params(&p); /* :29 */
    orc_nm_result r;
    const double x0[2] = {0.0, 0.0};
    orc_nelder_mead(2, fov_objective, &ctx, x0, &p, &r); /* :30-31 */
    double dir[3], dn[3];
    fov_to_dir(r.x, dir); /* :33 */
    normalized3(dir, dn);
    const double fov = acos(dn[2]); /* :43 */
    if (fov > max_fov) max_fov = fov;
  }
  return max_fov;
}

/* ------------------------------------------------------------------------------------------
 * CostCalculatorNID::calculate   src/vlcal/calib/cost_calculator_nid.cpp:21-67
 * ---------------------------------------------------------------------------------------- */

double orc_nid_from_hist(const int32_t* hist, int bins, double* Hr_out, double* Hs_out, double* Hrs_out, double* MI_out) {
  /* marginals are the row / column sums of the joint (all three incremented together, :49-51) */
  int32_t* hist_image = (int32_t*)calloc((size_t)bins, sizeof(int32_t));
  int32_t* hist_points = (int32_t*)calloc((size_t)bins, sizeof(int32_t));
  for (int lb = 0; lb < bins; lb++) {
    for (int ib = 0; ib < bins; ib++) {
      const int32_t c = hist[ib + lb * bins];
      hist_image[ib] += c;
      hist_points[lb] += c;
    }
  }
  int sum = 0; /* :54 */
  for (int i = 0; i < bins; i++) sum += hist_image[i];

  double Hr = 0.0, Hs = 0.0, Hrs = 0.0; /* :59-61, sums in storage order */
  for (int i = 0; i < bins; i++) {
    const double p = (double)hist_image[i] / sum;
    Hr = Hr + p * log(p + 1e-6);
  }
  for (int i = 0; i < bins; i++) {
    const double p = (double)hist_points[i] / sum;
    Hs = Hs + p * log(p + 1e-6);
  }
  for (int i = 0; i < bins * bins; i++) {
    const double p = (double)hist[i] / sum;
    Hrs = Hrs + p * log(p + 1e-6);
  }
  Hr = -Hr, Hs = -Hs, Hrs = -Hrs;
  const double MI = Hr + Hs - Hrs;     /* :63 */
  const double NID = (Hrs - MI) / Hrs; /* :64 */
  if (Hr_out) *Hr_out = Hr;
  if (Hs_out) *Hs_out = Hs;
  if (Hrs_out) *Hrs_out = Hrs;
  if (MI_out) *MI_out = MI;
  free(hist_image);
  free(hist_points);
  return NID;
}

/* one point of the loop body :31-51; returns 1 and the bin pair if the point is an inlier */
static inline int nid_point(
  const orc_camera* cam, const uint8_t* image, int width, int height, int row_stride, const double* pt, double intensity, int bins, double cos_fov, const double* T, int* image_bin, int* lidar_bin) {
  /* :31 pt_camera = T * p  (4x4 homogeneous, w = 1): ((m0*x + m1*y) + m2*z) + m3*1 */
  double pc[3];
  for (int r = 0; r < 3; r++) {
    pc[r] = ((M4(T, r, 0) * pt[0] + M4(T, r, 1) * pt[1]) + M4(T, r, 2) * pt[2]) + M4(T, r, 3);
  }
  /* :32 pt_camera.head<3>().normalized().z() < cos(max_fov) */
  const double z2 = sqnorm3(pc);
  const double nz = z2 > 0.0 ? pc[2] / sqrt(z2) : pc[2];
  if (nz < cos_fov) {
    return 0;
  }
  /* :37 */
  double uv[2];
  orc_project(cam, pc, uv);
  const int ix = orc_cast_int(uv[0]);
  const int iy = orc_cast_int(uv[1]);
  /* :38 */
  if (ix < 0 || iy < 0 || ix >= width || iy >= height) {
    return 0;
  }
  /* :43-47 */
  const double pixel = image[(size_t)iy * (size_t)row_stride + (size_t)ix] / 255.0;
  int ib = orc_cast_int(pixel * bins);
  int lb = orc_cast_int(intensity * bins);
  ib = ib < bins - 1 ? ib : bins - 1;
  ib = ib > 0 ? ib : 0;
  lb = lb < bins - 1 ? lb : bins - 1;
  lb = lb > 0 ? lb : 0;
  *image_bin = ib;
  *lidar_bin = lb;
  return 1;
}

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
  const double T[16],
  int32_t* hist_out) {
  int32_t* hist = (int32_t*)calloc((size_t)bins * bins, sizeof(int32_t));
  const double cos_fov = cos(max_fov);
  for (int64_t i = 0; i < n; i++) { /* :30 */
    int ib, lb;
    if (nid_point(cam, image, width, height, row_stride, points_xyzw + 4 * i, intensities[i], bins, cos_fov, T, &ib, &lb)) {
      hist[ib + lb * bins]++; /* :49 */
    }
  }
  const double nid = orc_nid_from_hist(hist, bins, NULL, NULL, NULL, NULL);
  if (hist_out) memcpy(hist_out, hist, sizeof(int32_t) * (size_t)bins * bins);
  free(hist);
  return nid;
}

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
  const double T[16],
  int32_t* hist_out) {
  const size_t nb = (size_t)bins * bins;
  int32_t* hist = (int32_t*)calloc(nb, sizeof(int32_t));
  const double cos_fov = cos(max_fov);
#pragma omp parallel
  {
    int32_t* local = (int32_t*)calloc(nb, sizeof(int32_t));
#pragma omp for schedule(static)
    for (int64_t i = 0; i < n; i++) {
      int ib, lb;
      if (nid_point(cam, image, width, height, row_stride, points_xyzw + 4 * i, intensities[i], bins, cos_fov, T, &ib, &lb)) {
        local[ib + lb * bins]++;
      }
    }
#pragma omp critical
    for (size_t k = 0; k < nb; k++) hist[k] += local[k];
    free(local);
  }
  const double nid = orc_nid_from_hist(hist, bins, NULL, NULL, NULL, NULL);
  if (hist_out) memcpy(hist_out, hist, sizeof(int32_t) * nb);
  free(hist);
  return nid;
}

/* ----------------------------------------------------------------------------------------
 * generate_lidar_image   src/vlcal/preprocess/generate_lidar_image.cpp:8-41
 * LiDAR intensity image (CV_64FC1, 0 where no point lands) and point-index map (CV_32SC1, -1 where no point lands): per
 * pixel the point with the smallest squared range wins; of several points with the SAME squared range the last one does
 * (:31 skips only when the stored value is strictly smaller).
 * ---------------------------------------------------------------------------------------- */
void orc_generate_lidar_image(
  const orc_camera* cam,
  int width,
  int height,
  const double T[16],
  const double* points_xyzw,
  const double* intensities,
  int64_t n,
  double* intensity_image,
  int32_t* index_image) {
  const double camera_fov = orc_estimate_camera_fov(cam, width, height); /* :10 */
  const double min_z = cos(camera_fov);                                  /* :11 */
  const size_t npix = (size_t)width * (size_t)height;
  double* sq_dist_image = (double*)malloc(sizeof(double) * (npix > 0 ? npix : 1));
  for (size_t i = 0; i < npix; i++) { /* :13-15 */
    sq_dist_image[i] = DBL_MAX;
    intensity_image[i] = 0.0;
    index_image[i] = -1;
  }
  for (int64_t i = 0; i < n; i++) { /* :17 */
    const double* pt = points_xyzw + 4 * i;
    double pc[3];
    for (int r = 0; r < 3; r++) { /* :19 */
      pc[r] = ((M4(T, r, 0) * pt[0] + M4(T, r, 1) * pt[1]) + M4(T, r, 2) * pt[2]) + M4(T, r, 3) * pt[3];
    }
    const double n2 = sqnorm3(pc); /* :21 head<3>().normalized().z() */
    const double nz = n2 > 0.0 ? pc[2] / sqrt(n2) : pc[2];
    if (nz < min_z) {
      continue;
    }
    double uv[2];
    orc_project(cam, pc, uv); /* :25 */
    const int ix = orc_cast_int(uv[0]);
    const int iy = orc_cast_int(uv[1]);
    if (ix < 0 || iy < 0 || ix >= width || iy >= height) { /* :26-28 */
      continue;
    }
    const double sq_dist = sqnorm3(pc); /* :30 */
    const size_t p = (size_t)iy * (size_t)width + (size_t)ix;
    if (sq_dist_image[p] < sq_dist) { /* :31-33 */
      continue;
    }
    sq_dist_image[p] = sq_dist; /* :35-37 */
    intensity_image[p] = intensities[i];
    index_image[p] = (int32_t)i;
  }
  free(sq_dist_image);
}

/* ------------------------------------------------------------------------------------------
 * ViewCulling::cull   src/vlcal/calib/view_culling.cpp:21-92
 * ---------------------------------------------------------------------------------------- */

int64_t orc_view_cull(
  const orc_camera* cam,
  int width,
  int height,
  double max_fov,
  int enable_depth_buffer_culling,
  const double* points_xyzw,
  int64_t n,
  const double T[16],
  int32_t* indices_out) {
  const double min_z = cos(max_fov); /* :17 */
  const size_t npix = (size_t)width * (size_t)height;
  float* dist_map = (float*)malloc(sizeof(float) * npix);
  /* :40 CV_32FC1 filled with cv::Scalar(DBL_MAX): saturate_cast<float>(double) = (float)DBL_MAX = +inf */
  for (size_t i = 0; i < npix; i++) dist_map[i] = (float)INFINITY;
  int32_t* proj = (int32_t*)malloc(sizeof(int32_t) * 2 * (size_t)(n > 0 ? n : 1));
  double* pcs = (double*)malloc(sizeof(double) * 3 * (size_t)(n > 0 ? n : 1));
  int64_t count = 0;

  for (int64_t i = 0; i < n; i++) { /* :43 */
    const double* pt = points_xyzw + 4 * i;
    double pc[4];
    for (int r = 0; r < 3; r++) { /* :25-28 */
      pc[r] = ((M4(T, r, 0) * pt[0] + M4(T, r, 1) * pt[1]) + M4(T, r, 2) * pt[2]) + M4(T, r, 3) * pt[3];
    }
    pc[3] = ((M4(T, 3, 0) * pt[0] + M4(T, 3, 1) * pt[1]) + M4(T, 3, 2) * pt[2]) + M4(T, 3, 3) * pt[3];
    /* :45 pt_camera.normalized().head<3>().z(): normalises the homogeneous 4-vector (w included) */
    const double z4 = (pc[0] * pc[0] + pc[1] * pc[1]) + (pc[2] * pc[2] + pc[3] * pc[3]);
    const double nz = z4 > 0.0 ? pc[2] / sqrt(z4) : pc[2];
    if (nz < min_z) {
      continue;
    }
    double uv[2];
    orc_project(cam, pc, uv); /* :50 */
    const int ix = orc_cast_int(uv[0]);
    const int iy = orc_cast_int(uv[1]);
    if (ix < 0 || iy < 0 || ix >= width || iy >= height) { /* :51-54 */
      continue;
    }
    indices_out[count] = (int32_t)i; /* :56-57 kept even if it loses the z-test below */
    proj[2 * count] = ix, proj[2 * count + 1] = iy;
    pcs[3 * count] = pc[0], pcs[3 * count + 1] = pc[1], pcs[3 * count + 2] = pc[2];
    count++;

    if (enable_depth_buffer_culling) { /* :59-67 */
      const double dist = sqrt(sqnorm3(pc));
      float* cell = &dist_map[(size_t)iy * (size_t)width + (size_t)ix];
      if (dist > *cell) {
        continue;
      }
      *cell = (float)dist;
    }
  }

  if (enable_depth_buffer_culling) { /* :70-89 */
    int64_t kept = 0;
    for (int64_t k = 0; k < count; k++) {
      const double dist = sqrt(sqnorm3(pcs + 3 * k));
      const float cell = dist_map[(size_t)proj[2 * k + 1] * (size_t)width + (size_t)proj[2 * k]];
      if (dist > cell + 0.1) { /* :81 float + double */
        continue;
      }
      indices_out[kept++] = indices_out[k];
    }
    count = kept;
  }
  free(dist_map);
  free(proj);
  free(pcs);
  return count;
}

void orc_project_n(const orc_camera* cam, const double* p, int64_t n, double* uv) {
  for (int64_t i = 0; i < n; i++) orc_project(cam, p + 3 * i, uv + 2 * i);
}

/* ------------------------------------------------------------------------------------------
 * NIDCost::operator()<double>   include/vlcal/costs/nid_cost.hpp:36-107  (mode B)
 * ---------------------------------------------------------------------------------------- */

int orc_nid_cost_bspline(
  const orc_camera* cam,
  const double* image64,
  int width,
  int height,
  const double* points_xyzw,
  const double* intensities,
  int64_t n,
  int bins,
  const double Tp[7],
  double* nid_out,
  double* hist_out) {
  /* :27-33 spline_coeffs / 6 */
  static const double C6[4][4] = {{1.0, -3.0, 3.0, -1.0}, {4.0, 0.0, -6.0, 3.0}, {1.0, 3.0, 3.0, -3.0}, {0.0, 0.0, 0.0, 1.0}};
  double C[4][4];
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++) C[i][j] = C6[i][j] / 6.0;

  const size_t nb = (size_t)bins * bins;
  double* hist = (double*)calloc(nb, sizeof(double));
  double* hist_image = (double*)calloc((size_t)bins, sizeof(double));
  double* hist_points = (double*)calloc((size_t)bins, sizeof(double));
  const double qx = Tp[0], qy = Tp[1], qz = Tp[2], qw = Tp[3];
  const double t[3] = {Tp[4], Tp[5], Tp[6]};

  for (int64_t i = 0; i < n; i++) { /* :46 */
    const double* p = points_xyzw + 4 * i;
    /* :47 Sophus SO3::operator*: uv = q.vec x p; uv += uv; p + w*uv + q.vec x uv; then + t */
    double uv[3] = {qy * p[2] - qz * p[1], qz * p[0] - qx * p[2], qx * p[1] - qy * p[0]};
    uv[0] += uv[0], uv[1] += uv[1], uv[2] += uv[2];
    const double c[3] = {qy * uv[2] - qz * uv[1], qz * uv[0] - qx * uv[2], qx * uv[1] - qy * uv[0]};
    double pc[3];
    for (int k = 0; k < 3; k++) pc[k] = (p[k] + qw * uv[k] + c[k]) + t[k];

    int bin_points = orc_cast_int(intensities[i] * bins); /* :49 */
    bin_points = bin_points < bins - 1 ? bin_points : bins - 1;
    bin_points = bin_points > 0 ? bin_points : 0;

    double pr[2];
    orc_project(cam, pc, pr); /* :51 */
    const int kx = orc_cast_int(floor(pr[0])); /* :52 */
    const int ky = orc_cast_int(floor(pr[1]));
    const double s[2] = {pr[0] - (double)kx, pr[1] - (double)ky}; /* :53 */
    if (kx < 0 || ky < 0 || kx >= width || ky >= height) { /* :55-58 */
      continue;
    }
    hist_points[bin_points] += 1.0; /* :60 */

    double beta[4][2]; /* :62-68 beta = C * [1 s s^2 s^3]^T */
    for (int a = 0; a < 2; a++) {
      const double se[4] = {1.0, s[a], s[a] * s[a], (s[a] * s[a]) * s[a]};
      for (int r = 0; r < 4; r++) {
        beta[r][a] = ((C[r][0] * se[0] + C[r][1] * se[1]) + C[r][2] * se[2]) + C[r][3] * se[3];
      }
    }
    int knots_x[4], knots_y[4]; /* :70-73 */
    for (int k = 0; k < 4; k++) {
      int vx = kx - 1 + k, vy = ky - 1 + k;
      vx = vx > 0 ? vx : 0;
      vx = vx < width - 1 ? vx : width - 1;
      vy = vy > 0 ? vy : 0;
      vy = vy < height - 1 ? vy : height - 1;
      knots_x[k] = vx, knots_y[k] = vy;
    }
    for (int a = 0; a < 4; a++) { /* :75-83 */
      for (int b = 0; b < 4; b++) {
        const double w = beta[a][0] * beta[b][1];
        const double pix = image64[(size_t)knots_y[b] * (size_t)width + (size_t)knots_x[a]];
        int bin_image = orc_cast_int(pix * bins);
        bin_image = bin_image < bins - 1 ? bin_image : bins - 1; /* :79 std::min only */
        hist[bin_image + bin_points * bins] += w;
        hist_image[bin_image] += w;
      }
    }
  }

  double sum = 0.0; /* :86 */
  for (int i = 0; i < bins; i++) sum = sum + hist_points[i];
  if (hist_out) memcpy(hist_out, hist, sizeof(double) * nb);

  double Hi = 0.0, Hp = 0.0, Hip = 0.0; /* :88-94 */
  for (int i = 0; i < bins; i++) {
    const double p = hist_image[i] / sum;
    Hi = Hi + p * log(p + 1e-6);
  }
  for (int i = 0; i < bins; i++) {
    const double p = hist_points[i] / sum;
    Hp = Hp + p * log(p + 1e-6);
  }
  for (size_t i = 0; i < nb; i++) {
    const double p = hist[i] / sum;
    Hip = Hip + p * log(p + 1e-6);
  }
  Hi = -Hi, Hp = -Hp, Hip = -Hip;
  const double MI = Hi + Hp - Hip;
  const double NID = (Hip - MI) / Hip;
  free(hist);
  free(hist_image);
  free(hist_points);
  if (!isfinite(NID)) { /* :98-102 */
    return 0;
  }
  *nid_out = NID;
  return 1;
}

/* ------------------------------------------------------------------------------------------
 * VisualCameraCalibration (NID_NELDER_MEAD branch)   src/vlcal/calib/visual_camera_calibration.cpp:35-139
 * ---------------------------------------------------------------------------------------- */

void orc_calib_default_params(orc_calib_params* p) { /* visual_camera_calibration.hpp:12-26 */
  p->max_outer_iterations = 10;
  p->max_inner_iterations = 256;
  p->delta_trans_thresh = 0.1;
  p->delta_rot_thresh = 0.5 * M_PI / 180.0;
  p->disable_z_buffer_culling = 0;
  p->nid_bins = 16;
  p->nelder_mead_init_step = 1e-3;
  p->nelder_mead_convergence_criteria = 1e-8;
}

/* threads of the objective's loop over bags (visual_camera_calibration.cpp:107): 0 = one per bag, 1 = serial */
#define ORC_MAX_BAGS 64
static int g_bag_threads = 0;
void orc_set_bag_threads(int n) { g_bag_threads = n < 0 ? 0 : n; }

typedef struct {
  const orc_camera* cam;
  int n_bags;
  const orc_bag* bags;        /* culled */
  const double* max_fovs;     /* per cost object (:82-84 -> cost_calculator_nid.cpp:17) */
  int bins;
  const double* init_T;
  double best_cost;
  orc_trace* trace;
} calib_ctx;

static double calib_objective(const double* x, void* user) { /* :103-119 */
  calib_ctx* c = (calib_ctx*)user;
  double E[16], T[16];
  orc_se3_expmap_gtsam(x, E);
  orc_isometry_mul(c->init_T, E, T); /* :104 */
  double sum_costs = 0.0;
  /* :107-110 `#pragma omp parallel for reduction(+ : sum_costs)` over the bags: one thread per cost object, each serial
   * over its points.  The per-bag values are added in bag order afterwards, so the result does not depend on the team
   * size (the reference's reduction order is unspecified; with one bag there is nothing to reorder). */
  double per_bag[ORC_MAX_BAGS];
  const int nb = c->n_bags;
  if (nb <= ORC_MAX_BAGS && g_bag_threads != 1 && nb > 1) {
    const int team = g_bag_threads > 0 ? (g_bag_threads < nb ? g_bag_threads : nb) : nb;
#pragma omp parallel for schedule(static) num_threads(team)
    for (int i = 0; i < nb; i++) {
      const orc_bag* b = &c->bags[i];
      per_bag[i] = orc_nid_calculate(c->cam, b->image, b->width, b->height, b->row_stride, b->points_xyzw, b->intensities, b->n, c->bins, c->max_fovs[i], T, NULL);
    }
    for (int i = 0; i < nb; i++) sum_costs += per_bag[i];
  } else {
    for (int i = 0; i < nb; i++) {
      const orc_bag* b = &c->bags[i];
      sum_costs += orc_nid_calculate(c->cam, b->image, b->width, b->height, b->row_stride, b->points_xyzw, b->intensities, b->n, c->bins, c->max_fovs[i], T, NULL);
    }
  }
  if (sum_costs < c->best_cost) { /* :112-116 */
    c->best_cost = sum_costs;
  }
  if (c->trace && c->trace->count < c->trace->capacity) {
    double* e = c->trace->evals + 7 * (size_t)c->trace->count;
    memcpy(e, x, 6 * sizeof(double));
    e[6] = sum_costs;
  }
  if (c->trace) c->trace->count++;
  return sum_costs;
}

void orc_estimate_pose_nelder_mead(
  const orc_camera* cam,
  const orc_bag* bags,
  int n_bags,
  const orc_calib_params* params,
  const double init_T[16],
  double T_out[16],
  orc_nm_result* nm_result,
  orc_trace* trace) {
  /* :71-73 ViewCulling on dataset.front()'s image size */
  const double cull_fov = orc_estimate_camera_fov(cam, bags[0].width, bags[0].height);
  orc_bag* culled = (orc_bag*)calloc((size_t)n_bags, sizeof(orc_bag));
  double* max_fovs = (double*)calloc((size_t)n_bags, sizeof(double));
  for (int b = 0; b < n_bags; b++) { /* :76-84 */
    const orc_bag* src = &bags[b];
    int32_t* idx = (int32_t*)malloc(sizeof(int32_t) * (size_t)(src->n > 0 ? src->n : 1));
    const int64_t m = orc_view_cull(cam, bags[0].width, bags[0].height, cull_fov, !params->disable_z_buffer_culling, src->points_xyzw, src->n, init_T, idx);
    double* pts = (double*)malloc(sizeof(double) * 4 * (size_t)(m > 0 ? m : 1));
    double* ins = (double*)malloc(sizeof(double) * (size_t)(m > 0 ? m : 1));
    for (int64_t k = 0; k < m; k++) { /* sample(): frame_cpu.cpp:281-331 gather */
      memcpy(pts + 4 * k, src->points_xyzw + 4 * (size_t)idx[k], 4 * sizeof(double));
      ins[k] = src->intensities[idx[k]];
    }
    free(idx);
    culled[b] = *src;
    culled[b].points_xyzw = pts;
    culled[b].intensities = ins;
    culled[b].n = m;
    max_fovs[b] = orc_estimate_camera_fov(cam, src->width, src->height); /* cost_calculator_nid.cpp:17 */
  }

  calib_ctx ctx;
  ctx.cam = cam, ctx.n_bags = n_bags, ctx.bags = culled, ctx.max_fovs = max_fovs;
  ctx.bins = params->nid_bins, ctx.init_T = init_T, ctx.best_cost = DBL_MAX, ctx.trace = trace;

  orc_nm_params nm; /* :122-125 */
  orc_nm_default_params(&nm);
  nm.init_step = params->nelder_mead_init_step;
  nm.convergence_var_thresh = params->nelder_mead_convergence_criteria;
  nm.max_iterations = params->max_inner_iterations;
  const double x0[6] = {0, 0, 0, 0, 0, 0};
  orc_nm_result r;
  orc_nelder_mead(6, calib_objective, &ctx, x0, &nm, &r); /* :126-127 */

  double E[16];
  orc_se3_expmap_gtsam(r.x, E);
  orc_isometry_mul(init_T, E, T_out); /* :129 */
  if (nm_result) *nm_result = r;

  for (int b = 0; b < n_bags; b++) {
    free((void*)culled[b].points_xyzw);
    free((void*)culled[b].intensities);
  }
  free(culled);
  free(max_fovs);
}

void orc_calibrate(
  const orc_camera* cam,
  const orc_bag* bags,
  int n_bags,
  const orc_calib_params* params,
  const double init_T[16],
  double T_out[16],
  orc_calib_stats* stats,
  orc_trace* trace) {
  double T[16];
  memcpy(T, init_T, sizeof(T));
  if (stats) memset(stats, 0, sizeof(*stats));
  for (int i = 0; i < params->max_outer_iterations; i++) { /* :39 */
    double new_T[16];
    orc_nm_result r;
    orc_estimate_pose_nelder_mead(cam, bags, n_bags, params, T, new_T, &r, trace); /* :46 */
    double inv[16], delta[16];
    orc_isometry_inverse(new_T, inv);
    orc_isometry_mul(inv, T, delta); /* :50 */
    memcpy(T, new_T, sizeof(T));     /* :51 */
    const double delta_t = sqrt((M4(delta, 0, 3) * M4(delta, 0, 3) + M4(delta, 1, 3) * M4(delta, 1, 3)) + M4(delta, 2, 3) * M4(delta, 2, 3)); /* :53 */
    const double delta_r = orc_rotation_angle(delta);                                                                                           /* :54 */
    const int converged = delta_t < params->delta_trans_thresh && delta_r < params->delta_rot_thresh;                                       /* :55 */
    if (stats) {
      stats->outer_iterations = i + 1;
      stats->total_evaluations += r.num_evaluations;
      if (i < 16) {
        stats->inner_iterations[i] = r.num_iterations;
        stats->inner_final_cost[i] = r.y;
      }
      stats->best_cost_last = r.y;
    }
    if (converged) { /* :62-64 */
      break;
    }
  }
  memcpy(T_out, T, sizeof(T));
}
