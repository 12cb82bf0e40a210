/*
 * pose_oracle.c -- CPU checker for PoseEstimation (csrc/pose_estimation.cu), test infrastructure only.
 *
 * A plain-C restatement, linked against the CPU oracle (oracle/vlcal_oracle.c: orc_project, orc_nelder_mead), of
 *   - estimate_direction (src/vlcal/common/estimate_fov.cpp:17-34) and the LiDAR bearings (estimate_pose.cpp:47-51);
 *   - the per-hypothesis rotation (the closed-form two-pair Umeyama solution), the squared reprojection errors and the
 *     inlier count (:108-116), in the operation order of the kernel, so that every squared error equals the kernel's up to the last-ulp differences of
 *     the device's transcendental functions (fisheye, atan, equirectangular);
 *   - InitialGuessAuto::read_correspondences' rules (initial_guess_auto.cpp:81-125).
 * Built with -ffp-contract=off (no FMA), like the oracle.
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "vlcal_oracle.h"

/* AngleAxisd(x0, UnitX) * AngleAxisd(x1, UnitY) * UnitZ (estimate_fov.cpp:18-20), evaluated as Eigen does */
static void to_dir(const double x[2], double dir[3]) {
  const double ha = 0.5 * x[0], hb = 0.5 * x[1];
  const double aw = cos(ha), ax = sin(ha);
  const double bw = cos(hb), by = sin(hb);
  const double qw = aw * bw - ax * 0.0 - 0.0 * by - 0.0 * 0.0;
  const double qx = aw * 0.0 + ax * bw + 0.0 * 0.0 - 0.0 * by;
  const double qy = aw * by + 0.0 * bw + 0.0 * 0.0 - ax * 0.0;
  const double qz = aw * 0.0 + 0.0 * bw + ax * by - 0.0 * 0.0;
  const double v[3] = {0.0, 0.0, 1.0};
  double uv[3] = {qy * v[2] - qz * v[1], qz * v[0] - qx * v[2], qx * v[1] - qy * v[0]};
  uv[0] += uv[0], uv[1] += uv[1], uv[2] += uv[2];
  const double c[3] = {qy * uv[2] - qz * uv[1], qz * uv[0] - qx * uv[2], qx * uv[1] - qy * uv[0]};
  for (int i = 0; i < 3; i++) dir[i] = v[i] + qw * uv[i] + c[i];
}

typedef struct {
  const orc_camera* cam;
  double target[2];
} dir_ctx;

static double dir_objective(const double* x, void* user) { /* :22-26 */
  const dir_ctx* c = (const dir_ctx*)user;
  double d[3], uv[2];
  to_dir(x, d);
  orc_project(c->cam, d, uv);
  const double ex = c->target[0] - uv[0], ey = c->target[1] - uv[1];
  const double err = ex * ex + ey * ey;
  return isfinite(err) ? err : DBL_MAX;
}

void pose_oracle_direction(const orc_camera* cam, const double pixel[2], double dir[3]) {
  dir_ctx ctx;
  ctx.cam = cam;
  ctx.target[0] = pixel[0], ctx.target[1] = pixel[1];
  orc_nm_params p;
  orc_nm_default_params(&p);
  orc_nm_result r;
  const double x0[2] = {0.0, 0.0};
  orc_nelder_mead(2, dir_objective, &ctx, x0, &p, &r);
  to_dir(r.x, dir);
}

static double sq3(const double v[3]) { return (v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]; }

/* the kernel's pair rotation: R = a^ p^T + b^ q^T + (a^ x b^)(p^ x q^)^T, a = c1 + c2, b = c1 - c2, p = l1 + l2, q = l1 - l2 */
static int pair_rotation(const double* c1, const double* c2, const double* l1, const double* l2, double R[9]) {
  double a[3], b[3], p[3], q[3];
  for (int k = 0; k < 3; k++) a[k] = c1[k] + c2[k], b[k] = c1[k] - c2[k], p[k] = l1[k] + l2[k], q[k] = l1[k] - l2[k];
  const double na = sq3(a), nb = sq3(b), np = sq3(p), nq = sq3(q), eps = 1e-18;
  if (!(na >= eps && nb >= eps && np >= eps && nq >= eps)) return 0;
  const double ia = 1.0 / sqrt(na), ib = 1.0 / sqrt(nb), ip = 1.0 / sqrt(np), iq = 1.0 / sqrt(nq);
  for (int k = 0; k < 3; k++) a[k] = a[k] * ia, b[k] = b[k] * ib, p[k] = p[k] * ip, q[k] = q[k] * iq;
  const double u3[3] = {a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]};
  const double v3[3] = {p[1] * q[2] - p[2] * q[1], p[2] * q[0] - p[0] * q[2], p[0] * q[1] - p[1] * q[0]};
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) R[3 * r + c] = (a[r] * p[c] + b[r] * q[c]) + u3[r] * v3[c];
  return 1;
}

/* bearings (m x 3 each, row-major): camera from estimate_direction(kp0), LiDAR = normalized point */
void pose_oracle_bearings(const orc_camera* cam, const double* kp0, const double* points, int m, double* dc, double* dl) {
#pragma omp parallel for schedule(dynamic, 64)
  for (int i = 0; i < m; i++) {
    pose_oracle_direction(cam, kp0 + 2 * i, dc + 3 * i);
    const double* p = points + 3 * i;
    const double n = sqrt(sq3(p));
    for (int k = 0; k < 3; k++) dl[3 * i + k] = p[k] / n;
  }
}

/* the kernel's rotation of one hypothesis from its two bearing pairs (c_k = R l_k): 1 and R (row-major), or 0 where the
 * pair is degenerate (R untouched) */
int pose_oracle_rotation(const double c1[3], const double c2[3], const double l1[3], const double l2[3], double R[9]) { return pair_rotation(c1, c2, l1, l2, R); }

/* |kp0_j - project(R dl_j)|^2 (:110-113), in the kernel's operation order */
static double sq_error(const orc_camera* cam, const double R[9], const double* kp, const double* d) {
  const double pc[3] = {(R[0] * d[0] + R[1] * d[1]) + R[2] * d[2], (R[3] * d[0] + R[4] * d[1]) + R[5] * d[2], (R[6] * d[0] + R[7] * d[1]) + R[8] * d[2]};
  double uv[2];
  orc_project(cam, pc, uv);
  const double du = kp[0] - uv[0], dv = kp[1] - uv[1];
  return du * du + dv * dv;
}

/* e[j] = the squared reprojection error of every correspondence under R: correspondence j is an inlier iff e[j] < thresh^2 */
void pose_oracle_errors(const orc_camera* cam, const double R[9], const double* kp0, const double* dl, int m, double* e) {
#pragma omp parallel for schedule(static)
  for (int j = 0; j < m; j++) e[j] = sq_error(cam, R, kp0 + 2 * j, dl + 3 * j);
}

/* per hypothesis h: counts[h] = #{j : |kp0_j - project(R_h dl_j)|^2 < thresh^2}, degenerate[h], near[h] = #{j : the squared
 * error lies within 1e-9 px^2 of thresh^2} (where device and host transcendental functions may decide differently) */
void pose_oracle_score(
  const orc_camera* cam, const double* kp0, const double* dc, const double* dl, int m, const int32_t* pairs, int h, double thresh, int32_t* counts,
  uint8_t* degenerate, int32_t* near) {
  const double thresh_sq = pow(thresh, 2);
#pragma omp parallel for schedule(dynamic, 16)
  for (int k = 0; k < h; k++) {
    const int i1 = pairs[2 * k], i2 = pairs[2 * k + 1];
    double R[9];
    const int ok = i1 != i2 && pair_rotation(dc + 3 * i1, dc + 3 * i2, dl + 3 * i1, dl + 3 * i2, R);
    degenerate[k] = ok ? 0 : 1;
    int count = 0, close = 0;
    for (int j = 0; ok && j < m; j++) {
      const double e = sq_error(cam, R, kp0 + 2 * j, dl + 3 * j);
      count += e < thresh_sq;
      close += fabs(e - thresh_sq) <= 1e-9;
    }
    counts[k] = count;
    near[k] = close;
  }
}

/* read_correspondences (initial_guess_auto.cpp:81-125) on already-parsed inputs: kpts0 (n0 x 2), kpts1 (n1 x 2) and
 * matches (n0) as the JSON's numbers, converted with (int) like nlohmann's get<int>; index image H x W int32.
 * Writes the used kpts0 index and point index of each correspondence; returns their number, or -1 for a match index
 * past kpts1, -2 for a kpts1 keypoint outside the image, -3 for a point index past n_points.  *blank_warnings counts
 * the matches skipped with the reference's warning (no point at the pixel nor at any of its 8 neighbours). */
int pose_oracle_correspondences(
  const int32_t* index_image, int width, int height, const double* kpts0, int n0, const double* kpts1, int n1, const double* matches, int64_t n_points,
  int32_t* kp_index_out, int32_t* point_index_out, int* blank_warnings) {
  (void)kpts0;
  int k = 0;
  *blank_warnings = 0;
  for (int i = 0; i < n0; i++) {
    const int match = (int)matches[i];
    if (match < 0) continue;
    if (match >= n1) return -1;
    const int x = (int)kpts1[2 * match], y = (int)kpts1[2 * match + 1];
    if (x < 0 || x >= width || y < 0 || y >= height) return -2;
    const int index = index_image[(int64_t)y * width + x];
    if (index < 0) {
      int found = 0;
      for (int dy = -1; dy <= 1; dy++)
        for (int dx = -1; dx <= 1; dx++) {
          const int xx = x + dx, yy = y + dy;
          if ((dx || dy) && xx >= 0 && xx < width && yy >= 0 && yy < height && index_image[(int64_t)yy * width + xx] >= 0) found = 1;
        }
      if (!found) (*blank_warnings)++;
      continue; /* the reference discards what the neighbour search found */
    }
    if (index >= n_points) return -3;
    kp_index_out[k] = i;
    point_index_out[k] = index;
    k++;
  }
  return k;
}
