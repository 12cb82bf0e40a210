// CPU check of the equirectangular delta step (csrc/lean_filter.cuh: classify_lean_anchor / classify_lean_delta) against
// the exact double path (csrc/exact_classify.cuh): pose 0 of a batch is the anchor, poses 1..7 lie on a line through it
// at 1e-6 .. 5e-3 rad / m (as Nelder-Mead's xr, xe, xc lie on a line through xo).  Every verdict the delta step keeps
// must be the exact path's.  Points are nudged to within 1e-3 .. 1e-8 px of a pixel edge AT POSE k >= 1; some sit near the
// poles and near the seam.  Prints counts as JSON.  Built host-only by tests/test_lean_delta_host.py.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <vector>

#include "exact_classify.cuh"
#include "fast_filter.hpp"
#include "host_math.hpp"

using namespace vlcal;

constexpr int P = 8;

static void pose_rows(const double xi[6], const double* T0, double* rows, float* rows32) {
  double E[16], T[16];
  host::se3_expmap_gtsam(xi, E);
  if (T0) {
    host::isometry_mul(T0, E, T);
  } else {
    std::memcpy(T, E, sizeof(T));
  }
  double tm = 0.0;
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 4; c++) rows[4 * r + c] = T[r + 4 * c];
    for (int c = 0; c < 3; c++) rows32[3 * r + c] = static_cast<float>(T[r + 4 * c]);
    rows32[9 + r] = static_cast<float>(T[r + 12]);
    tm = std::max(tm, std::fabs(T[r + 12]));
  }
  rows32[12] = std::nextafter(static_cast<float>(tm), INFINITY);
}

// out: point-poses and deferrals of the delta step, mismatches, accepted, max error / bound (ppm), batches in the gate,
// enabled, deferrals of the plain classifier on the same point-poses
static void run_case(int W, int H, double max_fov, unsigned seed, long long n_points, long long out[8]) {
  CameraParams cam;
  std::memset(&cam, 0, sizeof(cam));
  cam.model = CAM_EQUIRECTANGULAR;
  cam.n_intr = 2;
  cam.intr[0] = W, cam.intr[1] = H;
  const FastCam f = make_fast_cam(cam, W, H, max_fov);
  const LeanCam lc = make_lean_cam(cam, f, W, H, max_fov);
  if (!lc.enabled) return;
  const double cos_fov = std::cos(max_fov);
  std::mt19937_64 rng(seed);
  std::uniform_real_distribution<double> U(-1.0, 1.0);
  long long total = 0, unc = 0, mism = 0, acc = 0, gated = 0, plain_unc = 0;
  double max_ratio = 0.0;
  const long long per_batch = 2000;
  for (long long b0 = 0; b0 < n_points; b0 += per_batch) {
    // anchor: a perturbation of the identity; poses 1..7 along one direction of the tangent space, mixed signs
    double xi0[6] = {0.05 * U(rng), 0.05 * U(rng), 0.05 * U(rng), 0.3 * U(rng), 0.3 * U(rng), 0.3 * U(rng)};
    double dir[6];
    double nr = 0.0;
    for (double& d : dir) d = U(rng), nr += d * d;
    for (double& d : dir) d /= std::sqrt(nr);
    double T0[16];
    host::se3_expmap_gtsam(xi0, T0);
    double poses[P][12];
    float p32[P][16];
    pose_rows(xi0, nullptr, poses[0], p32[0]);
    for (int k = 1; k < P; k++) {
      const double s = std::pow(10.0, -6.0 + (std::log10(5e-3) + 6.0) * std::fabs(U(rng))) * (U(rng) > 0 ? 1 : -1);
      double xi[6];
      for (int i = 0; i < 6; i++) xi[i] = s * dir[i];
      pose_rows(xi, T0, poses[k], p32[k]);
    }
    float tmax_all = 0.f;
    for (int k = 0; k < P; k++) tmax_all = std::max(tmax_all, p32[k][12]);
    float Q[P][16];
    bool close = true;
    for (int k = 1; k < P; k++) close = lean_delta_pose(poses[k], poses[0], Q[k]) && close;
    gated += close ? 1 : 0;
    for (long long i = b0; i < std::min(n_points, b0 + per_batch); i++) {
      // directions: anywhere on the sphere; every 8th near a pole, every 8th near the seam (camera frame x ~ 0, z < 0)
      double d[3] = {U(rng), U(rng), U(rng)};
      if (i % 8 == 1) d[0] *= 1e-3, d[2] *= 1e-3;
      if (i % 8 == 2) d[0] *= std::pow(10.0, -2.0 - 4.0 * std::fabs(U(rng))), d[2] = -std::fabs(d[2]);
      const double nd = std::sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
      const double range = 0.3 + 40.0 * std::fabs(U(rng)) * std::fabs(U(rng));
      // camera frame of pose 0 -> lidar frame
      const double pc[3] = {range * d[0] / nd - poses[0][3], range * d[1] / nd - poses[0][7], range * d[2] / nd - poses[0][11]};
      double pl[3];
      for (int c = 0; c < 3; c++) pl[c] = poses[0][c] * pc[0] + poses[0][4 + c] * pc[1] + poses[0][8 + c] * pc[2];
      float x = static_cast<float>(pl[0]), y = static_cast<float>(pl[1]), z = static_cast<float>(pl[2]);
      if ((i & 1) == 0) {
        // nudge u (or v) to within 1e-3 .. 1e-8 px of an integer at a random pose k >= 1
        const int k = 1 + static_cast<int>(std::fabs(U(rng)) * (P - 1)) % (P - 1);
        const bool along_v = (i & 2) != 0;
        double u0, v0, u1, v1;
        exact_pixel_hd<CAM_EQUIRECTANGULAR>(cam, -2.0, 1 << 30, 1 << 30, poses[k], x, y, z, &u0, &v0);
        const double c0 = along_v ? v0 : u0;
        if (std::isfinite(c0)) {
          const double target = std::nearbyint(c0) + std::pow(10.0, -3.0 - 5.0 * std::fabs(U(rng))) * (U(rng) > 0 ? 1 : -1);
          float* coord = along_v ? &y : &x;
          const float h = 1e-3f * std::max(1.0f, std::fabs(*coord));
          const float keep = *coord;
          *coord = keep + h;
          exact_pixel_hd<CAM_EQUIRECTANGULAR>(cam, -2.0, 1 << 30, 1 << 30, poses[k], x, y, z, &u1, &v1);
          const double g = ((along_v ? v1 : u1) - c0) / h;
          *coord = keep;
          if (std::isfinite(g) && std::fabs(g) > 1e-3) *coord = static_cast<float>(keep + (target - c0) / g);
        }
      }
      const float delta = (5.25f * F32_U) * (std::fabs(x) + std::fabs(y) + std::fabs(z) + tmax_all);
      LeanAnchor an;
      for (int k = 0; k < P; k++) {
        const LeanVerdict v = k == 0 ? classify_lean_anchor<CAM_EQUIRECTANGULAR>(f, lc, W, p32[0], x, y, z, delta, an)
                                     : classify_lean_delta<CAM_EQUIRECTANGULAR>(lc, W, Q[k], x, y, z, delta, an);
        double ue, ve;
        const int pe = exact_pixel_hd<CAM_EQUIRECTANGULAR>(cam, cos_fov, W, H, poses[k], x, y, z, &ue, &ve);
        if (k == 0) {  // the anchor's verdict is the plain classifier's
          const LeanVerdict w = classify_lean<CAM_EQUIRECTANGULAR>(f, lc, W, p32[0], x, y, z, delta);
          if (w.accept != v.accept || w.uncertain != v.uncertain || (w.accept && w.idx != v.idx)) mism++;
          continue;
        }
        total++;
        plain_unc += classify_lean<CAM_EQUIRECTANGULAR>(f, lc, W, p32[k], x, y, z, delta).uncertain ? 1 : 0;
        if (v.uncertain) {
          unc++;
        } else if (v.accept) {
          acc++;
          if (v.idx != pe) mism++;
          else max_ratio = std::max(max_ratio, std::max(std::fabs(v.up - (ue - 0.5)) / (0.5 - v.hx), std::fabs(v.vp - (ve - 0.5)) / (0.5 - v.hy)));
        } else if (pe != -1) {
          mism++;
        }
      }
    }
  }
  out[0] = total, out[1] = unc, out[2] = mism, out[3] = acc, out[4] = static_cast<long long>(max_ratio * 1e6), out[5] = gated, out[6] = lc.enabled, out[7] = plain_unc;
}

int main(int argc, char** argv) {
  const long long n = argc > 1 ? std::atoll(argv[1]) : 200000;
  struct {
    int W, H;
    double fov;
  } cases[] = {{3840, 1920, M_PI}, {1024, 512, M_PI}, {3840, 1920, 1.9}};
  std::printf("[");
  int k = 0;
  for (const auto& c : cases) {
    long long out[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    run_case(c.W, c.H, c.fov, 300 + k, n, out);
    std::printf("%s{\"case\": %d, \"enabled\": %lld, \"point_poses\": %lld, \"uncertain\": %lld, \"mismatches\": %lld, \"accepted\": %lld, \"max_error_over_bound_ppm\": %lld, \"batches_in_gate\": %lld, \"plain_uncertain\": %lld}",
                k ? ", " : "", k, out[6], out[0], out[1], out[2], out[3], out[4], out[5], out[7]);
    k++;
  }
  std::printf("]\n");
  return 0;
}
