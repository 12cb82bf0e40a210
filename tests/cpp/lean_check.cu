// CPU check of the lean fp32 classifier (csrc/lean_filter.cuh) against the exact double path (csrc/exact_classify.cuh):
// every verdict the filter keeps (accept at pixel i / reject) must be the exact path's; prints counts as JSON.
// Built host-only by tests/test_lean_filter_host.py (nvcc, no device code is run).
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

struct Case {
  int model;
  int W, H;
  double intr[5];
  double dist[8];
  int n_intr, n_dist;
};

static bool adversarial = true;

template <int MODEL>
static void run_case(const Case& cs, unsigned seed, long long n_points, int n_poses, double spread, long long out[7]) {
  CameraParams cam;
  std::memset(&cam, 0, sizeof(cam));
  cam.model = MODEL;
  cam.n_intr = cs.n_intr, cam.n_dist = cs.n_dist;
  for (int i = 0; i < cs.n_intr; i++) cam.intr[i] = cs.intr[i];
  for (int i = 0; i < cs.n_dist; i++) cam.dist[i] = cs.dist[i];
  // estimate_camera_fov without the CUDA TU: same three probes, brute-force direction search is overkill here; use
  // the angle of the farthest of the three probe pixels through a numeric inversion of the exact projection
  double max_fov = 0.0;
  {
    const double probes[3][2] = {{0.0, 0.0}, {double(cs.W / 2), 0.0}, {0.0, double(cs.H / 2)}};
    for (auto& pr : probes) {
      double best = 1e300, best_fov = 0.0;
      for (int ia = -900; ia <= 900; ia++)
        for (int ib = -900; ib <= 900; ib += 1) {
          const double a = ia * (M_PI / 1800.0) * 1.0, b = ib * (M_PI / 1800.0) * 1.0;
          const double dir[3] = {std::sin(b), -std::sin(a) * std::cos(b), std::cos(a) * std::cos(b)};
          double u, v;
          project_exact_dyn(cam, dir[0], dir[1], dir[2], &u, &v);
          const double e = (u - pr[0]) * (u - pr[0]) + (v - pr[1]) * (v - pr[1]);
          if (e < best) best = e, best_fov = std::acos(dir[2]);
        }
      if (best_fov > max_fov) max_fov = best_fov;
    }
  }
  const FastCam f = make_fast_cam(cam, cs.W, cs.H, max_fov);
  const LeanCam lc = make_lean_cam(cam, f, cs.W, cs.H, max_fov);
  out[5] = lc.enabled;
  if (!lc.enabled) return;
  const double cos_fov = std::cos(max_fov);
  std::mt19937_64 rng(seed);
  std::uniform_real_distribution<double> U(-1.0, 1.0);
  // poses: small perturbations of identity-ish camera looking along +z of the lidar frame
  std::vector<double> poses(12 * n_poses);
  std::vector<float> poses32(16 * n_poses);
  float tmax_all = 0.f;
  for (int p = 0; p < n_poses; p++) {
    const double xi[6] = {0.05 * U(rng), 0.05 * U(rng), 0.05 * U(rng), 0.3 * U(rng), 0.3 * U(rng), 0.3 * U(rng)};
    double T[16];
    host::se3_expmap_gtsam(xi, T);
    double tm = 0.0;
    for (int r = 0; r < 3; r++) {
      for (int c = 0; c < 4; c++) poses[12 * p + 4 * r + c] = T[r + 4 * c];
      for (int c = 0; c < 3; c++) poses32[16 * p + 3 * r + c] = static_cast<float>(T[r + 4 * c]);
      poses32[16 * p + 9 + r] = static_cast<float>(T[r + 12]);
      tm = std::max(tm, std::fabs(T[r + 12]));
    }
    poses32[16 * p + 12] = std::nextafter(static_cast<float>(tm), INFINITY);
    tmax_all = std::max(tmax_all, poses32[16 * p + 12]);
  }
  long long total = 0, unc = 0, mism = 0, acc = 0, strip = 0;
  double max_ratio = 0.0;
  for (long long i = 0; i < n_points; i++) {
    // a direction inside a cone a bit wider than the FoV (so that FoV / border rejects occur), random range;
    // every 4th point is nudged so that its u (or v) lands within 1e-3 .. 1e-8 px of an integer at pose 0
    const double ang = spread * max_fov * std::sqrt(std::fabs(U(rng))), az = M_PI * U(rng);
    const double range = 0.5 + 30.0 * std::fabs(U(rng));
    double d[3] = {std::sin(ang) * std::cos(az), std::sin(ang) * std::sin(az), std::cos(ang)};
    float x = static_cast<float>(range * d[0]), y = static_cast<float>(range * d[1]), z = static_cast<float>(range * d[2]);
    if (adversarial && (i & 3) == 0) {
      double u0, v0;
      const int px = exact_pixel_hd<MODEL>(cam, -2.0, 1 << 30, 1 << 30, &poses[0], x, y, z, &u0, &v0);
      if (px >= 0 || std::isfinite(u0)) {
        const double target = std::nearbyint(u0) + std::pow(10.0, -3.0 - 5.0 * std::fabs(U(rng))) * (U(rng) > 0 ? 1 : -1);
        // du/dx ~ (u(x + h) - u(x)) / h
        double u1, v1;
        const float h = 1e-3f * std::max(1.0f, std::fabs(x));
        exact_pixel_hd<MODEL>(cam, -2.0, 1 << 30, 1 << 30, &poses[0], x + h, y, z, &u1, &v1);
        const double g = (u1 - u0) / h;
        if (std::isfinite(g) && std::fabs(g) > 1e-3) x = static_cast<float>(x + (target - u0) / g);
      }
    }
    const float a_p = std::fabs(x) + std::fabs(y) + std::fabs(z);
    const float delta = (5.25f * F32_U) * (a_p + tmax_all);
    for (int p = 0; p < n_poses; p++) {
      const LeanVerdict v = classify_lean<MODEL>(f, lc, cs.W, &poses32[16 * p], x, y, z, delta);
      double ue, ve;
      const int pe = exact_pixel_hd<MODEL>(cam, cos_fov, cs.W, cs.H, &poses[12 * p], x, y, z, &ue, &ve);
      total++;
      if (v.uncertain) {
        unc++;
      } else if (v.accept) {
        acc++;
        if (v.idx != pe) mism++;
        else max_ratio = std::max(max_ratio, std::max(std::fabs(v.up - (ue - 0.5)) / (0.5 - v.hx), std::fabs(v.vp - (ve - 0.5)) / (0.5 - v.hy)));
        if (pe >= 0 && (ue < 0.0 || ve < 0.0)) strip++;
      } else if (pe != -1) {
        mism++;
      }
    }
  }
  out[0] = total, out[1] = unc, out[2] = mism, out[3] = acc, out[4] = strip, out[6] = static_cast<long long>(max_ratio * 1e6);
}

// Cone mode: points at angle max_fov (1 +- 10^[-12, -3]) from the optical axis, i.e. inside (and just outside) the
// uncertain band of the FoV decision (cost_calculator_nid.cpp:32), at an explicit max_fov.  Four poses with small random
// rotations and translations within +-tscale (0.3 m as in run_case; 30 or 300 m for a camera that stands far from the
// LiDAR origin, as in a map frame, where the max|t| term of delta is a large part of the bound): the fp32 transform then
// carries the rounding error the delta terms of the FoV margins bound (a pure translation would leave the camera-frame
// point nearly exact).  Point i is placed on the cone at pose i % 4 and classified there.
template <int MODEL>
static void run_cone(const Case& cs, double fov, unsigned seed, long long n_points, double tscale, long long out[5]) {
  CameraParams cam;
  std::memset(&cam, 0, sizeof(cam));
  cam.model = MODEL;
  cam.n_intr = cs.n_intr, cam.n_dist = cs.n_dist;
  for (int i = 0; i < cs.n_intr; i++) cam.intr[i] = cs.intr[i];
  for (int i = 0; i < cs.n_dist; i++) cam.dist[i] = cs.dist[i];
  const FastCam f = make_fast_cam(cam, cs.W, cs.H, fov);
  const LeanCam lc = make_lean_cam(cam, f, cs.W, cs.H, fov);
  out[4] = lc.enabled;
  if (!lc.enabled) return;
  const double cos_fov = std::cos(fov);
  std::mt19937_64 rng(seed);
  std::uniform_real_distribution<double> U(0.0, 1.0);
  constexpr int n_poses = 4;
  double poses[12 * n_poses];
  float poses32[16 * n_poses];
  float tmax_all = 0.f;
  for (int p = 0; p < n_poses; p++) {
    const double xi[6] = {0.05 * (2 * U(rng) - 1), 0.05 * (2 * U(rng) - 1), 0.05 * (2 * U(rng) - 1), tscale * (2 * U(rng) - 1), tscale * (2 * U(rng) - 1), tscale * (2 * U(rng) - 1)};
    double T[16];
    host::se3_expmap_gtsam(xi, T);
    double tm = 0.0;
    for (int r = 0; r < 3; r++) {
      for (int c = 0; c < 4; c++) poses[12 * p + 4 * r + c] = T[r + 4 * c];
      for (int c = 0; c < 3; c++) poses32[16 * p + 3 * r + c] = static_cast<float>(T[r + 4 * c]);
      poses32[16 * p + 9 + r] = static_cast<float>(T[r + 12]);
      tm = std::max(tm, std::fabs(T[r + 12]));
    }
    poses32[16 * p + 12] = std::nextafter(static_cast<float>(tm), INFINITY);
    tmax_all = std::max(tmax_all, poses32[16 * p + 12]);
  }
  long long unc = 0, mism = 0, inimg = 0;
  for (long long i = 0; i < n_points; i++) {
    const int p = static_cast<int>(i % n_poses);
    const double* P = &poses[12 * p];
    const double eps = std::pow(10.0, -12.0 + 9.0 * U(rng)) * (U(rng) < 0.5 ? -1 : 1);
    const double a = fov * (1.0 + eps), az = 2 * M_PI * U(rng), range = 0.5 + 30 * U(rng);
    // camera-frame point at angle a, moved to the cloud frame: R^T (pc - t)
    const double pc[3] = {range * std::sin(a) * std::cos(az) - P[3], range * std::sin(a) * std::sin(az) - P[7], range * std::cos(a) - P[11]};
    const float x = float(P[0] * pc[0] + P[4] * pc[1] + P[8] * pc[2]);
    const float y = float(P[1] * pc[0] + P[5] * pc[1] + P[9] * pc[2]);
    const float z = float(P[2] * pc[0] + P[6] * pc[1] + P[10] * pc[2]);
    const float delta = (5.25f * F32_U) * (std::fabs(x) + std::fabs(y) + std::fabs(z) + tmax_all);
    const LeanVerdict v = classify_lean<MODEL>(f, lc, cs.W, &poses32[16 * p], x, y, z, delta);
    double ue, ve;
    const int pe = exact_pixel_hd<MODEL>(cam, cos_fov, cs.W, cs.H, P, x, y, z, &ue, &ve);
    if (exact_pixel_hd<MODEL>(cam, -2.0, cs.W, cs.H, P, x, y, z, &ue, &ve) >= 0) inimg++;  // the FoV test left out
    if (v.uncertain) unc++;
    else if (v.accept ? v.idx != pe : pe != -1) mism++;
  }
  out[0] = n_points, out[1] = unc, out[2] = mism, out[3] = inimg;
}

static int cone_mode(long long n, double tscale) {
  const Case pb = {CAM_PLUMB_BOB, 640, 480, {400, 410, 320, 240, 0}, {-0.04, 0.08, 1e-4, -3e-4, -0.04, 0, 0, 0}, 4, 5};
  const Case pb0 = {CAM_PLUMB_BOB, 640, 480, {400, 410, 320, 240, 0}, {0, 0, 0, 0, 0, 0, 0, 0}, 4, 5};
  const Case at = {CAM_ATAN, 640, 480, {400, 400, 320, 240, 0}, {0.9, 0, 0, 0, 0, 0, 0, 0}, 4, 1};
  const Case rp = {CAM_RATIONAL_POLYNOMIAL, 640, 480, {400, 410, 320, 240, 0}, {-0.04, 0.08, 1e-4, -3e-4, -0.04, 0.01, 0.02, -0.005}, 4, 8};
  const Case fe = {CAM_FISHEYE, 640, 480, {300, 300, 320, 240, 0}, {0.01, -0.02, 0.003, -0.001, 0, 0, 0, 0}, 4, 4};
  const Case om = {CAM_OMNIDIR, 640, 480, {300, 300, 320, 240, 1.1}, {-0.1, 0.02, 1e-3, -2e-3, 0, 0, 0, 0}, 5, 4};
  const Case eq = {CAM_EQUIRECTANGULAR, 640, 320, {640, 320, 0, 0, 0}, {0, 0, 0, 0, 0, 0, 0, 0}, 2, 0};
  struct ConeCase {
    const Case* cs;
    double fov;
  };
  // pinhole-type models below their enable threshold cos(max_fov) >= 0.05; the others also beyond 90 degrees
  const ConeCase cases[] = {{&pb, 0.3}, {&pb, 0.6}, {&pb0, 0.6}, {&at, 0.3}, {&at, 0.6}, {&rp, 0.3}, {&rp, 0.6},
                            {&fe, 0.5}, {&fe, 0.9}, {&fe, 2.1}, {&om, 0.5}, {&om, 1.2}, {&om, 1.9}, {&eq, 0.5}, {&eq, 1.0}, {&eq, 2.2}};
  std::printf("[");
  int k = 0;
  for (const ConeCase& cc : cases) {
    long long out[5] = {0, 0, 0, 0, 0};
    const unsigned seed = 300 + k;
    switch (cc.cs->model) {
      case CAM_PLUMB_BOB: run_cone<CAM_PLUMB_BOB>(*cc.cs, cc.fov, seed, n, tscale, out); break;
      case CAM_FISHEYE: run_cone<CAM_FISHEYE>(*cc.cs, cc.fov, seed, n, tscale, out); break;
      case CAM_ATAN: run_cone<CAM_ATAN>(*cc.cs, cc.fov, seed, n, tscale, out); break;
      case CAM_OMNIDIR: run_cone<CAM_OMNIDIR>(*cc.cs, cc.fov, seed, n, tscale, out); break;
      case CAM_EQUIRECTANGULAR: run_cone<CAM_EQUIRECTANGULAR>(*cc.cs, cc.fov, seed, n, tscale, out); break;
      default: run_cone<CAM_RATIONAL_POLYNOMIAL>(*cc.cs, cc.fov, seed, n, tscale, out); break;
    }
    std::printf("%s{\"case\": %d, \"model\": %d, \"max_fov\": %.3f, \"translation\": %g, \"enabled\": %lld, \"points\": %lld, \"uncertain\": %lld, \"mismatches\": %lld, \"in_image_without_fov\": %lld}",
                k ? ", " : "", k, cc.cs->model, cc.fov, tscale, out[4], out[0], out[1], out[2], out[3]);
    k++;
  }
  std::printf("]\n");
  return 0;
}

// argv: [points per case] [mode: 1 edge-adversarial (default), 0 random, 2 FoV cone] [cone mode: translation scale, m]
int main(int argc, char** argv) {
  const long long n = argc > 1 ? std::atoll(argv[1]) : 200000;
  if (argc > 2 && std::atoi(argv[2]) == 2) return cone_mode(n, argc > 3 ? std::atof(argv[3]) : 0.3);
  adversarial = !(argc > 2 && std::atoi(argv[2]) == 0);
  const Case cases[] = {
    // C2 camera (plumb_bob 1920x1080, f = 1000)
    {CAM_PLUMB_BOB, 1920, 1080, {1000, 1000, 960, 540, 0}, {-0.04, 0.08, 1e-4, -3e-4, -0.04, 0, 0, 0}, 4, 5},
    // C1 camera (640x480, f = 400)
    {CAM_PLUMB_BOB, 640, 480, {400, 400, 320, 240, 0}, {-0.04, 0.08, 1e-4, -3e-4, -0.04, 0, 0, 0}, 4, 5},
    // off-centre principal point, stronger distortion, non-square pixels
    {CAM_PLUMB_BOB, 1280, 720, {700, 820, 500.3, 410.7, 0}, {-0.25, 0.12, 2e-3, -1e-3, -0.02, 0, 0, 0}, 4, 5},
    // no distortion, tiny image (borders dominate)
    {CAM_PLUMB_BOB, 64, 48, {50, 50, 31.5, 23.5, 0}, {0, 0, 0, 0, 0, 0, 0, 0}, 4, 5},
    {CAM_FISHEYE, 1280, 960, {380, 380, 640, 480, 0}, {-0.01, 0.005, -0.002, 0.0005, 0, 0, 0, 0}, 4, 4},
    {CAM_ATAN, 1280, 960, {500, 500, 640, 480, 0}, {0.9, 0, 0, 0, 0, 0, 0, 0}, 4, 1},
    {CAM_OMNIDIR, 1280, 960, {600, 600, 640, 480, 1.2}, {-0.1, 0.02, 1e-3, -1e-3, 0, 0, 0, 0}, 5, 4},
    {CAM_EQUIRECTANGULAR, 3840, 1920, {3840, 1920, 0, 0, 0}, {0, 0, 0, 0, 0, 0, 0, 0}, 2, 0},
    {CAM_RATIONAL_POLYNOMIAL, 1920, 1080, {1000, 1000, 960, 540, 0}, {0.1, -0.05, 1e-4, -3e-4, 0.01, 0.12, -0.04, 0.008}, 4, 8},
  };
  std::printf("[");
  int k = 0;
  for (const Case& cs : cases) {
    long long out[7] = {0, 0, 0, 0, 0, 0, 0};
    switch (cs.model) {
      case CAM_PLUMB_BOB: run_case<CAM_PLUMB_BOB>(cs, 100 + k, n, 4, 1.15, out); break;
      case CAM_FISHEYE: run_case<CAM_FISHEYE>(cs, 100 + k, n, 4, 1.1, out); break;
      case CAM_ATAN: run_case<CAM_ATAN>(cs, 100 + k, n, 4, 1.1, out); break;
      case CAM_OMNIDIR: run_case<CAM_OMNIDIR>(cs, 100 + k, n, 4, 1.1, out); break;
      case CAM_EQUIRECTANGULAR: run_case<CAM_EQUIRECTANGULAR>(cs, 100 + k, n, 4, 1.0, out); break;
      default: run_case<CAM_RATIONAL_POLYNOMIAL>(cs, 100 + k, n, 4, 1.1, out); break;
    }
    std::printf("%s{\"case\": %d, \"model\": %d, \"enabled\": %lld, \"point_poses\": %lld, \"uncertain\": %lld, \"mismatches\": %lld, \"accepted\": %lld, \"accepted_in_minus_one_strip\": %lld, \"max_error_over_bound_ppm\": %lld}", k ? ", " : "", k, cs.model,
                out[5], out[0], out[1], out[2], out[3], out[4], out[6]);
    k++;
  }
  std::printf("]\n");
  return 0;
}
