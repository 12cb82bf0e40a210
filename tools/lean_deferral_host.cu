// Host-compiled equirectangular lean classifier (csrc/lean_filter.cuh) on a real cloud: the share of point-poses it defers
// to the exact path, with the constants of this tree and with those of the looser bound it replaced (arctangent charge
// argv[3] turns, one ulp per FMA rounding; loose_constants).  Driven by tools/lean_deferral_host.py, which writes the input file:
//   int32 W, H, n_points, n_batches; float32 xyz[n_points][3]; float64 rows[n_batches][4][12] (pose 0 = anchor, 1..3 close)
// Prints one JSON object: plain-classifier deferrals over every pose, delta-step deferrals over poses 1..3, mean E_u + E_v.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "fast_filter.hpp"

using namespace vlcal;

// the constants of the earlier, looser bound: the arctangent charged `err_turns` and the FMA roundings one ulp each,
// 2u (W + 1) for u', 2u (H + 1) for v' and 2u (1.03 W + 1), 2u (1.03 H + 1) for up0 + s in the delta step
static LeanCam loose_constants(const CameraParams& cam, LeanCam c, double err_turns) {
  constexpr double U = 5.9604644775390625e-08, SAFETY = 2.0;
  auto up = [](double v) { return std::nextafter(static_cast<float>(v), INFINITY); };
  auto dn = [](double v) { return std::nextafter(static_cast<float>(v), -INFINITY); };
  const double W = std::fabs(cam.intr[0]), H = std::fabs(cam.intr[1]);
  c.hx0 = dn(0.5 - SAFETY * (W * err_turns + 2.0 * U * (W + 1.0)));
  c.hy0 = dn(0.5 - SAFETY * (2.0 * H * err_turns + 2.0 * U * (H + 1.0)));
  c.eq_cu = up(SAFETY * (64.0 * U * W / (32.0 * M_PI) + 2.0 * U * (1.03 * W + 1.0)) + 1e-6);
  c.eq_cv = up(SAFETY * (64.0 * U * 2.0 * H / (32.0 * M_PI) + 2.0 * U * (1.03 * H + 1.0)) + 1e-6);
  c.eq_hxd = dn(static_cast<double>(c.hx0) - static_cast<double>(c.eq_cu));
  return c;
}

int main(int argc, char** argv) {
  if (argc < 4) {
    std::fprintf(stderr, "usage: %s input.bin stride other_err_turns\n", argv[0]);
    return 2;
  }
  FILE* fp = std::fopen(argv[1], "rb");
  if (!fp) return 2;
  const int stride = std::atoi(argv[2]);
  const double other = std::atof(argv[3]);
  int hdr[4];
  if (std::fread(hdr, sizeof(int), 4, fp) != 4) return 2;
  const int W = hdr[0], H = hdr[1], n = hdr[2], nb = hdr[3];
  std::vector<float> xyz(3 * static_cast<size_t>(n));
  std::vector<double> rows(48 * static_cast<size_t>(nb));
  if (std::fread(xyz.data(), sizeof(float), xyz.size(), fp) != xyz.size() || std::fread(rows.data(), sizeof(double), rows.size(), fp) != rows.size()) return 2;
  std::fclose(fp);
  CameraParams cam;
  std::memset(&cam, 0, sizeof(cam));
  cam.model = CAM_EQUIRECTANGULAR;
  cam.n_intr = 2;
  cam.intr[0] = W, cam.intr[1] = H;
  const FastCam f = make_fast_cam(cam, W, H, M_PI);
  const LeanCam lc[2] = {make_lean_cam(cam, f, W, H, M_PI), loose_constants(cam, make_lean_cam(cam, f, W, H, M_PI), other)};
  long long plain_pp = 0, delta_pp = 0, plain_unc[2] = {0, 0}, delta_unc[2] = {0, 0}, gated = 0;
  double esum[2] = {0.0, 0.0};
  for (int b = 0; b < nb; b++) {
    const double* R = &rows[48 * static_cast<size_t>(b)];
    float P[4][12], Q[4][16];
    float tmax = 0.0f;
    for (int k = 0; k < 4; k++) {
      for (int r = 0; r < 3; r++) {
        for (int c = 0; c < 3; c++) P[k][3 * r + c] = static_cast<float>(R[12 * k + 4 * r + c]);
        P[k][9 + r] = static_cast<float>(R[12 * k + 4 * r + 3]);
        tmax = std::max(tmax, std::nextafter(std::fabs(P[k][9 + r]), INFINITY));
      }
    }
    bool close = true;
    for (int k = 1; k < 4; k++) close = lean_delta_pose(R + 12 * k, R, Q[k]) && close;
    gated += close ? 1 : 0;
    for (int i = b % stride; i < n; i += stride) {
      const float x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
      const float delta = (5.25f * F32_U) * (std::fabs(x) + std::fabs(y) + std::fabs(z) + tmax);
      for (int v = 0; v < 2; v++) {
        LeanAnchor an;
        for (int k = 0; k < 4; k++) {
          const LeanVerdict w = classify_lean<CAM_EQUIRECTANGULAR>(f, lc[v], W, P[k], x, y, z, delta);
          plain_unc[v] += w.uncertain;
          if (v == 0) plain_pp++;
          if (w.accept) esum[v] += (0.5 - w.hx) + (0.5 - w.hy);
          if (!close) continue;
          if (k == 0) {
            classify_lean_anchor<CAM_EQUIRECTANGULAR>(f, lc[v], W, P[0], x, y, z, delta, an);
          } else {
            delta_unc[v] += classify_lean_delta<CAM_EQUIRECTANGULAR>(lc[v], W, Q[k], x, y, z, delta, an).uncertain;
            if (v == 0) delta_pp++;
          }
        }
      }
    }
  }
  std::printf("{\"W\": %d, \"H\": %d, \"points\": %d, \"stride\": %d, \"batches\": %d, \"batches_in_gate\": %lld, \"charged_this_tree\": %.4e, \"charged_loose\": %.4e, "
              "\"plain_point_poses\": %lld, \"plain_deferred\": [%lld, %lld], \"plain_rate\": [%.6f, %.6f], \"delta_point_poses\": %lld, \"delta_deferred\": [%lld, %lld], "
              "\"delta_rate\": [%.6f, %.6f], \"mean_Eu_plus_Ev_px\": [%.6e, %.6e], \"hx0\": [%.9g, %.9g], \"hy0\": [%.9g, %.9g]}\n",
              W, H, n, stride, nb, gated, LEAN_ATAN_ERR_TURNS, other, plain_pp, plain_unc[0], plain_unc[1], plain_unc[0] / double(plain_pp), plain_unc[1] / double(plain_pp), delta_pp,
              delta_unc[0], delta_unc[1], delta_unc[0] / double(std::max(1LL, delta_pp)), delta_unc[1] / double(std::max(1LL, delta_pp)), esum[0] / double(plain_pp - plain_unc[0]),
              esum[1] / double(plain_pp - plain_unc[1]), lc[0].hx0, lc[1].hx0, lc[0].hy0, lc[1].hy0);
  return 0;
}
