// Host-compiled equirectangular lean classifier (csrc/lean_filter.cuh) on a real cloud: the share of point-poses it defers
// to the exact path, with the constants of this tree and with those of the looser bound it replaced (arctangent charge
// argv[3] turns, one ulp per FMA rounding; loose_constants), and the delta step anchored at pose 0 and at the pose
// lean_delta_anchor picks.  Driven by tools/lean_deferral_host.py, which writes the input file:
//   int32 W, H, n_points, n_batches; float32 xyz[n_points][3]; float64 rows[n_batches][4][12] (four nearby poses, e.g. a
//   Nelder-Mead iteration {xo, xr, xe, xc})
// Prints one JSON object: plain-classifier deferrals over every pose, mean E_u + E_v, and per anchor [pose 0, rule] the
// batches inside the gate, the delta-step deferrals over the three other poses and the deferrals over all four poses of
// those batches (the anchor's are the plain classifier's).
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
  long long plain_pp = 0, plain_unc[2] = {0, 0}, gated[2] = {0, 0};
  long long delta_pp[2] = {0, 0}, delta_unc[2][2] = {{0, 0}, {0, 0}}, pass_unc[2][2] = {{0, 0}, {0, 0}};  // [anchor][constants]
  double esum[2] = {0.0, 0.0};
  for (int b = 0; b < nb; b++) {
    const double* R = &rows[48 * static_cast<size_t>(b)];
    float P[4][12], Q[2][4][16];
    float tmax = 0.0f;
    for (int k = 0; k < 4; k++) {
      for (int r = 0; r < 3; r++) {
        for (int c = 0; c < 3; c++) P[k][3 * r + c] = static_cast<float>(R[12 * k + 4 * r + c]);
        P[k][9 + r] = static_cast<float>(R[12 * k + 4 * r + 3]);
        tmax = std::max(tmax, std::nextafter(std::fabs(P[k][9 + r]), INFINITY));
      }
    }
    const int anc[2] = {0, lean_delta_anchor(reinterpret_cast<const double(*)[12]>(R), 4)};
    bool close[2] = {true, true};
    for (int a = 0; a < 2; a++) {
      for (int k = 0; k < 4; k++)
        if (k != anc[a]) close[a] = lean_delta_pose(R + 12 * k, R + 12 * anc[a], Q[a][k]) && close[a];
      gated[a] += close[a] ? 1 : 0;
    }
    for (int i = b % stride; i < n; i += stride) {
      const float x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
      const float delta = (5.25f * F32_U) * (std::fabs(x) + std::fabs(y) + std::fabs(z) + tmax);
      for (int v = 0; v < 2; v++) {
        for (int k = 0; k < 4; k++) {
          const LeanVerdict w = classify_lean<CAM_EQUIRECTANGULAR>(f, lc[v], W, P[k], x, y, z, delta);
          plain_unc[v] += w.uncertain;
          if (v == 0) plain_pp++;
          if (w.accept) esum[v] += (0.5 - w.hx) + (0.5 - w.hy);
        }
        for (int a = 0; a < 2; a++) {
          if (!close[a]) continue;
          LeanAnchor an;
          pass_unc[a][v] += classify_lean_anchor<CAM_EQUIRECTANGULAR>(f, lc[v], W, P[anc[a]], x, y, z, delta, an).uncertain;
          for (int k = 0; k < 4; k++) {
            if (k == anc[a]) continue;
            const bool u = classify_lean_delta<CAM_EQUIRECTANGULAR>(lc[v], W, Q[a][k], x, y, z, delta, an).uncertain;
            delta_unc[a][v] += u, pass_unc[a][v] += u;
            if (v == 0) delta_pp[a]++;
          }
        }
      }
    }
  }
  // rates per [constants: this tree, loose]; delta entries per anchor [pose 0, lean_delta_anchor]
  auto rate = [](long long a, long long b) { return a / double(std::max(1LL, b)); };
  std::printf("{\"W\": %d, \"H\": %d, \"points\": %d, \"stride\": %d, \"batches\": %d, \"charged_this_tree\": %.4e, \"charged_loose\": %.4e, "
              "\"plain_point_poses\": %lld, \"plain_deferred\": [%lld, %lld], \"plain_rate\": [%.6f, %.6f], \"mean_Eu_plus_Ev_px\": [%.6e, %.6e], \"hx0\": [%.9g, %.9g], \"hy0\": [%.9g, %.9g]",
              W, H, n, stride, nb, LEAN_ATAN_ERR_TURNS, other, plain_pp, plain_unc[0], plain_unc[1], rate(plain_unc[0], plain_pp), rate(plain_unc[1], plain_pp),
              esum[0] / double(plain_pp - plain_unc[0]), esum[1] / double(plain_pp - plain_unc[1]), lc[0].hx0, lc[1].hx0, lc[0].hy0, lc[1].hy0);
  const char* names[2] = {"anchor_pose0", "anchor_rule"};
  for (int a = 0; a < 2; a++)
    std::printf(", \"%s\": {\"batches_in_gate\": %lld, \"delta_point_poses\": %lld, \"delta_deferred\": [%lld, %lld], \"delta_rate\": [%.6f, %.6f], \"pass_rate\": [%.6f, %.6f]}",
                names[a], gated[a], delta_pp[a], delta_unc[a][0], delta_unc[a][1], rate(delta_unc[a][0], delta_pp[a]), rate(delta_unc[a][1], delta_pp[a]),
                rate(pass_unc[a][0], delta_pp[a] * 4 / 3), rate(pass_unc[a][1], delta_pp[a] * 4 / 3));
  std::printf("}\n");
  return 0;
}
