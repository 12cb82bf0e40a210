// CPU check of the anchor rule of the equirectangular delta step (csrc/lean_filter.cuh: lean_delta_anchor), built
// host-only.  Prints one JSON object: the anchor picked for a Nelder-Mead iteration {xo, xr, xe, xc}, for the initial
// simplex, for a batch of equal poses and for an 8-pose line whose central pose sits at index 3.
#include <cmath>
#include <cstdio>
#include <cstring>

#include "host_math.hpp"
#include "lean_filter.cuh"

using namespace vlcal;

// row-major 3x4 rows of T0 * Exp(xi)
static void pose_rows(const double T0[16], const double xi[6], double out[12]) {
  double E[16], T[16];
  host::se3_expmap_gtsam(xi, E);
  host::isometry_mul(T0, E, T);
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 4; c++) out[4 * r + c] = T[r + 4 * c];
}

int main() {
  const double xi0[6] = {0.3, -0.2, 0.1, 0.5, -1.0, 0.2};
  double T0[16];
  host::se3_expmap_gtsam(xi0, T0);
  const double dir[6] = {0.4e-3, -0.7e-3, 0.5e-3, 0.9e-3, 0.2e-3, -0.3e-3};
  auto line = [&](const double* s, int n, double (*rows)[12]) {
    for (int k = 0; k < n; k++) {
      double xi[6];
      for (int i = 0; i < 6; i++) xi[i] = s[k] * dir[i];
      pose_rows(T0, xi, rows[k]);
    }
  };
  double rows[8][12];
  const double iteration[4] = {0.0, 1.0, 2.0, 0.5};
  line(iteration, 4, rows);
  const int a_iter = lean_delta_anchor(rows, 4);
  for (int k = 0; k < 7; k++) {
    double xi[6] = {0, 0, 0, 0, 0, 0};
    if (k > 0) xi[k - 1] = 1e-3;
    pose_rows(T0, xi, rows[k]);
  }
  const int a_simplex = lean_delta_anchor(rows, 7);
  for (int k = 1; k < 5; k++) std::memcpy(rows[k], rows[0], sizeof(rows[0]));
  const int a_equal = lean_delta_anchor(rows, 5);
  const double central[8] = {-3.0, -2.0, -1.0, 0.0, 1.0, 2.0, 3.0, 0.5};
  line(central, 8, rows);
  const int a_central = lean_delta_anchor(rows, 8);
  std::printf("{\"iteration\": %d, \"simplex\": %d, \"equal\": %d, \"central\": %d, \"single\": %d}\n", a_iter, a_simplex, a_equal, a_central, lean_delta_anchor(rows, 1));
  return 0;
}
