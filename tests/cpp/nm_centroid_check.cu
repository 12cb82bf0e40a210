// CPU check of the centroid elision of the Nelder-Mead state machine (csrc/nm_machine.cuh): the same solve stepped with
// the centroid xo scored (score_centroid = true, the reference's batch {xo, xr, xe, xc}) and without it ({xr, xe, xc})
// must reach the same simplex, the same result and the same counters, save the poses scored, and the evaluations the
// machine reports must be the scored run's with every centroid left out.  Objectives: quadratic, Rosenbrock, a plateau
// of exact ties, a NaN region, a constant; n = 2 and n = 6, several starts and iteration limits.  Prints one JSON object
// per case.  Built host-only by tests/test_nm_centroid_host.py.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

#include "nm_machine.cuh"

using namespace vlcal;

static double objective(int kind, const double* x, int n) {
  double q = 0.0;
  for (int d = 0; d < n; d++) q += (d + 1.0) * (x[d] - 0.3 * (d % 3) + 0.1) * (x[d] - 0.3 * (d % 3) + 0.1);
  switch (kind) {
    case 0:  // quadratic
      return q;
    case 1: {  // Rosenbrock
      double s = 0.0;
      for (int d = 0; d + 1 < n; d++) s += 100.0 * (x[d + 1] - x[d] * x[d]) * (x[d + 1] - x[d] * x[d]) + (1.0 - x[d]) * (1.0 - x[d]);
      return s;
    }
    case 2:  // plateaus: exact ties between vertices
      return std::floor(q * 8.0) / 8.0;
    case 3:  // NaN region on one side of a plane the simplex crosses
      return x[0] + 0.5 * x[n - 1] > 0.02 ? NAN : q;
    default:  // constant: every comparison ties
      return 1.0;
  }
}

struct Run {
  NmMachine nm;
  int iteration_batches = 0;
  std::vector<double> obs;  // (x[0..n), y) per reported evaluation
  std::vector<double> obs_without_centroid;
};

static Run solve(int kind, int n, const double* x0, const NmParams& p, bool score_centroid) {
  Run r;
  r.nm.begin(n, p, x0, score_centroid);
  double ys[NM_MAX_N + 1];
  while (r.nm.phase != 3) {
    const bool iteration = r.nm.phase == 1;
    r.iteration_batches += iteration ? 1 : 0;
    for (int k = 0; k < r.nm.n_cand; k++) ys[k] = objective(kind, &r.nm.cand[k][1], n);
    r.nm.step(ys);
    for (int k = 0; k < r.nm.n_obs; k++) {
      for (int d = 0; d < n; d++) r.obs.push_back(r.nm.obs_x[k][d]);
      r.obs.push_back(r.nm.obs_y[k]);
      if (iteration && k == 0) continue;  // the centroid is the first evaluation the reference makes of an iteration
      for (int d = 0; d < n; d++) r.obs_without_centroid.push_back(r.nm.obs_x[k][d]);
      r.obs_without_centroid.push_back(r.nm.obs_y[k]);
    }
  }
  return r;
}

static bool same_bits(const void* a, const void* b, size_t bytes) {
  return std::memcmp(a, b, bytes) == 0;
}

int main() {
  const char* names[] = {"quadratic", "rosenbrock", "plateau", "nan_region", "constant"};
  const int limits[] = {1024, 7, 1, 0};
  std::printf("[\n");
  bool first = true;
  for (int kind = 0; kind < 5; kind++) {
    for (int n : {2, 6}) {
      for (int start = 0; start < 3; start++) {
        for (int limit : limits) {
          double x0[NM_MAX_N];
          for (int d = 0; d < n; d++) x0[d] = 0.25 * start - 0.2 * d + 0.05 * (start * d % 3);
          NmParams p;
          p.init_step = start == 2 ? 1e-3 : 0.1;
          p.max_iterations = limit;
          p.convergence_var_thresh = kind == 1 ? 1e-12 : 1e-8;
          const Run on = solve(kind, n, x0, p, true);
          const Run off = solve(kind, n, x0, p, false);
          const bool same_x = same_bits(on.nm.result_x, off.nm.result_x, sizeof(double) * n);
          const bool same_y = same_bits(&on.nm.result_y, &off.nm.result_y, sizeof(double));
          bool same_simplex = true;  // the n + 1 live rows {value, sample}
          for (int k = 0; k <= n; k++) same_simplex = same_simplex && same_bits(on.nm.x[k], off.nm.x[k], sizeof(double) * (n + 1));
          const bool obs_match = on.obs_without_centroid.size() == off.obs.size() &&
                                 (off.obs.empty() || same_bits(on.obs_without_centroid.data(), off.obs.data(), sizeof(double) * off.obs.size()));
          std::printf("%s{\"objective\": \"%s\", \"n\": %d, \"start\": %d, \"max_iterations\": %d, \"same_x\": %d, \"same_y\": %d, \"same_simplex\": %d, "
                      "\"obs_match\": %d, \"converged\": [%d, %d], \"num_iterations\": [%d, %d], \"num_evaluations\": [%d, %d], \"num_batches\": [%d, %d], "
                      "\"computed\": [%d, %d], \"iteration_batches\": [%d, %d], \"reported\": [%zu, %zu]}",
                      first ? "" : ",\n", names[kind], n, start, limit, same_x, same_y, same_simplex, obs_match, on.nm.converged, off.nm.converged,
                      on.nm.num_iterations, off.nm.num_iterations, on.nm.num_evaluations, off.nm.num_evaluations, on.nm.num_batches, off.nm.num_batches,
                      on.nm.num_evaluations_computed, off.nm.num_evaluations_computed, on.iteration_batches, off.iteration_batches,
                      on.obs.size() / (n + 1), off.obs.size() / (n + 1));
          first = false;
        }
      }
    }
  }
  std::printf("\n]\n");
  return 0;
}
