// nm_machine.cuh -- dfo::NelderMead<N> (reference: include/dfo/nelder_mead.hpp:32-113) as a resumable state machine.
//
// The host solver loop (host_math.hpp) steps it; the persistent kernel (nid_persistent.cuh) keeps its solver state in the
// same struct and steps it with a warp-parallel twin of step().  Decisions are those of the serial reference, evaluation
// for evaluation:
//   - libstdc++'s insertion-sort order for std::sort on <= 16 elements (ties and NaNs land where the reference puts them)
//   - the centroid xo is requested although its value is never used in a decision (:58): it is counted as a reference
//     evaluation always, but scored only when its value can be observed (begin(): score_centroid)
//   - the "contraction" point lies on the reflected side, xo + rho (xo - worst) (:75)
//   - the shrink step uses rho, not sigma (:82)
//   - convergence = sum over the N coordinates of sum_k (x_k - mean)^2 < threshold, no 1/n (:105-113)
//   - the result is x[0] as of the last sort (:99-100), num_iterations the last loop index (:50)
// {xo, xr, xe, xc} are affine in the sorted simplex, so they are known before any is scored: one batch per iteration
// (N+1 for the initial simplex, N for a shrink); only the values the reference would have requested are consumed, and
// `obs_*` lists them in the reference's order so that the objective's side effects can be replayed.  An iteration batch
// is cand = {xr, xe, xc, xo}: 4 poses when the caller observes the objective's side effects (a best-cost callback, a
// recorded trace, ranks that must issue equal batches), else 3 -- xo's value then reaches nobody, so it is not scored,
// and its entry is left out of `obs_*`.  Every score depends on its own pose alone, so both give the same trajectory.
// All arithmetic goes through exact_math.cuh (no FMA contraction on either side).
#pragma once

#include "exact_math.cuh"

namespace vlcal {

constexpr int NM_MAX_N = 8;

struct NmParams {  // nelder_mead.hpp:11-22
  double init_step = 0.1;
  double alpha = 1.0;
  double gamma = 2.0;
  double rho = 0.5;
  double sigma = 0.5;  // unused by the reference
  int max_iterations = 1024;
  double convergence_var_thresh = 1e-5;
};

struct NmMachine {
  // configuration
  int n;
  int score_centroid;  // iteration batches score xo too (4 poses instead of 3)
  NmParams params;
  // state
  int phase;      // 0 initial simplex pending, 1 iteration batch pending, 2 shrink batch pending, 3 finished
  int it;         // loop index of nelder_mead.hpp:49
  int converged;
  int num_iterations;
  double x[NM_MAX_N + 1][NM_MAX_N + 1];     // simplex, VectorM layout: [k][0] value, [k][1..n] sample
  double cand[NM_MAX_N + 1][NM_MAX_N + 1];  // pending batch, same layout (value slot unused until scored)
  int n_cand;
  // bookkeeping
  int num_evaluations;           // evaluations the serial reference would have requested
  int num_batches;
  int num_evaluations_computed;  // speculative ones included
  // evaluations of the batch just consumed that the reference made, in its order
  int n_obs;
  double obs_x[NM_MAX_N + 1][NM_MAX_N];
  double obs_y[NM_MAX_N + 1];
  // result
  double result_x[NM_MAX_N];
  double result_y;

  VL_HD void observe(const double* vertex, double y) {
    for (int d = 0; d < n; d++) obs_x[n_obs][d] = vertex[1 + d];
    obs_y[n_obs] = y;
    n_obs++;
    num_evaluations++;
  }

  // :35-46 initial simplex -> first batch.  score_centroid_: whether the caller reads xo's value (through obs_*)
  VL_HD void begin(int n_, const NmParams& p, const double* x0, bool score_centroid_ = true) {
    n = n_;
    score_centroid = score_centroid_ ? 1 : 0;
    params = p;
    phase = 0, it = 0, converged = 0, num_iterations = 0;
    num_evaluations = num_batches = num_evaluations_computed = 0;
    n_obs = 0;
    result_y = 0.0;
    const int m = n + 1;
    for (int k = 0; k < m; k++) {
      cand[k][0] = 0.0;
      for (int d = 0; d < n; d++) cand[k][1 + d] = x0[d];
      if (k > 0) cand[k][k] = (xd(cand[k][k]) + xd(params.init_step)).v;
    }
    n_cand = m;
  }

  VL_HD void finish() {
    for (int d = 0; d < n; d++) result_x[d] = x[0][1 + d];  // :99
    result_y = x[0][0];                                      // :100
    n_cand = 0;
    phase = 3;
  }

  // top of the loop body (:49-61): sort, convergence test, next candidates
  VL_HD void loop_top() {
    const int m = n + 1;
    if (it >= params.max_iterations) {
      finish();
      return;
    }
    num_iterations = it;  // :50
    // :51 std::sort, libstdc++ insertion sort
    for (int i = 1; i < m; i++) {
      double val[NM_MAX_N + 1];
      for (int d = 0; d < m; d++) val[d] = x[i][d];
      if (val[0] < x[0][0]) {
        for (int j = i; j > 0; j--)
          for (int d = 0; d < m; d++) x[j][d] = x[j - 1][d];
        for (int d = 0; d < m; d++) x[0][d] = val[d];
      } else {
        int j = i;
        while (val[0] < x[j - 1][0]) {
          for (int d = 0; d < m; d++) x[j][d] = x[j - 1][d];
          j--;
        }
        for (int d = 0; d < m; d++) x[j][d] = val[d];
      }
    }
    {  // :52-55, :105-113
      double mean[NM_MAX_N + 1], var[NM_MAX_N + 1];
      for (int d = 0; d < m; d++) {
        xd s(0.0);
        for (int k = 0; k < m; k++) s = s + xd(x[k][d]);
        mean[d] = (s / xd(static_cast<double>(m))).v;
        var[d] = 0.0;
      }
      for (int k = 0; k < m; k++) {
        for (int d = 0; d < m; d++) {
          const xd e = xd(x[k][d]) - xd(mean[d]);
          var[d] = (xd(var[d]) + e * e).v;
        }
      }
      xd total(0.0);
      for (int d = 1; d < m; d++) total = total + xd(var[d]);
      if (total.v < params.convergence_var_thresh) {
        converged = 1;
        finish();
        return;
      }
    }
    // :57, :60, :66, :75  xo, xr, xe, xc -> cand = {xr, xe, xc, xo}
    for (int d = 0; d < m; d++) {
      xd s(0.0);
      for (int k = 0; k < n; k++) s = s + xd(x[k][d]);
      const xd xo = s / xd(static_cast<double>(n));
      const xd diff = xo - xd(x[n][d]);
      cand[0][d] = (xo + xd(params.alpha) * diff).v;
      cand[1][d] = (xo + xd(params.gamma) * diff).v;
      cand[2][d] = (xo + xd(params.rho) * diff).v;
      cand[3][d] = xo.v;
    }
    n_cand = score_centroid ? 4 : 3;
    phase = 1;
  }

  // consume the scores ys[0..n_cand) of the pending batch; afterwards either phase == 3 (finished) or cand/n_cand hold
  // the next batch.  obs_* list the evaluations the reference made out of this batch.
  VL_HD void step(const double* ys) {
    const int m = n + 1;
    n_obs = 0;
    num_batches++;
    num_evaluations_computed += n_cand;
    if (phase == 0) {
      for (int k = 0; k < m; k++) {
        for (int d = 0; d < m; d++) x[k][d] = cand[k][d];
        x[k][0] = ys[k];
        observe(x[k], ys[k]);
      }
      loop_top();
    } else if (phase == 1) {
      double* xr = cand[0];
      double* xe = cand[1];
      double* xc = cand[2];
      double* xo = cand[3];
      xr[0] = ys[0];
      if (score_centroid) {
        xo[0] = ys[3];
        observe(xo, xo[0]);  // :58 evaluated, value never used in a decision
      } else {
        num_evaluations++;  // :58 requested by the reference; nobody reads its value
      }
      observe(xr, xr[0]);  // :61
      bool shrink = false;
      if (x[0][0] <= xr[0] && xr[0] < x[n - 1][0]) {  // :63-64
        for (int d = 0; d < m; d++) x[n][d] = xr[d];
      } else if (xr[0] < x[0][0]) {  // :65-73 expansion
        xe[0] = ys[1];
        observe(xe, xe[0]);
        const double* pick = (xe[0] < xr[0]) ? xe : xr;
        for (int d = 0; d < m; d++) x[n][d] = pick[d];
      } else {  // :74-86
        xc[0] = ys[2];
        observe(xc, xc[0]);
        if (xc[0] < x[n][0]) {
          for (int d = 0; d < m; d++) x[n][d] = xc[d];
        } else {
          shrink = true;
          for (int j = 1; j < m; j++)
            for (int d = 0; d < m; d++) x[j][d] = (xd(x[0][d]) + xd(params.rho) * (xd(x[j][d]) - xd(x[0][d]))).v;  // :82 (rho)
          for (int j = 1; j < m; j++)
            for (int d = 0; d < m; d++) cand[j - 1][d] = x[j][d];
          n_cand = n;
          phase = 2;
        }
      }
      if (!shrink) {
        it++;
        loop_top();
      }
    } else if (phase == 2) {
      for (int j = 1; j < m; j++) {
        x[j][0] = ys[j - 1];
        observe(x[j], ys[j - 1]);
      }
      it++;
      loop_top();
    }
  }
};

}  // namespace vlcal
