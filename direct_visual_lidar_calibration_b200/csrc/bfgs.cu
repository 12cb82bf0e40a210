// bfgs.cu -- host side of the reference's NID_BFGS branch (VisualCameraCalibration::estimate_pose_bfgs,
// src/vlcal/calib/visual_camera_calibration.cpp:187-238).
//
// The reference hands sum_bags NIDCost (MultiNIDCost, :141-173) to ceres::GradientProblemSolver with
// line_search_direction_type = BFGS on the Sophus::Manifold<SE3> (x (+) delta = x * exp(delta), :208-221).  Ceres is a
// third-party dependency that is neither in this image nor under /root/reference, so this is NOT a restatement of
// Ceres' code and its iterates are not expected to coincide with Ceres' (parity unpinned -- DESIGN.md); it is a
// Ceres-free quasi-Newton solver for the same problem with the same structure and Ceres' documented defaults:
//   * objective  : sum over bags of the mode-B NID, value + ambient gradient from K3 (vlcal_nid_evaluate_bspline_grad);
//                  an evaluation is invalid when any bag's functor returns false or the pose left the reference's trust
//                  region around the start pose (|dt| > 0.2 m or angle > 2 deg, :152-156)
//   * manifold   : tangent delta = (upsilon, omega); gradient pulled back with J = d(x * exp(delta))/d delta at 0
//   * direction  : dense BFGS on the inverse Hessian (6 x 6), H0 = I, steepest descent on the first iteration and after
//                  a failed update (s.y <= 0)
//   * line search: strong Wolfe (c1 = 1e-4, c2 = 0.9), bracketing with expansion <= 10x, zoom with safeguarded cubic
//                  interpolation, first trial step min(1, 1/|g|_inf), at most 20 trial steps
//   * stops      : max_num_iterations 50, function_tolerance 1e-6 (relative), gradient_tolerance 1e-10 (max norm),
//                  parameter_tolerance 1e-8
#include <algorithm>
#include <cmath>
#include <cstring>
#include <limits>
#include <vector>

#include "../../include/vlcal_nid.h"
#include "nid_context.cuh"

namespace vlcal {
namespace {

struct Pose7 {
  double v[7];  // qx qy qz qw tx ty tz (Sophus::SE3d storage)
};

void quat_to_R(const double* q, double R[3][3]) {
  const double x = q[0], y = q[1], z = q[2], w = q[3];
  R[0][0] = 1.0 - 2.0 * (y * y + z * z), R[0][1] = 2.0 * (x * y - z * w), R[0][2] = 2.0 * (x * z + y * w);
  R[1][0] = 2.0 * (x * y + z * w), R[1][1] = 1.0 - 2.0 * (x * x + z * z), R[1][2] = 2.0 * (y * z - x * w);
  R[2][0] = 2.0 * (x * z - y * w), R[2][1] = 2.0 * (y * z + x * w), R[2][2] = 1.0 - 2.0 * (x * x + y * y);
}

// rotation matrix -> unit quaternion (x y z w), largest-pivot branch selection
void R_to_quat(const double R[3][3], double* q) {
  const double tr = R[0][0] + R[1][1] + R[2][2];
  if (tr > 0.0) {
    const double s = std::sqrt(tr + 1.0) * 2.0;
    q[3] = 0.25 * s;
    q[0] = (R[2][1] - R[1][2]) / s, q[1] = (R[0][2] - R[2][0]) / s, q[2] = (R[1][0] - R[0][1]) / s;
  } else {
    int i = 0;
    if (R[1][1] > R[0][0]) i = 1;
    if (R[2][2] > R[i][i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    const double s = std::sqrt(R[i][i] - R[j][j] - R[k][k] + 1.0) * 2.0;
    q[i] = 0.25 * s;
    q[3] = (R[k][j] - R[j][k]) / s;
    q[j] = (R[j][i] + R[i][j]) / s;
    q[k] = (R[k][i] + R[i][k]) / s;
  }
  const double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  for (int c = 0; c < 4; c++) q[c] /= n;
}

Pose7 pose_from_colmajor(const double* T) {
  Pose7 p;
  double R[3][3];
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) R[r][c] = T[r + 4 * c];
  R_to_quat(R, p.v);
  for (int r = 0; r < 3; r++) p.v[4 + r] = T[r + 12];
  return p;
}

void pose_to_colmajor(const Pose7& p, double* T) {
  double R[3][3];
  quat_to_R(p.v, R);
  std::memset(T, 0, 16 * sizeof(double));
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) T[r + 4 * c] = R[r][c];
    T[r + 12] = p.v[4 + r];
  }
  T[15] = 1.0;
}

// x (+) delta = x * exp(delta), delta = (upsilon, omega)   (Sophus::Manifold<SE3>::Plus)
Pose7 pose_plus(const Pose7& x, const double* delta) {
  const double* up = delta;
  const double* om = delta + 3;
  const double th2 = om[0] * om[0] + om[1] * om[1] + om[2] * om[2];
  const double th = std::sqrt(th2);
  double b, c;  // (1 - cos th)/th^2, (th - sin th)/th^3
  if (th < 1e-5) {
    b = 0.5 - th2 / 24.0, c = 1.0 / 6.0 - th2 / 120.0;
  } else {
    b = (1.0 - std::cos(th)) / th2, c = (th - std::sin(th)) / (th2 * th);
  }
  // t_delta = V upsilon, V = I + b [om]x + c [om]x^2
  const double ox[3] = {om[1] * up[2] - om[2] * up[1], om[2] * up[0] - om[0] * up[2], om[0] * up[1] - om[1] * up[0]};
  const double oox[3] = {om[1] * ox[2] - om[2] * ox[1], om[2] * ox[0] - om[0] * ox[2], om[0] * ox[1] - om[1] * ox[0]};
  const double td[3] = {up[0] + b * ox[0] + c * oox[0], up[1] + b * ox[1] + c * oox[1], up[2] + b * ox[2] + c * oox[2]};
  // q_delta = (sin(th/2)/th om, cos(th/2))
  const double half = 0.5 * th;
  const double sh = th < 1e-5 ? 0.5 - th2 / 48.0 : std::sin(half) / th;
  const double qd[4] = {sh * om[0], sh * om[1], sh * om[2], std::cos(half)};
  const double* q = x.v;
  Pose7 out;
  out.v[0] = q[3] * qd[0] + q[0] * qd[3] + q[1] * qd[2] - q[2] * qd[1];
  out.v[1] = q[3] * qd[1] - q[0] * qd[2] + q[1] * qd[3] + q[2] * qd[0];
  out.v[2] = q[3] * qd[2] + q[0] * qd[1] - q[1] * qd[0] + q[2] * qd[3];
  out.v[3] = q[3] * qd[3] - q[0] * qd[0] - q[1] * qd[1] - q[2] * qd[2];
  const double n = std::sqrt(out.v[0] * out.v[0] + out.v[1] * out.v[1] + out.v[2] * out.v[2] + out.v[3] * out.v[3]);
  for (int k = 0; k < 4; k++) out.v[k] /= n;
  double R[3][3];
  quat_to_R(q, R);
  for (int r = 0; r < 3; r++) out.v[4 + r] = x.v[4 + r] + R[r][0] * td[0] + R[r][1] * td[1] + R[r][2] * td[2];
  return out;
}

// g6 = J^T g7 with J = d(x * exp(delta))/d delta at delta = 0:
//   d t / d upsilon = R(q),  d q / d omega_i = 1/2 q (x) (e_i, 0)
void pull_back_gradient(const Pose7& x, const double* g7, double* g6) {
  const double qx = x.v[0], qy = x.v[1], qz = x.v[2], qw = x.v[3];
  double R[3][3];
  quat_to_R(x.v, R);
  for (int i = 0; i < 3; i++) g6[i] = R[0][i] * g7[4] + R[1][i] * g7[5] + R[2][i] * g7[6];
  g6[3] = 0.5 * (qw * g7[0] + qz * g7[1] - qy * g7[2] - qx * g7[3]);
  g6[4] = 0.5 * (-qz * g7[0] + qw * g7[1] + qx * g7[2] - qy * g7[3]);
  g6[5] = 0.5 * (qy * g7[0] - qx * g7[1] + qw * g7[2] - qz * g7[3]);
}

// |translation|, rotation angle of init^-1 * x   (visual_camera_calibration.cpp:150-156)
void distance_from(const Pose7& init, const Pose7& x, double* dt, double* dr) {
  double Ri[3][3], Rx[3][3];
  quat_to_R(init.v, Ri);
  quat_to_R(x.v, Rx);
  const double d[3] = {x.v[4] - init.v[4], x.v[5] - init.v[5], x.v[6] - init.v[6]};
  double t[3];
  for (int i = 0; i < 3; i++) t[i] = Ri[0][i] * d[0] + Ri[1][i] * d[1] + Ri[2][i] * d[2];
  *dt = std::sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]);
  double tr = 0.0;  // trace(Ri^T Rx)
  for (int i = 0; i < 3; i++)
    for (int k = 0; k < 3; k++) tr += Ri[k][i] * Rx[k][i];
  const double cs = std::max(-1.0, std::min(1.0, 0.5 * (tr - 1.0)));
  *dr = std::acos(cs);
}

struct Sample {
  Pose7 x;
  double cost = std::numeric_limits<double>::infinity();
  double g[6] = {0, 0, 0, 0, 0, 0};
  bool valid = false;
};

using AmbientObjective = int (*)(const double x[7], double* cost, double grad7[7], void* user);

struct Solver {
  AmbientObjective f;
  void* user;
  vlcal_bfgs_params p;
  Pose7 init;
  int evaluations = 0;

  Sample eval(const Pose7& x) {
    Sample s;
    s.x = x;
    double dt, dr;
    distance_from(init, x, &dt, &dr);
    evaluations++;
    if (dt > p.max_translation_from_init || dr > p.max_rotation_from_init) return s;  // :152-156 -> false
    double g7[7], cost = 0.0;
    if (!f(x.v, &cost, g7, user) || !std::isfinite(cost)) return s;
    for (int k = 0; k < 7; k++)
      if (!std::isfinite(g7[k])) return s;
    s.cost = cost;
    pull_back_gradient(x, g7, s.g);
    s.valid = true;
    return s;
  }
};

double dot6(const double* a, const double* b) {
  double s = 0.0;
  for (int i = 0; i < 6; i++) s += a[i] * b[i];
  return s;
}

// minimiser of the cubic through (a, fa, ga) and (b, fb, gb), clamped into the middle 80 % of the interval
double cubic_step(double a, double fa, double ga, double b, double fb, double gb) {
  const double lo = std::min(a, b), hi = std::max(a, b);
  const double d1 = ga + gb - 3.0 * (fa - fb) / (a - b);
  const double rad = d1 * d1 - ga * gb;
  double t = 0.5 * (a + b);
  if (rad >= 0.0 && std::isfinite(rad)) {
    const double d2 = (b > a ? 1.0 : -1.0) * std::sqrt(rad);
    const double den = gb - ga + 2.0 * d2;
    if (den != 0.0) t = b - (b - a) * (gb + d2 - d1) / den;
  }
  const double margin = 0.1 * (hi - lo);
  if (!(t > lo + margin && t < hi - margin)) t = 0.5 * (lo + hi);
  return t;
}

}  // namespace
}  // namespace vlcal

using namespace vlcal;

extern "C" void vlcal_bfgs_default_params(vlcal_bfgs_params* p) {
  if (!p) return;
  p->max_num_iterations = 50;
  p->function_tolerance = 1e-6;
  p->gradient_tolerance = 1e-10;
  p->parameter_tolerance = 1e-8;
  p->sufficient_decrease = 1e-4;
  p->sufficient_curvature_decrease = 0.9;
  p->max_step_expansion = 10.0;
  p->max_line_search_steps = 20;
  p->max_translation_from_init = 0.2;                 // visual_camera_calibration.cpp:154
  p->max_rotation_from_init = 2.0 * M_PI / 180.0;     // :154
}

extern "C" int vlcal_bfgs_minimize_se3(
  vlcal_se3_objective objective, void* user, const vlcal_bfgs_params* params, const double init_T[16], vlcal_pose_callback callback, void* callback_user, double T_out[16],
  vlcal_bfgs_result* result) {
  if (!objective || !init_T || !T_out) {
    set_last_error("invalid arguments");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  Solver S;
  S.f = objective;
  S.user = user;
  if (params) {
    S.p = *params;
  } else {
    vlcal_bfgs_default_params(&S.p);
  }
  S.init = pose_from_colmajor(init_T);
  vlcal_bfgs_result res;
  std::memset(&res, 0, sizeof(res));

  Sample cur = S.eval(S.init);
  if (!cur.valid) {
    set_last_error("the objective cannot be evaluated at the initial pose");
    res.termination = VLCAL_BFGS_FAILURE;
    res.evaluations = S.evaluations;
    if (result) *result = res;
    std::memcpy(T_out, init_T, 16 * sizeof(double));
    return VLCAL_OK;
  }
  res.initial_cost = cur.cost;
  double H[6][6];
  auto reset_H = [&]() {
    for (int i = 0; i < 6; i++)
      for (int j = 0; j < 6; j++) H[i][j] = i == j ? 1.0 : 0.0;
  };
  reset_H();
  bool fresh = true;  // H is the identity: first trial step is scaled by the gradient
  double T[16];
  int it = 0;
  res.termination = VLCAL_BFGS_NO_CONVERGENCE;
  for (;; it++) {
    double gmax = 0.0;
    for (int i = 0; i < 6; i++) gmax = std::max(gmax, std::fabs(cur.g[i]));
    res.gradient_max_norm = gmax;
    if (gmax <= S.p.gradient_tolerance) {
      res.termination = VLCAL_BFGS_CONVERGED_GRADIENT;
      break;
    }
    if (it >= S.p.max_num_iterations) break;
    double d[6];
    for (int i = 0; i < 6; i++) {
      d[i] = 0.0;
      for (int j = 0; j < 6; j++) d[i] -= H[i][j] * cur.g[j];
    }
    double slope = dot6(d, cur.g);
    if (!(slope < 0.0)) {  // not a descent direction: restart from steepest descent
      reset_H();
      fresh = true;
      for (int i = 0; i < 6; i++) d[i] = -cur.g[i];
      slope = dot6(d, cur.g);
    }
    // ---- strong-Wolfe line search along x (+) (alpha d) ----
    auto phi = [&](double alpha) {
      double step[6];
      for (int i = 0; i < 6; i++) step[i] = alpha * d[i];
      return S.eval(pose_plus(cur.x, step));
    };
    const double c1 = S.p.sufficient_decrease, c2 = S.p.sufficient_curvature_decrease;
    double alpha = fresh ? std::min(1.0, 1.0 / gmax) : 1.0;
    double a_lo = 0.0, f_lo = cur.cost, g_lo = slope;
    double a_hi = 0.0, f_hi = 0.0, g_hi = 0.0;
    bool bracketed = false, accepted = false;
    Sample best;  // accepted trial
    double best_alpha = 0.0;
    double a_prev = 0.0, f_prev = cur.cost, g_prev = slope;
    for (int ls = 0; ls < S.p.max_line_search_steps; ls++) {
      Sample s = phi(alpha);
      if (!s.valid) {  // outside the trust region / invalid: treat as an upper bracket end with a large value
        if (!bracketed) {
          a_lo = a_prev, f_lo = f_prev, g_lo = g_prev;
          bracketed = true;
        }
        a_hi = alpha, f_hi = std::numeric_limits<double>::infinity(), g_hi = 0.0;
        alpha = 0.5 * (a_lo + a_hi);
        continue;
      }
      const double gs = dot6(s.g, d);
      if (!bracketed) {
        if (s.cost > cur.cost + c1 * alpha * slope || (ls > 0 && s.cost >= f_prev)) {
          a_lo = a_prev, f_lo = f_prev, g_lo = g_prev;
          a_hi = alpha, f_hi = s.cost, g_hi = gs;
          bracketed = true;
        } else if (std::fabs(gs) <= -c2 * slope) {
          best = s, best_alpha = alpha, accepted = true;
          break;
        } else if (gs >= 0.0) {
          a_lo = alpha, f_lo = s.cost, g_lo = gs;
          a_hi = a_prev, f_hi = f_prev, g_hi = g_prev;
          bracketed = true;
        } else {
          a_prev = alpha, f_prev = s.cost, g_prev = gs;
          best = s, best_alpha = alpha;  // sufficient decrease holds: keep as a fallback
          alpha = alpha * S.p.max_step_expansion;
          continue;
        }
      } else {  // zoom: [a_lo, a_hi] brackets a Wolfe point, a_lo satisfies sufficient decrease
        if (s.cost > cur.cost + c1 * alpha * slope || s.cost >= f_lo) {
          a_hi = alpha, f_hi = s.cost, g_hi = gs;
        } else {
          if (std::fabs(gs) <= -c2 * slope) {
            best = s, best_alpha = alpha, accepted = true;
            break;
          }
          if (gs * (a_hi - a_lo) >= 0.0) a_hi = a_lo, f_hi = f_lo, g_hi = g_lo;
          a_lo = alpha, f_lo = s.cost, g_lo = gs;
          best = s, best_alpha = alpha;
        }
      }
      if (std::fabs(a_hi - a_lo) < 1e-16 * std::max(1.0, std::fabs(a_lo))) break;
      alpha = std::isfinite(f_hi) ? cubic_step(a_lo, f_lo, g_lo, a_hi, f_hi, g_hi) : 0.5 * (a_lo + a_hi);
    }
    if (!accepted && !(best.valid && best.cost < cur.cost)) {
      if (!fresh) {  // the quasi-Newton direction failed: one retry from steepest descent
        reset_H();
        fresh = true;
        it--;
        res.line_search_restarts++;
        if (res.line_search_restarts > 5) {
          res.termination = VLCAL_BFGS_NO_CONVERGENCE;
          break;
        }
        continue;
      }
      res.termination = VLCAL_BFGS_LINE_SEARCH_FAILED;
      break;
    }
    // ---- BFGS update of the inverse Hessian with s = alpha d, y = g_new - g_old ----
    double sv[6], yv[6];
    for (int i = 0; i < 6; i++) sv[i] = best_alpha * d[i], yv[i] = best.g[i] - cur.g[i];
    const double sy = dot6(sv, yv);
    if (sy > 1e-14 * std::sqrt(dot6(sv, sv) * dot6(yv, yv))) {
      double Hy[6];
      for (int i = 0; i < 6; i++) {
        Hy[i] = 0.0;
        for (int j = 0; j < 6; j++) Hy[i] += H[i][j] * yv[j];
      }
      const double yHy = dot6(yv, Hy);
      const double rho = 1.0 / sy;
      for (int i = 0; i < 6; i++)
        for (int j = 0; j < 6; j++) H[i][j] += (1.0 + yHy * rho) * rho * sv[i] * sv[j] - rho * (Hy[i] * sv[j] + sv[i] * Hy[j]);
      fresh = false;
    } else {
      reset_H();
      fresh = true;
    }
    const double step_norm = std::sqrt(dot6(sv, sv));
    const double cost_change = cur.cost - best.cost;
    const double prev_cost = cur.cost;
    cur = best;
    res.iterations = it + 1;
    if (callback) {  // IterationCallbackWrapper with update_state_every_iteration (:219-226)
      pose_to_colmajor(cur.x, T);
      callback(T, cur.cost, callback_user);
    }
    double xnorm = 0.0;
    for (int k = 0; k < 7; k++) xnorm += cur.x.v[k] * cur.x.v[k];
    xnorm = std::sqrt(xnorm);
    if (step_norm <= S.p.parameter_tolerance * (xnorm + S.p.parameter_tolerance)) {
      res.termination = VLCAL_BFGS_CONVERGED_PARAMETER;
      it++;
      break;
    }
    if (std::fabs(cost_change) <= S.p.function_tolerance * std::fabs(prev_cost)) {
      res.termination = VLCAL_BFGS_CONVERGED_FUNCTION;
      it++;
      break;
    }
  }
  res.final_cost = cur.cost;
  res.evaluations = S.evaluations;
  double gmax = 0.0;
  for (int i = 0; i < 6; i++) gmax = std::max(gmax, std::fabs(cur.g[i]));
  res.gradient_max_norm = gmax;
  pose_to_colmajor(cur.x, T_out);
  if (result) *result = res;
  return VLCAL_OK;
}

namespace {
struct CtxObjective {
  vlcal_nid_ctx* const* ctxs;
  int n;
  int status;
  vlcal_allreduce_fn allreduce;  // optional: bags sharded over ranks (one process per GPU)
  void* allreduce_user;
};

int ctx_objective(const double x[7], double* cost, double grad7[7], void* user) {
  CtxObjective* o = static_cast<CtxObjective*>(user);
  double total = 0.0, g[7] = {0, 0, 0, 0, 0, 0, 0};
  bool all_ok = true;
  for (int b = 0; b < o->n; b++) {  // MultiNIDCost: residuals[0] += residuals[i] in bag order (:163-169)
    double nid = 0.0, gb[7];
    int32_t ok = 0;
    const int rc = o->status == VLCAL_OK ? vlcal_nid_evaluate_bspline_grad(o->ctxs[b], x, 1, &nid, gb, &ok) : o->status;
    if (rc != VLCAL_OK) {
      // a local failure must still reach the collective below (the other ranks are already waiting in it): record it,
      // report "invalid here" through the failed-bag count, and let every rank abort the solve consistently
      o->status = rc;
      all_ok = false;
      break;
    }
    all_ok = all_ok && ok != 0;
    total += nid;
    for (int k = 0; k < 7; k++) g[k] += gb[k];
  }
  if (o->allreduce) {  // sum_bags over all ranks: cost, 7 partials and the number of bags whose functor returned false
    double vals[9] = {total, g[0], g[1], g[2], g[3], g[4], g[5], g[6], all_ok ? 0.0 : 1.0};
    o->allreduce(vals, 9, o->allreduce_user);
    total = vals[0];
    for (int k = 0; k < 7; k++) g[k] = vals[1 + k];
    all_ok = vals[8] == 0.0;
  }
  *cost = total;
  for (int k = 0; k < 7; k++) grad7[k] = g[k];
  if (o->status != VLCAL_OK) return 0;
  return all_ok ? 1 : 0;
}
}  // namespace

extern "C" int vlcal_estimate_pose_bfgs_ctx(
  vlcal_nid_ctx* const* ctxs, int n_ctx, const vlcal_bfgs_params* params, const double init_T_camera_lidar[16], vlcal_pose_callback callback,
  vlcal_allreduce_fn allreduce, void* user, double T_out[16], vlcal_bfgs_result* result) {
  if (!ctxs || n_ctx <= 0 || !init_T_camera_lidar || !T_out) {
    set_last_error("invalid arguments");
    return VLCAL_ERR_INVALID_ARGUMENT;
  }
  for (int b = 0; b < n_ctx; b++) {
    if (!ctxs[b] || ctxs[b]->mode != VLCAL_NID_MODE_BSPLINE) {
      set_last_error("vlcal_estimate_pose_bfgs_ctx needs contexts created with VLCAL_NID_MODE_BSPLINE");
      return VLCAL_ERR_INVALID_ARGUMENT;
    }
  }
  CtxObjective o{ctxs, n_ctx, VLCAL_OK, allreduce, user};
  const int rc = vlcal_bfgs_minimize_se3(ctx_objective, &o, params, init_T_camera_lidar, callback, user, T_out, result);
  return o.status != VLCAL_OK ? o.status : rc;
}
