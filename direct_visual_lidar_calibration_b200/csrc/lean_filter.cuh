// lean_filter.cuh -- second-generation fp32 filter of the NID hot loop (reference decisions:
// src/vlcal/calib/cost_calculator_nid.cpp:31-38): same contract as classify_fast (nid_kernels.cuh) -- a verdict is
// final only when it is provably the reference's, everything else is re-decided by the exact fp64 path -- but written
// for instruction count:
//
//   * rounding by the magic constant M = 1.5 * 2^23: t = u' + M holds rint(u') in its low mantissa bits for
//     |u'| < 2^22, so the pixel index, the distance to the pixel edge and the image-bounds test all come out of two
//     FADDs per axis on the FMA pipe -- no FRND / F2I (quarter-rate conversion pipe), no integer compare chain;
//     u' = u - 0.5 is produced directly by the intrinsics FMA (cx - 0.5 folded on the host), hence
//     floor(u) = rint(u') wherever u is farther than E from an integer, and the reference's truncation TOWARD ZERO
//     (u in (-1, 0) -> column 0, cost_calculator_nid.cpp:37) is the clamp max(rint(u'), 0) with the lower bound at -1;
//   * pinhole-type models decide the FoV cone (:32) from r^2 = x^2 + y^2 of the normalised point, which the
//     distortion polynomial needs anyway:  z/|p| >= cos(fov)  <=>  z > 0 and r^2 <= tan^2(fov).  No |p|, no rsqrt;
//   * the error bound E is the round-1 bound (fast_filter.hpp, camera_models.cuh:project_fast), e = L exy + M16 with
//     exy = rho (1 + mh) + 4u mh, multiplied out on the host into e = rho A(r2b) + B(r2b): two degree-4 Horner chains
//     and one FMA instead of five dependent polynomial / product steps (same value up to the upward rounding of the
//     coefficients, so soundness carries over);
//   * verdicts are three predicates (accept / uncertain / otherwise rejected) built from FSETP chains: no SEL / integer
//     verdict codes.
//
// Everything here is __host__ __device__ so that tests/cpp_lean_check.cu can run the classifier against the exact path
// on the CPU (division and sqrt stand in for MUFU.RCP / MUFU.RSQ there; both are within the 1-ulp the bounds assume).
#pragma once

#include <cstdint>

#include "camera_models.cuh"

namespace vlcal {

constexpr float LEAN_MAGIC = 12582912.0f;      // 1.5 * 2^23
constexpr int LEAN_MAGIC_BITS = 0x4B400000;    // bit pattern of LEAN_MAGIC; bits(M + k) = LEAN_MAGIC_BITS + k, |k| < 2^22

struct LeanCam {
  int enabled;            // 0: no lean classifier for this camera / FoV / image size (fall back to the round-1 filter)
  float cxh, cyh;         // cx - 0.5, cy - 0.5 (equirectangular: W/2 - 0.5, H/2 - 0.5)
  float t_lo, t_hi;       // bounds tests on t = u' + M:  t >= M - 1 (truncation toward zero) and t <= M + (size - 1)
  float s_lo, s_hi;       // same for v
  int idx_bias;           // LEAN_MAGIC_BITS * (W + 1): idx = bits(ty) * W + bits(tx) - idx_bias
  // pinhole-type FoV test on r^2
  float T2lo;             // pass   iff r2 + 3 exy (1 + r2) < T2lo
  float T2hi, K3;         // reject iff rho < 0.01 and r2 > T2hi + K3 rho
  // error bound of the plumb_bob projection: e = rho A(r2b) + B(r2b), A = L (1 + mh), B = 4u L mh + M16 (fast_filter.hpp)
  float ea[5], eb[5];
  float C1x3, C2x3;       // FoV margin only: 3 exy <= rho C1x3 + C2x3 on the FoV disc (the band it widens holds ~0.001 % of the points)
  float hx0, hy0;         // 0.5 - cu, 0.5 - cv
  float nsfx, nsfy;       // -sfx, -sfy
  float eq_su, eq_sv;     // equirectangular: u' = lon_turns * W + cxh, v' = lat_turns * 2H + cyh
  // equirectangular delta step (classify_lean_delta): gradient scales W / 2pi, 2H / 2pi; remainder, d-error and
  // constant terms of its bound (derivation above classify_lean_delta)
  float eq_gu, eq_gv;
  float eq_ku, eq_kv;
  float eq_lu, eq_lv;
  float eq_cu, eq_cv;
  float eq_hxd, eq_nsx15;  // hx0 - eq_cu and -1.5 sfx: the anchor's half-width hx is recomputed from delta and 1 / r_xz
};

// atan2(a, b) / (2 pi) in turns, (-0.5, 0.5]: octant reduction + odd minimax polynomial of degree 13 on [0, 1] (fitted for
// this file, tools/fit_atan_turns.py) -- 20 instructions and one MUFU.RCP against ~40 for atan2f, whose special cases
// (infinities, signed zeros, denormals) the filter does not need: every degenerate input comes out NaN or lands on a pixel
// edge, i.e. "uncertain".
//
// Error certificate (u = 2^-24; LEAN_ATAN_ERR_TURNS is what the error bounds charge):
//   1. the polynomial: |fl(t P(t^2)) - atan(t) / 2pi| <= LEAN_ATAN_POLY_ERR_TURNS for EVERY float t in [0, 1 + 2^-20],
//      measured exhaustively (tests/cpp/atan_certificate.cu: the Horner chain of lean_atan_poly_turns as compiled,
//      fmaf = one rounding, against a long double atan; also with the last product t * P left unrounded, which is what a
//      contraction of p * t into the fold's subtraction would compute);
//   2. the quotient t = fl(mn * rcp(mx)): MUFU.RCP is within 1 ulp (relative 2^-23 = 2u), the product rounds once (u), so
//      t = (mn / mx)(1 + eta), |eta| <= 3u + 2u^2, and t <= 1 + 2^-23 (inside the swept range).  atan(t) / 2pi moves by at most
//      max_t t / (1 + t^2) |eta| / 2pi <= |eta| / 4pi (1 + 1e-6) <= 1.4234e-8 turns.  A denormal t rounds by at most 2^-150
//      absolutely (nothing in turns).  mx below 2^-126 or above 2^126 makes MUFU.RCP flush to inf / 0: the first gives
//      NaN / inf downstream, and neither can occur for a point the classifier accepts (n2 > 2e-3 and a finite |p|^2);
//   3. the octant folds: 0.25 - p lies in [0.124, 0.25] and rounds by at most half an ulp of [2^-3, 2^-2), 2^-27; 0.5 - q
//      lies in [0.25, 0.5] and rounds by at most 2^-26 (round to nearest; 0.25 and 0.5 are exact).  Both at once: 2.236e-8;
//   4. copysignf and fabsf, fmaxf, fminf are exact.
// Sum: LEAN_ATAN_POLY_ERR_TURNS + 1.4234e-8 + 2.236e-8 <= LEAN_ATAN_CERT_TURNS; charged with a margin of about 10 %.
// coefficients of P, c0 + c1 s + ... + c6 s^6 (scalars: device code may read constexpr scalars, not constexpr arrays)
constexpr float LEAN_ATAN_C0 = 0.15915432572364807f, LEAN_ATAN_C1 = -0.0530262365937233f, LEAN_ATAN_C2 = 0.03152511641383171f;
constexpr float LEAN_ATAN_C3 = -0.021061519160866737f, LEAN_ATAN_C4 = 0.012672499753534794f, LEAN_ATAN_C5 = -0.005348276346921921f;
constexpr float LEAN_ATAN_C6 = 0.0010841299081221223f;
constexpr double LEAN_ATAN_POLY_ERR_TURNS = 5.31e-8;   // bound of term 1 (the exhaustive sweep measures 5.264e-8)
constexpr double LEAN_ATAN_QUOT_ERR_TURNS = 1.4234e-8;  // term 2: (3u + 2u^2) / 4pi * (1 + 1e-6), rounded up
constexpr double LEAN_ATAN_FOLD_ERR_TURNS = 2.2352e-8;  // term 3: 2^-27 + 2^-26, rounded up
constexpr double LEAN_ATAN_CERT_TURNS = LEAN_ATAN_POLY_ERR_TURNS + LEAN_ATAN_QUOT_ERR_TURNS + LEAN_ATAN_FOLD_ERR_TURNS;
constexpr double LEAN_ATAN_ERR_TURNS = 1.0e-7;
static_assert(LEAN_ATAN_ERR_TURNS >= 1.05 * LEAN_ATAN_CERT_TURNS, "the charged arctangent error must cover its certificate");

// P(s), Horner
VL_HD float lean_atan_horner(float s) {
  float p = fmaf(s, LEAN_ATAN_C6, LEAN_ATAN_C5);
  p = fmaf(s, p, LEAN_ATAN_C4);
  p = fmaf(s, p, LEAN_ATAN_C3);
  p = fmaf(s, p, LEAN_ATAN_C2);
  p = fmaf(s, p, LEAN_ATAN_C1);
  return fmaf(s, p, LEAN_ATAN_C0);
}

// atan(t) / 2pi for t = mn / mx in [0, 1]: t P(t^2)
VL_HD float lean_atan_poly_turns(float t) { return lean_atan_horner(t * t) * t; }  // in [0, 1/8]

VL_HD float lean_atan2_turns(float a, float b) {
  const float ax = fabsf(a), bx = fabsf(b);
  const float mx = fmaxf(ax, bx), mn = fminf(ax, bx);
  float p = lean_atan_poly_turns(mn * VL_RCPF(mx));
  p = ax > bx ? 0.25f - p : p;        // first quadrant
  p = b < 0.0f ? 0.5f - p : p;        // upper half plane
  return copysignf(p, a);
}

struct LeanVerdict {
  bool accept;     // the reference certainly counts this point at pixel `idx`
  bool uncertain;  // within the error bound of a decision edge: ask the exact path
  int idx;         // iy * W + ix, meaningful when accept
  float up, vp;    // the fp32 projection minus 0.5, and
  float hx, hy;    // 0.5 - E: what the verify kernel needs to measure how much of the bound the fp32 error uses
};

#define LEAN_RCP(x) VL_RCPF(x)
#define LEAN_RSQRT(x) VL_RSQRTF(x)
#if defined(__CUDA_ARCH__)
#define LEAN_F2I(x) __float_as_int(x)
#else
static inline int lean_host_f2i(float f) {
  int i;
  memcpy(&i, &f, sizeof(i));
  return i;
}
#define LEAN_F2I(x) lean_host_f2i(x)
#endif

// common tail: half-pixel-shifted coordinates (up, vp) = (u - 0.5, v - 0.5) with half-widths (hx, hy) = 0.5 - E of the
// certain zone around the pixel centre; `pass`: FoV certainly passed and the projection is valid; `rej`: certainly
// rejected before the projection (FoV / behind the camera).
VL_HD LeanVerdict lean_tail(const LeanCam& c, int width, float up, float vp, float hx, float hy, bool pass, bool rej) {
  const float tx = up + LEAN_MAGIC, ty = vp + LEAN_MAGIC;
  const float rx = tx - LEAN_MAGIC, ry = ty - LEAN_MAGIC;  // rint(up), rint(vp) for |.| < 2^22
  const float dx = up - rx, dy = vp - ry;
  // certain: FoV passed, and both coordinates sit farther than E from every pixel edge.  (NaN anywhere -> false.)
  // (bitwise & | on bools: no short-circuit, so the compiler emits predicate logic instead of branches)
  const bool cert = pass & (fabsf(dx) < hx) & (fabsf(dy) < hy);
  const bool inside = (tx >= c.t_lo) & (tx <= c.t_hi) & (ty >= c.s_lo) & (ty <= c.s_hi);
  LeanVerdict v;
  v.accept = cert & inside;
  v.uncertain = !cert & !rej;
  // truncation toward zero: rint(u') == -1 (u in (-1, 0)) is column 0
  const int ixb = max(LEAN_F2I(tx), LEAN_MAGIC_BITS), iyb = max(LEAN_F2I(ty), LEAN_MAGIC_BITS);
  v.idx = iyb * width + ixb - c.idx_bias;
  v.up = up, v.vp = vp, v.hx = hx, v.hy = hy;
  return v;
}

// ---- equirectangular: the poses of a batch as first-order updates from one of them (the anchor) --------------------------
//
// The poses of a Nelder-Mead batch lie close together (xr, xe, xc on a line through xo; the initial simplex x0 + 1e-3
// along each axis), so for pose k the camera-frame point moves by D = p_k - p_0 = dR_k p + dt_k, dR_k = R_k - R_0,
// dt_k = t_k - t_0 (index 0: the anchor, lean_delta_anchor), which is small against the point's distance from the
// camera's y axis r_xz.  The anchor step is the plain classifier at the anchor (same verdict) and keeps, per point, the
// projection (up0, vp0), its gradient g at the fp32 point q0 = p~_0, 1 / r_xz and a radius within which the guards of the
// plain classifier provably hold.  The delta step
// projects pose k as  up = up0 + g_u . d,  vp = vp0 + g_v . d  with d = fl32(dR~_k p + dt~_k) (dR~, dt~ rounded once from
// the double poses), a handful of FMAs instead of two rsqrt and two arctangents, and keeps the verdict only where
// |up - u_ref(p_k) + 0.5| < 0.5 - |frac|, i.e. under the half-widths hx_k = hx_0 - (terms 2-4 below), as lean_tail tests.
//
// Soundness.  Let m = |D| + sqrt3 delta, so the ball B of radius m around q0 holds p_0 (|p_0 - q0| <= sqrt3 delta),
// p_k and the segment between them.  With xi = p_0 - q0 and h a bound on the Hessian norm of u on B,
//   u(p_k) - u(p_0) - grad u(q0) . D = int_0^1 (grad u(p_0 + sD) - grad u(q0)) . D ds,  |.| <= h (|xi||D| + |D|^2/2) <= h m^2/2.
// The error of up splits into
//   1. the anchor's own bound (0.5 - hx_0: the plain classifier's E, unchanged; hx_0 = hx0 - 1.5 sfx delta / r_xz
//      is recomputed by the delta step in another rounding order, which the safety factor 2 of that term absorbs);
//   2. the remainder h m^2 / 2.  lon = atan2(x, z) has Hessian norm 1 / r_xz^2.  lat = atan2(y, r_xz(x, z)): its Hessian
//      is J^T H_2 J + phi_r grad^2 r_xz with J's rows (e_y, grad r_xz) orthonormal, |H_2| = 1 / n^2 (polar angle),
//      |phi_r| = |y| / n^2 and |grad^2 r_xz| = 1 / r_xz, so |H_lat| <= (cos^2 b + |sin b| cos b) / r_xz^2 <= (1 + sqrt2) / 2
//      / r_xz^2 (y = n sin b, r_xz = n cos b).  On B, r_xz >= r_xz(q0) - m >= (15/16 - 4e-7) r_xz~ because the delta
//      step requires m < r_xz~ / 16, so 1 / r_xz,min^2 <= 1.138 / r_xz~^2; charged 1.15 (the fp32 1 / r_xz~^2 included).
//      In pixels: eq_ku = S W / 4pi * 1.15, eq_kv = S 2H / 4pi * 1.2072 * 1.15 (S = 2, the safety factor of the anchor);
//   3. the error of d: per component |d~ - D| <= 5u (sum_j |dR_ij| |p_j| + |dt_i|) (rounding of dR, dt and three FMAs);
//      |p|_1 <= delta / 5.25u, so |d~ - D|_2 <= eps := 1.7 max|dR~| delta + 9u max|dt~|  (per pose: A, B of lean_delta_pose,
//      both times 8.07).  It enters |D| <= |d~| + eps (hence m) and, through the gradient, |grad u| eps <= S W / 2pi eps / r_xz
//      (|grad v| <= 2H / 2pi / |p| <= 2H / 2pi / r_xz): eq_lu, eq_lv.  This term is far below the others by construction
//      (eps / r_xz ~ 1e-7 |dR|): no test can observe it, its charge rests on this derivation alone;
//   4. the fp32 gradient (relative error <= 16u incl. MUFU.RSQ, charged 64u) times |d| <= r_xz / 16, the products of
//      g . d, and the rounding of up0 + s, at most u |up0 + s| with |up0| <= W~ / 2 + |cxh~| (make_lean_cam) and
//      |s| <= W / 32pi: eq_cu = S (64u W / 32pi + u (W~ / 2 + |cxh~| + 0.02 W + 1)) + 1e-6 (the reference's own double
//      rounding, the rounding of hx_k), likewise eq_cv with 2H~ / 4 + |cyh~| and 2H.
// m^2 <= (1 + 1/64) |d~|^2 + 65 (eps + sqrt3 delta)^2 (the delta step computes it as fma(|d~|^2, 1.016, e8^2) with
// e8 = 8.07 (eps + sqrt3 delta)).  Guards at pose k, all from  m < radius  (radius^2 kept per point, shrunk by 1e-4):
//   * r_xz~ / 16: the remainder bound above; |p_k| >= 15/16 |q0| keeps n^2 > 2e-3 * 0.87 > 1e-3 (the reference's branch);
//   * the seam: B must not meet the cut {x = 0, z <= 0} of atan2(x, z): distance r_xz~ if z~ > 0, else |x~|;
//   * FoV: g = z - cos_fov |p| is 2-Lipschitz and the anchor's margin mf covers its fp32 and the reference's rounding,
//     so g~_0 - mf > 2|D| keeps the pass at pose k (radius 0.49 (g~_0 - mf)) and -g~_0 - mf > 2|D| keeps the reject.
// The anchor's own guards (n^2, r_xz > 40 delta, pole) must have held at the anchor for a pass; otherwise the radius is 0
// and the delta step defers every pose.  A NaN anywhere makes both predicates false: uncertain.
struct LeanAnchor {
  float up0, vp0;       // the anchor's projection (pixel coordinates minus 0.5)
  float gux, guz;       // d up / d (x, z) of the camera-frame point, pixels per metre (lon has no y term)
  float gvx, gvy, gvz;  // d vp / d (x, y, z)
  float irxz;           // 1 / r_xz at the anchor
  float hy;             // the anchor's half-width hy minus eq_cv (hx: hx0 - 1.5 sfx delta / r_xz, recomputed)
  float rad2;           // > 0: pass radius^2; < 0: -(reject radius^2); 0: every pose k is uncertain
};

constexpr float LEAN_DELTA_SQ3 = 13.98f;   // 8.07 sqrt3
constexpr float LEAN_DELTA_M2 = 1.016f;    // (1 + 1/64) and the rounding of |d~|^2

// P: pose32 row of the anchor, as classify_lean.  Same operations as the plain classifier for the verdict.
template <int MODEL>
VL_HD LeanVerdict classify_lean_anchor(const FastCam& f, const LeanCam& c, int width, const float* __restrict__ P, float x, float y, float z, float delta, LeanAnchor& an) {
  static_assert(MODEL == CAM_EQUIRECTANGULAR, "the delta step is derived for the equirectangular model");
  const float pcx = fmaf(P[0], x, fmaf(P[1], y, fmaf(P[2], z, P[9])));
  const float pcy = fmaf(P[3], x, fmaf(P[4], y, fmaf(P[5], z, P[10])));
  const float pcz = fmaf(P[6], x, fmaf(P[7], y, fmaf(P[8], z, P[11])));
  // u = W (0.5 + atan2(x, z) / 2pi),  v = H (0.5 + asin(y / |p|) / pi) = H (0.5 + 2 atan2(y, |(x, z)|) / 2pi)
  // (equirectangular.hpp:21-27).  Input-error terms as validated in round 1 (project_fast): |d lon| <= 1.5 delta / rxz,
  // |d asin| <= 1.03 (2.9 delta / |p| + 4u) |p| / rxz (an upper bound for the atan2 form as well, rxz <= |p|).
  const float xx = pcx * pcx;
  const float rxz2 = fmaf(pcz, pcz, xx);
  const float n2 = fmaf(pcy, pcy, rxz2);
  const float inv_n = LEAN_RSQRT(n2);
  const float nrm = n2 * inv_n;
  const float inv_rxz = LEAN_RSQRT(rxz2);
  const float rxz = rxz2 * inv_rxz;
  const float g = fmaf(-f.cos_fov, nrm, pcz);  // :32 (cos_fov = -1 for the full sphere: only the antipode is uncertain)
  const float mf = fmaf(3.0f, delta, (12.0f * F32_U) * nrm);
  const float lon = lean_atan2_turns(pcx, pcz);
  const float lat = lean_atan2_turns(pcy, rxz);
  const float up = fmaf(lon, c.eq_su, c.cxh);
  const float vp = fmaf(lat, c.eq_sv, c.cyh);
  const float t_lon = (1.5f * delta) * inv_rxz;
  const float t_by = fmaf(2.9f * delta, inv_n, 4.0f * F32_U);
  const float t_asn = (1.03f * t_by) * (nrm * inv_rxz);
  const float hx = fmaf(c.nsfx, t_lon, c.hx0);
  const float hy = fmaf(c.nsfy, t_asn, c.hy0);
  // away from the |p|^2 < 1e-3 branch (:15), from the poles and from the seam's ill-conditioning
  const bool ok = (n2 > 2e-3f) & (rxz > 40.0f * delta) & (rxz > 0.05f * nrm);
  const bool pass = ok & (g > mf);
  const bool rej = g < -mf;
  // what the delta step needs: gradient (lon: (z, -x) / r_xz^2; lat: (-x y / r_xz, r_xz, -z y / r_xz) / n^2, per 2pi)
  const float gu = c.eq_gu * (inv_rxz * inv_rxz);
  const float gv = c.eq_gv * (inv_n * inv_n);
  const float gvr = -(gv * pcy) * inv_rxz;
  an.up0 = up, an.vp0 = vp;
  an.gux = gu * pcz, an.guz = -(gu * pcx);
  an.gvx = gvr * pcx, an.gvy = gv * rxz, an.gvz = gvr * pcz;
  an.irxz = inv_rxz;
  an.hy = hy - c.eq_cv;
  const float r_seam = pcz > 0.0f ? rxz : fabsf(pcx);
  const float r_pass = fminf(fminf(0.0625f * rxz, r_seam), 0.49f * (g - mf));
  const float r_rej = 0.49f * (-g - mf);
  an.rad2 = pass ? (0.9999f * r_pass) * r_pass : (rej ? -((0.9999f * r_rej) * r_rej) : 0.0f);
  return lean_tail(c, width, up, vp, hx, hy, pass, rej);
}

// Q: pose k of the batch as written by lean_delta_pose: [dR row-major 9 | dt 3 | A | B], A, B: 8.07 eps = A delta + B
template <int MODEL>
VL_HD LeanVerdict classify_lean_delta(const LeanCam& c, int width, const float* __restrict__ Q, float x, float y, float z, float delta, const LeanAnchor& an) {
  static_assert(MODEL == CAM_EQUIRECTANGULAR, "the delta step is derived for the equirectangular model");
  const float dx = fmaf(Q[0], x, fmaf(Q[1], y, fmaf(Q[2], z, Q[9])));
  const float dy = fmaf(Q[3], x, fmaf(Q[4], y, fmaf(Q[5], z, Q[10])));
  const float dz = fmaf(Q[6], x, fmaf(Q[7], y, fmaf(Q[8], z, Q[11])));
  const float nd2 = fmaf(dx, dx, fmaf(dy, dy, dz * dz));
  const float e1 = fmaf(delta, Q[12], Q[13]);       // 8.07 eps
  const float e8 = fmaf(delta, LEAN_DELTA_SQ3, e1);  // 8.07 (eps + sqrt3 delta)
  const float m2 = fmaf(nd2, LEAN_DELTA_M2, e8 * e8);
  const float up = an.up0 + fmaf(an.gux, dx, an.guz * dz);
  const float vp = an.vp0 + fmaf(an.gvx, dx, fmaf(an.gvy, dy, an.gvz * dz));
  const float r2m2 = (an.irxz * an.irxz) * m2;
  const float lin = an.irxz * e1;
  const float tlx = fmaf(-c.eq_lu, e1, c.eq_nsx15 * delta);  // -(input-error term of the anchor + term 3) * r_xz
  const float hx = fmaf(-c.eq_ku, r2m2, fmaf(an.irxz, tlx, c.eq_hxd));
  const float hy = fmaf(-c.eq_kv, r2m2, fmaf(-c.eq_lv, lin, an.hy));
  const bool pass = m2 < an.rad2;
  const bool rej = m2 < -an.rad2;
  return lean_tail(c, width, up, vp, hx, hy, pass, rej);
}

// Spread of a batch for the delta step (a performance policy, not part of the bound): beyond it the remainder term would
// defer too many point-poses, and the batch takes the plain classifier.  Nelder-Mead batches start at ~1e-3 and shrink.
constexpr double LEAN_DELTA_MAX_DR = 4e-3;  // max |R_k - R_a| entry (a: the anchor)
constexpr double LEAN_DELTA_MAX_DT = 2e-2;  // max |t_k - t_a| entry, metres
constexpr float LEAN_DELTA_T_SCALE = static_cast<float>(LEAN_DELTA_MAX_DR / LEAN_DELTA_MAX_DT);

// gate entry between row r of two poses, fp32 rows [R_r0 R_r1 R_r2 t_r]: the largest |difference|, translation scaled to
// the rotation's limit (fmaxf: NaN entries are ignored, so a score is never NaN)
VL_HD float lean_delta_row_spread(const float* __restrict__ a, const float* __restrict__ b) {
  return fmaxf(fmaxf(fabsf(a[0] - b[0]), fabsf(a[1] - b[1])), fmaxf(fabsf(a[2] - b[2]), LEAN_DELTA_T_SCALE * fabsf(a[3] - b[3])));
}

// The anchor of a batch of n <= 8 poses (row-major 3x4 doubles; the rule runs on their fp32 roundings): the pose whose
// largest gate entry to the other poses is smallest, ties to the lowest index, so every block, every rank and the host
// pick the same pose.  The bound of the delta step holds for any anchor; this choice puts as many batches as possible
// inside the gate and keeps the remainder term, which grows with the squared distance to the anchor, small.  For a
// Nelder-Mead iteration {xr, xe, xc, xo} (s = 1, 2, 1/2, 0 along one line) it is xr, index 0: the farthest pose is
// |diff| away instead of 2 |diff|, and the squared offsets sum to 2.25 |diff|^2 instead of 5.25 (1.25 |diff|^2 when the
// centroid xo is not scored, nm_machine.cuh).  For the initial simplex it is x0.
// pk_delta_rows computes the same scores warp-parallel (max and min are exact, so any grouping gives the same bits).
VL_HD float lean_delta_anchor_score(const double (*__restrict__ T)[12], int n, int i) {
  float s = 0.0f;
  for (int r = 0; r < 3; r++) {
    float a[4];
    for (int c = 0; c < 4; c++) a[c] = static_cast<float>(T[i][4 * r + c]);
    for (int j = 0; j < n; j++) {
      float b[4];
      for (int c = 0; c < 4; c++) b[c] = static_cast<float>(T[j][4 * r + c]);
      s = fmaxf(s, lean_delta_row_spread(a, b));
    }
  }
  return s;
}
VL_HD int lean_delta_anchor(const double (*__restrict__ T)[12], int n) {
  int best = 0;
  float best_s = n > 0 ? lean_delta_anchor_score(T, n, 0) : 0.0f;
  for (int i = 1; i < n; i++) {
    const float s = lean_delta_anchor_score(T, n, i);
    if (s < best_s) best = i, best_s = s;
  }
  return best;
}

// pose k of a batch relative to the anchor T0 (row-major 3x4 doubles) -> Q[16] for classify_lean_delta (Q[14], Q[15]
// zero, free for the caller); true if within the spread
VL_HD bool lean_delta_pose(const double* __restrict__ T, const double* __restrict__ T0, float* __restrict__ Q) {
  float rmax = 0.0f, tmax = 0.0f;
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) {
      Q[3 * r + c] = static_cast<float>(T[4 * r + c] - T0[4 * r + c]);
      rmax = fmaxf(rmax, fabsf(Q[3 * r + c]));
    }
    Q[9 + r] = static_cast<float>(T[4 * r + 3] - T0[4 * r + 3]);
    tmax = fmaxf(tmax, fabsf(Q[9 + r]));
  }
  // 8.07 (1.7 max|dR| delta + 9u max|dt|), rounded up by the 1e-3 margins
  Q[12] = static_cast<float>(8.08 * 1.7 * static_cast<double>(rmax));
  Q[13] = static_cast<float>(8.08 * 9.0 * static_cast<double>(F32_U) * static_cast<double>(tmax));
  Q[14] = Q[15] = 0.0f;
  bool close = true;
  for (int i = 0; i < 12; i++) close = close && (fabsf(Q[i]) <= static_cast<float>(i < 9 ? LEAN_DELTA_MAX_DR : LEAN_DELTA_MAX_DT));
  return close;
}

// P: pose32 row (R row-major 9, t 3); delta >= |pc_fp32 - pc_exact|_inf for this point and every pose of the batch
template <int MODEL>
VL_HD LeanVerdict classify_lean(const FastCam& f, const LeanCam& c, int width, const float* __restrict__ P, float x, float y, float z, float delta) {
  const float pcx = fmaf(P[0], x, fmaf(P[1], y, fmaf(P[2], z, P[9])));
  const float pcy = fmaf(P[3], x, fmaf(P[4], y, fmaf(P[5], z, P[10])));
  const float pcz = fmaf(P[6], x, fmaf(P[7], y, fmaf(P[8], z, P[11])));
  if constexpr (MODEL == CAM_PLUMB_BOB) {
    // enabled only when cos(max_fov) >= 0.05: FoV pass <=> pcz > 0 and r2 <= tan^2(max_fov)
    const float inv = LEAN_RCP(pcz);
    const float xn = pcx * inv, yn = pcy * inv;
    const float rho = delta * inv;
    const float x2 = xn * xn, y2 = yn * yn, xy = xn * yn;
    const float r2 = x2 + y2;
    const float rc = fmaf(r2, fmaf(r2, fmaf(r2, f.d[4], f.d[1]), f.d[0]), 1.0f);  // 1 + k1 r2 + k2 r4 + k3 r6
    const float p1 = f.d[2], p2 = f.d[3];
    const float xd = fmaf(xn, rc, fmaf(2.0f * p1, xy, p2 * fmaf(2.0f, x2, r2)));
    const float yd = fmaf(yn, rc, fmaf(2.0f * p2, xy, p1 * fmaf(2.0f, y2, r2)));
    const float up = fmaf(f.fx, xd, c.cxh);
    const float vp = fmaf(f.fy, yd, c.cyh);
    // error bound: e = L exy + M16 of the round-1 filter, exy = rho (1 + mh) + 4u mh, with the products expanded on the host
    // into two polynomials of r2b: e = rho A(r2b) + B(r2b)  (positive coefficients, rounded up).  Evaluated PER POINT: maxima
    // or chords over the FoV disc are 3-4x looser on lenses whose distortion folds back (the C2 camera: max_fov = 59 deg
    // although the image corner sits at 48 deg) and deferred 10 % of the point-poses instead of 3 %.
    const float r2b = fmaf(r2, 1.001f, 1e-6f);
    const float A = fmaf(r2b, fmaf(r2b, fmaf(r2b, fmaf(r2b, c.ea[4], c.ea[3]), c.ea[2]), c.ea[1]), c.ea[0]);
    const float B = fmaf(r2b, fmaf(r2b, fmaf(r2b, fmaf(r2b, c.eb[4], c.eb[3]), c.eb[2]), c.eb[1]), c.eb[0]);
    const float e = fmaf(rho, A, B);
    const float hx = fmaf(c.nsfx, e, c.hx0);
    const float hy = fmaf(c.nsfy, e, c.hy0);
    // FoV cone from r2 (derivation: DESIGN.md section 4; needs z certainly positive and rho small)
    const float exy3 = fmaf(rho, c.C1x3, c.C2x3);
    const float fov_m = fmaf(exy3, 1.0f + r2, r2);
    const bool base = (pcz > delta) & (rho < 0.01f);
    const bool pass = base & (fov_m < c.T2lo);
    const bool rej = (base & (r2 > fmaf(c.K3, rho, c.T2hi))) | (pcz < -delta);
    return lean_tail(c, width, up, vp, hx, hy, pass, rej);
  } else if constexpr (MODEL == CAM_EQUIRECTANGULAR) {
    LeanAnchor unused;
    return classify_lean_anchor<MODEL>(f, c, width, P, x, y, z, delta, unused);
  } else {
    // other models: round-1 projection + bound (project_fast), FoV from |p| (these models need it anyway)
    const float n2 = fmaf(pcx, pcx, fmaf(pcy, pcy, pcz * pcz));
    const float nrm = n2 * LEAN_RSQRT(n2);
    const float g = fmaf(-f.cos_fov, nrm, pcz);
    const float mf = fmaf(3.0f, delta, (12.0f * F32_U) * nrm);
    float u, v, Eu, Ev;
    const bool ok = project_fast<MODEL>(f, pcx, pcy, pcz, nrm, delta, u, v, Eu, Ev);
    const bool pass = ok & (g > mf);
    const bool rej = g < -mf;
    return lean_tail(c, width, u - 0.5f, v - 0.5f, 0.5f - Eu, 0.5f - Ev, pass, rej);
  }
}

}  // namespace vlcal
