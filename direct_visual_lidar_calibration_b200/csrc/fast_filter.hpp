// fast_filter.hpp -- host-side (double) derivation of the fp32-filter error constants for one camera.
//
// Notation: u = 2^-24.  For a point p = (x,y,z) (exactly representable floats) and a pose (R,t):
//   pc_exact = R p + t in real arithmetic (the reference's double evaluation is within 1e-15 relative of it)
//   pc_fp32  = three fused multiply-adds on float(R), float(t):  |pc_fp32 - pc_exact|_inf <= delta
//   delta    = 5u (|x|+|y|+|z| + max|t|)     [1u rounding of R and t, 3u for the three FMAs, 1u slack]
// Pinhole-type models (plumb_bob, rational_polynomial), enabled when cos(max_fov) >= 0.05:
//   a point that certainly passes the FoV test has z >= cos(max_fov)|pc| > 0 and r = |(x/z, y/z)| <= Rmax = tan(max_fov)
//   e_xy = |(x/z)_fp32 - (x/z)_exact| <= rho (1 + r) + 4u r,  rho = delta / z,  r = |(x/z, y/z)|
//   distortion D(x,y): |J_D| <= L(r) = RC + 3 r^2 Q + 8 (|p1|+|p2|) r,   RC >= |r_coeff|, Q >= |d r_coeff / d r^2|
//       (polynomials with absolute coefficients, monotone in r^2, evaluated PER POINT in the kernel at r^2 * 1.001 + 1e-6;
//        a global bound at Rmax = tan(max_fov) would be 5x looser on a distorted wide lens and defer 15 % of the points)
//   fp32 evaluation of D rounds by at most 16u M(r),   M = r RC + 3 (|p1|+|p2|) r^2
//   pixel error  E = SAFETY * ( f (L e_xy + 16u M) + 4u (size + |c| + 1) )
// SAFETY = 2 (the constants are already worst case; the factor also covers the rounding of the fp32 evaluation of E).  The verify kernel (vlcal_nid_debug_filter_check) measures max |uv_fp32-uv_exact|/E.
#pragma once

#include <algorithm>
#include <cmath>

#include "camera_models.cuh"
#include "lean_filter.cuh"

namespace vlcal {

inline FastCam make_fast_cam(const CameraParams& cam, int width, int height, double max_fov) {
  constexpr double U = 5.9604644775390625e-08;
  constexpr double SAFETY = 2.0;
  FastCam f{};
  f.enabled = 0;
  const double cos_fov = std::cos(max_fov);
  f.cos_fov = static_cast<float>(cos_fov);
  f.fx = static_cast<float>(cam.intr[0]);
  f.fy = static_cast<float>(cam.intr[1]);
  f.cx = static_cast<float>(cam.intr[2]);
  f.cy = static_cast<float>(cam.intr[3]);
  f.xi = static_cast<float>(cam.intr[4]);
  for (int i = 0; i < 8; i++) f.d[i] = static_cast<float>(cam.dist[i]);
  for (int i = 0; i < 5; i++)
    if (!std::isfinite(cam.intr[i])) return f;
  for (int i = 0; i < 8; i++)
    if (!std::isfinite(cam.dist[i])) return f;
  if (!std::isfinite(max_fov)) return f;
  auto up = [](double v) { return std::nextafter(static_cast<float>(v), INFINITY); };  // round the bound constants up

  if (cam.model == CAM_PLUMB_BOB || cam.model == CAM_RATIONAL_POLYNOMIAL) {
    if (!(cos_fov >= 0.05)) return f;  // the pinhole division needs z > 0 for every point that passes the FoV test
    const double* d = cam.dist;
    const double P = std::fabs(d[2]) + std::fabs(d[3]);
    f.a1 = up(std::fabs(d[0])), f.a2 = up(std::fabs(d[1])), f.a3 = up(std::fabs(d[4]));
    f.b1 = up(std::fabs(d[5])), f.b2 = up(std::fabs(d[6])), f.b3 = up(std::fabs(d[7]));
    f.p3 = up(3.0 * P), f.p4 = up(4.0 * P);
    f.sfx = up(SAFETY * std::fabs(cam.intr[0]));
    f.sfy = up(SAFETY * std::fabs(cam.intr[1]));
    // u = fma(fx, xd, cx): one rounding of the result (|u| <= size + 1 wherever the verdict matters), rounding of the
    // float copies of fx (folded into the 16u M term) and cx
    f.cu = up(SAFETY * 4.0 * U * (width + std::fabs(cam.intr[2]) + 1.0));
    f.cv = up(SAFETY * 4.0 * U * (height + std::fabs(cam.intr[3]) + 1.0));
    {  // plumb_bob: L = RC + r2 (3Q + 4P) + 4P and M = (1+r2)/2 RC + 3P r2 expanded in powers of r2 (see project_fast)
      const double a1 = f.a1, a2 = f.a2, a3 = f.a3, p3 = f.p3, p4 = f.p4;
      f.l0 = up(1.0 + p4), f.l1 = up(4.0 * a1 + p4), f.l2 = up(7.0 * a2), f.l3 = up(10.0 * a3);
      const double s = 16.0 * U;
      f.m0 = up(s * 0.5), f.m1 = up(s * (0.5 + 0.5 * a1 + p3)), f.m2 = up(s * 0.5 * (a1 + a2)), f.m3 = up(s * 0.5 * (a2 + a3)), f.m4 = up(s * 0.5 * a3);
    }
    f.enabled = 1;
  }
  const double Wd = width, Hd = height;
  if (cam.model == CAM_EQUIRECTANGULAR) {
    // intr = [W, H] (the projection scales by the intrinsics, not by the image size passed to the cost)
    const double W = std::fabs(cam.intr[0]), H = std::fabs(cam.intr[1]);
    f.fx = static_cast<float>(cam.intr[0]);
    f.fy = static_cast<float>(cam.intr[1]);
    f.sfx = up(SAFETY * W / (2.0 * M_PI));
    f.sfy = up(SAFETY * H / M_PI);
    f.cu = up(SAFETY * (W / (2.0 * M_PI) * 8.0 * U * M_PI + 4.0 * U * (W + Wd + 1.0)));
    f.cv = up(SAFETY * (H / M_PI * 8.0 * U + 4.0 * U * (H + Hd + 1.0)));
    f.enabled = 1;
  } else if (cam.model == CAM_FISHEYE) {
    const double* d = cam.dist;
    f.a1 = up(std::fabs(d[0])), f.a2 = up(std::fabs(d[1])), f.a3 = up(std::fabs(d[2])), f.a4 = up(std::fabs(d[3]));
    f.sfx = up(SAFETY * std::fabs(cam.intr[0]));
    f.sfy = up(SAFETY * std::fabs(cam.intr[1]));
    f.cu = up(SAFETY * 4.0 * U * (Wd + std::fabs(cam.intr[2]) + 1.0));
    f.cv = up(SAFETY * 4.0 * U * (Hd + std::fabs(cam.intr[3]) + 1.0));
    f.enabled = 1;
  } else if (cam.model == CAM_OMNIDIR) {
    const double* d = cam.dist;
    const double a1 = std::fabs(d[0]), a2 = std::fabs(d[1]), P = std::fabs(d[2]) + std::fabs(d[3]);
    const double p3 = 3.0 * P, p4 = 4.0 * P;
    f.l0 = up(1.0 + p4), f.l1 = up(4.0 * a1 + p4), f.l2 = up(7.0 * a2), f.l3 = 0.0f;
    const double s16 = 16.0 * U;
    f.m0 = up(s16 * 0.5), f.m1 = up(s16 * (0.5 + 0.5 * a1 + p3)), f.m2 = up(s16 * 0.5 * (a1 + a2)), f.m3 = up(s16 * 0.5 * a2), f.m4 = 0.0f;
    f.sfx = up(SAFETY * std::fabs(cam.intr[0]));
    f.sfy = up(SAFETY * std::fabs(cam.intr[1]));
    f.cu = up(SAFETY * 4.0 * U * (Wd + std::fabs(cam.intr[2]) + 1.0));
    f.cv = up(SAFETY * 4.0 * U * (Hd + std::fabs(cam.intr[3]) + 1.0));
    f.enabled = 1;
  } else if (cam.model == CAM_ATAN) {
    if (!(cos_fov >= 0.05)) return f;  // pinhole division
    const double d0 = cam.dist[0];
    double G = 1.0;
    f.aux0 = 0.0f, f.aux1 = 0.0f;
    if (!(d0 < 1e-7)) {  // atan.hpp:17 (second operand): distortion active
      const double d1 = 1.0 / d0, d2 = 2.0 * std::tan(d0 / 2.0);
      if (!(std::isfinite(d1) && std::isfinite(d2)) || d1 <= 0.0 || d2 <= 0.0) return f;
      f.aux0 = static_cast<float>(d1);
      f.aux1 = static_cast<float>(d2);
      G = std::max(1.0, d1 * d2);
    }
    f.l0 = up(1.5 * G);
    f.m0 = up(8.0 * U * G);
    f.sfx = up(SAFETY * std::fabs(cam.intr[0]));
    f.sfy = up(SAFETY * std::fabs(cam.intr[1]));
    f.cu = up(SAFETY * 4.0 * U * (Wd + std::fabs(cam.intr[2]) + 1.0));
    f.cv = up(SAFETY * 4.0 * U * (Hd + std::fabs(cam.intr[3]) + 1.0));
    f.enabled = 1;
  }
  return f;
}

// constants of the lean classifier (lean_filter.cuh) from the validated round-1 constants `f` = make_fast_cam(...).
// Every quantity is an upper bound of the round-1 one on the set of points that can be accepted, rounded outward.
inline LeanCam make_lean_cam(const CameraParams& cam, const FastCam& f, int width, int height, double max_fov) {
  constexpr double U = 5.9604644775390625e-08;
  LeanCam c{};
  c.enabled = 0;
  if (!f.enabled) return c;
  // magic-constant rounding needs |u'| < 2^22 wherever a verdict is accepted, and 32-bit pixel indices
  if (width < 1 || height < 1 || width >= (1 << 21) || height >= (1 << 21) || static_cast<long long>(width) * height >= (1LL << 31)) return c;
  auto up = [](double v) { return std::nextafter(static_cast<float>(v), INFINITY); };
  auto dn = [](double v) { return std::nextafter(static_cast<float>(v), -INFINITY); };
  c.t_lo = LEAN_MAGIC - 1.0f;
  c.t_hi = LEAN_MAGIC + static_cast<float>(width - 1);
  c.s_lo = LEAN_MAGIC - 1.0f;
  c.s_hi = LEAN_MAGIC + static_cast<float>(height - 1);
  c.idx_bias = static_cast<int>(static_cast<unsigned int>(LEAN_MAGIC_BITS) * static_cast<unsigned int>(width + 1));  // modulo 2^32, like the kernel's IMAD
  c.hx0 = dn(0.5 - static_cast<double>(f.cu));
  c.hy0 = dn(0.5 - static_cast<double>(f.cv));
  c.nsfx = -f.sfx;
  c.nsfy = -f.sfy;
  if (cam.model == CAM_PLUMB_BOB) {
    const double cs = std::cos(max_fov);
    if (!(cs >= 0.05)) return c;  // make_fast_cam already requires it
    const double T2 = 1.0 / (cs * cs) - 1.0;  // tan^2(max_fov)
    const double sT = std::sqrt(T2);
    // e = L (rho (1 + mh) + 4u mh) + M16 with L = sum l_i t^i, mh = (1 + t) / 2, M16 = sum m_i t^i  (t = r2b), expanded:
    //   A(t) = L(t) (1.5 + 0.5 t),  B(t) = L(t) (2u + 2u t) + M16(t)   -- all coefficients non-negative
    const double l[5] = {f.l0, f.l1, f.l2, f.l3, 0.0};
    const double m[5] = {f.m0, f.m1, f.m2, f.m3, f.m4};
    for (int i = 0; i < 5; i++) {
      const double lm1 = i > 0 ? l[i - 1] : 0.0;
      c.ea[i] = up((1.5 * l[i] + 0.5 * lm1) * (1.0 + 8 * U));
      c.eb[i] = up((2.0 * U * (l[i] + lm1) + m[i]) * (1.0 + 8 * U));
    }
    // FoV margin: 3 exy over the disc a point that certainly passes the FoV test can lie in (r2 < T2, r2b <= R2B)
    const double R2B = (1.001 * T2 + 1e-6) * (1.0 + 1e-6);
    const double MH = 0.5 * R2B + 0.5;  // mh = (1 + r2b) / 2 <= MH
    c.C1x3 = up(3.0 * (1.0 + MH));
    c.C2x3 = up(12.0 * U * MH);
    c.T2lo = dn(T2 * (1.0 - 1e-6));
    c.T2hi = up(T2 * (1.0 + 2e-6));
    c.K3 = up(3.0 * (1.0 + sT) * (1.0 + sT));
    c.cxh = static_cast<float>(cam.intr[2] - 0.5);
    c.cyh = static_cast<float>(cam.intr[3] - 0.5);
    // the chord / maxima must be finite and the certain zone non-empty somewhere
    for (int i = 0; i < 5; i++)
      if (!std::isfinite(c.ea[i]) || !std::isfinite(c.eb[i])) return c;
    if (!std::isfinite(c.K3) || !std::isfinite(c.C1x3) || !(c.hx0 > 0.0f) || !(c.hy0 > 0.0f)) return c;
  }
  if (cam.model == CAM_EQUIRECTANGULAR) {
    // own rounding budget: the custom atan2 (LEAN_ATAN_ERR_TURNS) instead of the atan2f / asinf allowances of project_fast
    constexpr double SAFETY = 2.0;
    const double Wd = width, Hd = height;
    const double W = std::fabs(cam.intr[0]), H = std::fabs(cam.intr[1]);
    if (!(cam.intr[0] > 0.0) || !(cam.intr[1] > 0.0) || W >= (1 << 21) || H >= (1 << 21)) return c;
    c.eq_su = static_cast<float>(cam.intr[0]);
    c.eq_sv = static_cast<float>(2.0 * cam.intr[1]);
    c.cxh = static_cast<float>(0.5 * cam.intr[0] - 0.5);
    c.cyh = static_cast<float>(0.5 * cam.intr[1] - 0.5);
    // u' = fma(lon_turns, W~, cxh~) (W~ = eq_su, cxh~ = cxh: the float copies of W and W/2 - 0.5) against the exact
    // W L + W/2 - 0.5 (L: the longitude in turns).  With L~ the fp32 angle (|L~| <= 1/2: lean_atan2_turns returns at most
    // 0.5 in magnitude) and z = L~ W~ + cxh~ the unrounded FMA,
    //   u' - (W L + W/2 - 0.5) = (fl(z) - z) + L~ (W~ - W) + (cxh~ - (W/2 - 0.5)) + W (L~ - L),
    // |fl(z) - z| <= u |z| <= u (W~ / 2 + |cxh~|) (one rounding to nearest; 1e-9 px covers an underflow).  The last term is
    // the angle's error times W: LEAN_ATAN_ERR_TURNS here, the input-error term through sfx in the kernel.  Likewise v' =
    // fma(lat_turns, 2H~, cyh~) with |lat~| <= 1/4 (atan2(y, r_xz) with r_xz >= 0 never takes the b < 0 fold).  For
    // W = 3840 this is u (W - 1/2) + 0 + 0, half an ulp of the result at most.  (project_fast charges 4u (W + Wd + 1) for
    // its three-step form.)
    (void)Wd, (void)Hd;
    const double Wf = c.eq_su, Sf = c.eq_sv, cxf = c.cxh, cyf = c.cyh;
    const double ru = U * (0.5 * Wf + std::fabs(cxf)) + 0.5 * std::fabs(Wf - W) + std::fabs(cxf - (0.5 * W - 0.5)) + 1e-9;
    const double rv = U * (0.25 * Sf + std::fabs(cyf)) + 0.25 * std::fabs(Sf - 2.0 * H) + std::fabs(cyf - (0.5 * H - 0.5)) + 1e-9;
    const double cu = SAFETY * (W * LEAN_ATAN_ERR_TURNS + ru);
    const double cv = SAFETY * (2.0 * H * LEAN_ATAN_ERR_TURNS + rv);
    c.hx0 = dn(0.5 - cu);
    c.hy0 = dn(0.5 - cv);
    if (!(c.hx0 > 0.0f) || !(c.hy0 > 0.0f)) return c;
    // delta step (lean_filter.cuh, above classify_lean_delta): terms 2-4 of its bound.  The rounding of up0 + s is at most
    // u |up0 + s| with |up0| <= (W~ / 2 + |cxh~|)(1 + u) (as above) and |s| <= W / 32pi < 0.01 W; 0.02 W + 1 absorbs both
    // excesses (likewise v with 2H~ / 4 + |cyh~| and 2H / 32pi).
    const double su = W, sv = 2.0 * H;
    c.eq_gu = static_cast<float>(su / (2.0 * M_PI));
    c.eq_gv = static_cast<float>(sv / (2.0 * M_PI));
    c.eq_ku = up(SAFETY * su / (4.0 * M_PI) * 1.15);
    c.eq_kv = up(SAFETY * sv / (4.0 * M_PI) * 1.2072 * 1.15);
    c.eq_lu = up(SAFETY * su / (2.0 * M_PI) / 8.07 * (1.0 + 1e-5));
    c.eq_lv = up(SAFETY * sv / (2.0 * M_PI) / 8.07 * (1.0 + 1e-5));
    c.eq_cu = up(SAFETY * (64.0 * U * su / (32.0 * M_PI) + U * (0.5 * Wf + std::fabs(cxf) + 0.02 * su + 1.0)) + 1e-6);
    c.eq_cv = up(SAFETY * (64.0 * U * sv / (32.0 * M_PI) + U * (0.25 * Sf + std::fabs(cyf) + 0.02 * sv + 1.0)) + 1e-6);
    c.eq_hxd = dn(static_cast<double>(c.hx0) - static_cast<double>(c.eq_cu));
    c.eq_nsx15 = dn(1.5 * static_cast<double>(c.nsfx));
  }
  c.enabled = 1;
  return c;
}

}  // namespace vlcal
