// lean_filter2.cuh -- the lean classifier (lean_filter.cuh) for TWO points at a time.
//
// The persistent kernel is bound by instruction issue, and most of what it issues per point-pose are fp32 FMA / MUL / ADD
// of straight-line chains (rigid transform, distortion polynomial, error-bound polynomials, magic-constant rounding).  A
// lane already owns K = 2 points of its tile, so the two points ride in the two halves of an F2 and their chains are
// issued interleaved (two independent dependency chains per lane); comparisons, selects, MUFU and the integer tail stay
// scalar per half.
//
// Each half performs exactly the operation sequence of classify_lean (same order, same constants, each result rounded once
// or -- where the assembler contracts a product into the following sum -- not at all), so the error bounds of
// fast_filter.hpp / lean_filter.cuh hold for it unchanged; nid_lean_verify_kernel runs THIS code against the exact path.
// Device only.
#pragma once

#include "lean_filter.cuh"

namespace vlcal {

struct F2 {
  float lo, hi;
};

__device__ __forceinline__ F2 f2_pack(float lo, float hi) { return F2{lo, hi}; }
__device__ __forceinline__ F2 f2_dup(float a) { return f2_pack(a, a); }
__device__ __forceinline__ void f2_unpack(F2 a, float& lo, float& hi) { lo = a.lo, hi = a.hi; }
// Hopper has no packed fp32 pipe: each half is one FFMA / FMUL / FADD.  The _rn intrinsics are never contracted or
// reassociated, so every half rounds exactly once, as fma/mul/add.rn.f32x2 would, and the two chains interleave for ILP.
__device__ __forceinline__ F2 f2_fma(F2 a, F2 b, F2 c) { return F2{__fmaf_rn(a.lo, b.lo, c.lo), __fmaf_rn(a.hi, b.hi, c.hi)}; }
__device__ __forceinline__ F2 f2_mul(F2 a, F2 b) { return F2{__fmul_rn(a.lo, b.lo), __fmul_rn(a.hi, b.hi)}; }
__device__ __forceinline__ F2 f2_add(F2 a, F2 b) { return F2{__fadd_rn(a.lo, b.lo), __fadd_rn(a.hi, b.hi)}; }
__device__ __forceinline__ F2 f2_fma(float a, F2 b, F2 c) { return f2_fma(f2_dup(a), b, c); }
__device__ __forceinline__ F2 f2_fma(F2 a, F2 b, float c) { return f2_fma(a, b, f2_dup(c)); }
__device__ __forceinline__ F2 f2_fma(float a, F2 b, float c) { return f2_fma(f2_dup(a), b, f2_dup(c)); }
__device__ __forceinline__ F2 f2_mul(float a, F2 b) { return f2_mul(f2_dup(a), b); }
__device__ __forceinline__ F2 f2_add(F2 a, float b) { return f2_add(a, f2_dup(b)); }
__device__ __forceinline__ F2 f2_rcp(F2 a) {
  float lo, hi;
  f2_unpack(a, lo, hi);
  return f2_pack(LEAN_RCP(lo), LEAN_RCP(hi));
}
__device__ __forceinline__ F2 f2_rsqrt(F2 a) {
  float lo, hi;
  f2_unpack(a, lo, hi);
  return f2_pack(LEAN_RSQRT(lo), LEAN_RSQRT(hi));
}

// what the hot loop needs of a verdict (the verify kernel also reads the projection and the half-widths)
struct LeanVerdict2 {
  bool accept[2], uncertain[2];
  int idx[2];
  float up[2], vp[2], hx[2], hy[2];
};

__device__ __forceinline__ LeanVerdict2 lean_tail2(const LeanCam& c, int width, F2 up, F2 vp, F2 hx, F2 hy, const bool (&pass)[2], const bool (&rej)[2]) {
  const F2 tx = f2_add(up, LEAN_MAGIC), ty = f2_add(vp, LEAN_MAGIC);
  const F2 rx = f2_add(tx, -LEAN_MAGIC), ry = f2_add(ty, -LEAN_MAGIC);  // exact
  const F2 dx = f2_fma(-1.0f, rx, up), dy = f2_fma(-1.0f, ry, vp);      // up - rx, one rounding as the subtraction has
  float txs[2], tys[2], dxs[2], dys[2], hxs[2], hys[2];
  f2_unpack(tx, txs[0], txs[1]);
  f2_unpack(ty, tys[0], tys[1]);
  f2_unpack(dx, dxs[0], dxs[1]);
  f2_unpack(dy, dys[0], dys[1]);
  f2_unpack(hx, hxs[0], hxs[1]);
  f2_unpack(hy, hys[0], hys[1]);
  LeanVerdict2 v;
  f2_unpack(up, v.up[0], v.up[1]);
  f2_unpack(vp, v.vp[0], v.vp[1]);
#pragma unroll
  for (int h = 0; h < 2; h++) {
    const bool cert = pass[h] & (fabsf(dxs[h]) < hxs[h]) & (fabsf(dys[h]) < hys[h]);
    const bool inside = (txs[h] >= c.t_lo) & (txs[h] <= c.t_hi) & (tys[h] >= c.s_lo) & (tys[h] <= c.s_hi);
    v.accept[h] = cert & inside;
    v.uncertain[h] = !cert & !rej[h];
    const int ixb = max(__float_as_int(txs[h]), LEAN_MAGIC_BITS), iyb = max(__float_as_int(tys[h]), LEAN_MAGIC_BITS);
    v.idx[h] = iyb * width + ixb - c.idx_bias;
    v.hx[h] = hxs[h], v.hy[h] = hys[h];
  }
  return v;
}

// atan2(a, b) / 2pi of both halves: the quotient and the polynomial packed, the octant folds per half (lean_atan2_turns)
__device__ __forceinline__ F2 lean_atan2_turns2(F2 a, F2 b) {
  float as[2], bs[2], mx[2], mn[2];
  f2_unpack(a, as[0], as[1]);
  f2_unpack(b, bs[0], bs[1]);
#pragma unroll
  for (int h = 0; h < 2; h++) {
    const float ax = fabsf(as[h]), bx = fabsf(bs[h]);
    mx[h] = fmaxf(ax, bx), mn[h] = fminf(ax, bx);
  }
  const F2 t = f2_mul(f2_pack(mn[0], mn[1]), f2_pack(LEAN_RCP(mx[0]), LEAN_RCP(mx[1])));
  const F2 s = f2_mul(t, t);
  F2 p = f2_fma(s, f2_dup(LEAN_ATAN_C6), LEAN_ATAN_C5);  // lean_atan_poly_turns
  p = f2_fma(s, p, LEAN_ATAN_C4);
  p = f2_fma(s, p, LEAN_ATAN_C3);
  p = f2_fma(s, p, LEAN_ATAN_C2);
  p = f2_fma(s, p, LEAN_ATAN_C1);
  p = f2_fma(s, p, LEAN_ATAN_C0);
  p = f2_mul(p, t);
  float ps[2];
  f2_unpack(p, ps[0], ps[1]);
#pragma unroll
  for (int h = 0; h < 2; h++) {
    float q = ps[h];
    q = fabsf(as[h]) > fabsf(bs[h]) ? 0.25f - q : q;
    q = bs[h] < 0.0f ? 0.5f - q : q;
    ps[h] = copysignf(q, as[h]);
  }
  return f2_pack(ps[0], ps[1]);
}

template <int MODEL>
struct LeanPacked {
  static constexpr bool value = MODEL == CAM_PLUMB_BOB || MODEL == CAM_EQUIRECTANGULAR;
};

// LeanAnchor of both points
struct LeanAnchor2 {
  F2 up0, vp0, gux, guz, gvx, gvy, gvz, irxz, hy, rad2;
};

// classify_lean_anchor for two points (also the equirectangular branch of classify_lean2)
template <int MODEL>
__device__ __forceinline__ LeanVerdict2 classify_lean2_anchor(const FastCam& f, const LeanCam& c, int width, const float* __restrict__ P, F2 X, F2 Y, F2 Z, F2 D, LeanAnchor2& an) {
  static_assert(MODEL == CAM_EQUIRECTANGULAR, "the delta step is derived for the equirectangular model");
  const F2 pcx = f2_fma(P[0], X, f2_fma(P[1], Y, f2_fma(P[2], Z, P[9])));
  const F2 pcy = f2_fma(P[3], X, f2_fma(P[4], Y, f2_fma(P[5], Z, P[10])));
  const F2 pcz = f2_fma(P[6], X, f2_fma(P[7], Y, f2_fma(P[8], Z, P[11])));
  const F2 xx = f2_mul(pcx, pcx);
  const F2 rxz2 = f2_fma(pcz, pcz, xx);
  const F2 n2 = f2_fma(pcy, pcy, rxz2);
  const F2 inv_n = f2_rsqrt(n2);
  const F2 nrm = f2_mul(n2, inv_n);
  const F2 inv_rxz = f2_rsqrt(rxz2);
  const F2 rxz = f2_mul(rxz2, inv_rxz);
  const F2 g = f2_fma(-f.cos_fov, nrm, pcz);
  const F2 mf = f2_fma(3.0f, D, f2_mul(12.0f * F32_U, nrm));
  const F2 lon = lean_atan2_turns2(pcx, pcz);
  const F2 lat = lean_atan2_turns2(pcy, rxz);
  const F2 up = f2_fma(lon, f2_dup(c.eq_su), c.cxh);
  const F2 vp = f2_fma(lat, f2_dup(c.eq_sv), c.cyh);
  const F2 t_lon = f2_mul(f2_mul(1.5f, D), inv_rxz);
  const F2 t_by = f2_fma(f2_mul(2.9f, D), inv_n, 4.0f * F32_U);
  const F2 t_asn = f2_mul(f2_mul(1.03f, t_by), f2_mul(nrm, inv_rxz));
  const F2 hx = f2_fma(c.nsfx, t_lon, c.hx0);
  const F2 hy = f2_fma(c.nsfy, t_asn, c.hy0);
  const F2 far = f2_mul(40.0f, D), pole = f2_mul(0.05f, nrm);
  // delta-step state (classify_lean_anchor)
  const F2 gu = f2_mul(c.eq_gu, f2_mul(inv_rxz, inv_rxz));
  const F2 gv = f2_mul(c.eq_gv, f2_mul(inv_n, inv_n));
  const F2 gvr = f2_mul(f2_mul(-1.0f, f2_mul(gv, pcy)), inv_rxz);
  an.up0 = up, an.vp0 = vp;
  an.gux = f2_mul(gu, pcz), an.guz = f2_mul(-1.0f, f2_mul(gu, pcx));
  an.gvx = f2_mul(gvr, pcx), an.gvy = f2_mul(gv, rxz), an.gvz = f2_mul(gvr, pcz);
  an.irxz = inv_rxz;
  an.hy = f2_add(hy, -c.eq_cv);
  const F2 gm = f2_add(g, f2_mul(-1.0f, mf)), ngm = f2_fma(-1.0f, g, f2_mul(-1.0f, mf));  // g - mf, -g - mf
  float n2s[2], rxzs[2], gs[2], mfs[2], fars[2], poles[2], pczs[2], pcxs[2], gms[2], ngms[2], rad2[2];
  f2_unpack(n2, n2s[0], n2s[1]);
  f2_unpack(rxz, rxzs[0], rxzs[1]);
  f2_unpack(g, gs[0], gs[1]);
  f2_unpack(mf, mfs[0], mfs[1]);
  f2_unpack(far, fars[0], fars[1]);
  f2_unpack(pole, poles[0], poles[1]);
  f2_unpack(pcz, pczs[0], pczs[1]);
  f2_unpack(pcx, pcxs[0], pcxs[1]);
  f2_unpack(gm, gms[0], gms[1]);
  f2_unpack(ngm, ngms[0], ngms[1]);
  bool pass[2], rej[2];
#pragma unroll
  for (int h = 0; h < 2; h++) {
    const bool ok = (n2s[h] > 2e-3f) & (rxzs[h] > fars[h]) & (rxzs[h] > poles[h]);
    pass[h] = ok & (gs[h] > mfs[h]);
    rej[h] = gs[h] < -mfs[h];
    const float r_seam = pczs[h] > 0.0f ? rxzs[h] : fabsf(pcxs[h]);
    const float r_pass = fminf(fminf(0.0625f * rxzs[h], r_seam), 0.49f * gms[h]);
    const float r_rej = 0.49f * ngms[h];
    rad2[h] = pass[h] ? (0.9999f * r_pass) * r_pass : (rej[h] ? -((0.9999f * r_rej) * r_rej) : 0.0f);
  }
  an.rad2 = f2_pack(rad2[0], rad2[1]);
  return lean_tail2(c, width, up, vp, hx, hy, pass, rej);
}

// classify_lean_delta for two points; Q: as written by lean_delta_pose
template <int MODEL>
__device__ __forceinline__ LeanVerdict2 classify_lean2_delta(const LeanCam& c, int width, const float* __restrict__ Q, F2 X, F2 Y, F2 Z, F2 D, const LeanAnchor2& an) {
  static_assert(MODEL == CAM_EQUIRECTANGULAR, "the delta step is derived for the equirectangular model");
  const F2 dx = f2_fma(Q[0], X, f2_fma(Q[1], Y, f2_fma(Q[2], Z, Q[9])));
  const F2 dy = f2_fma(Q[3], X, f2_fma(Q[4], Y, f2_fma(Q[5], Z, Q[10])));
  const F2 dz = f2_fma(Q[6], X, f2_fma(Q[7], Y, f2_fma(Q[8], Z, Q[11])));
  const F2 nd2 = f2_fma(dx, dx, f2_fma(dy, dy, f2_mul(dz, dz)));
  const F2 e1 = f2_fma(D, f2_dup(Q[12]), Q[13]);
  const F2 e8 = f2_fma(D, f2_dup(LEAN_DELTA_SQ3), e1);
  const F2 m2 = f2_fma(nd2, f2_dup(LEAN_DELTA_M2), f2_mul(e8, e8));
  const F2 up = f2_add(an.up0, f2_fma(an.gux, dx, f2_mul(an.guz, dz)));
  const F2 vp = f2_add(an.vp0, f2_fma(an.gvx, dx, f2_fma(an.gvy, dy, f2_mul(an.gvz, dz))));
  const F2 r2m2 = f2_mul(f2_mul(an.irxz, an.irxz), m2);
  const F2 lin = f2_mul(an.irxz, e1);
  const F2 tlx = f2_fma(-c.eq_lu, e1, f2_mul(c.eq_nsx15, D));
  const F2 hx = f2_fma(-c.eq_ku, r2m2, f2_fma(an.irxz, tlx, c.eq_hxd));
  const F2 hy = f2_fma(-c.eq_kv, r2m2, f2_fma(-c.eq_lv, lin, an.hy));
  float m2s[2], rads[2];
  f2_unpack(m2, m2s[0], m2s[1]);
  f2_unpack(an.rad2, rads[0], rads[1]);
  bool pass[2], rej[2];
#pragma unroll
  for (int h = 0; h < 2; h++) {
    pass[h] = m2s[h] < rads[h];
    rej[h] = m2s[h] < -rads[h];
  }
  return lean_tail2(c, width, up, vp, hx, hy, pass, rej);
}

// P: pose32 row as in classify_lean; X, Y, Z, D: coordinates and input-error bounds of the two points
template <int MODEL>
__device__ __forceinline__ LeanVerdict2 classify_lean2(const FastCam& f, const LeanCam& c, int width, const float* __restrict__ P, F2 X, F2 Y, F2 Z, F2 D) {
  static_assert(LeanPacked<MODEL>::value, "packed classifier: plumb_bob and equirectangular");
  const F2 pcx = f2_fma(P[0], X, f2_fma(P[1], Y, f2_fma(P[2], Z, P[9])));
  const F2 pcy = f2_fma(P[3], X, f2_fma(P[4], Y, f2_fma(P[5], Z, P[10])));
  const F2 pcz = f2_fma(P[6], X, f2_fma(P[7], Y, f2_fma(P[8], Z, P[11])));
  float pczs[2], ds[2];
  f2_unpack(pcz, pczs[0], pczs[1]);
  f2_unpack(D, ds[0], ds[1]);
  bool pass[2], rej[2];
  if constexpr (MODEL == CAM_PLUMB_BOB) {
    const F2 inv = f2_pack(LEAN_RCP(pczs[0]), LEAN_RCP(pczs[1]));
    const F2 xn = f2_mul(pcx, inv), yn = f2_mul(pcy, inv);
    const F2 rho = f2_mul(D, inv);
    const F2 x2 = f2_mul(xn, xn), y2 = f2_mul(yn, yn), xy = f2_mul(xn, yn);
    const F2 r2 = f2_add(x2, y2);
    const F2 rc = f2_fma(r2, f2_fma(r2, f2_fma(r2, f2_dup(f.d[4]), f.d[1]), f.d[0]), 1.0f);
    const float p1 = f.d[2], p2 = f.d[3];
    const F2 xd = f2_fma(xn, rc, f2_fma(2.0f * p1, xy, f2_mul(p2, f2_fma(2.0f, x2, r2))));
    const F2 yd = f2_fma(yn, rc, f2_fma(2.0f * p2, xy, f2_mul(p1, f2_fma(2.0f, y2, r2))));
    const F2 up = f2_fma(f.fx, xd, c.cxh);
    const F2 vp = f2_fma(f.fy, yd, c.cyh);
    const F2 r2b = f2_fma(r2, f2_dup(1.001f), 1e-6f);
    const F2 A = f2_fma(r2b, f2_fma(r2b, f2_fma(r2b, f2_fma(r2b, f2_dup(c.ea[4]), c.ea[3]), c.ea[2]), c.ea[1]), c.ea[0]);
    const F2 B = f2_fma(r2b, f2_fma(r2b, f2_fma(r2b, f2_fma(r2b, f2_dup(c.eb[4]), c.eb[3]), c.eb[2]), c.eb[1]), c.eb[0]);
    const F2 e = f2_fma(rho, A, B);
    const F2 hx = f2_fma(c.nsfx, e, c.hx0);
    const F2 hy = f2_fma(c.nsfy, e, c.hy0);
    const F2 exy3 = f2_fma(rho, f2_dup(c.C1x3), c.C2x3);
    const F2 fov_m = f2_fma(exy3, f2_add(r2, 1.0f), r2);
    const F2 rej_t = f2_fma(c.K3, rho, c.T2hi);
    float rhos[2], fovs[2], r2s[2], rts[2];
    f2_unpack(rho, rhos[0], rhos[1]);
    f2_unpack(fov_m, fovs[0], fovs[1]);
    f2_unpack(r2, r2s[0], r2s[1]);
    f2_unpack(rej_t, rts[0], rts[1]);
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const bool base = (pczs[h] > ds[h]) & (rhos[h] < 0.01f);
      pass[h] = base & (fovs[h] < c.T2lo);
      rej[h] = (base & (r2s[h] > rts[h])) | (pczs[h] < -ds[h]);
    }
    return lean_tail2(c, width, up, vp, hx, hy, pass, rej);
  } else {
    LeanAnchor2 unused;
    return classify_lean2_anchor<MODEL>(f, c, width, P, X, Y, Z, D, unused);
  }
}

}  // namespace vlcal
