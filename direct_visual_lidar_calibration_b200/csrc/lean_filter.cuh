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
};

// atan2(a, b) / (2 pi) in turns, (-0.5, 0.5]: octant reduction + odd minimax polynomial of degree 13 on [0, 1] (fitted for
// this file, tools/fit_atan_turns.py; fp32 Horner error <= 5.3e-8 turns) -- 20 instructions and one MUFU.RCP against ~40
// for atan2f, whose special cases (infinities, signed zeros, denormals) the filter does not need: every degenerate input
// comes out NaN or lands on a pixel edge, i.e. "uncertain".  Absolute error <= 1.1e-7 turns (polynomial 5.3e-8, quotient
// rounding 1.4e-8, octant folds 4.5e-8); LEAN_ATAN_ERR_TURNS is what the error bound charges for it.
constexpr double LEAN_ATAN_ERR_TURNS = 2.5e-7;
VL_HD float lean_atan2_turns(float a, float b) {
  const float ax = fabsf(a), bx = fabsf(b);
  const float mx = fmaxf(ax, bx), mn = fminf(ax, bx);
  const float t = mn * VL_RCPF(mx);
  const float s = t * t;
  float p = fmaf(s, 0.0010841299081221223f, -0.005348276346921921f);
  p = fmaf(s, p, 0.012672499753534794f);
  p = fmaf(s, p, -0.021061519160866737f);
  p = fmaf(s, p, 0.03152511641383171f);
  p = fmaf(s, p, -0.0530262365937233f);
  p = fmaf(s, p, 0.15915432572364807f);
  p = p * t;                          // atan(mn / mx) / 2pi in [0, 1/8]
  p = ax > bx ? 0.25f - p : p;        // first quadrant
  p = b < 0.0f ? 0.5f - p : p;        // upper half plane
  return copysignf(p, a);
}

struct LeanVerdict {
  bool accept;     // the reference certainly counts this point at pixel `idx`
  bool uncertain;  // within the error bound of a decision edge: ask the exact path
  int idx;         // iy * W + ix, meaningful when accept
  int ixb, iyb;    // ix + LEAN_MAGIC_BITS, iy + LEAN_MAGIC_BITS (the rounded coordinates as they come out of the magic add)
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
  v.ixb = ixb, v.iyb = iyb;
  v.up = up, v.vp = vp, v.hx = hx, v.hy = hy;
  return v;
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
    return lean_tail(c, width, up, vp, hx, hy, pass, rej);
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
