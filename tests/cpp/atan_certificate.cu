// Exhaustive certificate of the arctangent polynomial of the lean classifier (csrc/lean_filter.cuh, lean_atan_poly_turns):
// for EVERY float t in [0, 1 + 2^-20] (1 065 353 225 values, denormals included), the fp32 evaluation as the kernel
// compiles it -- the same function, fmaf rounded once, no contraction (-ffp-contract=off) -- against atan(t) / 2pi in long
// double (64-bit significand: its error is ~1e-19 turns, four orders below what is measured).  Also measured: the same
// value with the last product t * P(t^2) left unrounded, which is what the device computes if the compiler contracts that
// product into the octant fold's subtraction.  Then the whole routine lean_atan2_turns on random (a, b) pairs against
// atan2l, which must stay within the certified sum LEAN_ATAN_CERT_TURNS.  Prints one JSON object.
// Built host-only with OpenMP by tests/test_atan_certificate_host.py (nvcc, no device code is run).
#include <omp.h>

#include <cinttypes>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <vector>

#include "lean_filter.cuh"

using namespace vlcal;

static float from_bits(uint32_t b) {
  float f;
  std::memcpy(&f, &b, sizeof(f));
  return f;
}
static uint32_t to_bits(float f) {
  uint32_t b;
  std::memcpy(&b, &f, sizeof(b));
  return b;
}

static const long double TWO_PI = 6.283185307179586476925286766559005768L;

struct Acc {
  long double err_r = 0.0L, err_u = 0.0L;  // max |error| with the last product rounded / unrounded
  float t_r = 0.0f, t_u = 0.0f;
  float p_min = INFINITY, p_max = -INFINITY;
  unsigned long long nan = 0;
  char pad[64];
};

int main(int argc, char** argv) {
  const long long n_pairs = argc > 1 ? std::atoll(argv[1]) : 20000000LL;
  const uint32_t hi = to_bits(1.0f) + 8u;  // 1 + 8 * 2^-23 = 1 + 2^-20
  const int nt = omp_get_max_threads();
  std::vector<Acc> acc(nt);
#pragma omp parallel
  {
    Acc& a = acc[omp_get_thread_num()];
#pragma omp for schedule(dynamic, 1 << 20)
    for (long long b = 0; b <= static_cast<long long>(hi); b++) {
      const float t = from_bits(static_cast<uint32_t>(b));
      const float p = lean_atan_poly_turns(t);
      const long double pu = static_cast<long double>(lean_atan_horner(t * t)) * static_cast<long double>(t);  // exact product
      const long double ref = atanl(static_cast<long double>(t)) / TWO_PI;
      const long double er = fabsl(static_cast<long double>(p) - ref), eu = fabsl(pu - ref);
      if (!(er <= 1.0L) || !(eu <= 1.0L)) a.nan++;
      if (er > a.err_r) a.err_r = er, a.t_r = t;
      if (eu > a.err_u) a.err_u = eu, a.t_u = t;
      a.p_min = std::fmin(a.p_min, p), a.p_max = std::fmax(a.p_max, p);
    }
  }
  Acc tot;
  for (const Acc& a : acc) {
    if (a.err_r > tot.err_r) tot.err_r = a.err_r, tot.t_r = a.t_r;
    if (a.err_u > tot.err_u) tot.err_u = a.err_u, tot.t_u = a.t_u;
    tot.p_min = std::fmin(tot.p_min, a.p_min), tot.p_max = std::fmax(tot.p_max, a.p_max);
    tot.nan += a.nan;
  }

  // the whole routine on random pairs: signs, octants and magnitudes spread over 2^-20 .. 2^20; a sprinkle of |a| == |b|
  std::vector<long double> worst(nt, 0.0L);
#pragma omp parallel
  {
    const int id = omp_get_thread_num();
    std::mt19937_64 rng(12345u + 7919u * static_cast<unsigned>(id));
    std::uniform_real_distribution<double> U(-1.0, 1.0), E(-20.0, 20.0);
    long double w = 0.0L;
#pragma omp for
    for (long long i = 0; i < n_pairs; i++) {
      const float a = static_cast<float>(U(rng) * std::exp2(E(rng)));
      const float b = (i % 64 == 0) ? std::copysign(a, static_cast<float>(U(rng))) : static_cast<float>(U(rng) * std::exp2(E(rng)));
      if (a == 0.0f) continue;
      const long double ref = atan2l(static_cast<long double>(a), static_cast<long double>(b)) / TWO_PI;
      const long double e = fabsl(static_cast<long double>(lean_atan2_turns(a, b)) - ref);
      if (!(e <= w)) w = (e == e) ? e : 1.0L;
    }
    worst[id] = w;
  }
  long double w = 0.0L;
  for (long double x : worst) w = std::fmax(w, x);

  const double U = 5.9604644775390625e-08;
  std::printf("{\"values\": %" PRIu32 ", \"t_hi\": %.9g, \"max_err_rounded\": %.6Le, \"t_at_max_rounded\": %.9g, \"max_err_unrounded\": %.6Le, \"t_at_max_unrounded\": %.9g, "
              "\"p_min\": %.9g, \"p_max\": %.9g, \"non_finite\": %llu, \"pairs\": %lld, \"pairs_max_err\": %.6Le, "
              "\"poly_bound\": %.6e, \"quot_bound\": %.6e, \"quot_formula\": %.6e, \"fold_bound\": %.6e, \"fold_formula\": %.6e, \"cert\": %.6e, \"charged\": %.6e}\n",
              hi + 1u, from_bits(hi), tot.err_r, tot.t_r, tot.err_u, tot.t_u, tot.p_min, tot.p_max, tot.nan, n_pairs, w, LEAN_ATAN_POLY_ERR_TURNS, LEAN_ATAN_QUOT_ERR_TURNS,
              (3.0 * U + 2.0 * U * U) / (4.0 * M_PI) * (1.0 + 1e-6), LEAN_ATAN_FOLD_ERR_TURNS, std::ldexp(1.0, -27) + std::ldexp(1.0, -26), LEAN_ATAN_CERT_TURNS, LEAN_ATAN_ERR_TURNS);
  return 0;
}
