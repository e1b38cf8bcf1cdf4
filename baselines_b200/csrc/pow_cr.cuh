// Correctly rounded pow(x, y) for the prioritized-replay arithmetic (replay.cu).
//
// The replay buffer's leaves are priority ** alpha and its importance weights (p * n) ** -beta.  The reference
// evaluates both with the host libm, so a leaf or weight is reproducible only if host and device round pow the same
// way.  CUDA's pow is documented to 2 ulp, and glibc's current pow to 0.52 ulp, so neither is an exact target.  The one
// value both can be held to is the correctly rounded result, which is what this computes:
//   log(x) as a double-double: x = m * 2^e with m in [1/sqrt2, sqrt2); log(m) = l0 + log1p(m * exp(-l0) - 1), one
//     Newton step from l0 = log(m) with exp evaluated in double-double (quadratic convergence: ~2^-100 absolute);
//   z = y * log(x) as a double-double;
//   exp(z): z = k*ln2 + r, exp(r) = (1 + q)^(2^8) with q = expm1(r / 2^8) from its Taylor series to degree 11, squared
//     eight times in the expm1 form q <- 2q + q^2 to keep its relative precision;
//   one final rounding of 1 + q, then the exact scaling by 2^k.
// The result is within ~2^-89 relative of x^y before that rounding, so it is the correctly rounded value unless x^y lies
// that close to a midpoint of two doubles; for |y| <= 1 and y != 0 the midpoints are never hit exactly (x^y would need
// 54 significant bits from a 53-bit x).  Results outside about [2^-1009, 2^1009] (never reached by the replay
// arithmetic), x <= 0, and non-finite arguments fall back to the platform pow.
//
// Every multiply-add is an explicit fma and, on the device, every other add and multiply an explicit _rn intrinsic, so
// the host build and the device build (-fmad=true) perform the same operations.
#pragma once
#include <cmath>

namespace b200rl {
namespace powcr {

#if defined(__CUDACC__)
#define B200RL_HD __host__ __device__ __forceinline__
#else
#define B200RL_HD inline
#endif

// The dd algorithms rely on each operation being rounded on its own: nvcc would contract a product feeding a later sum
// (fast_two_sum(p, e) after p = a * b) into an fma and break the error terms, so on the device every add and multiply
// is an explicit round-to-nearest intrinsic, which is never contracted.
#if defined(__CUDA_ARCH__)
#define ADD(a, b) __dadd_rn((a), (b))
#define SUB(a, b) __dsub_rn((a), (b))
#define MUL(a, b) __dmul_rn((a), (b))
#else
#define ADD(a, b) ((a) + (b))
#define SUB(a, b) ((a) - (b))
#define MUL(a, b) ((a) * (b))
#endif

struct dd { double hi, lo; };

B200RL_HD dd two_sum(double a, double b) {
  const double s = ADD(a, b), bb = SUB(s, a);
  return {s, ADD(SUB(a, SUB(s, bb)), SUB(b, bb))};
}
B200RL_HD dd fast_two_sum(double a, double b) {            // |a| >= |b| (or a == 0)
  const double s = ADD(a, b);
  return {s, SUB(b, SUB(s, a))};
}
B200RL_HD dd add(dd x, dd y) {
  dd s = two_sum(x.hi, y.hi);
  const dd t = two_sum(x.lo, y.lo);
  s = fast_two_sum(s.hi, ADD(s.lo, t.hi));
  return fast_two_sum(s.hi, ADD(s.lo, t.lo));
}
B200RL_HD dd mul(dd x, dd y) {
  const double p = MUL(x.hi, y.hi);
  double e = fma(x.hi, y.hi, -p);
  e = fma(x.hi, y.lo, e);
  e = fma(x.lo, y.hi, e);
  return fast_two_sum(p, e);
}
B200RL_HD dd mul_d(dd x, double y) {
  const double p = MUL(x.hi, y);
  double e = fma(x.hi, y, -p);
  e = fma(x.lo, y, e);
  return fast_two_sum(p, e);
}

// expm1(r) for |r| <= ~0.35, as a double-double
B200RL_HD dd expm1_small(dd r) {
  const dd s{MUL(r.hi, 0x1p-8), MUL(r.lo, 0x1p-8)};                  // exact
  const dd inv_fact[10] = {                                   // 1/n!, n = 2 .. 11
      {0x1p-1, 0.0},
      {0x1.5555555555555p-3, 0x1.5555555555555p-57},
      {0x1.5555555555555p-5, 0x1.5555555555555p-59},
      {0x1.1111111111111p-7, 0x1.1111111111111p-63},
      {0x1.6c16c16c16c17p-10, -0x1.f49f49f49f49fp-65},
      {0x1.a01a01a01a01ap-13, 0x1.a01a01a01a01ap-73},
      {0x1.a01a01a01a01ap-16, 0x1.a01a01a01a01ap-76},
      {0x1.71de3a556c734p-19, -0x1.c154f8ddc6c00p-73},
      {0x1.27e4fb7789f5cp-22, 0x1.cbbc05b4fa99ap-76},
      {0x1.ae64567f544e4p-26, -0x1.c062e06d1f209p-80}};
  dd p = inv_fact[9];
  for (int n = 8; n >= 0; --n) p = add(mul(p, s), inv_fact[n]);
  dd q = mul(add(mul(p, s), dd{1.0, 0.0}), s);               // s + s^2/2! + ... + s^11/11!
  for (int i = 0; i < 8; ++i) q = add(mul_d(q, 2.0), mul(q, q));     // (1 + q)^2 = 1 + (2q + q^2)
  return q;
}

B200RL_HD dd ln2_times(double k) {                            // k * ln2 for |k| < 2^11, to ~2^-150 absolute
  const double p1 = MUL(k, 0x1.62e42fefa39efp-1), p2 = MUL(k, 0x1.abc9e3b39803fp-56);
  const dd a = two_sum(p1, fma(k, 0x1.62e42fefa39efp-1, -p1));
  const dd b{p2, fma(k, 0x1.7b57a079a1934p-111, fma(k, 0x1.abc9e3b39803fp-56, -p2))};
  return add(a, b);
}

B200RL_HD dd log_dd(double x) {                               // x > 0, finite
  int e;
  double m = frexp(x, &e);                                    // [0.5, 1)
  if (m < 0x1.6a09e667f3bcdp-1) { m = MUL(m, 2.0); e -= 1; }         // [1/sqrt2, sqrt2)
  const double l0 = log(m);
  const dd q = expm1_small(dd{-l0, 0.0});                      // exp(-l0) = 1 + q
  const dd t = add(dd{SUB(m, 1.0), 0.0}, mul_d(q, m));            // m * exp(-l0) - 1; m - 1 is exact
  // log1p(t) = t - t^2/2 + O(t^3), |t| ~ 2^-52
  const dd lm = add(dd{l0, 0.0}, add(t, dd{MUL(-0.5, MUL(t.hi, t.hi)), 0.0}));
  return add(ln2_times((double)e), lm);
}

B200RL_HD double pow_cr(double x, double y) {
  if (y == 0.0 || x == 1.0) return 1.0;
  if (y == 1.0) return x;
  if (!(x > 0.0) || !(fabs(x) < INFINITY) || !(fabs(y) < INFINITY)) return pow(x, y);
  const dd z = mul_d(log_dd(x), y);
  if (!(fabs(z.hi) < 700.0)) return pow(x, y);
  const double k = rint(MUL(z.hi, 0x1.71547652b82fep0));         // z / ln2
  const dd kl = ln2_times(k);
  const dd r = add(z, dd{-kl.hi, -kl.lo});
  const dd v = add(dd{1.0, 0.0}, expm1_small(r));
  return ldexp(v.hi, (int)k);
}

#undef ADD
#undef SUB
#undef MUL
#undef B200RL_HD

}  // namespace powcr
}  // namespace b200rl
