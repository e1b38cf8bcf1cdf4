// numpy's summation order on the device: np.add.reduce of a contiguous vector (and along axis 0 of an [N, 1] array)
// is loops_utils.h pairwise_sum, from +0.  Blocks of <= 128 elements use eight strided accumulators
// ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)) and a sequential tail; longer runs split at n2 = n/2 - (n/2) % 8.
// Every add / multiply / divide is an explicit *_rn intrinsic, so no FMA is contracted.
#pragma once
#include "common.cuh"

namespace b200rl {

__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float div_rn(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double div_rn(double a, double b) { return __ddiv_rn(a, b); }

// pairwise_sum of the n <= 128 terms f(lo), ..., f(lo + n - 1) in the accumulator type R
template <typename R, typename F, typename I>
__device__ __forceinline__ R np_pairwise_block(F f, I lo, I n) {
  if (n < 8) {
    R res = R(0);
    for (I i = 0; i < n; ++i) res = add_rn(res, f(lo + i));
    return res;
  }
  R r[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) r[j] = f(lo + j);
  const I m = n - n % 8;
  for (I i = 8; i < m; i += 8) {
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = add_rn(r[j], f(lo + i + j));
  }
  R res = add_rn(add_rn(add_rn(r[0], r[1]), add_rn(r[2], r[3])), add_rn(add_rn(r[4], r[5]), add_rn(r[6], r[7])));
  for (I i = m; i < n; ++i) res = add_rn(res, f(lo + i));
  return res;
}

// pairwise_sum of the n terms f(lo), ..., f(lo + n - 1), by one thread
template <typename R, typename F, typename I>
__device__ R np_pairwise(F f, I lo, I n) {
  if (n <= 128) return np_pairwise_block<R>(f, lo, n);
  I n2 = n / 2;
  n2 -= n2 % 8;
  return add_rn(np_pairwise<R>(f, lo, n2), np_pairwise<R>(f, lo + n2, n - n2));
}

}  // namespace b200rl
