// Gumbel-max sampling of one categorical segment (CategoricalPd.sample, distributions.py:199-201), shared by the PPO2
// sampler (policy_heads.cu cat_step) and the ACER sampler (acer.cu acer_step) so that both draw the same action bits
// for the same seed and stream position.
#pragma once
#include "philox.cuh"

namespace b200rl {

// argmax_j (l[j] - log(-log(u_j))) over [lo, hi) of row b.  Uniform j is column j of the row's Philox stream at
// (seed, b, j / 4, offset), or uniforms[b * nA + j] when `uniforms` is given; rnd / held cache the 4 words of the
// last Philox counter across the segments of one row.  The first maximum wins (tf.argmax).
__device__ __forceinline__ int cat_gumbel_argmax(const float* l, int lo, int hi, int nA, const float* uniforms,
                                                 uint64_t seed, long long b, uint64_t offset, uint32_t (&rnd)[4],
                                                 int& held) {
  float best = -INFINITY;
  int a = lo;
  for (int j = lo; j < hi; ++j) {
    float u;
    if (uniforms) {
      u = uniforms[b * nA + j];
    } else {
      if ((j >> 2) != held) {
        held = j >> 2;
        philox4(seed, (uint64_t)b, (uint32_t)held, (uint32_t)offset, rnd);
      }
      u = u01_open(rnd[j & 3]);
    }
    const float sc = l[j] - logf(-logf(u));
    if (sc > best) { best = sc; a = j; }
  }
  return a;
}

}  // namespace b200rl
