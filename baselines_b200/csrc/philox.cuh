// The project's counter-based random stream: Philox4x32-10 keyed by a seed, counted by (row, column block, stream
// position).  Shared by the samplers of policy_heads.cu and the parameter perturbation of param_noise.cu.
#pragma once
#include <stdint.h>

namespace b200rl {

// ---------------------------------------------------------------- Philox4x32-10 (counter based)
__device__ __forceinline__ void philox_round(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
  const uint32_t hi0 = __umulhi(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
  const uint32_t hi1 = __umulhi(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
  const uint32_t n0 = hi1 ^ c[1] ^ k0, n1 = lo1, n2 = hi0 ^ c[3] ^ k1, n3 = lo0;
  c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
}
__device__ __forceinline__ void philox4(uint64_t seed, uint64_t row, uint32_t ctr, uint32_t stream,
                                        uint32_t (&out)[4]) {
  uint32_t c[4] = {(uint32_t)row, (uint32_t)(row >> 32), ctr, stream};
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    philox_round(c, k0, k1);
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) out[i] = c[i];
}
__device__ __forceinline__ float u01_open(uint32_t x) { return ((float)(x >> 8) + 0.5f) * (1.0f / 16777216.0f); }

}  // namespace b200rl
