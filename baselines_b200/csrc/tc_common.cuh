// Device helpers shared by the wgmma GEMM / convolution kernels.
#pragma once
#include "common.cuh"
#include "wgmma.cuh"

namespace b200rl {

enum : int { MODE_F16_ACT = 0, MODE_F32_STORE = 1, MODE_F32_ATOMIC = 2, MODE_F16_DACT = 3, MODE_F16_SHUFFLE = 4 };
enum : int { ACT_NONE = 0, ACT_RELU = 1, ACT_TANH = 2 };

// wgmma shared-memory matrix descriptor; layout: 1 = SWIZZLE_128B, 2 = SWIZZLE_64B, 3 = SWIZZLE_32B.
// The swizzle is a function of the shared-memory address, so a descriptor may start at any 16-byte column of any row.
__host__ __device__ constexpr uint32_t sdesc_layout(int row_bytes) {
  return row_bytes == 128 ? 1u : row_bytes == 64 ? 2u : 3u;
}
__device__ __forceinline__ uint64_t make_sdesc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t layout) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= (uint64_t)layout << 62;
  return d;
}

// Register position of accumulator element e (0 .. N/2-1) of a m64nN wgmma tile for thread t of the warpgroup:
// row = 16*(t/32) + (t%32)/4 + 8*((e/2)%2), column = 8*(e/4) + 2*(t%4) + e%2.
__device__ __forceinline__ int acc_row(int t, int e) { return 16 * (t >> 5) + ((t & 31) >> 2) + 8 * ((e >> 1) & 1); }
__device__ __forceinline__ int acc_col(int t, int e) { return 8 * (e >> 2) + 2 * (t & 3) + (e & 1); }

__device__ __forceinline__ void tma_load_im2col_4d(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar, int c, int w,
                                                   int h, int n, uint16_t off_w, uint16_t off_h) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};"
      ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c), "r"(w), "r"(h), "r"(n), "h"(off_w), "h"(off_h)
      : "memory");
}

__device__ __forceinline__ float apply_act(float x, int act) {
  if (act == ACT_RELU) return fmaxf(x, 0.0f);
  if (act == ACT_TANH) return tanhf(x);
  return x;
}
__device__ __forceinline__ float act_grad_from_saved(float h, int act) {
  if (act == ACT_RELU) return h > 0.0f ? 1.0f : 0.0f;
  if (act == ACT_TANH) return 1.0f - h * h;
  return 1.0f;
}

// Ordered MMA issue of the two consumer warpgroups under the ping-pong schedule (barrier 0 is __syncthreads, 1 joins the
// consumer warps where a kernel needs it).  Group g waits on barrier ORDER_BAR + g for its turn and hands the turn over
// with an arrive on the other group's barrier: every wait is matched by exactly one arrive, so neither group may skip
// one while the other waits.
static constexpr int ORDER_BAR = 2;
__device__ __forceinline__ void order_wait(int wg) {
  asm volatile("bar.sync %0, %1;" ::"r"(ORDER_BAR + wg), "n"(256) : "memory");
}
__device__ __forceinline__ void order_pass(int wg) {
  asm volatile("bar.arrive %0, %1;" ::"r"(ORDER_BAR + 1 - wg), "n"(256) : "memory");
}

// Epilogue transpose: the accumulator fragment of one warp (16 rows; thread t holds 2 columns of rows t/4 and t/4 + 8 per
// 8-column block) goes through a per-warp scratch of 16 rows x 64 B so that each lane then holds 8 consecutive columns
// of one row.  16-byte piece p of scratch row r lives at slot p ^ ((r >> 1) & 3): the 8 rows of one stmatrix matrix,
// and the 8 lanes of a quarter-warp load, hit 8 distinct 16-byte slots of 128 B (no bank conflict).
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, const uint32_t (&r)[4]) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r[0]), "r"(r[1]),
               "r"(r[2]), "r"(r[3])
               : "memory");
}
// stmatrix's inverse: the same lane addresses give back the fragment layout (used to read an operand tile of the
// epilogue, staged row by row in the scratch, into the accumulator layout)
__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr)
               : "memory");
}
__device__ __forceinline__ void st_shared_v4(uint32_t addr, const uint4& v) {
  asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint4 ld_shared_v4(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
  return v;
}
// (a plain uint4 store is split into four 4-byte stores by the compiler here)
__device__ __forceinline__ void st_global_v4(void* p, const uint4& v) {
  asm volatile("st.global.v4.b32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint32_t h2_bits(__half2 h) { return *reinterpret_cast<const uint32_t*>(&h); }
// bits 2k, 2k + 1 of b8 -> 0xffff in the low / high half of the word (the mask of fp16 elements 2k, 2k + 1)
__device__ __forceinline__ uint32_t mask_pair(uint32_t b8, int k) {
  const uint32_t b = b8 >> (2 * k);
  return ((b & 1u) | ((b & 2u) << 15)) * 0xffffu;
}


// host helpers implemented in gemm_wgmma.cu
int make_tmap_2d_f16(CUtensorMap* tm, const void* ptr, long long rows, long long cols, long long ld, int box_cols,
                     int box_rows);

}  // namespace b200rl
