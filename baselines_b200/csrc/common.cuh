// Shared device/host helpers for libb200rl (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

// The entry points are defined extern "C" against these prototypes: a definition whose parameter types differ from
// the header's is a compile error, not a second overload.
#include "../../include/b200rl.h"

namespace b200rl {

void set_last_error(const char* fmt, ...);

inline int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error("%s: %s", what, cudaGetErrorString(e));
    return B200RL_ERR_CUDA;
  }
  return B200RL_OK;
}

#define B200RL_REQUIRE(cond, ...)                 \
  do {                                            \
    if (!(cond)) {                                \
      ::b200rl::set_last_error(__VA_ARGS__);      \
      return B200RL_ERR_ARG;                      \
    }                                             \
  } while (0)

__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
__host__ __device__ inline long long ceil_div_ll(long long a, long long b) { return (a + b - 1) / b; }

// Deterministic cross-CTA reductions: instead of float atomics (whose order, and so whose rounding, changes from run
// to run) every CTA stores its partial result into a device workspace and sum_partials() adds the parts in index order.
// det_workspace() returns a per-device buffer of at least `floats` floats; it only grows outside stream capture, and a
// buffer is never freed, so captured graphs keep valid pointers.  Its users must be ordered on the device: every
// reduction of the training path is issued on the caller's current stream.
float* det_workspace(size_t floats, cudaStream_t stream);
// out[r * ldo + c] += sum_{p < parts} ws[(p * rows + r) * cols + c], parts summed in order
int sum_partials(const float* ws, int parts, long long rows, int cols, float* out, long long ldo, cudaStream_t stream);
int device_num_sms();   // streaming multiprocessors of the current device (grid sizing)
// grid of a grid-stride kernel over `work` items: one thread per item, at most per_sm CTAs per SM, at least one CTA
inline int grid_blocks(long long work, int threads, int per_sm) {
  const long long blocks = ceil_div_ll(work, threads), cap = (long long)per_sm * device_num_sms();
  return (int)(blocks < 1 ? 1 : (blocks < cap ? blocks : cap));
}

#ifdef __CUDACC__
// ------------------------------------------------------------------ mbarrier / TMA / wgmma PTX
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
// the transaction count of the current phase, without an arrival (the caller arrives once its own writes are done)
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.expect_tx.relaxed.cta.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// try_wait suspends the warp until the phase completes or the hint expires; without a hint the default time limit is
// short and the polling loop (YIELD / TRYWAIT / BRA) of the waiting warps takes issue slots the producer and
// consumer warps need.
static constexpr uint32_t MBAR_SUSPEND_NS = 20000;
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(MBAR_SUSPEND_NS)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ------------------------------------------------------------------ thread-block clusters
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t cluster_nctarank() {
  uint32_t n;
  asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(n));
  return n;
}
// every thread of every CTA of the cluster arrives (release) and waits (acquire)
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}
// arrive on the mbarrier at `bar`'s shared-memory offset in CTA `rank` of the cluster.  Default (CTA-scope) release:
// a cluster-scope release compiles to a GPU-wide MEMBAR in front of every arrival.  Releasing a stage needs none:
// the reads it orders are the caller's wgmma operand reads, complete once wgmma.wait_group returns.
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t rank) {
  asm volatile(
      "{\n\t.reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.shared::cluster.b64 _, [ra];\n\t}"
      ::"r"(smem_u32(bar)), "r"(rank)
      : "memory");
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}
// tma_load_2d into the same shared-memory offset of every CTA of the cluster in `mask` (bit r: rank r); each
// destination's barrier at `bar`'s offset receives the box's bytes
__device__ __forceinline__ void tma_load_2d_multicast(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar, int c0,
                                                      int c1, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(mask)
      : "memory");
}
// 1-D bulk copy global -> shared (no tensor map)
__device__ __forceinline__ void bulk_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// wgmma.mma_async ordering: fence before the first MMA that touches accumulator registers written by ordinary
// instructions; MMAs issued since the last commit form a group; wait until at most N groups are pending.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// ------------------------------------------------------------------ small reductions
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// One CTA of N threads: thread 0 returns the N values v added in thread order from +0 (the others return 0).  red: N
// floats of shared memory, free for reuse when the call returns.
template <int N>
__device__ __forceinline__ float cta_sum_in_order(float v, float* red) {
  red[threadIdx.x] = v;
  __syncthreads();
  float t = 0.0f;
  if (threadIdx.x == 0)
    for (int k = 0; k < N; ++k) t = __fadd_rn(t, red[k]);
  __syncthreads();
  return t;
}

// ------------------------------------------------------------------ fp16 [hi | lo] operand rows (obs_encode.cu)
// v = hi + lo with hi = fp16(v), lo = fp16(v - hi): v - hi is exact in fp32
__device__ __forceinline__ void split_f16(float v, __half& hi, __half& lo) {
  const __half h = __float2half_rn(v);
  hi = h;
  lo = __float2half_rn(v - __half2float(h));
}
// some |v[j]| >= 65520, which rounds hi to +-inf (a NaN compares false: it passes through)
__device__ __forceinline__ bool f16_overflow8(const float (&v)[8]) {
  bool over = false;
#pragma unroll
  for (int j = 0; j < 8; ++j) over |= fabsf(v[j]) >= 65520.0f;
  return over;
}
// eight columns of an operand row [hi(0..in_pad) | lo(0..in_pad)]: o points at the first (16-byte aligned) hi column
__device__ __forceinline__ void store_split_f16x8(__half* o, int in_pad, const float (&v)[8]) {
  __align__(16) __half hi[8], lo[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) split_f16(v[j], hi[j], lo[j]);
  *reinterpret_cast<uint4*>(o) = *reinterpret_cast<const uint4*>(hi);
  *reinterpret_cast<uint4*>(o + in_pad) = *reinterpret_cast<const uint4*>(lo);
}
#endif  // __CUDACC__

}  // namespace b200rl
