// GAE(lambda) backward scan over an HBM-resident [T, N] rollout (time-major, env contiguous).
//
// Replaces the numpy loop of baselines/ppo2/runner.py:53-65 (reference) and reproduces its dtype
// behaviour bit for bit: gamma*V(t+1) is a float32 product, delta / lastgaelam are carried in
// float64, advs are rounded to float32 on store, returns = advs + values is a float32 add.
// The recurrence is evaluated in the reference's association order with explicit *_rn intrinsics
// (no FMA contraction), so outputs are bit-identical to the reference.
//
// Algorithmic bytes per (t, env) element: r(4) + V(4) + done(1) read, adv(4) + ret(4) written = 17 B.
//
// Two kernels:
//   gae_tma_kernel   (default when N % 32 == 0): one warp per 32 envs; 32-step x 32-env tiles are staged
//       through a 4-deep shared-memory ring by 2-D TMA tile loads (cp.async.bulk.tensor + mbarrier
//       tx-count, three loads per tile), so ~36 KB per warp is in flight without holding registers; lanes
//       read their env's column conflict-free; outputs are 128 B coalesced streaming stores.
//   gae_direct_kernel (any N): thread per env with a 16-step register prefetch.
#include "common.cuh"

namespace b200rl {

struct GaeStep {
  double last;    // lastgaelam (float64 carry)
  float next_v;   // V(t+1)
  double nnt;     // 1.0 - done(t+1)
  float gamma_f;
  double gl;      // gamma*lam in float64 (python float product)

  __device__ __forceinline__ void step(float r, float v, uint8_t d, float& adv, float& ret) {
    const float gv = __fmul_rn(gamma_f, next_v);                           // float32 product (runner.py:63)
    const double delta = __dsub_rn(__dadd_rn((double)r, __dmul_rn((double)gv, nnt)), (double)v);
    last = __dadd_rn(delta, __dmul_rn(__dmul_rn(gl, nnt), last));          // runner.py:64
    adv = __double2float_rn(last);
    ret = __fadd_rn(adv, v);                                               // runner.py:65
    next_v = v;
    nnt = d ? 0.0 : 1.0;                                                   // 1.0 - mb_dones[t] for step t-1
  }
};

template <int U>
__global__ void __launch_bounds__(64)
gae_direct_kernel(const float* __restrict__ rew, const float* __restrict__ val, const uint8_t* __restrict__ done,
                  const float* __restrict__ last_val, const uint8_t* __restrict__ last_done,
                  float* __restrict__ adv, float* __restrict__ ret, int T, int N, float gamma_f, double gl) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= N) return;
  GaeStep st;
  st.last = 0.0;
  st.next_v = last_val[e];
  st.nnt = last_done[e] ? 0.0 : 1.0;
  st.gamma_f = gamma_f;
  st.gl = gl;
  for (int t1 = T; t1 > 0; t1 -= U) {
    float r[U], v[U];
    uint8_t d[U];
#pragma unroll
    for (int i = 0; i < U; ++i) {
      const int t = t1 - 1 - i;
      if (t >= 0) {
        const size_t o = (size_t)t * N + e;
        r[i] = __ldg(rew + o);
        v[i] = __ldg(val + o);
        d[i] = __ldg(done + o);
      }
    }
#pragma unroll
    for (int i = 0; i < U; ++i) {
      const int t = t1 - 1 - i;
      if (t >= 0) {
        float a, rt;
        st.step(r[i], v[i], d[i], a, rt);
        const size_t o = (size_t)t * N + e;
        adv[o] = a;
        ret[o] = rt;
      }
    }
  }
}

static constexpr int GAE_TT = 32;  // timesteps per stage
static constexpr int GAE_NS = 4;   // ring depth

struct __align__(128) GaeStage {
  float r[GAE_TT][32];
  float v[GAE_TT][32];
  uint8_t d[GAE_TT][32];
};

// One warp per 32 envs.  Each 32-step x 32-env tile is fetched by THREE 2-D TMA tile loads (rewards,
// values, dones) into a 4-deep smem ring; tiles beyond T are zero-filled by TMA and never read.
__global__ void __launch_bounds__(32)
gae_tma_kernel(const __grid_constant__ CUtensorMap tm_rew, const __grid_constant__ CUtensorMap tm_val,
               const __grid_constant__ CUtensorMap tm_done, const float* __restrict__ last_val,
               const uint8_t* __restrict__ last_done, float* __restrict__ adv, float* __restrict__ ret, int T, int N,
               float gamma_f, double gl) {
  __shared__ GaeStage stage[GAE_NS];
  __shared__ __align__(8) uint64_t full[GAE_NS];
  const int lane = threadIdx.x;
  const int e0 = blockIdx.x * 32;
  const int e = e0 + lane;
  const int nchunks = (T + GAE_TT - 1) / GAE_TT;

  if (lane == 0) {
    tma_prefetch_desc(&tm_rew);
    tma_prefetch_desc(&tm_val);
    tma_prefetch_desc(&tm_done);
    for (int s = 0; s < GAE_NS; ++s) mbar_init(&full[s], 1);
    fence_barrier_init();
  }
  __syncwarp();

  auto issue = [&](int c, int s) {
    if (lane == 0) {
      mbar_arrive_expect_tx(&full[s], (uint32_t)(GAE_TT * (128 + 128 + 32)));
      tma_load_2d(&stage[s].r[0][0], &tm_rew, &full[s], e0, c * GAE_TT);
      tma_load_2d(&stage[s].v[0][0], &tm_val, &full[s], e0, c * GAE_TT);
      tma_load_2d(&stage[s].d[0][0], &tm_done, &full[s], e0, c * GAE_TT);
    }
  };

  for (int i = 0; i < GAE_NS && i < nchunks; ++i) issue(nchunks - 1 - i, i);

  GaeStep st;
  st.last = 0.0;
  st.next_v = last_val[e];
  st.nnt = last_done[e] ? 0.0 : 1.0;
  st.gamma_f = gamma_f;
  st.gl = gl;

  int s = 0;
  uint32_t ph = 0;
  for (int c = nchunks - 1; c >= 0; --c) {
    mbar_wait(&full[s], ph);
    const int t0 = c * GAE_TT;
    const int rows = min(GAE_TT, T - t0);
#pragma unroll 8
    for (int i = rows - 1; i >= 0; --i) {
      float a, rt;
      st.step(stage[s].r[i][lane], stage[s].v[i][lane], stage[s].d[i][lane], a, rt);
      const size_t o = (size_t)(t0 + i) * N + e;
      __stcs(adv + o, a);
      __stcs(ret + o, rt);
    }
    __syncwarp();
    const int cn = c - GAE_NS;          // refill this slot with the chunk GAE_NS behind
    if (cn >= 0) {
      fence_proxy_async_smem();
      issue(cn, s);
    }
    if (++s == GAE_NS) { s = 0; ph ^= 1; }
  }
}

typedef CUresult (*PFN_encodeTiledGae)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                       const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                       CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                       CUtensorMapFloatOOBfill);

static int make_tmap_tn(CUtensorMap* tm, const void* ptr, int T, int N, int elem_bytes) {
  static PFN_encodeTiledGae enc = nullptr;
  if (!enc) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess) {
      set_last_error("cuTensorMapEncodeTiled entry point unavailable");
      return B200RL_ERR_DRIVER;
    }
    enc = reinterpret_cast<PFN_encodeTiledGae>(p);
  }
  cuuint64_t gdim[2] = {(cuuint64_t)N, (cuuint64_t)T};
  cuuint64_t gstr[1] = {(cuuint64_t)N * elem_bytes};
  cuuint32_t box[2] = {32, (cuuint32_t)GAE_TT};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(tm, elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_UINT8, 2,
                   const_cast<void*>(ptr), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("gae: cuTensorMapEncodeTiled failed (%d) T=%d N=%d elem=%d", (int)r, T, N, elem_bytes);
    return B200RL_ERR_DRIVER;
  }
  return B200RL_OK;
}

}  // namespace b200rl

using namespace b200rl;

extern "C" int b200rl_gae_scan(const float* rew, const float* val, const uint8_t* done, const float* last_val,
                               const uint8_t* last_done, float* adv, float* ret, int T, int N, double gamma, double lam,
                               int variant, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(rew && val && done && last_val && last_done && adv && ret, "gae: null pointer");
  B200RL_REQUIRE(T > 0 && N > 0, "gae: bad shape T=%d N=%d", T, N);
  const float gamma_f = (float)gamma;
  const double gl = gamma * lam;
  const bool aligned = (N % 32 == 0) && ((reinterpret_cast<uintptr_t>(rew) | reinterpret_cast<uintptr_t>(val) |
                                          reinterpret_cast<uintptr_t>(done)) % 16 == 0);
  if (variant == 1) B200RL_REQUIRE(aligned, "gae: bulk variant needs N %% 32 == 0 and 16 B aligned inputs");
  const bool bulk = (variant == 1) || (variant < 0 && aligned);
  if (bulk) {
    CUtensorMap tr, tv, td;
    int rc;
    if ((rc = make_tmap_tn(&tr, rew, T, N, 4)) != 0) return rc;
    if ((rc = make_tmap_tn(&tv, val, T, N, 4)) != 0) return rc;
    if ((rc = make_tmap_tn(&td, done, T, N, 1)) != 0) return rc;
    gae_tma_kernel<<<N / 32, 32, 0, stream>>>(tr, tv, td, last_val, last_done, adv, ret, T, N, gamma_f, gl);
    return check_launch("gae_tma_kernel");
  }
  const int threads = 64;
  gae_direct_kernel<16><<<ceil_div(N, threads), threads, 0, stream>>>(rew, val, done, last_val, last_done, adv, ret,
                                                                       T, N, gamma_f, gl);
  return check_launch("gae_direct_kernel");
}
