// Parameter-space noise for DQN exploration (deepq/build_graph.py:202-314, Plappert et al. 2017).
//   param_perturb          perturb_vars (:258-272): a network copy <- q_func, + N(0, scale^2) on the variables the
//                          filter selects (default_param_noise_filter :131-143: the fully_connected ones)
//   dqn_param_noise_adapt  mean_kl between the plain and the adaptively perturbed policy (:279-280) and the scale
//                          update against the threshold (:281-287)
// The scale, the threshold, mean_kl and the random stream position live in device memory, so an act call is a fixed
// launch sequence.  Both kernels are a few thousand elements of latency-bound work.
#include <algorithm>

#include "common.cuh"
#include "philox.cuh"

namespace b200rl {

struct PerturbJob {            // one variable: dst[dst_off + i] = src[src_off + i] (+ scale * n), i < len
  long long src_off, dst_off, len, perturb;
};

// Normal e of a perturbation is Box-Muller over words (2p, 2p + 1), p = (e & 3) >> 1, of Philox block e >> 2 at the
// stream position: cos for even e, sin for odd e (gauss_step's pairing).  The sum is an unfused multiply then add.
__global__ void __launch_bounds__(256)
param_perturb_kernel(const float* __restrict__ src, float* __restrict__ dst, const PerturbJob* __restrict__ jobs,
                     const float* __restrict__ scale_dev, const float* __restrict__ normals, uint64_t seed,
                     const unsigned long long* __restrict__ offset_dev) {
  const PerturbJob job = jobs[blockIdx.y];
  const float scale = *scale_dev;
  const uint32_t offset = (uint32_t)*offset_dev;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < job.len; i += (long long)gridDim.x * blockDim.x) {
    const long long e = job.dst_off + i;
    float v = src[job.src_off + i];
    if (job.perturb) {
      float n;
      if (normals) {
        n = normals[e];
      } else {
        uint32_t rnd[4];
        philox4(seed, (uint64_t)(e >> 2), 0u, offset, rnd);
        const int p = (int)(e & 3) >> 1;
        const float u1 = u01_open(rnd[2 * p]), u2 = u01_open(rnd[2 * p + 1]);
        const float r = sqrtf(-2.0f * logf(u1));
        n = (e & 1) ? r * sinpif(2.0f * u2) : r * cospif(2.0f * u2);
      }
      v = __fadd_rn(v, __fmul_rn(scale, n));
    }
    dst[e] = v;
  }
}

// log softmax(q)_a of row b without materialising q: q_a = A_a (+ S - mean(A) when dueling)
struct QRow {
  const float* a;
  float shift;                 // S - mean(A), or 0
  float lse;                   // log sum exp(q)
};
__device__ __forceinline__ QRow q_row(const float* out, long long ld, int b, int nA, int dueling) {
  QRow r;
  r.a = out + (long long)b * ld;
  r.shift = 0.0f;
  if (dueling) {
    float m = 0.0f;
    for (int j = 0; j < nA; ++j) m += r.a[j];
    r.shift = r.a[nA] - m / (float)nA;
  }
  float mx = -INFINITY;
  for (int j = 0; j < nA; ++j) mx = fmaxf(mx, r.a[j] + r.shift);
  float z = 0.0f;
  for (int j = 0; j < nA; ++j) z += expf(r.a[j] + r.shift - mx);
  r.lse = mx + logf(z);
  return r;
}

// One CTA: thread t adds the KL of rows t, t + 256, ... in order, thread 0 adds the 256 sums in order.
__global__ void __launch_bounds__(256)
dqn_param_noise_adapt_kernel(const float* __restrict__ q, const float* __restrict__ q_adapt, long long ld, int nA,
                             int dueling, int B, float* __restrict__ scale_dev, const float* __restrict__ threshold_dev,
                             float* __restrict__ mean_kl_dev) {
  __shared__ float red[256];
  float s = 0.0f;
  for (int b = threadIdx.x; b < B; b += 256) {
    const QRow p = q_row(q, ld, b, nA, dueling), r = q_row(q_adapt, ld, b, nA, dueling);
    float kl = 0.0f;
    for (int j = 0; j < nA; ++j) {
      const float lp = p.a[j] + p.shift - p.lse, lr = r.a[j] + r.shift - r.lse;
      kl += expf(lp) * (lp - lr);
    }
    s += kl;
  }
  red[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.0f;
    for (int k = 0; k < 256; ++k) t += red[k];
    const float mean_kl = t / (float)B;
    *mean_kl_dev = mean_kl;
    const float sc = *scale_dev;
    *scale_dev = mean_kl < *threshold_dev ? __fmul_rn(sc, 1.01f) : __fdiv_rn(sc, 1.01f);
  }
}

}  // namespace b200rl

using namespace b200rl;

extern "C" int b200rl_param_perturb(const float* src, float* dst, const void* jobs, int njobs, long long max_len,
                                    const float* scale_dev, const float* normals, unsigned long long seed,
                                    const unsigned long long* offset_dev, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(src && dst && jobs && njobs > 0 && max_len > 0 && scale_dev && offset_dev, "param_perturb: bad args");
  B200RL_REQUIRE(njobs <= 65535, "param_perturb: at most 65535 variables per launch");
  const dim3 grid((unsigned)std::min<long long>(ceil_div_ll(max_len, 256), 64), (unsigned)njobs);
  param_perturb_kernel<<<grid, 256, 0, stream>>>(src, dst, reinterpret_cast<const PerturbJob*>(jobs), scale_dev, normals,
                                                 seed, offset_dev);
  return check_launch("param_perturb_kernel");
}

extern "C" int b200rl_dqn_param_noise_adapt(const float* q, const float* q_adapt, long long ld, int nA, int dueling,
                                            int B, float* scale_dev, const float* threshold_dev, float* mean_kl_dev,
                                            void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(q && q_adapt && nA > 0 && B > 0 && scale_dev && threshold_dev && mean_kl_dev && ld >= nA + (dueling != 0),
                 "dqn_param_noise_adapt: bad args");
  dqn_param_noise_adapt_kernel<<<1, 256, 0, stream>>>(q, q_adapt, ld, nA, dueling, B, scale_dev, threshold_dev,
                                                      mean_kl_dev);
  return check_launch("dqn_param_noise_adapt_kernel");
}
