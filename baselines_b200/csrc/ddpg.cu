// DDPG (baselines/ddpg/ddpg_learner.py, Lillicrap et al. 2015) train-step and acting kernels.
//   ddpg_encode        the replay ring's rows (or acting observations) -> fp16 [hi | lo] operand rows of the towers'
//                      split_in first layers: clip((x - mean) / (std + 1e-8), -5, 5) (:17-20, :108-111), then the
//                      action columns of the critic's [obs | action] input (models.py:43)
//   ddpg_tanh          mu = tanh(z) in float32: the actor's output (models.py:31-32)
//   ddpg_denorm        q * std + mean (:23-26): the acting pass's critic_with_actor_tf
//   ddpg_target        y = r + (1 - d) * gamma * denormalize(Q') (:134-135)
//   ddpg_loss          critic_loss = mean((Q - normalize(y))^2) (:185-186) and actor_loss = -mean(denormalize(Q(s,
//                      mu(s)))) (:174) with their head gradients
//   ddpg_actor_dz      the actor's head gradient: dQ/dmu through tanh'
//   ddpg_l2            the critic's L2 term over the `/w:0` variables outside `output` (:187-196)
//   ddpg_obs_rms       mpi_running_mean_std RunningMeanStd.update once per stored row (:281-287) + mean / std
//   ddpg_ret_rms       the same update over a target batch (:299), then Pop-Art on the critics' output layers (:205-221)
//   ddpg_pn_adapt      sqrt(mean((mu - mu_adapt)^2)) (:170) and AdaptiveParamNoiseSpec.adapt (noise.py:12-18)
// Every reduction runs in one CTA in a fixed order, so a step is deterministic run to run.  All of them are a few
// thousand elements: the step is latency bound, and one launch per stage is what matters.  The soft target update
// (:36-47) is b200rl_soft_update (optim.cu).
#include "np_sum.cuh"

namespace b200rl {

constexpr int DD_THREADS = 256;

// float32 expressions of the reference, unfused
__device__ __forceinline__ float dd_normalize(float x, float mean, float std) {
  return __fdiv_rn(__fsub_rn(x, mean), __fadd_rn(std, 1e-8f));
}
__device__ __forceinline__ float dd_denormalize(float x, float mean, float std) {
  return __fadd_rn(__fmul_rn(x, std), mean);
}

__device__ __forceinline__ long long dd_ring_row(const long long* sel, long long b, long long limit) {
  // sel = [start, idx_0, idx_1, ...]: the ring row of sample b is (start + idx_b) % limit (memory.py:17-20)
  return sel ? (sel[0] + sel[1 + b]) % limit : b;
}

struct DdpgEncodeParams {
  const float* obs;            // [*, obs_dim] rows (the ring, or B acting rows)
  const long long* sel;        // optional [1 + B] ring selection
  long long limit;
  long long B;
  int obs_dim;
  const float* mean;           // optional obs_rms mean / std [obs_dim]
  const float* std;
  float clip;
  const float* act;            // optional [*, nA] action rows: ring rows (act_sel) or row b
  int act_sel;
  int nA;
  int in_pad;
  __half* out;                 // [B, 2 * in_pad]
  int* overflow;
};

__global__ void __launch_bounds__(DD_THREADS) ddpg_encode_kernel(const DdpgEncodeParams p) {
  const int groups = p.in_pad >> 3;
  const long long total = p.B * groups;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / groups;
    const int c0 = (int)(i - b * groups) << 3;
    const long long r = dd_ring_row(p.sel, b, p.limit);
    const float* src = p.obs + r * p.obs_dim;
    const float* a = p.act ? p.act + (p.act_sel ? r : b) * p.nA : nullptr;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = c0 + j;
      float t = 0.0f;
      if (c < p.obs_dim) {
        t = src[c];
        if (p.mean) t = dd_normalize(t, p.mean[c], p.std[c]);
        t = fminf(fmaxf(t, -p.clip), p.clip);
      } else if (a && c < p.obs_dim + p.nA) {
        t = a[c - p.obs_dim];
      }
      v[j] = t;
    }
    if (p.overflow && f16_overflow8(v)) *p.overflow = 1;
    store_split_f16x8(p.out + b * (2LL * p.in_pad) + c0, p.in_pad, v);
  }
}

__global__ void __launch_bounds__(DD_THREADS) ddpg_tanh_kernel(const float* __restrict__ z, long long ldz,
                                                               float* __restrict__ mu, long long B, int nA) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < B * nA; i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / nA;
    const int j = (int)(i - b * nA);
    mu[i] = tanhf(z[b * ldz + j]);
  }
}

__global__ void __launch_bounds__(DD_THREADS) ddpg_denorm_kernel(const float* __restrict__ q, long long ldq,
                                                                 const float* __restrict__ mean,
                                                                 const float* __restrict__ std, float* __restrict__ out,
                                                                 long long B) {
  for (long long b = blockIdx.x * (long long)blockDim.x + threadIdx.x; b < B; b += (long long)gridDim.x * blockDim.x) {
    const float v = q[b * ldq];
    out[b] = mean ? dd_denormalize(v, *mean, *std) : v;
  }
}

__global__ void __launch_bounds__(DD_THREADS)
ddpg_target_kernel(const float* __restrict__ q1, long long ldq, const long long* __restrict__ sel, long long limit,
                   const float* __restrict__ rewards, const float* __restrict__ terminals,
                   const float* __restrict__ mean, const float* __restrict__ std, float gamma, float* __restrict__ y,
                   long long B) {
  for (long long b = blockIdx.x * (long long)blockDim.x + threadIdx.x; b < B; b += (long long)gridDim.x * blockDim.x) {
    const long long r = dd_ring_row(sel, b, limit);
    float q = q1[b * ldq];
    if (mean) q = dd_denormalize(q, *mean, *std);
    // rewards + (1 - terminals1) * gamma * Q_obs1, left to right
    y[b] = __fadd_rn(rewards[r], __fmul_rn(__fmul_rn(__fsub_rn(1.0f, terminals[r]), gamma), q));
  }
}

// One CTA.  Rows [0, B) of q: Q(s, a) of the stored actions; rows [B, 2B): Q(s, mu(s)).  Thread t sums rows t, t + 256,
// ... in order; thread 0 adds the 256 partial sums in order.  dq holds the gradients of the SUMS over the rows (the
// caller scales the backward by 1/B): 2 (Q - y_n) and -std (-1 without return normalisation).
__global__ void __launch_bounds__(DD_THREADS)
ddpg_loss_kernel(const float* __restrict__ q, long long ldq, const float* __restrict__ y, const float* __restrict__ mean,
                 const float* __restrict__ std, int B, __half* __restrict__ dq, long long lddq, float* __restrict__ losses) {
  __shared__ float red[DD_THREADS];
  const float m = mean ? *mean : 0.0f, s = mean ? *std : 1.0f;
  float sc = 0.0f, sa = 0.0f;
  for (int b = threadIdx.x; b < B; b += DD_THREADS) {
    const float yn = mean ? dd_normalize(y[b], m, s) : y[b];
    const float d = __fsub_rn(q[(long long)b * ldq], yn);
    sc = __fadd_rn(sc, __fmul_rn(d, d));
    dq[(long long)b * lddq] = __float2half_rn(__fmul_rn(2.0f, d));
    const float qa = q[(long long)(B + b) * ldq];
    sa = __fadd_rn(sa, mean ? dd_denormalize(qa, m, s) : qa);
    dq[(long long)(B + b) * lddq] = __float2half_rn(-s);
  }
  const float tc = cta_sum_in_order<DD_THREADS>(sc, red);
  const float ta = cta_sum_in_order<DD_THREADS>(sa, red);
  if (threadIdx.x == 0) {
    losses[0] = __fdiv_rn(tc, (float)B);
    losses[1] = -__fdiv_rn(ta, (float)B);
  }
}

__global__ void __launch_bounds__(DD_THREADS)
ddpg_actor_dz_kernel(const float* __restrict__ g, long long ldg, const float* __restrict__ mu, long long B, int nA,
                     __half* __restrict__ dz, long long lddz) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < B * nA; i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / nA;
    const int j = (int)(i - b * nA);
    const float m = mu[i];
    dz[b * lddz + j] = __float2half_rn(__fmul_rn(g[b * ldg + j], __fsub_rn(1.0f, __fmul_rn(m, m))));
  }
}

struct DdpgSeg {                 // one variable of a flat parameter buffer
  long long off, len;
};

// One CTA over the segments in order: g += reg * w; loss += sum_s reg * (sum(w_s^2) / 2) (l2_regularizer, add_n).
__global__ void __launch_bounds__(1024)
ddpg_l2_kernel(const float* __restrict__ w, float* __restrict__ g, const DdpgSeg* __restrict__ segs, int nseg, float reg,
               float* __restrict__ loss) {
  __shared__ float red[1024];
  float total = 0.0f;
  for (int s = 0; s < nseg; ++s) {
    const DdpgSeg sg = segs[s];
    float acc = 0.0f;
    for (long long i = threadIdx.x; i < sg.len; i += blockDim.x) {
      const float v = w[sg.off + i];
      acc = __fadd_rn(acc, __fmul_rn(v, v));
      g[sg.off + i] = __fadd_rn(g[sg.off + i], __fmul_rn(reg, v));
    }
    const float t = cta_sum_in_order<1024>(acc, red);
    if (threadIdx.x == 0) total = __fadd_rn(total, __fmul_rn(reg, __fmul_rn(t, 0.5f)));
  }
  if (threadIdx.x == 0) *loss = __fadd_rn(*loss, total);
}

// RunningMeanStd state: float64 [sum(D) | sumsq(D) | count]; mean = float32(sum / count), std = sqrt(max(float32(sumsq /
// count) - mean^2, 1e-2)) in float32 (mpi_running_mean_std.py:29-30).
__device__ __forceinline__ void dd_rms_publish(const double* st, int D, int c, float* mean, float* std) {
  const double cnt = st[2 * D];
  const float m = (float)__ddiv_rn(st[c], cnt);
  const float q = (float)__ddiv_rn(st[D + c], cnt);
  mean[c] = m;
  std[c] = sqrtf(fmaxf(__fsub_rn(q, __fmul_rn(m, m)), 1e-2f));
}

// One CTA: the n rows at ring positions (pos0 + i) % limit, each an update of its own (sum += x, sumsq += x^2, count
// += 1, in row order).
__global__ void __launch_bounds__(DD_THREADS)
ddpg_obs_rms_kernel(const float* __restrict__ x, long long pos0, long long limit, long long n, int D,
                    double* __restrict__ st, float* __restrict__ mean, float* __restrict__ std) {
  if (threadIdx.x == 0) {
    double cnt = st[2 * D];
    for (long long i = 0; i < n; ++i) cnt = __dadd_rn(cnt, 1.0);
    st[2 * D] = cnt;
  }
  for (int c = threadIdx.x; c < D; c += blockDim.x) {
    double s = st[c], q = st[D + c];
    for (long long i = 0; i < n; ++i) {
      const double v = (double)x[((pos0 + i) % limit) * D + c];
      s = __dadd_rn(s, v);
      q = __dadd_rn(q, __dmul_rn(v, v));
    }
    st[c] = s;
    st[D + c] = q;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < D; c += blockDim.x) dd_rms_publish(st, D, c, mean, std);
}

// One CTA.  ret_rms.update(y) over the B targets, then (Pop-Art, w0 given) the output layers [K] + [1] of the critic and
// the target critic: M <- M * old_std / new_std, b <- (b * old_std + old_mean - new_mean) / new_std.
__global__ void __launch_bounds__(DD_THREADS)
ddpg_ret_rms_kernel(const float* __restrict__ y, long long B, double* __restrict__ st, float* __restrict__ mean,
                    float* __restrict__ std, float* __restrict__ w0, float* __restrict__ b0, float* __restrict__ w1,
                    float* __restrict__ b1, int K) {
  __shared__ float old[2], now[2];
  if (threadIdx.x == 0) {
    old[0] = *mean;
    old[1] = *std;
    // numpy's pairwise sums of the float64 vector y and of its squares
    const double s = np_pairwise<double>([y](long long i) { return (double)y[i]; }, 0LL, B);
    const double q = np_pairwise<double>([y](long long i) { const double v = y[i]; return __dmul_rn(v, v); }, 0LL, B);
    st[0] = __dadd_rn(st[0], __dadd_rn(0.0, s));
    st[1] = __dadd_rn(st[1], __dadd_rn(0.0, q));
    st[2] = __dadd_rn(st[2], (double)B);
    dd_rms_publish(st, 1, 0, mean, std);
    now[0] = *mean;
    now[1] = *std;
  }
  __syncthreads();
  if (w0 == nullptr) return;
  const float om = old[0], os = old[1], nm = now[0], ns = now[1];
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    w0[k] = __fdiv_rn(__fmul_rn(w0[k], os), ns);
    w1[k] = __fdiv_rn(__fmul_rn(w1[k], os), ns);
  }
  if (threadIdx.x == 0) {
    *b0 = __fdiv_rn(__fsub_rn(__fadd_rn(__fmul_rn(*b0, os), om), nm), ns);
    *b1 = __fdiv_rn(__fsub_rn(__fadd_rn(__fmul_rn(*b1, os), om), nm), ns);
  }
}

// One CTA: distance = sqrt(mean((mu - mu_adapt)^2)) over B x nA in a fixed order; current_stddev (float64) /= 1.01 when
// distance > desired, else *= 1.01; stddev32 = float32(current_stddev), the perturbations' scale.
__global__ void __launch_bounds__(DD_THREADS)
ddpg_pn_adapt_kernel(const float* __restrict__ mu, const float* __restrict__ mu_adapt, long long n, double desired,
                     double* __restrict__ stddev, float* __restrict__ stddev32, float* __restrict__ dist) {
  __shared__ float red[DD_THREADS];
  float s = 0.0f;
  for (long long i = threadIdx.x; i < n; i += DD_THREADS) {
    const float d = __fsub_rn(mu[i], mu_adapt[i]);
    s = __fadd_rn(s, __fmul_rn(d, d));
  }
  const float t = cta_sum_in_order<DD_THREADS>(s, red);
  if (threadIdx.x == 0) {
    const float dv = sqrtf(__fdiv_rn(t, (float)n));
    *dist = dv;
    const double sd = (double)dv > desired ? __ddiv_rn(*stddev, 1.01) : __dmul_rn(*stddev, 1.01);
    *stddev = sd;
    *stddev32 = (float)sd;
  }
}

}  // namespace b200rl

using namespace b200rl;

extern "C" int b200rl_ddpg_encode(const float* obs, const long long* sel, long long limit, long long B, int obs_dim,
                                  const float* mean, const float* std, float clip, const float* act, int act_sel,
                                  int nA, int in_pad, void* out, int* overflow, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(obs && out && B > 0 && obs_dim > 0 && nA >= 0, "ddpg_encode: bad args");
  B200RL_REQUIRE(in_pad % 8 == 0 && in_pad >= obs_dim + (act ? nA : 0), "ddpg_encode: in_pad must be a multiple of 8 "
                 "that holds the row");
  B200RL_REQUIRE((reinterpret_cast<uintptr_t>(out) & 15) == 0, "ddpg_encode: output must be 16-byte aligned");
  B200RL_REQUIRE((mean == nullptr) == (std == nullptr), "ddpg_encode: mean and std come together");
  B200RL_REQUIRE(sel == nullptr || limit > 0, "ddpg_encode: a ring selection needs limit > 0");
  B200RL_REQUIRE(!act_sel || sel, "ddpg_encode: ring actions need the ring selection");
  DdpgEncodeParams p{obs, sel, limit, B, obs_dim, mean, std, clip, act, act_sel, act ? nA : 0, in_pad,
                     reinterpret_cast<__half*>(out), overflow};
  ddpg_encode_kernel<<<grid_blocks(B * (in_pad / 8), DD_THREADS, 16), DD_THREADS, 0, stream>>>(p);
  return check_launch("ddpg_encode_kernel");
}

extern "C" int b200rl_ddpg_tanh(const float* z, long long ldz, float* mu, long long B, int nA, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(z && mu && B > 0 && nA > 0 && ldz >= nA, "ddpg_tanh: bad args");
  ddpg_tanh_kernel<<<grid_blocks(B * nA, DD_THREADS, 16), DD_THREADS, 0, stream>>>(z, ldz, mu, B, nA);
  return check_launch("ddpg_tanh_kernel");
}

extern "C" int b200rl_ddpg_denorm(const float* q, long long ldq, const float* mean, const float* std, float* out,
                                  long long B, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(q && out && B > 0 && ldq >= 1 && (mean == nullptr) == (std == nullptr), "ddpg_denorm: bad args");
  ddpg_denorm_kernel<<<grid_blocks(B, DD_THREADS, 16), DD_THREADS, 0, stream>>>(q, ldq, mean, std, out, B);
  return check_launch("ddpg_denorm_kernel");
}

extern "C" int b200rl_ddpg_target(const float* q1, long long ldq, const long long* sel, long long limit,
                                  const float* rewards, const float* terminals, const float* mean, const float* std,
                                  float gamma, float* y, long long B, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(q1 && rewards && terminals && y && B > 0 && ldq >= 1, "ddpg_target: bad args");
  B200RL_REQUIRE(sel == nullptr || limit > 0, "ddpg_target: a ring selection needs limit > 0");
  B200RL_REQUIRE((mean == nullptr) == (std == nullptr), "ddpg_target: mean and std come together");
  ddpg_target_kernel<<<grid_blocks(B, DD_THREADS, 16), DD_THREADS, 0, stream>>>(q1, ldq, sel, limit, rewards,
                                                                                 terminals, mean, std, gamma, y, B);
  return check_launch("ddpg_target_kernel");
}

extern "C" int b200rl_ddpg_loss(const float* q, long long ldq, const float* y, const float* mean, const float* std,
                                int B, void* dq, long long lddq, float* losses, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(q && y && dq && losses && B > 0 && ldq >= 1 && lddq >= 1, "ddpg_loss: bad args");
  B200RL_REQUIRE((mean == nullptr) == (std == nullptr), "ddpg_loss: mean and std come together");
  ddpg_loss_kernel<<<1, DD_THREADS, 0, stream>>>(q, ldq, y, mean, std, B, reinterpret_cast<__half*>(dq), lddq, losses);
  return check_launch("ddpg_loss_kernel");
}

extern "C" int b200rl_ddpg_actor_dz(const float* g, long long ldg, const float* mu, long long B, int nA, void* dz,
                                    long long lddz, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(g && mu && dz && B > 0 && nA > 0 && ldg >= nA && lddz >= nA, "ddpg_actor_dz: bad args");
  ddpg_actor_dz_kernel<<<grid_blocks(B * nA, DD_THREADS, 16), DD_THREADS, 0, stream>>>(
      g, ldg, mu, B, nA, reinterpret_cast<__half*>(dz), lddz);
  return check_launch("ddpg_actor_dz_kernel");
}

extern "C" int b200rl_ddpg_l2(const float* w, float* g, const long long* segs, int nseg, float reg, float* loss,
                              void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(w && g && segs && loss && nseg > 0, "ddpg_l2: bad args");
  ddpg_l2_kernel<<<1, 1024, 0, stream>>>(w, g, reinterpret_cast<const DdpgSeg*>(segs), nseg, reg, loss);
  return check_launch("ddpg_l2_kernel");
}

extern "C" int b200rl_ddpg_obs_rms(const float* x, long long pos0, long long limit, long long n, int D, double* st,
                                   float* mean, float* std, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(x && st && mean && std && n > 0 && D > 0 && limit > 0 && pos0 >= 0, "ddpg_obs_rms: bad args");
  ddpg_obs_rms_kernel<<<1, DD_THREADS, 0, stream>>>(x, pos0, limit, n, D, st, mean, std);
  return check_launch("ddpg_obs_rms_kernel");
}

extern "C" int b200rl_ddpg_ret_rms(const float* y, long long B, double* st, float* mean, float* std, float* w0,
                                   float* b0, float* w1, float* b1, int K, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(y && st && mean && std && B > 0, "ddpg_ret_rms: bad args");
  B200RL_REQUIRE(w0 == nullptr || (b0 && w1 && b1 && K > 0), "ddpg_ret_rms: Pop-Art needs both output layers");
  ddpg_ret_rms_kernel<<<1, DD_THREADS, 0, stream>>>(y, B, st, mean, std, w0, b0, w1, b1, K);
  return check_launch("ddpg_ret_rms_kernel");
}

extern "C" int b200rl_ddpg_pn_adapt(const float* mu, const float* mu_adapt, long long n, double desired,
                                    double* stddev, float* stddev32, float* dist, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(mu && mu_adapt && stddev && stddev32 && dist && n > 0, "ddpg_pn_adapt: bad args");
  ddpg_pn_adapt_kernel<<<1, DD_THREADS, 0, stream>>>(mu, mu_adapt, n, desired, stddev, stddev32, dist);
  return check_launch("ddpg_pn_adapt_kernel");
}
