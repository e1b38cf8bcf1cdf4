// Hindsight Experience Replay (baselines/her/, Andrychowicz et al. 2017) train-step and acting kernels.
//   her_sample         one launch per train batch: gather o, o_2, ag, ag_2, g, u of the sampled (episode, t) from the
//                      float64 episode ring, relabel g <- ag[ep, future_t] (her_sampler.py:34-43), recompute the goal
//                      distance reward in float64 (np.linalg.norm, gym robotics' compute_reward), _preprocess_og
//                      (ddpg.py:112-121) in float64, round to float32 (the staging area), normalise with the device
//                      statistics and clip (normalizer.py:72-77), and write the fp16 [hi | lo] operand rows of
//                      [o | g], [o_2 | g_2] and [o | g | u / max_u] (actor_critic.py:30-46)
//   her_obs_encode     the same normalise + encode for acting rows already preprocessed on the host (get_actions)
//   her_pi             pi = max_u * tanh(z), and pi / max_u into the action columns of a critic's operand rows
//   her_target         y = clip(r + gamma * Q', -clip_return, 0 or inf) (ddpg.py:356-358)
//   her_loss           Q_loss = mean((y - Q)^2) and the critic head gradients; the -mean(Q_pi) head gradient
//   her_actor_dz       the actor's head gradient: dQ/du_in / max_u + action_l2's term, through max_u * tanh'
//   her_norm           Normalizer.update over a sample of new episodes + recompute_stats (normalizer.py:64-118)
// Every reduction runs in one CTA in a fixed order, so a step is deterministic run to run.  The target update
// (ddpg.py:398-399) is b200rl_soft_update (optim.cu).
#include "np_sum.cuh"

namespace b200rl {

constexpr int HER_THREADS = 256;

__device__ __forceinline__ double her_clip64(double x, double c) { return fmin(fmax(x, -c), c); }

// normalizer.py:77: clip((v - mean) / std, -clip, clip) in float32
__device__ __forceinline__ float her_normalize(float x, const float* mean, const float* std, int c, float clip) {
  const float v = __fdiv_rn(__fsub_rn(x, mean[c]), std[c]);
  return fminf(fmaxf(v, -clip), clip);
}

struct HerSampleParams {
  const double *o, *ag, *g, *u, *info;  // ring [S, T+1, dimo], [S, T+1, dimg], [S, T, dimg], [S, T, dimu], [S, T, ninfo]
  int T, dimo, dimg, dimu, ninfo;
  const long long* sel;                 // [B, 3]: episode slot, t, future_t (-1: keep the stored goal)
  int B;
  int relative;
  double clip_obs;
  const float *o_mean, *o_std, *g_mean, *g_std;
  float norm_clip;
  const float* max_u;                   // [dimu]
  int reward_type;                      // 0: none (the host computes r), 1: sparse, 2: dense
  double threshold;
  float* r;
  __half *xa, *xta;                     // [B, 2 * pad_a]
  __half *xc, *xtc;                     // [2B, 2 * pad_c] (rows [B, 2B) get [o | g] only), [B, 2 * pad_c]
  int pad_a, pad_c;
  double *ag2_out, *g_out, *info_out;   // optional [B, dimg], [B, dimg], [B, ninfo]
};

__global__ void __launch_bounds__(HER_THREADS) her_sample_kernel(const HerSampleParams p) {
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < p.B; b += gridDim.x * blockDim.x) {
    const long long ep = p.sel[3 * b], t = p.sel[3 * b + 1], ft = p.sel[3 * b + 2];
    const long long T1 = p.T + 1;
    const double* o0 = p.o + (ep * T1 + t) * p.dimo;
    const double* o1 = o0 + p.dimo;
    const double* ag0 = p.ag + (ep * T1 + t) * p.dimg;
    const double* ag1 = ag0 + p.dimg;
    const double* gs = ft >= 0 ? p.ag + (ep * T1 + ft) * p.dimg : p.g + (ep * p.T + t) * p.dimg;
    if (p.reward_type) {
      // np.linalg.norm: numpy's pairwise sum of the squares
      const double d2 = np_pairwise<double>([&](int i) { const double d = __dsub_rn(ag1[i], gs[i]); return __dmul_rn(d, d); },
                                            0, p.dimg);
      const double d = __dsqrt_rn(__dadd_rn(0.0, d2));
      p.r[b] = p.reward_type == 1 ? (d > p.threshold ? -1.0f : -0.0f) : (float)(-d);
    }
    if (p.ag2_out)
      for (int i = 0; i < p.dimg; ++i) {
        p.ag2_out[(long long)b * p.dimg + i] = ag1[i];
        p.g_out[(long long)b * p.dimg + i] = gs[i];
      }
    if (p.info_out)
      for (int i = 0; i < p.ninfo; ++i)
        p.info_out[(long long)b * p.ninfo + i] = p.info[(ep * p.T + t) * p.ninfo + i];
    __half* ra = p.xa + (long long)b * 2 * p.pad_a;
    __half* rta = p.xta + (long long)b * 2 * p.pad_a;
    __half* rc = p.xc + (long long)b * 2 * p.pad_c;
    __half* rc2 = p.xc + (long long)(p.B + b) * 2 * p.pad_c;
    __half* rtc = p.xtc + (long long)b * 2 * p.pad_c;
    for (int c = 0; c < p.dimo; ++c) {
      const float v0 = her_normalize((float)her_clip64(o0[c], p.clip_obs), p.o_mean, p.o_std, c, p.norm_clip);
      const float v1 = her_normalize((float)her_clip64(o1[c], p.clip_obs), p.o_mean, p.o_std, c, p.norm_clip);
      split_f16(v0, ra[c], ra[p.pad_a + c]);
      split_f16(v0, rc[c], rc[p.pad_c + c]);
      split_f16(v0, rc2[c], rc2[p.pad_c + c]);
      split_f16(v1, rta[c], rta[p.pad_a + c]);
      split_f16(v1, rtc[c], rtc[p.pad_c + c]);
    }
    for (int i = 0; i < p.dimg; ++i) {
      const double g0 = p.relative ? __dsub_rn(gs[i], ag0[i]) : gs[i];
      const double g1 = p.relative ? __dsub_rn(gs[i], ag1[i]) : gs[i];
      const float v0 = her_normalize((float)her_clip64(g0, p.clip_obs), p.g_mean, p.g_std, i, p.norm_clip);
      const float v1 = her_normalize((float)her_clip64(g1, p.clip_obs), p.g_mean, p.g_std, i, p.norm_clip);
      const int c = p.dimo + i;
      split_f16(v0, ra[c], ra[p.pad_a + c]);
      split_f16(v0, rc[c], rc[p.pad_c + c]);
      split_f16(v0, rc2[c], rc2[p.pad_c + c]);
      split_f16(v1, rta[c], rta[p.pad_a + c]);
      split_f16(v1, rtc[c], rtc[p.pad_c + c]);
    }
    const double* us = p.u + (ep * p.T + t) * p.dimu;
    for (int j = 0; j < p.dimu; ++j) {
      const int c = p.dimo + p.dimg + j;
      split_f16(__fdiv_rn((float)us[j], p.max_u[j]), rc[c], rc[p.pad_c + c]);
    }
  }
}

__global__ void __launch_bounds__(HER_THREADS)
her_obs_encode_kernel(const float* __restrict__ o, const float* __restrict__ g, int n, int dimo, int dimg,
                      const float* __restrict__ o_mean, const float* __restrict__ o_std,
                      const float* __restrict__ g_mean, const float* __restrict__ g_std, float norm_clip,
                      __half* __restrict__ xa, int pad_a, __half* __restrict__ xc, int pad_c) {
  const int w = dimo + dimg;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (long long)n * w;
       i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / w;
    const int c = (int)(i - b * w);
    const float v = c < dimo ? her_normalize(o[b * dimo + c], o_mean, o_std, c, norm_clip)
                             : her_normalize(g[b * dimg + c - dimo], g_mean, g_std, c - dimo, norm_clip);
    __half* ra = xa + b * 2 * pad_a;
    split_f16(v, ra[c], ra[pad_a + c]);
    if (xc) {
      __half* rc = xc + b * 2 * pad_c;
      split_f16(v, rc[c], rc[pad_c + c]);
    }
  }
}

__global__ void __launch_bounds__(HER_THREADS)
her_pi_kernel(const float* __restrict__ z, long long ldz, int B, int dimu, const float* __restrict__ max_u,
              float* __restrict__ pi, __half* __restrict__ xc, int pad_c, int col0) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (long long)B * dimu;
       i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / dimu;
    const int j = (int)(i - b * dimu);
    const float v = __fmul_rn(max_u[j], tanhf(z[b * ldz + j]));
    pi[i] = v;
    if (xc) {
      __half* rc = xc + b * 2 * pad_c;
      split_f16(__fdiv_rn(v, max_u[j]), rc[col0 + j], rc[pad_c + col0 + j]);
    }
  }
}

__global__ void __launch_bounds__(HER_THREADS)
her_target_kernel(const float* __restrict__ q, long long ldq, const float* __restrict__ r, int B, float gamma,
                  float lo, float hi, float* __restrict__ y) {
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < B; b += gridDim.x * blockDim.x)
    y[b] = fminf(fmaxf(__fadd_rn(r[b], __fmul_rn(gamma, q[(long long)b * ldq])), lo), hi);
}

// One CTA.  Rows [0, B) of q: Q(o, g, u / max_u); rows [B, 2B): Q_pi.  Thread t sums rows t, t + 256, ... in order;
// thread 0 adds the 256 partial sums in order.  dq holds the gradients of the SUMS over the rows (the backward scales
// by 1/B): -2 (y - Q) on the first B rows, -1 (of -sum(Q_pi)) on the second.
__global__ void __launch_bounds__(HER_THREADS)
her_loss_kernel(const float* __restrict__ q, long long ldq, const float* __restrict__ y, int B, __half* __restrict__ dq,
                long long lddq, float* __restrict__ loss, float* __restrict__ q_pi) {
  __shared__ float red[HER_THREADS];
  float s = 0.0f;
  for (int b = threadIdx.x; b < B; b += HER_THREADS) {
    const float d = __fsub_rn(y[b], q[(long long)b * ldq]);
    s = __fadd_rn(s, __fmul_rn(d, d));
    dq[(long long)b * lddq] = __float2half_rn(__fmul_rn(-2.0f, d));
    dq[(long long)(B + b) * lddq] = __float2half_rn(-1.0f);
    q_pi[b] = q[(long long)(B + b) * ldq];
  }
  const float t = cta_sum_in_order<HER_THREADS>(s, red);
  if (threadIdx.x == 0) *loss = __fdiv_rn(t, (float)B);
}

// dz = (g / max_u + 2 action_l2 (pi / max_u) / (max_u dimu)) * max_u * (1 - tanh(z)^2), sum scaling over the batch:
// the actor's backward scales by 1/B, so the L2 mean's 1/(B dimu) leaves 1/dimu here.
__global__ void __launch_bounds__(HER_THREADS)
her_actor_dz_kernel(const float* __restrict__ g, long long ldg, const float* __restrict__ z, long long ldz,
                    const float* __restrict__ pi, int B, int dimu, const float* __restrict__ max_u, float action_l2,
                    __half* __restrict__ dz, long long lddz) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (long long)B * dimu;
       i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / dimu;
    const int j = (int)(i - b * dimu);
    const float mu = max_u[j];
    const float uin = __fdiv_rn(pi[i], mu);
    const float l2 = __fdiv_rn(__fmul_rn(__fmul_rn(2.0f, action_l2), uin), __fmul_rn(mu, (float)dimu));
    const float dpi = __fadd_rn(__fdiv_rn(g[b * ldg + j], mu), l2);
    const float t = tanhf(z[b * ldz + j]);
    dz[b * lddz + j] = __float2half_rn(__fmul_rn(__fmul_rn(dpi, mu), __fsub_rn(1.0f, __fmul_rn(t, t))));
  }
}

// Block 0: the o statistics, block 1: the g statistics.  Each thread owns columns and adds, over the N samples, the
// preprocessed value (float32 arithmetic when the stored episode was float32, float64 otherwise: numpy's dtype of the
// transitions) and its square in numpy's order for v.sum(axis=0): row after row, except for a single column, which numpy
// reduces pairwise; local = float32(sum).  Then recompute_stats: count += N, sum += local, sumsq += local_sq, mean =
// sum / count, std = sqrt(max(eps^2, sumsq / count - mean^2)), all float32.  state: float32 [sum(D) | sumsq(D) | count].
template <typename R>
__device__ void her_norm_sums(const double* o, const double* ag, const double* g, int T, int dimo, int dimg,
                              const long long* sel, int N, int relative, double clip_obs, bool is_o, int D, int c,
                              float* ls, float* lq) {
  const long long T1 = T + 1;
  auto val = [&](int i) -> R {
    const long long ep = sel[3 * i], t = sel[3 * i + 1], ft = sel[3 * i + 2];
    R v;
    if (is_o) {
      v = (R)o[(ep * T1 + t) * dimo + c];
    } else {
      v = (R)(ft >= 0 ? ag[(ep * T1 + ft) * dimg + c] : g[(ep * T + t) * dimg + c]);
      if (relative) v = sub_rn(v, (R)ag[(ep * T1 + t) * dimg + c]);
    }
    const R cl = (R)clip_obs;
    return v < -cl ? -cl : (v > cl ? cl : v);
  };
  R s = R(0), q = R(0);
  if (D == 1) {
    s = np_pairwise<R>(val, 0, N);
    q = np_pairwise<R>([&](int i) { const R v = val(i); return mul_rn(v, v); }, 0, N);
  } else {
    for (int i = 0; i < N; ++i) {
      const R x = val(i);
      s = add_rn(s, x);
      q = add_rn(q, mul_rn(x, x));
    }
  }
  *ls = (float)s;
  *lq = (float)q;
}

__global__ void __launch_bounds__(HER_THREADS)
her_norm_kernel(const double* __restrict__ o, const double* __restrict__ ag, const double* __restrict__ g, int T,
                int dimo, int dimg, const long long* __restrict__ sel, int N, int relative, double clip_obs,
                int f32_o, int f32_g, float* __restrict__ o_st, float* __restrict__ o_mean, float* __restrict__ o_std,
                float* __restrict__ g_st, float* __restrict__ g_mean, float* __restrict__ g_std, float eps) {
  const bool is_o = blockIdx.x == 0;
  const int D = is_o ? dimo : dimg;
  float* st = is_o ? o_st : g_st;
  float* mean = is_o ? o_mean : g_mean;
  float* std = is_o ? o_std : g_std;
  const bool f32 = is_o ? f32_o : f32_g;
  const float cnt = __fadd_rn(st[2 * D], (float)N);
  const float eps2 = __fmul_rn(eps, eps);
  for (int c = threadIdx.x; c < D; c += blockDim.x) {
    float ls, lq;
    if (f32)
      her_norm_sums<float>(o, ag, g, T, dimo, dimg, sel, N, relative, clip_obs, is_o, D, c, &ls, &lq);
    else
      her_norm_sums<double>(o, ag, g, T, dimo, dimg, sel, N, relative, clip_obs, is_o, D, c, &ls, &lq);
    const float sum = __fadd_rn(st[c], ls), sumsq = __fadd_rn(st[D + c], lq);
    st[c] = sum;
    st[D + c] = sumsq;
    const float m = __fdiv_rn(sum, cnt);
    mean[c] = m;
    std[c] = __fsqrt_rn(fmaxf(eps2, __fsub_rn(__fdiv_rn(sumsq, cnt), __fmul_rn(m, m))));
  }
  __syncthreads();
  if (threadIdx.x == 0) st[2 * D] = cnt;
}

}  // namespace b200rl

using namespace b200rl;

extern "C" int b200rl_her_sample(const double* o, const double* ag, const double* g, const double* u,
                                 const double* info, int T, int dimo, int dimg, int dimu, int ninfo,
                                 const long long* sel, int B, int relative, double clip_obs, const float* o_mean,
                                 const float* o_std, const float* g_mean, const float* g_std, float norm_clip,
                                 const float* max_u, int reward_type, double threshold, float* r, void* xa,
                                 void* xta, int pad_a, void* xc, void* xtc, int pad_c, double* ag2_out, double* g_out,
                                 double* info_out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(o && ag && g && u && sel && B > 0 && T > 0 && dimo > 0 && dimg > 0 && dimu > 0 && ninfo >= 0,
                 "her_sample: bad args");
  B200RL_REQUIRE(o_mean && o_std && g_mean && g_std && max_u && xa && xta && xc && xtc, "her_sample: bad args");
  B200RL_REQUIRE(pad_a >= dimo + dimg && pad_c >= dimo + dimg + dimu, "her_sample: operand rows too narrow");
  B200RL_REQUIRE(reward_type >= 0 && reward_type <= 2 && (reward_type == 0 || r), "her_sample: bad reward rule");
  B200RL_REQUIRE((ag2_out == nullptr) == (g_out == nullptr), "her_sample: ag2_out and g_out come together");
  B200RL_REQUIRE(info_out == nullptr || ninfo == 0 || info, "her_sample: info_out needs the info ring");
  HerSampleParams p{o, ag, g, u, info, T, dimo, dimg, dimu, ninfo, sel, B, relative, clip_obs, o_mean, o_std, g_mean,
                    g_std, norm_clip, max_u, reward_type, threshold, r, reinterpret_cast<__half*>(xa),
                    reinterpret_cast<__half*>(xta), reinterpret_cast<__half*>(xc), reinterpret_cast<__half*>(xtc),
                    pad_a, pad_c, ag2_out, g_out, ninfo ? info_out : nullptr};
  her_sample_kernel<<<grid_blocks(B, HER_THREADS, 16), HER_THREADS, 0, stream>>>(p);
  return check_launch("her_sample_kernel");
}

extern "C" int b200rl_her_obs_encode(const float* o, const float* g, int n, int dimo, int dimg, const float* o_mean,
                                     const float* o_std, const float* g_mean, const float* g_std, float norm_clip,
                                     void* xa, int pad_a, void* xc, int pad_c, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(o && g && xa && o_mean && o_std && g_mean && g_std && n > 0 && dimo > 0 && dimg > 0,
                 "her_obs_encode: bad args");
  B200RL_REQUIRE(pad_a >= dimo + dimg && (xc == nullptr || pad_c >= dimo + dimg), "her_obs_encode: rows too narrow");
  her_obs_encode_kernel<<<grid_blocks((long long)n * (dimo + dimg), HER_THREADS, 16), HER_THREADS, 0, stream>>>(
      o, g, n, dimo, dimg, o_mean, o_std, g_mean, g_std, norm_clip, reinterpret_cast<__half*>(xa), pad_a,
      reinterpret_cast<__half*>(xc), pad_c);
  return check_launch("her_obs_encode_kernel");
}

extern "C" int b200rl_her_pi(const float* z, long long ldz, int B, int dimu, const float* max_u, float* pi, void* xc,
                             int pad_c, int col0, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(z && max_u && pi && B > 0 && dimu > 0 && ldz >= dimu, "her_pi: bad args");
  B200RL_REQUIRE(xc == nullptr || (col0 >= 0 && pad_c >= col0 + dimu), "her_pi: action columns outside the row");
  her_pi_kernel<<<grid_blocks((long long)B * dimu, HER_THREADS, 16), HER_THREADS, 0, stream>>>(
      z, ldz, B, dimu, max_u, pi, reinterpret_cast<__half*>(xc), pad_c, col0);
  return check_launch("her_pi_kernel");
}

extern "C" int b200rl_her_target(const float* q, long long ldq, const float* r, int B, float gamma, float lo, float hi,
                                 float* y, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(q && r && y && B > 0 && ldq >= 1, "her_target: bad args");
  her_target_kernel<<<grid_blocks(B, HER_THREADS, 16), HER_THREADS, 0, stream>>>(q, ldq, r, B, gamma, lo, hi, y);
  return check_launch("her_target_kernel");
}

extern "C" int b200rl_her_loss(const float* q, long long ldq, const float* y, int B, void* dq, long long lddq,
                               float* loss, float* q_pi, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(q && y && dq && loss && q_pi && B > 0 && ldq >= 1 && lddq >= 1, "her_loss: bad args");
  her_loss_kernel<<<1, HER_THREADS, 0, stream>>>(q, ldq, y, B, reinterpret_cast<__half*>(dq), lddq, loss, q_pi);
  return check_launch("her_loss_kernel");
}

extern "C" int b200rl_her_actor_dz(const float* g, long long ldg, const float* z, long long ldz, const float* pi, int B,
                                   int dimu, const float* max_u, float action_l2, void* dz, long long lddz,
                                   void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(g && z && pi && max_u && dz && B > 0 && dimu > 0 && ldg >= dimu && ldz >= dimu && lddz >= dimu,
                 "her_actor_dz: bad args");
  her_actor_dz_kernel<<<grid_blocks((long long)B * dimu, HER_THREADS, 16), HER_THREADS, 0, stream>>>(
      g, ldg, z, ldz, pi, B, dimu, max_u, action_l2, reinterpret_cast<__half*>(dz), lddz);
  return check_launch("her_actor_dz_kernel");
}

extern "C" int b200rl_her_norm(const double* o, const double* ag, const double* g, int T, int dimo, int dimg,
                               const long long* sel, int N, int relative, double clip_obs, int f32_o, int f32_g,
                               float* o_st, float* o_mean, float* o_std, float* g_st, float* g_mean, float* g_std,
                               float eps, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(o && ag && g && sel && N > 0 && T > 0 && dimo > 0 && dimg > 0, "her_norm: bad args");
  B200RL_REQUIRE(o_st && o_mean && o_std && g_st && g_mean && g_std, "her_norm: bad statistics");
  her_norm_kernel<<<2, HER_THREADS, 0, stream>>>(o, ag, g, T, dimo, dimg, sel, N, relative, clip_obs, f32_o, f32_g, o_st,
                                                 o_mean, o_std, g_st, g_mean, g_std, eps);
  return check_launch("her_norm_kernel");
}
