// ACER kernels (acer/acer.py, acer/buffer.py):
//   * acer_step        : Gumbel-max action (the cat_step sampler, cat_sample.cuh) + mu = softmax(logits) rows
//                        (acer.py:105,214), which the runner stores
//   * acer_stack_obs   : gather one ring slot per env (Buffer.get/take, buffer.py:77-97) and re-stack its frames
//                        (_stack_obs, buffer.py:124-140) into the train batch, env-major, bit for bit
//   * acer_loss        : the whole loss head of acer.py:103-178 for one env per CTA: softmax of the train and Polyak
//                        logits, v, the Retrace recursion (float32, the reference's order), the truncated-importance
//                        and bias-correction policy losses, entropy, the Q loss, the trust-region projection of the
//                        gradient w.r.t. f, and d loss / d [logits | q] in fp16 "sum" scaling (the backward applies
//                        1/N); float64 statistics reduced in env order by the last CTA
//   * clip_rmsprop_ema : global-norm clip + TF RMSProp (ms starts at 1) + the Polyak ExponentialMovingAverage of the
//                        parameters after the step (acer.py:181-188), one pass over the flat buffers
#include "common.cuh"
#include "cat_sample.cuh"

namespace b200rl {

// ---------------------------------------------------------------- act
__global__ void __launch_bounds__(256)
acer_step_kernel(const float* __restrict__ logits, long long ld, int nA, uint64_t seed, uint64_t offset,
                 const unsigned long long* __restrict__ offset_dev, long long* __restrict__ actions,
                 float* __restrict__ mu, long long B) {
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  if (offset_dev) offset = *offset_dev;
  const float* l = logits + b * ld;
  float m = -INFINITY;
  for (int j = 0; j < nA; ++j) m = fmaxf(m, l[j]);
  float z = 0.0f;
  for (int j = 0; j < nA; ++j) z += expf(l[j] - m);
  uint32_t rnd[4];
  int held = -1;
  actions[b] = cat_gumbel_argmax(l, 0, nA, nA, nullptr, seed, b, offset, rnd, held);
  for (int j = 0; j < nA; ++j) mu[b * nA + j] = expf(l[j] - m) / z;
}

// ---------------------------------------------------------------- segment gather + re-stack
// ring: [slots, nenv, nsteps + nstack, F, nc] (F = frame elements per channel); out row e * (nsteps + 1) + t, element
// (f, i * nc + c) = ring[idx[e], e, t + i, f, c] * M_i(t), with M_i(t) = prod over the dones[t - 1 - j],
// j < nstack - 1 - i, j <= t - 1, of (1 - done): the cumulative masks of _stack_obs (the newest block is unmasked).
// The multiply is done as the reference does it, so float frames keep -0.0 / NaN exactly as numpy leaves them.
template <typename T>
__global__ void __launch_bounds__(256)
acer_stack_kernel(const T* __restrict__ ring, long long slot_stride, const long long* __restrict__ idx, int nsteps,
                  int nstack, long long F, int nc, const uint8_t* __restrict__ dones_ring, T* __restrict__ out) {
  const int row = blockIdx.y;                         // e * (nsteps + 1) + t
  const int e = row / (nsteps + 1), t = row % (nsteps + 1);
  const int nenv = gridDim.y / (nsteps + 1);
  const long long slot = idx ? idx[e] : 0;
  const long long seg = nsteps + nstack;
  const uint8_t* d = dones_ring + (slot * nenv + e) * nsteps;
  // keep[i]: 1 while no done lies within the window of block i
  uint32_t keep = 0;
  for (int i = 0; i < nstack; ++i) {
    bool k = true;
    for (int j = 0; j < nstack - 1 - i && j <= t - 1; ++j) k = k && (d[t - 1 - j] == 0);
    keep |= (uint32_t)k << i;
  }
  const T* src = ring + slot * slot_stride + (long long)e * seg * F * nc;
  const long long W = (long long)nstack * nc, n = F * W;
  T* o = out + (long long)row * n;
  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
    const long long f = k / W;
    const int r = (int)(k - f * W), i = r / nc, c = r - i * nc;
    const T x = src[((long long)(t + i) * F + f) * nc + c];
    o[k] = (i == nstack - 1) ? x : (T)(x * (T)((keep >> i) & 1u));
  }
}

// the slot's per-step arrays: actions / rewards / dones [nenv, nsteps], mus [nenv, nsteps, nA], masks [nenv, nsteps+1]
__global__ void __launch_bounds__(256)
acer_take_kernel(const long long* __restrict__ idx, int nenv, int nsteps, int nA, const long long* __restrict__ a_r,
                 const float* __restrict__ r_r, const float* __restrict__ mu_r, const uint8_t* __restrict__ d_r,
                 const uint8_t* __restrict__ m_r, long long* __restrict__ a, float* __restrict__ r,
                 float* __restrict__ mu, uint8_t* __restrict__ dn, uint8_t* __restrict__ mk) {
  const int e = blockIdx.x;
  const long long s = (idx ? idx[e] : 0) * nenv + e;
  for (int t = threadIdx.x; t < nsteps; t += blockDim.x) {
    a[e * nsteps + t] = a_r[s * nsteps + t];
    r[e * nsteps + t] = r_r[s * nsteps + t];
    dn[e * nsteps + t] = d_r[s * nsteps + t];
  }
  for (int t = threadIdx.x; t <= nsteps; t += blockDim.x) mk[e * (nsteps + 1) + t] = m_r[s * (nsteps + 1) + t];
  for (int k = threadIdx.x; k < nsteps * nA; k += blockDim.x) mu[(long long)e * nsteps * nA + k] = mu_r[s * nsteps * nA + k];
}

// ---------------------------------------------------------------- loss head
static constexpr int ACER_NSTAT = 13;          // per-env partial sums (see acer_loss_kernel)
static constexpr int ACER_MAX_ENVS = 4096;
// One scratch and one completion counter per device (the sumsq pattern): acer_loss launches must not overlap, so a
// process issues them on one stream.
__device__ double g_acer_part[ACER_MAX_ENVS * ACER_NSTAT];
__device__ unsigned int g_acer_done = 0;

struct AcerArgs {
  int nsteps, nA, trust_region;
  float gamma, c, delta, q_coef, ent_coef;
};

__device__ __forceinline__ void softmax_row(const float* l, int nA, float& m, float& z) {
  m = -INFINITY;
  for (int j = 0; j < nA; ++j) m = fmaxf(m, l[j]);
  z = 0.0f;
  for (int j = 0; j < nA; ++j) z += expf(l[j] - m);
}

// One CTA per env e: rows r0 + t, t in [0, nsteps], r0 = e * (nsteps + 1); step rows e * nsteps + t.
// Dynamic shared memory: 4 * (nsteps + 1) floats.
__global__ void __launch_bounds__(128)
acer_loss_kernel(const float* __restrict__ pi, long long ldpi, const float* __restrict__ q, long long ldq,
                 const float* __restrict__ pol, long long ldpol, const long long* __restrict__ actions,
                 const float* __restrict__ rewards, const uint8_t* __restrict__ dones, const float* __restrict__ mus,
                 AcerArgs a, __half* __restrict__ dpi, long long lddpi, __half* __restrict__ dq, long long lddq,
                 double* __restrict__ stats, float* __restrict__ f_out, float* __restrict__ v_out,
                 float* __restrict__ qret_out) {
  extern __shared__ float sh[];
  const int T = a.nsteps, nA = a.nA, e = blockIdx.x, nenv = gridDim.x;
  float* v_s = sh;                    // [T + 1]
  float* qi_s = v_s + (T + 1);        // [T]
  float* rho_s = qi_s + (T + 1);      // [T]  rho_i
  float* qret_s = rho_s + (T + 1);    // [T]
  const float eps = 1e-6f;
  const long long r0 = (long long)e * (T + 1), s0 = (long long)e * T;
  for (int t = threadIdx.x; t <= T; t += blockDim.x) {
    const float* l = pi + (r0 + t) * ldpi;
    const float* qq = q + (r0 + t) * ldq;
    float m, z;
    softmax_row(l, nA, m, z);
    float v = 0.0f;
    for (int j = 0; j < nA; ++j) {
      const float f = expf(l[j] - m) / z;
      v = __fadd_rn(v, __fmul_rn(f, qq[j]));
      if (f_out) f_out[(r0 + t) * nA + j] = f;
    }
    v_s[t] = v;
    if (v_out) v_out[r0 + t] = v;
    if (t < T) {
      const int ai = (int)actions[s0 + t];
      qi_s[t] = qq[ai];
      rho_s[t] = expf(l[ai] - m) / z / (mus[(s0 + t) * nA + ai] + eps);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {                     // q_retrace, acer.py:36-50, float32 in the reference's order
    float qret = v_s[T];
    for (int i = T - 1; i >= 0; --i) {
      const float notdone = 1.0f - (float)dones[s0 + i];
      qret = __fadd_rn(rewards[s0 + i], __fmul_rn(__fmul_rn(a.gamma, qret), notdone));
      qret_s[i] = qret;
      const float rho_bar = fminf(1.0f, rho_s[i]);
      qret = __fadd_rn(__fmul_rn(rho_bar, __fsub_rn(qret, qi_s[i])), v_s[i]);
    }
  }
  __syncthreads();
  double acc[ACER_NSTAT];
  for (int k = 0; k < ACER_NSTAT; ++k) acc[k] = 0.0;
  for (int t = threadIdx.x; t <= T; t += blockDim.x) {
    __half* dl = dpi + (r0 + t) * lddpi;
    __half* dqr = dq + (r0 + t) * lddq;
    if (t == T) {                             // strip(): the last row of each env carries no loss
      for (int j = 0; j < nA; ++j) { dl[j] = __float2half_rn(0.0f); dqr[j] = __float2half_rn(0.0f); }
      continue;
    }
    const float* l = pi + (r0 + t) * ldpi;
    const float* qq = q + (r0 + t) * ldq;
    const float* lp = pol + (r0 + t) * ldpol;
    const float* mu = mus + (s0 + t) * nA;
    const int ai = (int)actions[s0 + t];
    float m, z, mp, zp;
    softmax_row(l, nA, m, z);
    softmax_row(lp, nA, mp, zp);
    const float v = v_s[t], qret = qret_s[t], qi = qi_s[t], rho_i = rho_s[t];
    const float fa = expf(l[ai] - m) / z;
    const float Af = (qret - v) * fminf(a.c, rho_i);           // stop_gradient(adv * min(c, rho_i))
    float loss_bc = 0.0f, H = 0.0f, kg = 0.0f, kk = 0.0f, gg = 0.0f;
    // pass 1: g = d[-(loss_policy - ent_coef * entropy) * N] / df, k = -f_pol / (f + eps)
    for (int j = 0; j < nA; ++j) {
      const float f = expf(l[j] - m) / z, fp = expf(lp[j] - mp) / zp;
      const float rho = f / (mu[j] + eps);
      const float Bj = (qq[j] - v) * fmaxf(0.0f, 1.0f - a.c / (rho + eps)) * f;
      const float lf6 = logf(f + 1e-6f);
      loss_bc -= logf(f + eps) * Bj;
      H -= f * lf6;
      float g = Bj / (f + eps) - a.ent_coef * (lf6 + f / (f + 1e-6f));
      if (j == ai) g += Af / (fa + eps);
      const float k = -fp / (f + eps);
      kg += k * g;
      kk += k * k;
      gg += g * g;
    }
    const float adj = a.trust_region ? fmaxf(0.0f, (kg - a.delta) / (kk + eps)) : 0.0f;
    // pass 2: g' = g - adj k; d/dlogits = f * (<f, g'> - g') in sum scaling
    float fg = 0.0f, gpn = 0.0f;
    for (int j = 0; j < nA; ++j) {
      const float f = expf(l[j] - m) / z, fp = expf(lp[j] - mp) / zp;
      const float rho = f / (mu[j] + eps);
      const float Bj = (qq[j] - v) * fmaxf(0.0f, 1.0f - a.c / (rho + eps)) * f;
      float g = Bj / (f + eps) - a.ent_coef * (logf(f + 1e-6f) + f / (f + 1e-6f));
      if (j == ai) g += Af / (fa + eps);
      const float gp = g - adj * (-fp / (f + eps));
      fg += f * gp;
      gpn += gp * gp;
    }
    for (int j = 0; j < nA; ++j) {
      const float f = expf(l[j] - m) / z, fp = expf(lp[j] - mp) / zp;
      const float rho = f / (mu[j] + eps);
      const float Bj = (qq[j] - v) * fmaxf(0.0f, 1.0f - a.c / (rho + eps)) * f;
      float g = Bj / (f + eps) - a.ent_coef * (logf(f + 1e-6f) + f / (f + 1e-6f));
      if (j == ai) g += Af / (fa + eps);
      const float gp = g - adj * (-fp / (f + eps));
      dl[j] = __float2half_rn(f * (fg - gp));
      dqr[j] = __float2half_rn(j == ai ? -a.q_coef * (qret - qi) : 0.0f);
    }
    const double dqi = (double)qret - (double)qi;
    acc[0] += -(double)logf(fa + eps) * Af;     // loss_f * N
    acc[1] += loss_bc;                          // loss_bc * N
    acc[2] += 0.5 * dqi * dqi;                  // loss_q * N
    acc[3] += H;                                // entropy * N
    acc[4] += sqrt((double)kk);                 // ||k||
    acc[5] += sqrt((double)gg);                 // ||g|| (before the adjustment)
    acc[6] += fabs((double)kg);
    acc[7] += fabs((double)adj);
    acc[8] += sqrt((double)gpn);                // ||g'|| = N ||grads_f||
    acc[9] += qret;
    acc[10] += (double)qret * qret;
    acc[11] += dqi;
    acc[12] += dqi * dqi;
  }
  // block reduction in thread order, then the last CTA adds the envs' parts in env order
  __shared__ double red[4][ACER_NSTAT];
  __shared__ bool last;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int k = 0; k < ACER_NSTAT; ++k) {
    const double s = warp_sum_d(acc[k]);
    if (lane == 0) red[w][k] = s;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 0; k < ACER_NSTAT; ++k) {
      double s = 0.0;
      for (int ww = 0; ww < (int)(blockDim.x >> 5); ++ww) s += red[ww][k];
      g_acer_part[e * ACER_NSTAT + k] = s;
    }
    __threadfence();
    last = (atomicAdd(&g_acer_done, 1u) == (unsigned)nenv - 1);
  }
  __syncthreads();
  if (last && threadIdx.x == 0) {
    __threadfence();
    double S[ACER_NSTAT];
    for (int k = 0; k < ACER_NSTAT; ++k) S[k] = 0.0;
    for (int ee = 0; ee < nenv; ++ee)
      for (int k = 0; k < ACER_NSTAT; ++k) S[k] += *((volatile double*)&g_acer_part[ee * ACER_NSTAT + k]);
    const double N = (double)nenv * T;
    const double loss_f = S[0] / N, loss_bc = S[1] / N, loss_q = S[2] / N, ent = S[3] / N;
    const double loss_policy = loss_f + loss_bc;
    const double my = S[9] / N, vary = S[10] / N - my * my;
    const double md = S[11] / N, vard = S[12] / N - md * md;
    stats[0] = loss_policy + (double)a.q_coef * loss_q - (double)a.ent_coef * ent;
    stats[1] = loss_q;
    stats[2] = ent;
    stats[3] = loss_policy;
    stats[4] = loss_f;
    stats[5] = loss_bc;
    stats[6] = 1.0 - vard / vary;
    stats[7] = S[4] / N;
    stats[8] = S[5] / N;
    stats[9] = S[6] / N;
    stats[10] = S[7] / N;
    stats[11] = S[8] / N;
    g_acer_done = 0;
  }
  if (qret_out)
    for (int t = threadIdx.x; t < T; t += blockDim.x) qret_out[s0 + t] = qret_s[t];
}

// ---------------------------------------------------------------- optimiser
// g *= clip / max(||g||, clip); ms += (g^2 - ms) (1 - decay); p -= lr g / sqrt(ms + eps); shadow -= (shadow - p) (1-alpha)
__global__ void __launch_bounds__(256)
clip_rmsprop_ema_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ ms,
                        float* __restrict__ shadow, long long n, const float* __restrict__ lr_dev, float clip,
                        const double* __restrict__ sumsq, float one_minus_decay, float eps, float one_minus_alpha) {
  const float lr = *lr_dev;
  float sc = 1.0f;
  if (clip > 0.0f) sc = clip / fmaxf((float)sqrt(sumsq[0]), clip);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float gi = __fmul_rn(g[i], sc);
    float m = ms[i];
    m = __fadd_rn(m, __fmul_rn(__fsub_rn(__fmul_rn(gi, gi), m), one_minus_decay));
    ms[i] = m;
    const float pn = __fsub_rn(p[i], __fdiv_rn(__fmul_rn(gi, lr), __fsqrt_rn(__fadd_rn(m, eps))));
    p[i] = pn;
    const float s = shadow[i];
    shadow[i] = __fsub_rn(s, __fmul_rn(__fsub_rn(s, pn), one_minus_alpha));
  }
}

}  // namespace b200rl

using namespace b200rl;

extern "C" int b200rl_acer_step(const float* logits, long long ld, int nA, unsigned long long seed,
                                unsigned long long offset, const unsigned long long* offset_dev, long long* actions,
                                float* mu, long long B, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(logits && actions && mu && B > 0 && nA > 0 && ld >= nA, "acer_step: bad args");
  acer_step_kernel<<<(int)ceil_div_ll(B, 256), 256, 0, stream>>>(logits, ld, nA, seed, offset, offset_dev, actions,
                                                                 mu, B);
  return check_launch("acer_step_kernel");
}

extern "C" int b200rl_acer_stack_obs(const void* ring, int f32, long long slot_stride, const long long* idx, int nenv,
                                     int nsteps, int nstack, long long F, int nc, const uint8_t* dones_ring,
                                     void* out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(ring && dones_ring && out && nenv > 0 && nsteps > 0 && nstack > 0 && nstack <= 32 && F > 0 && nc > 0,
                 "acer_stack_obs: bad args");
  B200RL_REQUIRE((long long)nenv * (nsteps + 1) <= 65535, "acer_stack_obs: %d rows exceed the grid",
                 nenv * (nsteps + 1));
  const long long n = F * nstack * nc;
  const dim3 grid((unsigned)ceil_div_ll(n, 256 * 4) < 64u ? (unsigned)ceil_div_ll(n, 256 * 4) : 64u,
                  (unsigned)(nenv * (nsteps + 1)));
  if (f32)
    acer_stack_kernel<float><<<grid, 256, 0, stream>>>(static_cast<const float*>(ring), slot_stride, idx, nsteps,
                                                       nstack, F, nc, dones_ring, static_cast<float*>(out));
  else
    acer_stack_kernel<uint8_t><<<grid, 256, 0, stream>>>(static_cast<const uint8_t*>(ring), slot_stride, idx, nsteps,
                                                         nstack, F, nc, dones_ring, static_cast<uint8_t*>(out));
  return check_launch("acer_stack_kernel");
}

extern "C" int b200rl_acer_take(const long long* idx, int nenv, int nsteps, int nA, const long long* actions_ring,
                                const float* rewards_ring, const float* mus_ring, const uint8_t* dones_ring,
                                const uint8_t* masks_ring, long long* actions, float* rewards, float* mus,
                                uint8_t* dones, uint8_t* masks, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(actions_ring && rewards_ring && mus_ring && dones_ring && masks_ring && actions && rewards && mus &&
                 dones && masks && nenv > 0 && nsteps > 0 && nA > 0, "acer_take: bad args");
  acer_take_kernel<<<nenv, 128, 0, stream>>>(idx, nenv, nsteps, nA, actions_ring, rewards_ring, mus_ring, dones_ring,
                                             masks_ring, actions, rewards, mus, dones, masks);
  return check_launch("acer_take_kernel");
}

extern "C" int b200rl_acer_loss(const float* pi, long long ldpi, const float* q, long long ldq, const float* pol,
                                long long ldpol, const long long* actions, const float* rewards, const uint8_t* dones,
                                const float* mus, int nenv, int nsteps, int nA, float gamma, float c, float delta,
                                float q_coef, float ent_coef, int trust_region, void* dpi, long long lddpi, void* dq,
                                long long lddq, double* stats, float* f_out, float* v_out, float* qret_out,
                                void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(pi && q && pol && actions && rewards && dones && mus && dpi && dq && stats && nenv > 0 &&
                 nsteps > 0 && nA > 0, "acer_loss: bad args");
  B200RL_REQUIRE(nenv <= ACER_MAX_ENVS, "acer_loss: %d envs exceed %d", nenv, ACER_MAX_ENVS);
  AcerArgs a{nsteps, nA, trust_region, gamma, c, delta, q_coef, ent_coef};
  const size_t shm = 4 * (size_t)(nsteps + 1) * sizeof(float);
  B200RL_REQUIRE(shm <= 48 * 1024, "acer_loss: nsteps %d is too long", nsteps);
  acer_loss_kernel<<<nenv, 128, shm, stream>>>(pi, ldpi, q, ldq, pol, ldpol, actions, rewards, dones, mus, a,
                                               static_cast<__half*>(dpi), lddpi, static_cast<__half*>(dq), lddq,
                                               stats, f_out, v_out, qret_out);
  return check_launch("acer_loss_kernel");
}

extern "C" int b200rl_clip_rmsprop_ema(float* p, const float* g, float* ms, float* shadow, long long n,
                                       const float* lr_dev, float clip, const double* sumsq, float decay, float eps,
                                       float alpha, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(p && g && ms && shadow && lr_dev && n > 0, "clip_rmsprop_ema: bad args");
  B200RL_REQUIRE(clip <= 0.0f || sumsq != nullptr, "clip_rmsprop_ema: clipping needs the device sumsq");
  long long blocks = ceil_div_ll(n, 256);
  if (blocks > 8LL * device_num_sms()) blocks = 8LL * device_num_sms();
  clip_rmsprop_ema_kernel<<<(unsigned)blocks, 256, 0, stream>>>(p, g, ms, shadow, n, lr_dev, clip, sumsq,
                                                                1.0f - decay, eps, 1.0f - alpha);
  return check_launch("clip_rmsprop_ema_kernel");
}
