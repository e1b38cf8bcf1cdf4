// Row-wise policy-head kernels (one thread per sample; all HBM/latency bound, no reuse):
//   * act path  (PolicyWithValue.step, common/policies.py:77-96): Gumbel-max sample per categorical segment
//     (distributions.py:199-201, MultiCategorical :76-94), neglogp (:164-183) / Bernoulli sample+neglogp (:115-128) /
//     DiagGaussian sample+neglogp (:238-248)
//   * train path (ppo2/model.py:57-91): clipped-surrogate + clipped-value + entropy loss, its five
//     statistics, and the hand-derived gradient w.r.t. the head outputs (logits / mean, value), written
//     as fp16 in "sum" scaling (the 1/M of tf.reduce_mean is applied as alpha in the wgrad epilogues so
//     fp16 gradients do not underflow)
//   * per-minibatch advantage moments (ppo2/model.py:136-139)
// The rollout arrays are gathered in place through src_idx (no materialised minibatch, ppo2.py:165).
#include "common.cuh"
#include "cat_sample.cuh"

namespace b200rl {

// ---------------------------------------------------------------- categorical / multi-categorical: act
// A row of nA logits is cut into segments [seg_off[s], seg_off[s+1]) (MultiCategoricalPd, distributions.py:76-94,
// 206-225: one independent categorical per MultiDiscrete component); Discrete(n) is the single segment [0, n).
// MULTI = false is that single segment with its bounds known at compile time.  Uniform j of a row is always column j
// of the row's Philox stream (or of `uniforms`), whichever segment it falls in.
template <bool MULTI>
__device__ __forceinline__ void seg_bounds(const int* seg_off, int nA, int s, int& lo, int& hi) {
  lo = MULTI ? seg_off[s] : 0;
  hi = MULTI ? seg_off[s + 1] : nA;
}

// max, partition function and entropy (distributions.py:193-198) of the softmax over l[lo, hi)
__device__ __forceinline__ void seg_softmax(const float* l, int lo, int hi, float& m, float& z, float& logz, float& H) {
  m = -INFINITY;
  for (int j = lo; j < hi; ++j) m = fmaxf(m, l[j]);
  z = 0.0f;
  for (int j = lo; j < hi; ++j) z += expf(l[j] - m);
  logz = logf(z);
  H = 0.0f;
  for (int j = lo; j < hi; ++j) {
    const float a0 = l[j] - m;
    H += (expf(a0) / z) * (logz - a0);
  }
}

template <bool MULTI>
__global__ void __launch_bounds__(256)
cat_step_kernel(const float* __restrict__ logits, long long ld, int nA, const int* __restrict__ seg_off, int nseg,
                const float* __restrict__ vpred, long long ldv, const float* __restrict__ uniforms, uint64_t seed,
                uint64_t offset, const unsigned long long* __restrict__ offset_dev, long long* __restrict__ actions,
                float* __restrict__ values, float* __restrict__ neglogp, long long B) {
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  if (offset_dev) offset = *offset_dev;            // stream position kept on the device (CUDA-graph replays)
  if (!MULTI) nseg = 1;
  const float* l = logits + b * ld;
  uint32_t rnd[4];
  int held = -1;                                   // Philox counter whose 4 words are in rnd
  float nlp = 0.0f;
  for (int s = 0; s < nseg; ++s) {
    int lo, hi;
    seg_bounds<MULTI>(seg_off, nA, s, lo, hi);
    float m = -INFINITY;
    for (int j = lo; j < hi; ++j) m = fmaxf(m, l[j]);
    float z = 0.0f;
    for (int j = lo; j < hi; ++j) z += expf(l[j] - m);
    const int a = cat_gumbel_argmax(l, lo, hi, nA, uniforms, seed, b, offset, rnd, held);
    actions[b * nseg + s] = a - lo;
    nlp += (m + logf(z)) - l[a];             // sum of the components' neglogp (distributions.py:86-87)
  }
  neglogp[b] = nlp;
  values[b] = vpred[b * ldv];
}

// ---------------------------------------------------------------- Bernoulli (MultiBinary): act
// BernoulliPd (distributions.py:115-128, 254-276): p = sigmoid(l); x = float(u < p); neglogp = sum sigmoid_xent(l, x)
__device__ __forceinline__ float sigmoid_xent(float l, float y) {   // tf.nn.sigmoid_cross_entropy_with_logits
  return fmaxf(l, 0.0f) - l * y + log1pf(expf(-fabsf(l)));
}
__device__ __forceinline__ float sigmoidf(float l) { return 1.0f / (1.0f + expf(-l)); }

__global__ void __launch_bounds__(256)
bern_step_kernel(const float* __restrict__ logits, long long ld, int n, const float* __restrict__ vpred, long long ldv,
                 const float* __restrict__ uniforms, uint64_t seed, uint64_t offset,
                 const unsigned long long* __restrict__ offset_dev, float* __restrict__ actions,
                 float* __restrict__ values, float* __restrict__ neglogp, long long B) {
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  if (offset_dev) offset = *offset_dev;
  const float* l = logits + b * ld;
  uint32_t rnd[4];
  float nlp = 0.0f;
  for (int j = 0; j < n; ++j) {
    float u;
    if (uniforms) {
      u = uniforms[b * n + j];
    } else {
      if ((j & 3) == 0) philox4(seed, (uint64_t)b, (uint32_t)(j >> 2), (uint32_t)offset, rnd);
      u = u01_open(rnd[j & 3]);
    }
    const float lj = l[j];
    const float x = (u < sigmoidf(lj)) ? 1.0f : 0.0f;
    actions[b * n + j] = x;
    nlp += sigmoid_xent(lj, x);
  }
  neglogp[b] = nlp;
  values[b] = vpred[b * ldv];
}

// ---------------------------------------------------------------- gaussian: act
__global__ void __launch_bounds__(256)
gauss_step_kernel(const float* __restrict__ mean, long long ld, const float* __restrict__ logstd, int d,
                  const float* __restrict__ vpred, long long ldv, const float* __restrict__ normals, uint64_t seed,
                  uint64_t offset, const unsigned long long* __restrict__ offset_dev, float* __restrict__ actions,
                  float* __restrict__ values, float* __restrict__ neglogp, long long B) {
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  if (offset_dev) offset = *offset_dev;
  float q = 0.0f, sl = 0.0f;
  uint32_t rnd[4];
  float z0 = 0.f, z1 = 0.f;
  for (int j = 0; j < d; ++j) {
    float n;
    if (normals) {
      n = normals[b * d + j];
    } else {
      if ((j & 1) == 0) {
        if ((j & 3) == 0) philox4(seed, (uint64_t)b, (uint32_t)(j >> 2), (uint32_t)offset, rnd);
        const float u1 = u01_open(rnd[j & 3]), u2 = u01_open(rnd[(j & 3) + 1]);
        const float r = sqrtf(-2.0f * logf(u1));
        z0 = r * cospif(2.0f * u2);
        z1 = r * sinpif(2.0f * u2);
      }
      n = (j & 1) ? z1 : z0;
    }
    const float mu = mean[b * ld + j], ls = logstd[j];
    const float sd = expf(ls);
    const float x = mu + sd * n;                     // distributions.py:247-248
    actions[b * d + j] = x;
    const float t = (x - mu) / sd;
    q += t * t;
    sl += ls;
  }
  neglogp[b] = 0.5f * q + 0.5f * 1.8378770664093453f * (float)d + sl;   // log(2*pi)
  values[b] = vpred[b * ldv];
}

// ---------------------------------------------------------------- advantage moments (fp64, deterministic)
// ADV_BLOCKS blocks each reduce a FIXED contiguous slice in a fixed order; the block that finishes last adds the
// partials in index order, so the result does not depend on scheduling (same bits on every run).  The gathers are
// dependent loads (index -> returns, values): each thread keeps 8 in flight.  Sum and sum of squares are accumulated
// together in fp64 (inputs are fp32 differences of O(1): E[x^2] - mean^2 in fp64 loses nothing fp32 numpy would keep).
static constexpr int ADV_BLOCKS = 128;
__device__ double g_adv_part[2 * ADV_BLOCKS];
__device__ unsigned int g_adv_done = 0;

__global__ void __launch_bounds__(512)
adv_stats_kernel(const float* __restrict__ returns, const float* __restrict__ values,
                 const long long* __restrict__ src_idx, long long M, double* __restrict__ out) {
  __shared__ double red[2][16];
  __shared__ bool last;
  const int tid = threadIdx.x;
  constexpr int U = 8;
  const long long per = (M + gridDim.x - 1) / gridDim.x;
  const long long lo = (long long)blockIdx.x * per, hi = (lo + per < M) ? lo + per : M;
  double s1 = 0.0, s2 = 0.0;
  for (long long i0 = lo + tid; i0 < hi; i0 += (long long)blockDim.x * U) {
    float d[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long i = i0 + (long long)u * blockDim.x;
      d[u] = 0.0f;
      if (i < hi) {
        const long long s = src_idx ? src_idx[i] : i;
        d[u] = __fsub_rn(returns[s], values[s]);                 // float32 subtraction (model.py:136)
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      s1 += (double)d[u];
      s2 += (double)d[u] * (double)d[u];
    }
  }
  s1 = warp_sum_d(s1);
  s2 = warp_sum_d(s2);
  if ((tid & 31) == 0) { red[0][tid >> 5] = s1; red[1][tid >> 5] = s2; }
  __syncthreads();
  if (tid == 0) {
    double a = 0.0, b = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { a += red[0][w]; b += red[1][w]; }
    g_adv_part[2 * blockIdx.x] = a;
    g_adv_part[2 * blockIdx.x + 1] = b;
    __threadfence();
    last = (atomicAdd(&g_adv_done, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (last && tid == 0) {
    __threadfence();
    double a = 0.0, b = 0.0;
    for (int k = 0; k < (int)gridDim.x; ++k) {
      a += *((volatile double*)&g_adv_part[2 * k]);
      b += *((volatile double*)&g_adv_part[2 * k + 1]);
    }
    const double mean = a / (double)M;
    const double var = fmax(b / (double)M - mean * mean, 0.0);
    out[0] = mean;
    out[1] = sqrt(var);                                          // population std (numpy default ddof=0)
    g_adv_done = 0;
  }
}

// ---------------------------------------------------------------- shared pieces of the PPO loss
struct PpoCommon {
  const long long* src_idx;
  const float* returns;
  const float* old_values;
  const float* old_neglogp;
  const double* adv_stats;        // {mean, std}
  float cliprange, ent_coef, vf_coef;
  double* stats;                  // [5] sums: pg, vf, entropy, approxkl, clipfrac
  const float* cliprange_dev;     // optional: read the clip range from device memory (CUDA-graph replays)
};

__device__ __forceinline__ void block_accumulate5(double (&v)[5], double* stats) {
  __shared__ double red[5][8];
  const int tid = threadIdx.x;
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    const double s = warp_sum_d(v[k]);
    if ((tid & 31) == 0) red[k][tid >> 5] = s;
  }
  __syncthreads();
  if (tid < 5) {
    double s = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[tid][w];
    atomicAdd(stats + tid, s);
  }
}

// value-loss part: returns dL/dv (sum scaling, already times vf_coef) and the per-sample loss
__device__ __forceinline__ float value_loss_grad(float v, float oldv, float R, float clip, float vf_coef,
                                                 float& vloss) {
  const float dv = v - oldv;
  const float vclipped = oldv + fminf(fmaxf(dv, -clip), clip);
  const float l1 = (v - R) * (v - R), l2 = (vclipped - R) * (vclipped - R);
  vloss = 0.5f * fmaxf(l1, l2);
  float g;
  if (l1 >= l2) g = (v - R);                                       // tf.maximum: ties -> first argument
  else g = (dv >= -clip && dv <= clip) ? (vclipped - R) : 0.0f;    // clip_by_value passes grad inside [lo, hi]
  return vf_coef * g;
}

// policy-gradient part: returns dL/dneglogp (sum scaling)
__device__ __forceinline__ float pg_loss_grad(float nlp, float oldnlp, float adv, float clip, float& pgloss,
                                              float& kl, float& clipped) {
  const float ratio = expf(oldnlp - nlp);
  const float rc = fminf(fmaxf(ratio, 1.0f - clip), 1.0f + clip);
  const float p1 = -adv * ratio, p2 = -adv * rc;
  pgloss = fmaxf(p1, p2);
  const float dn = nlp - oldnlp;
  kl = 0.5f * dn * dn;
  clipped = (fabsf(ratio - 1.0f) > clip) ? 1.0f : 0.0f;
  // d(-A*ratio)/dnlp = A*ratio ; the clipped branch only passes inside the clip interval
  if (p1 >= p2) return adv * ratio;
  return (ratio >= 1.0f - clip && ratio <= 1.0f + clip) ? adv * ratio : 0.0f;
}

// ---------------------------------------------------------------- categorical / multi-categorical: loss + gradient
// actions: [*, nseg] rows (component index inside its segment), gathered through src_idx.  For logit j of segment s:
//   d nlp/dl_j = p_j - 1{j = off_s + a_s};  d(-ent_coef * sum_s H_s)/dl_j = ent_coef * p_j * (log p_j + H_s)
// with the segment's own entropy H_s.  The gradient pass recomputes each segment's softmax (MULTI = false: the single
// segment's values of the first pass are reused).
template <bool MULTI>
__global__ void __launch_bounds__(256)
cat_loss_kernel(const float* __restrict__ logits, long long ld, int nA, const int* __restrict__ seg_off, int nseg,
                const float* __restrict__ vpred, long long ldv, const long long* __restrict__ actions, PpoCommon pc,
                __half* __restrict__ dlogits, long long ld_dl, __half* __restrict__ dv, long long ld_dv, long long B) {
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  double st[5] = {0, 0, 0, 0, 0};
  if (!MULTI) nseg = 1;
  if (b < B) {
    const long long s = pc.src_idx ? pc.src_idx[b] : b;
    const float* l = logits + b * ld;
    const long long* arow = actions + s * nseg;
    float m, z, logz, Hs;                              // softmax of the current segment
    int lo, hi, a;
    float nlp = 0.0f, H = 0.0f;
    for (int g = 0; g < nseg; ++g) {
      seg_bounds<MULTI>(seg_off, nA, g, lo, hi);
      seg_softmax(l, lo, hi, m, z, logz, Hs);
      a = lo + (int)arow[g];
      nlp += (m + logz) - l[a];
      H += Hs;
    }
    const float R = pc.returns[s], oldv = pc.old_values[s];
    const float adv_raw = __fsub_rn(R, oldv);
    const float adv = (float)(((double)adv_raw - pc.adv_stats[0]) / (pc.adv_stats[1] + 1e-8));
    float pgl, kl, cf, vl;
    const float clip = pc.cliprange_dev ? *pc.cliprange_dev : pc.cliprange;
    const float g_nlp = pg_loss_grad(nlp, pc.old_neglogp[s], adv, clip, pgl, kl, cf);
    const float g_v = value_loss_grad(vpred[b * ldv], oldv, R, clip, pc.vf_coef, vl);
    // gradients leave as 16-byte stores (8 fp16 per store; one 2-byte store per column made the kernel
    // store-instruction bound: 32 rows x 2 B per instruction).  Columns past nA inside the last group are zero.
    __half* drow = dlogits + b * ld_dl;
    const bool vec = ((ld_dl & 7) == 0) && ((reinterpret_cast<uintptr_t>(dlogits) & 15) == 0) && (((nA + 7) & ~7) <= ld_dl);
    if (MULTI) {
      // segment by segment; the fp16 values pass through a 4-word shift register that leaves as one 16-byte store per
      // 8-column group (registers only: the row's segment layout is not known at compile time)
      uint32_t w0 = 0, w1 = 0, w2 = 0, w3 = 0;
      auto push = [&](__half h) {
        w0 = (w0 >> 16) | (w1 << 16);
        w1 = (w1 >> 16) | (w2 << 16);
        w2 = (w2 >> 16) | (w3 << 16);
        w3 = (w3 >> 16) | ((uint32_t)__half_as_ushort(h) << 16);
      };
      for (int g = 0; g < nseg; ++g) {
        seg_bounds<MULTI>(seg_off, nA, g, lo, hi);
        seg_softmax(l, lo, hi, m, z, logz, Hs);
        a = lo + (int)arow[g];
        for (int j = lo; j < hi; ++j) {
          const float a0 = l[j] - m;
          const float pj = expf(a0) / z;
          const float logpj = a0 - logz;
          const __half h = __float2half_rn(g_nlp * (pj - (j == a ? 1.0f : 0.0f)) + pc.ent_coef * pj * (logpj + Hs));
          if (vec) {
            push(h);
            if ((j & 7) == 7) *reinterpret_cast<uint4*>(drow + (j - 7)) = make_uint4(w0, w1, w2, w3);
          } else {
            drow[j] = h;
          }
        }
      }
      if (vec && (nA & 7)) {                           // last partial group: columns past nA are zero
        for (int j = nA; j & 7; ++j) push(__float2half_rn(0.0f));
        *reinterpret_cast<uint4*>(drow + (nA & ~7)) = make_uint4(w0, w1, w2, w3);
      }
    } else {
      for (int j0 = 0; j0 < nA; j0 += 8) {
        __align__(16) __half g8[8];
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int j = j0 + jj;
          float gj = 0.0f;
          if (j < nA) {
            const float a0 = l[j] - m;
            const float pj = expf(a0) / z;
            const float logpj = a0 - logz;
            gj = g_nlp * (pj - (j == a ? 1.0f : 0.0f)) + pc.ent_coef * pj * (logpj + Hs);
          }
          g8[jj] = __float2half_rn(gj);
        }
        if (vec) {
          *reinterpret_cast<uint4*>(drow + j0) = *reinterpret_cast<const uint4*>(g8);
        } else {
          for (int jj = 0; jj < 8 && j0 + jj < nA; ++jj) drow[j0 + jj] = g8[jj];
        }
      }
    }
    dv[b * ld_dv] = __float2half_rn(g_v);
    st[0] = pgl; st[1] = vl; st[2] = H; st[3] = kl; st[4] = cf;
  }
  block_accumulate5(st, pc.stats);
}

// ---------------------------------------------------------------- Bernoulli (MultiBinary): loss + gradient
// actions: float32 [*, n] rows of 0 / 1.  neglogp = sum_j sigmoid_xent(l_j, x_j), entropy = sum_j sigmoid_xent(l_j, p_j)
// (distributions.py:120-125).  TF differentiates the entropy through its labels p = sigmoid(l) too, so
//   d nlp/dl_j = p_j - x_j;  d(-ent_coef * H)/dl_j = ent_coef * l_j * p_j * (1 - p_j)   (total derivative)
__global__ void __launch_bounds__(256)
bern_loss_kernel(const float* __restrict__ logits, long long ld, int n, const float* __restrict__ vpred, long long ldv,
                 const float* __restrict__ actions, PpoCommon pc, __half* __restrict__ dlogits, long long ld_dl,
                 __half* __restrict__ dv, long long ld_dv, long long B) {
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  double st[5] = {0, 0, 0, 0, 0};
  if (b < B) {
    const long long s = pc.src_idx ? pc.src_idx[b] : b;
    const float* l = logits + b * ld;
    const float* x = actions + s * n;
    float nlp = 0.0f, H = 0.0f;
    for (int j = 0; j < n; ++j) {
      const float lj = l[j];
      nlp += sigmoid_xent(lj, x[j]);
      H += sigmoid_xent(lj, sigmoidf(lj));
    }
    const float R = pc.returns[s], oldv = pc.old_values[s];
    const float adv_raw = __fsub_rn(R, oldv);
    const float adv = (float)(((double)adv_raw - pc.adv_stats[0]) / (pc.adv_stats[1] + 1e-8));
    float pgl, kl, cf, vl;
    const float clip = pc.cliprange_dev ? *pc.cliprange_dev : pc.cliprange;
    const float g_nlp = pg_loss_grad(nlp, pc.old_neglogp[s], adv, clip, pgl, kl, cf);
    const float g_v = value_loss_grad(vpred[b * ldv], oldv, R, clip, pc.vf_coef, vl);
    __half* drow = dlogits + b * ld_dl;
    const bool vec = ((ld_dl & 7) == 0) && ((reinterpret_cast<uintptr_t>(dlogits) & 15) == 0) && (((n + 7) & ~7) <= ld_dl);
    for (int j0 = 0; j0 < n; j0 += 8) {
      __align__(16) __half g8[8];
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const int j = j0 + jj;
        float gj = 0.0f;
        if (j < n) {
          const float lj = l[j];
          const float pj = sigmoidf(lj);
          gj = g_nlp * (pj - x[j]) + pc.ent_coef * lj * pj * (1.0f - pj);
        }
        g8[jj] = __float2half_rn(gj);
      }
      if (vec) {
        *reinterpret_cast<uint4*>(drow + j0) = *reinterpret_cast<const uint4*>(g8);
      } else {
        for (int jj = 0; jj < 8 && j0 + jj < n; ++jj) drow[j0 + jj] = g8[jj];
      }
    }
    dv[b * ld_dv] = __float2half_rn(g_v);             // after the logit stores: column n of the same row when fused
    st[0] = pgl; st[1] = vl; st[2] = H; st[3] = kl; st[4] = cf;
  }
  block_accumulate5(st, pc.stats);
}

// ---------------------------------------------------------------- gaussian: loss + gradient
// One thread per sample.  DMAX > 0: the whole action row lives in registers -- all 2*d global loads of a thread are
// issued back to back (the generic loop, DMAX = 0, waits for each element's loads in turn: measured 143 us for 262144
// rows of d = 17, all of it load latency) and exp(logstd) is computed once per block instead of once per element.
template <int DMAX>
__global__ void __launch_bounds__(256)
gauss_loss_kernel(const float* __restrict__ mean, long long ld, const float* __restrict__ logstd, int d,
                  const float* __restrict__ vpred, long long ldv, const float* __restrict__ actions, PpoCommon pc,
                  __half* __restrict__ dmean, long long ld_dm, __half* __restrict__ dv, long long ld_dv,
                  float* __restrict__ dls_part, float inv_M, long long B) {
  // [8 warps][d] per-warp partials of dL/dlogstd, then [d] std, [d] logstd; dls_part[block, j] gets the block's sum
  extern __shared__ float s_dls[];
  float* s_std = s_dls + 8 * d;
  float* s_ls = s_dls + 9 * d;
  for (int j = threadIdx.x; j < 8 * d; j += blockDim.x) s_dls[j] = 0.0f;
  for (int j = threadIdx.x; j < d; j += blockDim.x) {
    const float ls = logstd[j];
    s_ls[j] = ls;
    s_std[j] = expf(ls);
  }
  __syncthreads();
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  double st[5] = {0, 0, 0, 0, 0};
  float g_nlp = 0.0f, g_v = 0.0f;
  long long srow = 0;
  constexpr int TN = DMAX > 0 ? DMAX : 1;
  float t[TN];                                       // (x - mu) / sigma of this sample (DMAX > 0)
  if (b < B) {
    const long long s = pc.src_idx ? pc.src_idx[b] : b;
    srow = s;
    float q = 0.0f, sl = 0.0f;
    if (DMAX > 0) {
      float av[TN], mv[TN];
#pragma unroll
      for (int j = 0; j < TN; ++j) {
        av[j] = (j < d) ? actions[s * d + j] : 0.0f;
        mv[j] = (j < d) ? mean[b * ld + j] : 0.0f;
      }
#pragma unroll
      for (int j = 0; j < TN; ++j) {
        t[j] = (j < d) ? (av[j] - mv[j]) / s_std[j] : 0.0f;
        q += t[j] * t[j];
        sl += (j < d) ? s_ls[j] : 0.0f;
      }
    } else {
      for (int j = 0; j < d; ++j) {
        const float tt = (actions[s * d + j] - mean[b * ld + j]) / s_std[j];
        q += tt * tt;
        sl += s_ls[j];
      }
    }
    const float nlp = 0.5f * q + 0.5f * 1.8378770664093453f * (float)d + sl;
    const float H = sl + 0.5f * 2.8378770664093453f * (float)d;       // sum(logstd + .5*log(2*pi*e))
    const float R = pc.returns[s], oldv = pc.old_values[s];
    const float adv_raw = __fsub_rn(R, oldv);
    const float adv = (float)(((double)adv_raw - pc.adv_stats[0]) / (pc.adv_stats[1] + 1e-8));
    float pgl, kl, cf, vl;
    const float clip = pc.cliprange_dev ? *pc.cliprange_dev : pc.cliprange;
    g_nlp = pg_loss_grad(nlp, pc.old_neglogp[s], adv, clip, pgl, kl, cf);
    g_v = value_loss_grad(vpred[b * ldv], oldv, R, clip, pc.vf_coef, vl);
    st[0] = pgl; st[1] = vl; st[2] = H; st[3] = kl; st[4] = cf;
  } else if (DMAX > 0) {
#pragma unroll
    for (int j = 0; j < TN; ++j) t[j] = 0.0f;
  }
  // every lane takes part in the warp reductions of dL/dlogstd (inactive rows contribute 0); each warp adds into its own
  // shared-memory slot, so the block's sum has a fixed order
  const bool vec = ((ld_dm & 7) == 0) && ((reinterpret_cast<uintptr_t>(dmean) & 15) == 0) && (((d + 7) & ~7) <= ld_dm);
  auto chunk8 = [&](int j0, const float* t8) {       // t8: this sample's 8 standardised residuals (null: recompute)
    __align__(16) __half g8[8];
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const int j = j0 + jj;
      float gl = 0.0f, gm = 0.0f;
      if (b < B && j < d) {
        const float sd = s_std[j];
        const float tt = t8 ? t8[jj] : (actions[srow * d + j] - mean[b * ld + j]) / sd;
        gm = g_nlp * (-tt / sd);                     // d nlp/d mu = -(x-mu)/sigma^2
        gl = g_nlp * (1.0f - tt * tt) - pc.ent_coef; // d nlp/d logstd = 1 - t^2 ; d(-ent_coef*H)/d logstd = -ent_coef
      }
      g8[jj] = __float2half_rn(gm);
      if (j < d) {                                   // uniform across the warp
        gl = warp_sum(gl);
        if ((threadIdx.x & 31) == 0) s_dls[(threadIdx.x >> 5) * d + j] += gl;
      }
    }
    if (b < B) {
      if (vec) {
        *reinterpret_cast<uint4*>(dmean + b * ld_dm + j0) = *reinterpret_cast<const uint4*>(g8);
      } else {
        for (int jj = 0; jj < 8 && j0 + jj < d; ++jj) dmean[b * ld_dm + j0 + jj] = g8[jj];
      }
    }
  };
  if (DMAX > 0) {
#pragma unroll
    for (int j0 = 0; j0 < TN; j0 += 8)
      if (j0 < d) chunk8(j0, &t[j0]);
  } else {
    for (int j0 = 0; j0 < d; j0 += 8) chunk8(j0, nullptr);
  }
  if (b < B) dv[b * ld_dv] = __float2half_rn(g_v);   // after dmean: with a fused [pi | vf] head dv is column d of the same row
  __syncthreads();
  for (int j = threadIdx.x; j < d; j += blockDim.x) {
    float t = 0.0f;
    for (int w = 0; w < 8; ++w) t += s_dls[w * d + j];
    dls_part[(long long)blockIdx.x * d + j] = t * inv_M;
  }
  block_accumulate5(st, pc.stats);
}

}  // namespace b200rl

using namespace b200rl;

// ---------------------------------------------------------------- launchers
extern "C" int b200rl_cat_step(const float* logits, long long ld, int nA, const int* seg_off, int nseg,
                               const float* vpred, long long ldv, const float* uniforms, unsigned long long seed,
                               unsigned long long offset, const unsigned long long* offset_dev, long long* actions,
                               float* values, float* neglogp, long long B, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(logits && vpred && actions && values && neglogp && B > 0 && nA > 0, "cat_step: bad args");
  B200RL_REQUIRE(seg_off == nullptr || (nseg >= 1 && nseg <= nA), "cat_step: a segment table needs 1 <= nseg <= nA");
  const int grid = (int)ceil_div_ll(B, 256);
  if (seg_off)
    cat_step_kernel<true><<<grid, 256, 0, stream>>>(logits, ld, nA, seg_off, nseg, vpred, ldv, uniforms, seed, offset,
                                                    offset_dev, actions, values, neglogp, B);
  else
    cat_step_kernel<false><<<grid, 256, 0, stream>>>(logits, ld, nA, nullptr, 1, vpred, ldv, uniforms, seed, offset,
                                                     offset_dev, actions, values, neglogp, B);
  return check_launch("cat_step_kernel");
}

extern "C" int b200rl_bern_step(const float* logits, long long ld, int n, const float* vpred, long long ldv,
                                const float* uniforms, unsigned long long seed, unsigned long long offset,
                                const unsigned long long* offset_dev, float* actions, float* values, float* neglogp,
                                long long B, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(logits && vpred && actions && values && neglogp && B > 0 && n > 0, "bern_step: bad args");
  bern_step_kernel<<<(int)ceil_div_ll(B, 256), 256, 0, stream>>>(logits, ld, n, vpred, ldv, uniforms, seed, offset,
                                                                  offset_dev, actions, values, neglogp, B);
  return check_launch("bern_step_kernel");
}

extern "C" int b200rl_gauss_step(const float* mean, long long ld, const float* logstd, int d, const float* vpred,
                                 long long ldv, const float* normals, unsigned long long seed,
                                 unsigned long long offset, const unsigned long long* offset_dev, float* actions,
                                 float* values, float* neglogp, long long B, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(mean && logstd && vpred && actions && values && neglogp && B > 0 && d > 0, "gauss_step: bad args");
  gauss_step_kernel<<<(int)ceil_div_ll(B, 256), 256, 0, stream>>>(mean, ld, logstd, d, vpred, ldv, normals, seed,
                                                                   offset, offset_dev, actions, values, neglogp, B);
  return check_launch("gauss_step_kernel");
}

extern "C" int b200rl_adv_stats(const float* returns, const float* values, const long long* src_idx, long long M,
                                double* out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(returns && values && out && M > 0, "adv_stats: bad args");
  const int blocks = (int)((M + 4095) / 4096 < ADV_BLOCKS ? (M + 4095) / 4096 : ADV_BLOCKS);
  adv_stats_kernel<<<blocks, 512, 0, stream>>>(returns, values, src_idx, M, out);
  return check_launch("adv_stats_kernel");
}

extern "C" int b200rl_cat_loss(const float* logits, long long ld, int nA, const int* seg_off, int nseg,
                               const float* vpred, long long ldv, const long long* actions, const long long* src_idx,
                               const float* returns, const float* old_values, const float* old_neglogp,
                               const double* adv_stats, float cliprange, float ent_coef, float vf_coef, void* dlogits,
                               long long ld_dl, void* dv, long long ld_dv, double* stats, long long B,
                               const float* cliprange_dev, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(logits && vpred && actions && returns && old_values && old_neglogp && adv_stats && dlogits && dv &&
                     stats && B > 0 && nA > 0,
                 "cat_loss: bad args");
  B200RL_REQUIRE(seg_off == nullptr || (nseg >= 1 && nseg <= nA), "cat_loss: a segment table needs 1 <= nseg <= nA");
  PpoCommon pc{src_idx, returns, old_values, old_neglogp, adv_stats, cliprange, ent_coef, vf_coef, stats, cliprange_dev};
  const int grid = (int)ceil_div_ll(B, 256);
  if (seg_off)
    cat_loss_kernel<true><<<grid, 256, 0, stream>>>(logits, ld, nA, seg_off, nseg, vpred, ldv, actions, pc,
                                                    reinterpret_cast<__half*>(dlogits), ld_dl,
                                                    reinterpret_cast<__half*>(dv), ld_dv, B);
  else
    cat_loss_kernel<false><<<grid, 256, 0, stream>>>(logits, ld, nA, nullptr, 1, vpred, ldv, actions, pc,
                                                     reinterpret_cast<__half*>(dlogits), ld_dl,
                                                     reinterpret_cast<__half*>(dv), ld_dv, B);
  return check_launch("cat_loss_kernel");
}

extern "C" int b200rl_bern_loss(const float* logits, long long ld, int n, const float* vpred, long long ldv,
                                const float* actions, const long long* src_idx, const float* returns,
                                const float* old_values, const float* old_neglogp, const double* adv_stats,
                                float cliprange, float ent_coef, float vf_coef, void* dlogits, long long ld_dl,
                                void* dv, long long ld_dv, double* stats, long long B, const float* cliprange_dev,
                                void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(logits && vpred && actions && returns && old_values && old_neglogp && adv_stats && dlogits && dv &&
                     stats && B > 0 && n > 0,
                 "bern_loss: bad args");
  PpoCommon pc{src_idx, returns, old_values, old_neglogp, adv_stats, cliprange, ent_coef, vf_coef, stats, cliprange_dev};
  bern_loss_kernel<<<(int)ceil_div_ll(B, 256), 256, 0, stream>>>(logits, ld, n, vpred, ldv, actions, pc,
                                                                  reinterpret_cast<__half*>(dlogits), ld_dl,
                                                                  reinterpret_cast<__half*>(dv), ld_dv, B);
  return check_launch("bern_loss_kernel");
}

extern "C" int b200rl_gauss_loss(const float* mean, long long ld, const float* logstd, int d, const float* vpred,
                                 long long ldv, const float* actions, const long long* src_idx, const float* returns,
                                 const float* old_values, const float* old_neglogp, const double* adv_stats,
                                 float cliprange, float ent_coef, float vf_coef, void* dmean, long long ld_dm, void* dv,
                                 long long ld_dv, float* dlogstd, float inv_M, double* stats, long long B,
                                 const float* cliprange_dev, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(mean && logstd && vpred && actions && returns && old_values && old_neglogp && adv_stats && dmean &&
                     dv && dlogstd && stats && B > 0,
                 "gauss_loss: bad args");
  PpoCommon pc{src_idx, returns, old_values, old_neglogp, adv_stats, cliprange, ent_coef, vf_coef, stats, cliprange_dev};
  const int grid = (int)ceil_div_ll(B, 256);
  const size_t sm = 10 * (size_t)d * sizeof(float);
  float* part = det_workspace((size_t)grid * d, stream);
  if (!part) return B200RL_ERR_CUDA;
  if (d <= 8)
    gauss_loss_kernel<8><<<grid, 256, sm, stream>>>(mean, ld, logstd, d, vpred, ldv, actions, pc,
                                                    reinterpret_cast<__half*>(dmean), ld_dm,
                                                    reinterpret_cast<__half*>(dv), ld_dv, part, inv_M, B);
  else if (d <= 24)
    gauss_loss_kernel<24><<<grid, 256, sm, stream>>>(mean, ld, logstd, d, vpred, ldv, actions, pc,
                                                     reinterpret_cast<__half*>(dmean), ld_dm,
                                                     reinterpret_cast<__half*>(dv), ld_dv, part, inv_M, B);
  else
    gauss_loss_kernel<0><<<grid, 256, sm, stream>>>(mean, ld, logstd, d, vpred, ldv, actions, pc,
                                                    reinterpret_cast<__half*>(dmean), ld_dm,
                                                    reinterpret_cast<__half*>(dv), ld_dv, part, inv_M, B);
  const int rc = check_launch("gauss_loss_kernel");
  return rc == B200RL_OK ? sum_partials(part, grid, 1, d, dlogstd, d, stream) : rc;
}
