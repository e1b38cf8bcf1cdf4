// Device-resident prioritized replay (fp64 sum / min segment trees) and the DQN TD / Huber step.
//
// Replaces the pure-python baselines/common/segment_tree.py and the sampling arithmetic of
// baselines/deepq/replay_buffer.py:100-191 (reference).  Trees keep the reference's layout
// (2*capacity float64 nodes, root at 1, leaves at [capacity, 2*capacity)) and every ancestor is
// recomputed as op(left child, right child), so after a batch of writes the trees are bit-identical
// to the reference's sequential updates (last write to a duplicated index wins, as in the python loop).
// Sampling is latency bound (batch x log2(capacity) dependent 8-byte reads that stay in L2).
//
// Priorities follow the reference's dtypes: its new priorities are |td| + eps on the float32 TD errors, so float32
// values, and the leaves are float64 powers of them (priority ** alpha, NumPy 1.x scalar promotion).  Every pow here
// (leaves, the add path's max_priority ** alpha, importance weights) is the correctly rounded pow_cr of pow_cr.cuh, so
// the leaves and weights do not depend on which libm rounds them.  A priority that is not > 0 (the reference's
// `assert priority > 0`, e.g. a NaN TD error) sets a sticky device flag that the buffer raises on; sampling never
// returns an index outside the stored range, even from such a tree.
#include "common.cuh"
#include "pow_cr.cuh"

namespace b200rl {

// one block; n <= 1024 per launch (host chunks larger batches, which keeps sequential semantics)
__global__ void __launch_bounds__(1024)
tree_set_kernel(double* __restrict__ sum_tree, double* __restrict__ min_tree, long long capacity,
                const long long* __restrict__ idx, const double* __restrict__ vals, int n) {
  __shared__ long long s_idx[1024];
  const int i = threadIdx.x;
  long long my = -1;
  if (i < n) { my = idx[i]; s_idx[i] = my; }
  __syncthreads();
  if (i < n) {
    bool last = true;
    for (int j = i + 1; j < n; ++j) if (s_idx[j] == my) { last = false; break; }
    if (last) {
      sum_tree[capacity + my] = vals[i];
      min_tree[capacity + my] = vals[i];
    }
  }
  __syncthreads();
  for (long long span = capacity >> 1, node = (capacity + (my < 0 ? 0 : my)) >> 1; span >= 1; span >>= 1, node >>= 1) {
    if (i < n) {
      const double a = sum_tree[2 * node], b = sum_tree[2 * node + 1];
      const double c = min_tree[2 * node], d = min_tree[2 * node + 1];
      sum_tree[node] = __dadd_rn(a, b);
      min_tree[node] = fmin(c, d);
    }
    __threadfence_block();
    __syncthreads();
  }
}

// Range sum with the SAME association of additions as the reference's recursive top-down decomposition
// (segment_tree.py:36-49), evaluated iteratively (device recursion overflowed the stack at capacity 2^20):
//   * descend to the node where the range splits;
//   * the left part is a right-aligned range  -> ((innermost + v) + v) ...   (complete right siblings outward)
//   * the right part is a left-aligned range  -> v + (v + (... innermost))   (complete left siblings outward)
__device__ double fold_left_aligned(const double* v, long long hi, long long node, long long nlo, long long nhi) {
  double st[48];
  int n = 0;
  while (hi != nhi) {
    const long long mid = (nlo + nhi) / 2;
    if (hi <= mid) { node = 2 * node; nhi = mid; }
    else { st[n++] = v[2 * node]; node = 2 * node + 1; nlo = mid + 1; }
  }
  double acc = v[node];
  while (n > 0) acc = __dadd_rn(st[--n], acc);
  return acc;
}
__device__ double fold_right_aligned(const double* v, long long lo, long long node, long long nlo, long long nhi) {
  double st[48];
  int n = 0;
  while (lo != nlo) {
    const long long mid = (nlo + nhi) / 2;
    if (mid + 1 <= lo) { node = 2 * node + 1; nlo = mid + 1; }
    else { st[n++] = v[2 * node + 1]; node = 2 * node; nhi = mid; }
  }
  double acc = v[node];
  while (n > 0) acc = __dadd_rn(acc, st[--n]);
  return acc;
}
__device__ double fold_sum(const double* v, long long lo, long long hi, long long node, long long nlo, long long nhi) {
  while (true) {
    if (lo == nlo && hi == nhi) return v[node];
    const long long mid = (nlo + nhi) / 2;
    if (hi <= mid) { node = 2 * node; nhi = mid; continue; }
    if (mid + 1 <= lo) { node = 2 * node + 1; nlo = mid + 1; continue; }
    const double l = fold_right_aligned(v, lo, 2 * node, nlo, mid);
    const double r = fold_left_aligned(v, hi, 2 * node + 1, mid + 1, nhi);
    return __dadd_rn(l, r);
  }
}

__global__ void tree_range_sum_kernel(const double* __restrict__ tree, long long capacity, long long start,
                                      long long end_inclusive, double* __restrict__ out) {
  if (threadIdx.x == 0 && blockIdx.x == 0) out[0] = fold_sum(tree, start, end_inclusive, 1, 0, capacity - 1);
}

using powcr::pow_cr;

// proportional stratified sampling + importance weights (replay_buffer.py:107-115,157-165).
// bad (optional): set to 1 when the tree holds a priority that is not > 0 (NaN root sum, zero minimum) or the descent
// ends past the stored range, which only such a tree can make it do; that slot returns index 0 instead.
__global__ void __launch_bounds__(256)
per_sample_kernel(const double* __restrict__ sum_tree, const double* __restrict__ min_tree, long long capacity,
                  long long n_stored, const double* __restrict__ uniforms, int batch, double beta,
                  long long* __restrict__ idx_out, double* __restrict__ w_out, float* __restrict__ w_out_f32,
                  int* __restrict__ bad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= batch) return;
  // NOTE the reference's quirk: sum(0, len-1) has an EXCLUSIVE end, so the last stored element is dropped
  const double p_total = fold_sum(sum_tree, 0, n_stored - 2, 1, 0, capacity - 1);
  const double every = p_total / (double)batch;
  double mass = __dadd_rn(__dmul_rn(uniforms[i], every), __dmul_rn((double)i, every));
  long long node = 1;
  while (node < capacity) {                                   // segment_tree.py:124-131
    const double left = sum_tree[2 * node];
    if (left > mass) node = 2 * node;
    else { mass = __dsub_rn(mass, left); node = 2 * node + 1; }
  }
  long long leaf = node - capacity;
  const double total = sum_tree[1];
  if (leaf >= n_stored || !(total > 0.0) || !(min_tree[1] > 0.0)) {
    if (bad) *bad = 1;
    if (leaf >= n_stored) { leaf = 0; node = capacity; }
  }
  idx_out[i] = leaf;
  const double p_min = min_tree[1] / total;
  const double max_w = pow_cr(p_min * (double)n_stored, -beta);
  const double p = sum_tree[node] / total;
  const double w = pow_cr(p * (double)n_stored, -beta) / max_w;
  w_out[i] = w;
  if (w_out_f32) w_out_f32[i] = (float)w;
}

// new priorities from TD errors, deepq.py:302 + replay_buffer.py:186-191: p = float32(|td| + float32(eps)) (float32
// TD errors plus a python float stay float32), leaf = p^alpha in float64, running max of p over every entry (duplicates
// included).  bad: set to 1 when some p is not > 0 (NaN or zero), where the reference asserts.
__global__ void __launch_bounds__(256)
per_priorities_kernel(const float* __restrict__ td, int n, double eps, double alpha, double* __restrict__ powered,
                      double* __restrict__ max_priority, int* __restrict__ bad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double p = (double)__fadd_rn(fabsf(td[i]), __double2float_rn(eps));
  powered[i] = pow_cr(p, alpha);
  if (!(p > 0.0)) { *bad = 1; return; }
  // atomic max on a positive double == atomic max on its bit pattern as signed 64-bit
  atomicMax(reinterpret_cast<long long*>(max_priority), __double_as_longlong(p));
}

// out[i] = x[i]^y with the same pow as the leaves (the add path's max_priority ** alpha)
__global__ void per_pow_kernel(const double* __restrict__ x, int n, double y, double* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = pow_cr(x[i], y);
}

// ------------------------------------------------------------------------------------------ DQN TD step
// build_graph.py:388-413 + tf_util.py:39-45.  Inputs are the raw head outputs; with dueling,
// q = s + (a - mean(a)) (deepq/models.py:38-40).  Gradients are written in "sum" scaling
// (d sum_i w_i*huber(td_i) / d head outputs); the 1/batch of reduce_mean is the wgrad alpha.
struct QHead {
  const float* a; long long lda;      // action scores [B, nA]
  const float* s; long long lds;      // state score [B] (nullptr when not dueling)
};

__device__ __forceinline__ float q_value(const QHead& h, long long b, int j, int nA, float mean_a) {
  const float a = h.a[b * h.lda + j];
  return h.s ? h.s[b * h.lds] + (a - mean_a) : a;
}
__device__ __forceinline__ float mean_adv(const QHead& h, long long b, int nA) {
  if (!h.s) return 0.0f;
  float m = 0.0f;
  for (int j = 0; j < nA; ++j) m += h.a[b * h.lda + j];
  return m / (float)nA;
}

__global__ void __launch_bounds__(256)
dqn_td_kernel(QHead qt, QHead q1_online, QHead q1_target, int nA, const long long* __restrict__ idx,
              const long long* __restrict__ actions, const float* __restrict__ rewards,
              const float* __restrict__ dones, const float* __restrict__ weights, float gamma, int double_q,
              float* __restrict__ td_out, __half* __restrict__ d_a, long long ld_da, __half* __restrict__ d_s,
              long long ld_ds, double* __restrict__ loss_sum, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const long long s = idx ? idx[b] : b;
  const int act = (int)actions[s];
  const float m_t = mean_adv(qt, b, nA);
  const float q_sel = q_value(qt, b, act, nA, m_t);
  const float m_tg = mean_adv(q1_target, b, nA);
  float best;
  if (double_q) {
    const float m_on = mean_adv(q1_online, b, nA);
    int arg = 0;
    float bq = -INFINITY;
    for (int j = 0; j < nA; ++j) {
      const float q = q_value(q1_online, b, j, nA, m_on);
      if (q > bq) { bq = q; arg = j; }
    }
    best = q_value(q1_target, b, arg, nA, m_tg);
  } else {
    best = -INFINITY;
    for (int j = 0; j < nA; ++j) best = fmaxf(best, q_value(q1_target, b, j, nA, m_tg));
  }
  const float target = rewards[s] + gamma * ((1.0f - dones[s]) * best);
  const float td = q_sel - target;
  td_out[b] = td;
  const float w = weights[b];
  const float atd = fabsf(td);
  const float hub = atd < 1.0f ? 0.5f * td * td : (atd - 0.5f);
  atomicAdd(loss_sum, (double)(w * hub));
  const float g = w * (atd < 1.0f ? td : (td > 0.0f ? 1.0f : -1.0f));     // d huber / d td
  // dq_j = g * 1{j = act};  dueling: dA_j = dq_j - mean_j(dq) = g*(1{j=act} - 1/nA), dS = g
  for (int j = 0; j < nA; ++j) {
    float v = (j == act) ? g : 0.0f;
    if (qt.s) v -= g / (float)nA;
    d_a[b * ld_da + j] = __float2half_rn(v);
  }
  if (qt.s) d_s[b * ld_ds] = __float2half_rn(g);
}

// epsilon-greedy action selection (build_graph.py:184-191) with counter-based randomness
__global__ void dqn_act_kernel(QHead q, int nA, float eps, unsigned long long seed, unsigned long long step,
                               const float* __restrict__ eps_dev, const unsigned long long* __restrict__ step_dev,
                               long long* __restrict__ actions, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  if (eps_dev) eps = *eps_dev;                       // exploration rate / stream position kept on the device
  if (step_dev) step = *step_dev;                    // (CUDA-graph replays of the acting pass)
  const float m = mean_adv(q, b, nA);
  int arg = 0;
  float bq = -INFINITY;
  for (int j = 0; j < nA; ++j) {
    const float v = q_value(q, b, j, nA, m);
    if (v > bq) { bq = v; arg = j; }
  }
  // splitmix64 on (seed, step, b): two draws
  unsigned long long x = seed + 0x9E3779B97F4A7C15ull * (step * 1315423911ull + (unsigned long long)b + 1);
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  x ^= x >> 31;
  const float u = ((float)(x >> 40) + 0.5f) * (1.0f / 16777216.0f);
  const int r = (int)((x & 0xFFFFFFull) % (unsigned long long)nA);
  actions[b] = (u < eps) ? r : arg;
}

}  // namespace b200rl

using namespace b200rl;

// ------------------------------------------------------------------------------------------ launchers
extern "C" int b200rl_tree_set(double* sum_tree, double* min_tree, long long capacity, const long long* idx,
                               const double* vals, int n, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(sum_tree && min_tree && idx && vals && n > 0, "tree_set: bad args");
  B200RL_REQUIRE(capacity > 0 && (capacity & (capacity - 1)) == 0, "tree_set: capacity must be a power of two");
  for (int o = 0; o < n; o += 1024) {
    const int m = n - o < 1024 ? n - o : 1024;
    tree_set_kernel<<<1, 1024, 0, stream>>>(sum_tree, min_tree, capacity, idx + o, vals + o, m);
  }
  return check_launch("tree_set_kernel");
}

extern "C" int b200rl_tree_range_sum(const double* tree, long long capacity, long long start, long long end,
                                     double* out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(tree && out, "tree_range_sum: bad args");
  // reference semantics (segment_tree.py:69-74): end exclusive, negative wraps by +capacity
  if (end < 0) end += capacity;
  end -= 1;
  B200RL_REQUIRE(start >= 0 && end >= start && end < capacity, "tree_range_sum: bad range");
  tree_range_sum_kernel<<<1, 32, 0, stream>>>(tree, capacity, start, end, out);
  return check_launch("tree_range_sum_kernel");
}

extern "C" int b200rl_per_sample(const double* sum_tree, const double* min_tree, long long capacity, long long n_stored,
                                 const double* uniforms, int batch, double beta, long long* idx_out, double* w_out,
                                 float* w_out_f32, int* bad, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(sum_tree && min_tree && uniforms && idx_out && w_out && batch > 0, "per_sample: bad args");
  B200RL_REQUIRE(n_stored >= 2 && n_stored <= capacity, "per_sample: need 2 <= n_stored <= capacity");
  B200RL_REQUIRE(beta > 0, "per_sample: beta must be > 0");
  per_sample_kernel<<<ceil_div(batch, 256), 256, 0, stream>>>(sum_tree, min_tree, capacity, n_stored, uniforms, batch,
                                                              beta, idx_out, w_out, w_out_f32, bad);
  return check_launch("per_sample_kernel");
}

extern "C" int b200rl_per_priorities(const float* td, int n, double eps, double alpha, double* powered,
                                     double* max_priority, int* bad, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(td && powered && max_priority && bad && n > 0, "per_priorities: bad args");
  per_priorities_kernel<<<ceil_div(n, 256), 256, 0, stream>>>(td, n, eps, alpha, powered, max_priority, bad);
  return check_launch("per_priorities_kernel");
}

extern "C" int b200rl_per_pow(const double* x, int n, double y, double* out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(x && out && n > 0, "per_pow: bad args");
  per_pow_kernel<<<ceil_div(n, 256), 256, 0, stream>>>(x, n, y, out);
  return check_launch("per_pow_kernel");
}

extern "C" int b200rl_dqn_td(const float* a_t, long long lda_t, const float* s_t, long long lds_t, const float* a_on,
                             long long lda_on, const float* s_on, long long lds_on, const float* a_tg, long long lda_tg,
                             const float* s_tg, long long lds_tg, int nA, const long long* idx,
                             const long long* actions, const float* rewards, const float* dones, const float* weights,
                             float gamma, int double_q, float* td_out, void* d_a, long long ld_da, void* d_s,
                             long long ld_ds, double* loss_sum, int B, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(a_t && a_tg && actions && rewards && dones && weights && td_out && d_a && loss_sum && B > 0,
                 "dqn_td: bad args");
  B200RL_REQUIRE(!double_q || a_on, "dqn_td: double_q needs the online q(s')");
  B200RL_REQUIRE(!s_t || d_s, "dqn_td: dueling needs d_s");
  QHead qt{a_t, lda_t, s_t, lds_t}, qon{a_on, lda_on, s_on, lds_on}, qtg{a_tg, lda_tg, s_tg, lds_tg};
  dqn_td_kernel<<<ceil_div(B, 256), 256, 0, stream>>>(qt, qon, qtg, nA, idx, actions, rewards, dones, weights, gamma,
                                                      double_q, td_out, reinterpret_cast<__half*>(d_a), ld_da,
                                                      reinterpret_cast<__half*>(d_s), ld_ds, loss_sum, B);
  return check_launch("dqn_td_kernel");
}

extern "C" int b200rl_dqn_act(const float* a, long long lda, const float* s, long long lds, int nA, float eps,
                              unsigned long long seed, unsigned long long step, const float* eps_dev,
                              const unsigned long long* step_dev, long long* actions, int B, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(a && actions && B > 0 && nA > 0, "dqn_act: bad args");
  QHead q{a, lda, s, lds};
  dqn_act_kernel<<<ceil_div(B, 128), 128, 0, stream>>>(q, nA, eps, seed, step, eps_dev, step_dev, actions, B);
  return check_launch("dqn_act_kernel");
}
