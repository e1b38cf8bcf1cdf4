// VecNormalize on the device (common/vec_env/vec_normalize.py:26-47, common/running_mean_std.py:22-33): batch
// moments of the observations and of the discounted return, the float64 running-statistics update, the observation
// normalisation and the reward scaling, bit for bit with the numpy wrapper.
//
// numpy's summation order is reproduced exactly (np.mean / np.var along axis 0, in the dtype of x):
//   * D >= 2 columns: every column is one dependent chain of N adds in row order, starting from +0;
//   * D == 1 and the 1-D return vector: np.add.reduce's pairwise sum (loops_utils.h pairwise_sum) from +0: blocks
//     of <= 128 elements with eight strided accumulators ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)) and a sequential tail,
//     combined along the binary split n2 = n/2 - (n/2) % 8;
//   * mean = sum / N, var = sum((x - mean)^2) / N, each difference and square rounded to the dtype.
// Every add / multiply / divide is an explicit *_rn intrinsic, so no FMA is contracted.
//
// Running statistics: one float64 buffer per RunningMeanStd, [mean(D) | var(D) | std(D) | count], where
// std = sqrt(var + eps) is stored by the update for the normalisation that follows.  Batch moments go through a
// float64 workspace [mean(D) | var(D)] (the dtype's values, widened exactly).
//
// Kernels (all on the caller's stream, no host synchronisation):
//   vn_col_moments_kernel  one warp per 32 adjacent columns (each row slice is one coalesced 128 / 256 B piece), both
//       passes in one launch.  Rows are streamed through a shared-memory ring by cp.async (4 / 8 B per lane, which
//       works for any row stride), STAGES-1 chunks ahead of the adds, so no load sits on the add chain: the kernel
//       is bound by 2·N dependent add latencies.  A lane reads only the slots it copied itself, so cp.async.wait_group
//       alone orders the ring.
//   vn_pair_moments_kernel numpy's pairwise tree for D == 1 in one CTA: the leaves are summed in parallel, the tree
//       is combined by one thread.
//   vn_combine_kernel      the update of every column (one CTA: the shared count is written after all columns have
//       read it).  float64, except bvar * N, which numpy leaves in the batch's dtype.
//   vn_normalize_kernel    float32 rows clip((x - mean) / std, +-clip) computed in float64, NaN propagating.
//   vn_rewards_kernel      one CTA: ret = ret * gamma + rew, the pairwise moments of ret, the update of the return
//       statistics, rew = clip(rew / std, +-cliprew) rounded to float32, ret = 0 where news.
#include "np_sum.cuh"

namespace b200rl {

namespace {

// np.clip(v, -c, c) = minimum(maximum(v, -c), c): a NaN stays NaN (fminf / fmaxf would drop it)
__device__ __forceinline__ double clip_nan(double v, double c) {
  v = v < -c ? -c : v;
  return v > c ? c : v;
}

__device__ __forceinline__ void cp_async(void* smem, const void* g, int bytes) {
  if (bytes == 4)
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem)), "l"(g) : "memory");
  else
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(smem)), "l"(g) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// running_mean_std.py:22-31 for one column; `count` is the count before this batch
// bv * n stays in the batch's dtype (numpy: a float32 array times a Python int is a float32 product)
__device__ __forceinline__ void combine_col(double* rms, int D, int c, double count, double bm, double bv, double n,
                                            double eps, bool f32) {
  double* mean = rms;
  double* var = rms + D;
  double* stdv = rms + 2 * D;
  const double delta = __dsub_rn(bm, mean[c]);
  const double tot = __dadd_rn(count, n);
  mean[c] = __dadd_rn(mean[c], __ddiv_rn(__dmul_rn(delta, n), tot));
  const double bvn = f32 ? (double)__fmul_rn((float)bv, (float)n) : __dmul_rn(bv, n);
  const double m2 = __dadd_rn(__dadd_rn(__dmul_rn(var[c], count), bvn),
                              __ddiv_rn(__dmul_rn(__dmul_rn(__dmul_rn(delta, delta), count), n), tot));
  const double v = __ddiv_rn(m2, tot);
  var[c] = v;
  stdv[c] = __dsqrt_rn(__dadd_rn(v, eps));
}

// ------------------------------------------------------------------ column moments (D >= 2)
template <typename T, int ROWS, int STAGES>
__global__ void __launch_bounds__(32) vn_col_moments_kernel(const T* __restrict__ x, long long N, int D,
                                                            double* __restrict__ ws) {
  __shared__ T ring[STAGES][ROWS][32];
  const int lane = threadIdx.x;
  const int c = blockIdx.x * 32 + lane;
  if (c >= D) return;
  const T* col = x + c;
  const long long nchunks = (N + ROWS - 1) / ROWS;
  auto issue = [&](long long k) {
    if (k < nchunks) {
      const long long r0 = k * ROWS;
      const int rows = (int)min((long long)ROWS, N - r0);
      T(*slot)[32] = ring[k % STAGES];
      for (int r = 0; r < rows; ++r) cp_async(&slot[r][lane], col + (r0 + r) * D, (int)sizeof(T));
    }
    cp_async_commit();                                   // empty groups keep the wait count uniform
  };
  T mean = T(0), var = T(0);
#pragma unroll 1
  for (int pass = 0; pass < 2; ++pass) {
    T s = T(0);
    for (int k = 0; k < STAGES - 1; ++k) issue(k);
#pragma unroll 1
    for (long long k = 0; k < nchunks; ++k) {
      // refills the slot read in iteration k-1: in-order issue puts this after the adds that consumed its values
      issue(k + STAGES - 1);
      cp_async_wait<STAGES - 1>();                       // this lane's copies of chunk k have landed
      const T(*slot)[32] = ring[k % STAGES];
      const int rows = (int)min((long long)ROWS, N - k * ROWS);
      if (rows == ROWS) {
        T v[ROWS];
#pragma unroll
        for (int r = 0; r < ROWS; ++r) v[r] = slot[r][lane];
        if (pass == 0) {
#pragma unroll
          for (int r = 0; r < ROWS; ++r) s = add_rn(s, v[r]);
        } else {
#pragma unroll
          for (int r = 0; r < ROWS; ++r) {
            const T d = sub_rn(v[r], mean);
            s = add_rn(s, mul_rn(d, d));
          }
        }
      } else {
        for (int r = 0; r < rows; ++r) {
          const T v = slot[r][lane];
          if (pass == 0) {
            s = add_rn(s, v);
          } else {
            const T d = sub_rn(v, mean);
            s = add_rn(s, mul_rn(d, d));
          }
        }
      }
    }
    cp_async_wait<0>();
    if (pass == 0)
      mean = div_rn(s, (T)N);
    else
      var = div_rn(s, (T)N);
  }
  ws[c] = (double)mean;
  ws[D + c] = (double)var;
}

// ------------------------------------------------------------------ pairwise moments (one CTA)
constexpr int PW_BLOCK = 128;
constexpr int PW_MAX_LEAVES = 2048;      // leaves hold >= 64 elements once N > 128: N <= 131072
constexpr long long PW_MAX_N = PW_MAX_LEAVES * 64LL;
constexpr int PW_THREADS = 512;
constexpr int PW_STACK = 48;

template <typename T>
struct PairwiseSmem {
  int leaf_start[PW_MAX_LEAVES];
  int leaf_len[PW_MAX_LEAVES];
  T leaf_sum[PW_MAX_LEAVES];
  long long st_n[PW_STACK];
  long long st_s[PW_STACK];
  int st_ph[PW_STACK];
  T st_v[PW_STACK];
  int nleaves;
  T result;
};

__device__ __forceinline__ long long pw_split(long long n) {
  long long n2 = n / 2;
  return n2 - n2 % 8;
}

// thread 0: the leaves of pairwise_sum(0, N) in left-to-right order
template <typename T>
__device__ void pw_leaves(PairwiseSmem<T>& sm, long long N) {
  int top = 0, nl = 0;
  sm.st_s[0] = 0;
  sm.st_n[0] = N;
  top = 1;
  while (top > 0) {
    --top;
    const long long s = sm.st_s[top], n = sm.st_n[top];
    if (n <= PW_BLOCK) {
      sm.leaf_start[nl] = (int)s;
      sm.leaf_len[nl] = (int)n;
      ++nl;
    } else {
      const long long n2 = pw_split(n);
      sm.st_s[top] = s + n2;                              // right, popped after the whole left subtree
      sm.st_n[top] = n - n2;
      sm.st_s[top + 1] = s;
      sm.st_n[top + 1] = n2;
      top += 2;
    }
  }
  sm.nleaves = nl;
}

// pairwise_sum of one block of n <= 128 elements f(a[0..n))
template <typename T, typename F>
__device__ __forceinline__ T pw_leaf(const T* a, int n, F f) {
  return np_pairwise_block<T>([&](int i) { return f(a[i]); }, 0, n);
}

// thread 0: combine the leaf sums along the split tree (post-order), then add to the +0 the reduction starts from
template <typename T>
__device__ T pw_tree(PairwiseSmem<T>& sm, long long N) {
  int top = 1, leaf = 0;
  sm.st_n[0] = N;
  sm.st_ph[0] = 0;
  bool have = false;
  T val = T(0);
  while (true) {
    if (!have) {
      const int i = top - 1;
      if (sm.st_n[i] <= PW_BLOCK) {
        val = sm.leaf_sum[leaf++];
        have = true;
        --top;
      } else {
        sm.st_ph[i] = 1;
        sm.st_n[top] = pw_split(sm.st_n[i]);
        sm.st_ph[top] = 0;
        ++top;
      }
    } else {
      if (top == 0) break;
      const int i = top - 1;
      if (sm.st_ph[i] == 1) {                             // left subtree done: descend right
        sm.st_v[i] = val;
        sm.st_ph[i] = 2;
        sm.st_n[top] = sm.st_n[i] - pw_split(sm.st_n[i]);
        sm.st_ph[top] = 0;
        ++top;
        have = false;
      } else {
        val = add_rn(sm.st_v[i], val);
        --top;
      }
    }
  }
  return add_rn(T(0), val);
}

// np.add.reduce(f(a)) over a[0..N) by the whole CTA; the leaves must have been built.  Result in every thread.
template <typename T, typename F>
__device__ T pw_reduce(PairwiseSmem<T>& sm, const T* a, long long N, F f) {
  for (int l = threadIdx.x; l < sm.nleaves; l += blockDim.x)
    sm.leaf_sum[l] = pw_leaf(a + sm.leaf_start[l], sm.leaf_len[l], f);
  __syncthreads();
  if (threadIdx.x == 0) sm.result = pw_tree(sm, N);
  __syncthreads();
  const T r = sm.result;
  __syncthreads();
  return r;
}

// (mean, var) of a[0..N) as np.mean / np.var of a 1-D array
template <typename T>
__device__ void pw_moments(PairwiseSmem<T>& sm, const T* a, long long N, T& mean, T& var) {
  if (threadIdx.x == 0) pw_leaves(sm, N);
  __syncthreads();
  mean = div_rn(pw_reduce(sm, a, N, [](T v) { return v; }), (T)N);
  const T m = mean;
  var = div_rn(pw_reduce(sm, a, N, [m](T v) { const T d = sub_rn(v, m); return mul_rn(d, d); }), (T)N);
}

template <typename T>
__global__ void __launch_bounds__(PW_THREADS) vn_pair_moments_kernel(const T* __restrict__ x, long long N,
                                                                     double* __restrict__ ws) {
  __shared__ PairwiseSmem<T> sm;
  T m, v;
  pw_moments(sm, x, N, m, v);
  if (threadIdx.x == 0) {
    ws[0] = (double)m;
    ws[1] = (double)v;
  }
}

// ------------------------------------------------------------------ combine
__global__ void __launch_bounds__(256) vn_combine_kernel(double* __restrict__ rms, const double* __restrict__ ws,
                                                         long long N, int D, double eps, bool f32) {
  const double count = rms[3 * D];
  for (int c = threadIdx.x; c < D; c += blockDim.x)
    combine_col(rms, D, c, count, ws[c], ws[D + c], (double)N, eps, f32);
  __syncthreads();                                        // every column has read the old count
  if (threadIdx.x == 0) rms[3 * D] = __dadd_rn(count, (double)N);
}

// ------------------------------------------------------------------ normalise
template <typename T>
__global__ void __launch_bounds__(256) vn_normalize_kernel(const T* __restrict__ x, long long total, int D,
                                                           const double* __restrict__ rms, double clip,
                                                           float* __restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    double v = (double)x[i];
    if (rms) {
      const int c = (int)(i % D);
      v = clip_nan(__ddiv_rn(__dsub_rn(v, rms[c]), rms[2 * D + c]), clip);
    }
    out[i] = __double2float_rn(v);
  }
}

// ------------------------------------------------------------------ rewards
template <typename R>
__global__ void __launch_bounds__(PW_THREADS) vn_rewards_kernel(const R* __restrict__ rew, const uint8_t* __restrict__ news,
                                                                long long N, double* __restrict__ ret,
                                                                double* __restrict__ rms, double gamma, double eps,
                                                                double cliprew, float* __restrict__ out) {
  __shared__ PairwiseSmem<double> sm;
  for (long long e = threadIdx.x; e < N; e += blockDim.x)              // vec_normalize.py:37
    ret[e] = __dadd_rn(__dmul_rn(ret[e], gamma), (double)rew[e]);
  __syncthreads();
  double stdv = 1.0;
  if (rms) {                                                            // vec_normalize.py:38-40
    double m, v;
    pw_moments(sm, ret, N, m, v);
    if (threadIdx.x == 0) {
      combine_col(rms, 1, 0, rms[3], m, v, (double)N, eps, false);
      rms[3] = __dadd_rn(rms[3], (double)N);
    }
    __syncthreads();
    stdv = rms[2];
  }
  for (long long e = threadIdx.x; e < N; e += blockDim.x) {
    const double r = (double)rew[e];
    out[e] = __double2float_rn(rms ? clip_nan(__ddiv_rn(r, stdv), cliprew) : r);
    if (news && news[e]) ret[e] = 0.0;                                  // vec_normalize.py:41
  }
}

// latency probe: one thread, n dependent adds; out[0] = SM cycles per add (out[1] keeps the chain alive)
template <typename T>
__global__ void vn_add_chain_kernel(long long n, double* out) {
  T s = (T)out[1];
  const T inc = (T)1.0000001;
  const long long t0 = clock64();
#pragma unroll 8
  for (long long i = 0; i < n; ++i) s = add_rn(s, inc);
  const long long t1 = clock64();
  out[0] = (double)(t1 - t0) / (double)n;
  out[1] = (double)s;
}

template <typename T>
int moments_t(const void* x, long long N, int D, double* ws, cudaStream_t stream) {
  const T* xt = static_cast<const T*>(x);
  if (D == 1) {
    vn_pair_moments_kernel<T><<<1, PW_THREADS, 0, stream>>>(xt, N, ws);
    return check_launch("vn_pair_moments_kernel");
  }
  constexpr int ROWS = sizeof(T) == 4 ? 32 : 16;
  constexpr int STAGES = sizeof(T) == 4 ? 8 : 10;
  vn_col_moments_kernel<T, ROWS, STAGES><<<ceil_div(D, 32), 32, 0, stream>>>(xt, N, D, ws);
  return check_launch("vn_col_moments_kernel");
}

}  // namespace

}  // namespace b200rl

using namespace b200rl;

extern "C" int b200rl_vecnorm_moments(const void* x, int x_f64, long long N, int D, double* ws, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(x && ws, "vecnorm_moments: null operand");
  B200RL_REQUIRE(N > 0 && D > 0, "vecnorm_moments: empty batch");
  B200RL_REQUIRE((reinterpret_cast<uintptr_t>(x) & (x_f64 ? 7 : 3)) == 0, "vecnorm_moments: x must be aligned to its dtype");
  B200RL_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 7) == 0, "vecnorm_moments: ws must be 8-byte aligned");
  B200RL_REQUIRE(x_f64 || N < (1LL << 24), "vecnorm_moments: float32 batches need N < 2^24 (N exact in float32)");
  if (D == 1) B200RL_REQUIRE(N <= PW_MAX_N, "vecnorm_moments: D == 1 needs N <= %lld", PW_MAX_N);
  return x_f64 ? moments_t<double>(x, N, D, ws, stream) : moments_t<float>(x, N, D, ws, stream);
}

extern "C" int b200rl_vecnorm_combine(double* rms, const double* ws, int ws_f32, long long N, int D, double eps,
                                      void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(rms && ws && N > 0 && D > 0, "vecnorm_combine: bad operands");
  B200RL_REQUIRE(!ws_f32 || N < (1LL << 24), "vecnorm_combine: float32 batches need N < 2^24");
  vn_combine_kernel<<<1, 256, 0, stream>>>(rms, ws, N, D, eps, ws_f32 != 0);
  return check_launch("vn_combine_kernel");
}

extern "C" int b200rl_vecnorm_normalize(const void* x, int x_f64, long long N, int D, const double* rms, double clip,
                                        float* out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(x && out && N > 0 && D > 0, "vecnorm_normalize: bad operands");
  B200RL_REQUIRE((reinterpret_cast<uintptr_t>(x) & (x_f64 ? 7 : 3)) == 0, "vecnorm_normalize: x must be aligned to its dtype");
  const long long total = N * D;
  const int blocks = grid_blocks(total, 256, 16);
  if (x_f64)
    vn_normalize_kernel<double><<<blocks, 256, 0, stream>>>(static_cast<const double*>(x), total, D, rms, clip, out);
  else
    vn_normalize_kernel<float><<<blocks, 256, 0, stream>>>(static_cast<const float*>(x), total, D, rms, clip, out);
  return check_launch("vn_normalize_kernel");
}

extern "C" int b200rl_vecnorm_rewards(const void* rew, int rew_f64, const uint8_t* news, long long N, double* ret,
                                      double* rms, double gamma, double eps, double cliprew, float* out,
                                      void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(rew && ret && out && N > 0, "vecnorm_rewards: bad operands");
  B200RL_REQUIRE((reinterpret_cast<uintptr_t>(rew) & (rew_f64 ? 7 : 3)) == 0, "vecnorm_rewards: rew must be aligned to its dtype");
  B200RL_REQUIRE(N <= PW_MAX_N, "vecnorm_rewards: needs N <= %lld", PW_MAX_N);
  if (rew_f64)
    vn_rewards_kernel<double><<<1, PW_THREADS, 0, stream>>>(static_cast<const double*>(rew), news, N, ret, rms, gamma,
                                                            eps, cliprew, out);
  else
    vn_rewards_kernel<float><<<1, PW_THREADS, 0, stream>>>(static_cast<const float*>(rew), news, N, ret, rms, gamma,
                                                           eps, cliprew, out);
  return check_launch("vn_rewards_kernel");
}

extern "C" int b200rl_vecnorm_add_latency(int f64, long long n, double* out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(out && n > 0, "vecnorm_add_latency: bad operands");
  if (f64)
    vn_add_chain_kernel<double><<<1, 1, 0, stream>>>(n, out);
  else
    vn_add_chain_kernel<float><<<1, 1, 0, stream>>>(n, out);
  return check_launch("vn_add_chain_kernel");
}
