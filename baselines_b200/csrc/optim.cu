// Flat-buffer optimiser kernels (all HBM-bound; float4 accesses, grid = multiple of the SM count).
//   sumsq            : sum of squares of the flat gradient -> device double (tf.clip_by_global_norm,
//                      ppo2/model.py:105-107), or per-tensor norms (tf.clip_by_norm, deepq/build_graph.py:416-421)
//   clip_adam        : g *= clip/max(||g||, clip) fused with TF-Adam exactly as pinned by the reference's
//                      numpy statement baselines/common/mpi_adam.py:37-42:
//                          a = lr*sqrt(1-b2^t)/(1-b1^t); m = b1 m + (1-b1) g; v = b2 v + (1-b2) g*g;
//                          p -= a*m/(sqrt(v)+eps)            (eps OUTSIDE the bias correction)
//                      28 B of traffic per parameter.  The norm is read from device memory: no host sync.
//   cast / transpose : refresh the fp16 operand copies (W [in,out] for dgrad, W^T [out,in] for forward)
#include "common.cuh"

namespace b200rl {

static constexpr int SUMSQ_MAX_BLOCKS = 1024;
__device__ double g_sumsq_part[SUMSQ_MAX_BLOCKS];
__device__ unsigned int g_sumsq_done = 0;

__global__ void __launch_bounds__(256)
sumsq_kernel(const float* __restrict__ g, long long n, double* __restrict__ out) {
  __shared__ double red[8];
  __shared__ bool last;
  double acc = 0.0;
  const long long n4 = n >> 2;
  const float4* g4 = reinterpret_cast<const float4*>(g);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 q = g4[i];
    acc += (double)q.x * q.x + (double)q.y * q.y + (double)q.z * q.z + (double)q.w * q.w;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const float x = g[(n4 << 2) + threadIdx.x];
    acc += (double)x * x;
  }
  acc = warp_sum_d(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < 8; ++w) s += red[w];
    // the last block to finish adds the blocks' sums in block order: the norm is the same on every run
    g_sumsq_part[blockIdx.x] = s;
    __threadfence();
    last = (atomicAdd(&g_sumsq_done, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (last && threadIdx.x == 0) {
    __threadfence();
    double t = 0.0;
    for (int b = 0; b < (int)gridDim.x; ++b) t += *((volatile double*)&g_sumsq_part[b]);
    *out = t;
    g_sumsq_done = 0;
  }
}

// segment s covers [seg_off[s], seg_off[s+1]); block (s, y) stores its slice's sum at part[s * gridDim.y + y]
__global__ void __launch_bounds__(256)
seg_sumsq_kernel(const float* __restrict__ g, const long long* __restrict__ seg_off, double* __restrict__ part) {
  __shared__ double red[8];
  const int s = blockIdx.x;
  const long long a = seg_off[s], b = seg_off[s + 1];
  double acc = 0.0;
  for (long long i = a + (long long)blockIdx.y * blockDim.x + threadIdx.x; i < b; i += (long long)gridDim.y * blockDim.x) {
    const float x = g[i];
    acc += (double)x * x;
  }
  acc = warp_sum_d(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += red[w];
    part[s * gridDim.y + blockIdx.y] = t;
  }
}

// out[s] = sum of the segment's gridDim.y slice sums, in slice order
__global__ void seg_sumsq_finish_kernel(const double* __restrict__ part, int nseg, int slices, double* __restrict__ out) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s < nseg) {
    double t = 0.0;
    for (int k = 0; k < slices; ++k) t += part[(long long)s * slices + k];
    out[s] = t;
  }
}

struct AdamArgs {
  float lr_t;       // lr*sqrt(1-b2^t)/(1-b1^t), computed on the host from the step counter
  float beta1, beta2, eps;
  float clip;       // <= 0 : no clipping
};

__device__ __forceinline__ void adam1(float& p, float g, float& m, float& v, const AdamArgs& a) {
  m = a.beta1 * m + (1.0f - a.beta1) * g;
  v = a.beta2 * v + (1.0f - a.beta2) * (g * g);
  p = p + (-a.lr_t) * m / (sqrtf(v) + a.eps);
}

// mode 0: one global norm in sumsq[0]; mode 1: per-segment norms (seg_id gives the segment of each 4-block)
__global__ void __launch_bounds__(256)
clip_adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                 long long n, AdamArgs a, const double* __restrict__ sumsq, const long long* __restrict__ seg_off,
                 int nseg, const float* __restrict__ lr_t_dev) {
  if (lr_t_dev) a.lr_t = *lr_t_dev;                // step size kept on the device (CUDA-graph replays)
  float gscale = 1.0f;
  if (a.clip > 0.0f && seg_off == nullptr) {
    const float norm = (float)sqrt(sumsq[0]);
    gscale = a.clip / fmaxf(norm, a.clip);
  }
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float sc = gscale;
    if (a.clip > 0.0f && seg_off != nullptr) {
      int lo = 0, hi = nseg;                       // segment of element i (binary search, nseg is tiny)
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (seg_off[mid] <= i) lo = mid; else hi = mid;
      }
      const float norm = (float)sqrt(sumsq[lo]);
      sc = a.clip / fmaxf(norm, a.clip);
    }
    float pp = p[i], mm = m[i], vv = v[i];
    adam1(pp, g[i] * sc, mm, vv, a);
    p[i] = pp; m[i] = mm; v[i] = vv;
  }
}

// acc += g * (clip / max(||g||, clip)) * weight : the per-microbatch clipped gradients of the reference's
// MicrobatchedModel (ppo2/microbatched_model.py:60-70: self.grads are the clip_by_global_norm outputs of
// ppo2/model.py:105-107, summed over microbatches and divided by their number)
__global__ void __launch_bounds__(256)
clip_accumulate_kernel(const float* __restrict__ g, float* __restrict__ acc, long long n, float clip, float weight,
                       const double* __restrict__ sumsq) {
  float sc = weight;
  if (clip > 0.0f) sc *= clip / fmaxf((float)sqrt(sumsq[0]), clip);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    acc[i] += g[i] * sc;
}

// The 32 x 32 tile at (r0, c0) of dst16[r, c] = src[r, c]*scale (row pitch ld_dst), and optionally of
// dstT16[c, r] = src[r, c]*scale (pitch ld_t), by a block of 256 threads
__device__ __forceinline__ void cast_transpose_tile(const float* __restrict__ src, int R, int C,
                                                    __half* __restrict__ dst, long long ld_dst,
                                                    __half* __restrict__ dstT, long long ld_t, float scale, int r0,
                                                    int c0) {
  __shared__ float tile[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 32 x 8
  for (int i = ty; i < 32; i += 8) {
    const int r = r0 + i, c = c0 + tx;
    float x = 0.0f;
    if (r < R && c < C) {
      x = src[(long long)r * C + c] * scale;
      if (dst) dst[(long long)r * ld_dst + c] = __float2half_rn(x);
    }
    tile[i][tx] = x;
  }
  __syncthreads();
  if (dstT) {
    for (int i = ty; i < 32; i += 8) {
      const int c = c0 + i, r = r0 + tx;
      if (r < R && c < C) dstT[(long long)c * ld_t + r] = __float2half_rn(tile[tx][i]);
    }
  }
}

__global__ void __launch_bounds__(256)
cast_transpose_kernel(const float* __restrict__ src, int R, int C, __half* __restrict__ dst, long long ld_dst,
                      __half* __restrict__ dstT, long long ld_t, float scale) {
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  cast_transpose_tile(src, R, C, dst, ld_dst, dstT, ld_t, scale, r0, c0);
}

__global__ void __launch_bounds__(256)
cast_f32_f16_kernel(const float* __restrict__ src, __half* __restrict__ dst, long long rows, int cols,
                    long long ld_src, long long ld_dst, float scale) {
  const long long total = rows * cols;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols;
    const int c = (int)(i % cols);
    dst[r * ld_dst + c] = __float2half_rn(src[r * ld_src + c] * scale);
  }
}

// All operand refreshes of a network in ONE launch: job j of the table is a cast_transpose (blockIdx.z = j; blocks
// outside a job's tile range exit).  One PPO2 minibatch used to issue 18 of these launches (cfg-2), 8 per tower at
// cfg-3 and 23 per deepq step -- each a 4-10 us kernel.
struct CastJob {
  const float* src;
  __half* dst;
  __half* dstT;
  long long ld_dst, ld_t;
  int R, C;
  float scale;
  int pad;
};
__global__ void __launch_bounds__(256)
cast_transpose_batch_kernel(const CastJob* __restrict__ jobs) {
  const CastJob j = jobs[blockIdx.z];
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  if (c0 >= j.C || r0 >= j.R) return;
  cast_transpose_tile(j.src, j.R, j.C, j.dst, j.ld_dst, j.dstT, j.ld_t, j.scale, r0, c0);
}

// Weight operand of the implicit-GEMM data gradient of a strided convolution ("pixel shuffle" form):
//   out[(py, px, c), (a', b', co)] = W[s*(An-1-a') + py, s*(An-1-b') + px, c, co]   (0 when outside the filter)
// with W in HWIO [R, S, Cin, Cout] fp32, An = ceil(R/s); out is fp16 [s*s*Cin, An*An*Cout] (row pitch ld).
__global__ void __launch_bounds__(256)
dgrad_weights_kernel(const float* __restrict__ w, __half* __restrict__ out, int R, int S, int Cin, int Cout, int s,
                     int An, long long ld) {
  const long long cols = (long long)An * An * Cout;
  const long long total = (long long)s * s * Cin * cols;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / cols, col = i % cols;
    const int c = (int)(row % Cin), cls = (int)(row / Cin);
    const int py = cls / s, px = cls % s;
    const int co = (int)(col % Cout), tap = (int)(col / Cout);
    const int ap = tap / An, bp = tap % An;
    const int ky = s * (An - 1 - ap) + py, kx = s * (An - 1 - bp) + px;
    float v = 0.0f;
    if (ky < R && kx < S) v = w[(((long long)ky * S + kx) * Cin + c) * Cout + co];
    out[row * ld + col] = __float2half_rn(v);
  }
}

// Soft target update t <- keep * t + mix * s, unfused, of (t0, s0, n0) and, in grid row 1, (t1, s1, n1)
__global__ void __launch_bounds__(256)
soft_update_kernel(float* __restrict__ t0, const float* __restrict__ s0, long long n0, float* __restrict__ t1,
                   const float* __restrict__ s1, long long n1, float keep, float mix) {
  float* t = blockIdx.y ? t1 : t0;
  const float* s = blockIdx.y ? s1 : s0;
  const long long n = blockIdx.y ? n1 : n0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    t[i] = __fadd_rn(__fmul_rn(keep, t[i]), __fmul_rn(mix, s[i]));
}

__global__ void set_scalars_kernel(float* dst, float a, float b, float c, float d, int n) {
  const float v[4] = {a, b, c, d};
  if (threadIdx.x < n) dst[threadIdx.x] = v[threadIdx.x];
}
__global__ void counter_add_kernel(unsigned long long* ctr, unsigned long long inc) { *ctr += inc; }

// Minibatch shuffle on the device (replaces np.random.shuffle(inds) of ppo2/ppo2.py:160 + the index arithmetic of
// sf01, ppo2/runner.py:69-74): out[i] = buffer offset of the pi(i)-th sample, pi a keyed pseudo-random BIJECTION of
// [0, n) -- a 6-round Feistel network over the next power of four with cycle walking, the construction of
// thrust::shuffle -- so no permutation array is generated, sorted or uploaded.  Env-major flat index j = e*T + t maps
// to buffer offset t*N + e.  (The host MT19937 shuffle stays available for seed-for-seed parity runs.)
__device__ __forceinline__ uint32_t feistel_round(uint32_t x, uint32_t k) {
  x ^= k;
  x *= 0x9E3779B1u;
  x ^= x >> 15;
  x *= 0x85EBCA77u;
  x ^= x >> 13;
  return x;
}
__global__ void __launch_bounds__(256)
shuffle_indices_kernel(long long* __restrict__ out, long long n, unsigned long long key, int half_bits, long long T,
                       long long N) {
  const uint32_t mask = (1u << half_bits) - 1u;
  uint32_t rk[6];
#pragma unroll
  for (int r = 0; r < 6; ++r) rk[r] = (uint32_t)(key >> (8 * r)) * 0x9E3779B1u + (uint32_t)(key >> 32) + 0x7F4A7C15u * (r + 1);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    unsigned long long x = (unsigned long long)i;
    do {                                             // cycle walking: re-encrypt until the value lands in [0, n)
      uint32_t l = (uint32_t)(x >> half_bits) & mask, r = (uint32_t)x & mask;
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        const uint32_t t = l ^ (feistel_round(r, rk[k]) & mask);
        l = r;
        r = t;
      }
      x = ((unsigned long long)l << half_bits) | r;
    } while (x >= (unsigned long long)n);
    const long long j = (long long)x;
    out[i] = (T > 0) ? (j % T) * N + j / T : j;
  }
}

}  // namespace b200rl

using namespace b200rl;

extern "C" int b200rl_sumsq(const float* g, long long n, double* out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(g && out && n > 0, "sumsq: bad args");
  B200RL_REQUIRE((reinterpret_cast<uintptr_t>(g) & 15) == 0, "sumsq: gradient buffer must be 16 B aligned");
  cudaMemsetAsync(out, 0, sizeof(double), stream);
  const int grid = grid_blocks(n / 4 + 1, 256, 4);
  B200RL_REQUIRE(grid <= SUMSQ_MAX_BLOCKS, "sumsq: %d blocks exceed the partial-sum slots", grid);
  sumsq_kernel<<<grid, 256, 0, stream>>>(g, n, out);
  return check_launch("sumsq_kernel");
}

extern "C" int b200rl_seg_sumsq(const float* g, const long long* seg_off, int nseg, double* out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(g && seg_off && out && nseg > 0, "seg_sumsq: bad args");
  constexpr int SLICES = 16;
  double* part = reinterpret_cast<double*>(det_workspace((size_t)nseg * SLICES * 2, stream));
  if (!part) return B200RL_ERR_CUDA;
  seg_sumsq_kernel<<<dim3(nseg, SLICES), 256, 0, stream>>>(g, seg_off, part);
  seg_sumsq_finish_kernel<<<ceil_div(nseg, 128), 128, 0, stream>>>(part, nseg, SLICES, out);
  return check_launch("seg_sumsq_kernel");
}

extern "C" int b200rl_clip_adam(float* p, const float* g, float* m, float* v, long long n, float lr_t, float beta1,
                                float beta2, float eps, float clip, const double* sumsq, const long long* seg_off,
                                int nseg, const float* lr_t_dev, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(p && g && m && v && n > 0, "clip_adam: bad args");
  B200RL_REQUIRE(clip <= 0.0f || sumsq != nullptr, "clip_adam: clipping needs the device sumsq");
  AdamArgs a{lr_t, beta1, beta2, eps, clip};
  clip_adam_kernel<<<grid_blocks(n, 256, 8), 256, 0, stream>>>(p, g, m, v, n, a, sumsq, seg_off, nseg, lr_t_dev);
  return check_launch("clip_adam_kernel");
}

// dst[0..n) = {a, b, c, d}[0..n): scalars that change between replays of a captured launch sequence (Adam step size,
// clip range) travel as kernel arguments of this one-thread kernel, so no host buffer can be overwritten too early
extern "C" int b200rl_set_scalars(float* dst, int n, float a, float b, float c, float d, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(dst && n >= 1 && n <= 4, "set_scalars: 1..4 values");
  set_scalars_kernel<<<1, 32, 0, stream>>>(dst, a, b, c, d, n);
  return check_launch("set_scalars_kernel");
}

extern "C" int b200rl_counter_add(unsigned long long* ctr, unsigned long long inc, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(ctr != nullptr, "counter_add: null counter");
  counter_add_kernel<<<1, 1, 0, stream>>>(ctr, inc);
  return check_launch("counter_add_kernel");
}

extern "C" int b200rl_shuffle_indices(long long* out, long long n, unsigned long long key, long long T, long long N,
                                      void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(out && n > 0 && n < (1LL << 40), "shuffle_indices: bad args");
  B200RL_REQUIRE(T == 0 || T * N == n, "shuffle_indices: T*N must equal n");
  int half_bits = 1;
  while ((1LL << (2 * half_bits)) < n) ++half_bits;  // domain 4^half_bits >= n: at most 4x the range (<= 4 walks expected)
  shuffle_indices_kernel<<<grid_blocks(n, 256, 8), 256, 0, stream>>>(out, n, key, half_bits, T, N);
  return check_launch("shuffle_indices_kernel");
}

extern "C" int b200rl_clip_accumulate(const float* g, float* acc, long long n, float clip, float weight,
                                      const double* sumsq, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(g && acc && n > 0, "clip_accumulate: bad args");
  B200RL_REQUIRE(clip <= 0.0f || sumsq != nullptr, "clip_accumulate: clipping needs the device sumsq");
  clip_accumulate_kernel<<<grid_blocks(n, 256, 8), 256, 0, stream>>>(g, acc, n, clip, weight, sumsq);
  return check_launch("clip_accumulate_kernel");
}

extern "C" int b200rl_soft_update(float* t0, const float* s0, long long n0, float* t1, const float* s1, long long n1,
                                  double keep, double mix, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(t0 && s0 && n0 > 0 && (t1 == nullptr || (s1 && n1 > 0)), "soft_update: bad args");
  const long long n = n0 > n1 ? n0 : n1;
  const dim3 grid(grid_blocks(n, 256, 16), t1 ? 2u : 1u);
  // keep and mix are python floats; the reference's graph holds them as float32 constants
  soft_update_kernel<<<grid, 256, 0, stream>>>(t0, s0, n0, t1, s1, t1 ? n1 : 0, (float)keep, (float)mix);
  return check_launch("soft_update_kernel");
}

extern "C" int b200rl_cast_transpose(const float* src, int R, int C, void* dst, long long ld_dst, void* dstT,
                                     long long ld_t, float scale, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(src && R > 0 && C > 0 && (dst || dstT), "cast_transpose: bad args");
  dim3 grid(ceil_div(C, 32), ceil_div(R, 32));
  cast_transpose_kernel<<<grid, 256, 0, stream>>>(src, R, C, reinterpret_cast<__half*>(dst), ld_dst,
                                                  reinterpret_cast<__half*>(dstT), ld_t, scale);
  return check_launch("cast_transpose_kernel");
}

extern "C" int b200rl_cast_transpose_batch(const void* jobs, int njobs, int max_rows, int max_cols, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(jobs && njobs > 0 && njobs <= 65535 && max_rows > 0 && max_cols > 0, "cast_transpose_batch: bad args");
  static_assert(sizeof(CastJob) == 56, "CastJob layout is part of the C ABI (see include/b200rl.h)");
  dim3 grid(ceil_div(max_cols, 32), ceil_div(max_rows, 32), njobs);
  cast_transpose_batch_kernel<<<grid, 256, 0, stream>>>(reinterpret_cast<const CastJob*>(jobs));
  return check_launch("cast_transpose_batch_kernel");
}

extern "C" int b200rl_dgrad_weights(const float* w, void* out, int R, int S, int Cin, int Cout, int s, long long ld,
                                    void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(w && out && R > 0 && S > 0 && s > 0, "dgrad_weights: bad args");
  const int An = (R + s - 1) / s;
  const long long total = (long long)s * s * Cin * An * An * Cout;
  dgrad_weights_kernel<<<grid_blocks(total, 256, 8), 256, 0, stream>>>(w, reinterpret_cast<__half*>(out), R, S, Cin,
                                                                        Cout, s, An, ld);
  return check_launch("dgrad_weights_kernel");
}

extern "C" int b200rl_cast_f32_f16(const float* src, void* dst, long long rows, int cols, long long ld_src,
                                   long long ld_dst, float scale, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(src && dst && rows > 0 && cols > 0, "cast: bad args");
  cast_f32_f16_kernel<<<grid_blocks(rows * cols, 256, 8), 256, 0, stream>>>(src, reinterpret_cast<__half*>(dst), rows,
                                                                            cols, ld_src, ld_dst, scale);
  return check_launch("cast_f32_f16_kernel");
}
