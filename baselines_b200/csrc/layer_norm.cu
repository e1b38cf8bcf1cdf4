// Row layer normalisation (tf.contrib.layers.layer_norm(center=True, scale=True) after a fully connected layer:
// common/models.py:97-98, deepq/models.py:24-25,34-35), forward and backward.
//   y  = act(gamma * xhat + beta),  xhat = (z - mean) * rstd,  rstd = 1 / sqrt(var + eps),  var biased (tf.nn.moments)
//   dz = rstd * (g - mean(g) - xhat * mean(g * xhat)),  g = gamma * du;  dgamma = sum_r du * xhat;  dbeta = sum_r du
// A group of G lanes (a warp, or 8 lanes for rows of at most 64 columns, so that narrow rows keep every lane loading)
// owns a row and holds it in registers: lane l of the group has the 8-column chunks l, l + G, ... (16-byte loads and
// stores).  The mean comes first and the variance is the mean of the centred squares, so a row with a large mean and a
// small spread keeps its variance.  Both sums are xor-butterflies over fixed per-lane partial sums: a row's result is a
// function of the row alone, whatever the number of rows or the grid.  The backward saves nothing: it recomputes the
// two statistics from z, which stays in its fp32 workspace.  HBM bound (6 B / element forward, 8 B backward).
#include "common.cuh"

namespace b200rl {

static constexpr int LN_WARPS = 8;           // warps (rows in flight) per CTA
static constexpr int LN_BWD_ROWS = 128;      // rows per CTA of the backward: one dgamma / dbeta partial per 128-row slice

__device__ __forceinline__ float ln_act(float v, int act) {
  return act == 1 ? fmaxf(v, 0.0f) : (act == 2 ? tanhf(v) : v);
}

template <int G>
__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// x[k][0..8) = z[row, 8 * (lane + G k) ..), zeros beyond N or when the group has no row (`live` false); leaves xhat in
// x and the row's 1 / sqrt(var + eps) in rstd
template <int G, int NCH>
__device__ __forceinline__ void ln_row_stats(const float* __restrict__ zrow, bool live, int N, int lane, float eps,
                                             float (&x)[NCH][8], float& rstd) {
  float s = 0.0f;
#pragma unroll
  for (int k = 0; k < NCH; ++k) {
    const int c = 8 * (lane + G * k);
    if (live && c < N) {
      const float4 a = *reinterpret_cast<const float4*>(zrow + c);
      const float4 b = *reinterpret_cast<const float4*>(zrow + c + 4);
      x[k][0] = a.x; x[k][1] = a.y; x[k][2] = a.z; x[k][3] = a.w;
      x[k][4] = b.x; x[k][5] = b.y; x[k][6] = b.z; x[k][7] = b.w;
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) x[k][j] = 0.0f;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) s += x[k][j];
  }
  const float mean = group_sum<G>(s) / (float)N;
  float q = 0.0f;
#pragma unroll
  for (int k = 0; k < NCH; ++k) {
    const bool in = live && 8 * (lane + G * k) < N;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      x[k][j] = in ? x[k][j] - mean : 0.0f;
      q += x[k][j] * x[k][j];
    }
  }
  rstd = 1.0f / sqrtf(group_sum<G>(q) / (float)N + eps);
#pragma unroll
  for (int k = 0; k < NCH; ++k)
#pragma unroll
    for (int j = 0; j < 8; ++j) x[k][j] *= rstd;
}

template <int G, int NCH>
__global__ void __launch_bounds__(32 * LN_WARPS)
ln_fwd_kernel(const float* __restrict__ z, long long ld_z, const float* __restrict__ gamma,
              const float* __restrict__ beta, __half* __restrict__ y, long long ld_y, long long rows, int N, int act,
              float eps) {
  constexpr int RPW = 32 / G;                      // rows per warp
  const int lane = threadIdx.x & (G - 1);
  const long long row = ((long long)blockIdx.x * LN_WARPS + (threadIdx.x >> 5)) * RPW + ((threadIdx.x & 31) / G);
  const bool live = row < rows;
  float x[NCH][8], rstd;
  ln_row_stats<G, NCH>(z + row * ld_z, live, N, lane, eps, x, rstd);
#pragma unroll
  for (int k = 0; k < NCH; ++k) {
    const int c = 8 * (lane + G * k);
    if (live && c < N) {
      uint4 o;
      __half2* h = reinterpret_cast<__half2*>(&o);
#pragma unroll
      for (int j = 0; j < 8; j += 2) {
        const float v0 = ln_act(__ldg(gamma + c + j) * x[k][j] + __ldg(beta + c + j), act);
        const float v1 = ln_act(__ldg(gamma + c + j + 1) * x[k][j + 1] + __ldg(beta + c + j + 1), act);
        h[j >> 1] = __floats2half2_rn(v0, v1);
      }
      *reinterpret_cast<uint4*>(y + row * ld_y + c) = o;
    }
  }
}

// CTA b owns rows [128 b, 128 b + 128).  Lane group t = 0 .. 256 / G - 1 of the CTA takes rows t, t + 256 / G, ... of
// the slice in order; the groups' sums are added in group order, and part_g / part_b[b, :] = alpha * the slice's sums
// (sum_partials then adds the slices in order): dgamma and dbeta depend on the data alone, not on the grid or the
// device.  du and dz may be the same buffer: a lane reads its chunks of a row before it writes them.
template <int G, int NCH>
__global__ void __launch_bounds__(32 * LN_WARPS)
ln_bwd_kernel(const __half* du, long long ld_du, const float* __restrict__ z, long long ld_z,
              const float* __restrict__ gamma, __half* dz, long long ld_dz, float* __restrict__ part_g,
              float* __restrict__ part_b, long long rows, int N, float alpha, float eps) {
  constexpr int GROUPS = 32 * LN_WARPS / G;        // rows in flight per CTA
  constexpr int PASS = 8 * G;                      // columns the groups hold per chunk index k
  __shared__ float red[GROUPS][PASS];
  const int lane = threadIdx.x & (G - 1), grp = threadIdx.x / G;
  float ag[NCH][8], ab[NCH][8];
#pragma unroll
  for (int k = 0; k < NCH; ++k)
#pragma unroll
    for (int j = 0; j < 8; ++j) ag[k][j] = ab[k][j] = 0.0f;
  const long long r0 = (long long)blockIdx.x * LN_BWD_ROWS;
  for (int i = grp; i < LN_BWD_ROWS && r0 + i - (grp % (32 / G)) < rows; i += GROUPS) {   // uniform over the warp
    const long long row = r0 + i;
    const bool live = row < rows;
    float x[NCH][8], g[NCH][8], rstd;
    ln_row_stats<G, NCH>(z + row * ld_z, live, N, lane, eps, x, rstd);
    float s1 = 0.0f, s2 = 0.0f;
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
      const int c = 8 * (lane + G * k);
      if (live && c < N) {
        const uint4 q = *reinterpret_cast<const uint4*>(du + row * ld_du + c);
        const __half2* h = reinterpret_cast<const __half2*>(&q);
#pragma unroll
        for (int j = 0; j < 8; j += 2) {
          const float2 d = __half22float2(h[j >> 1]);
          ab[k][j] += d.x;
          ab[k][j + 1] += d.y;
          ag[k][j] += d.x * x[k][j];
          ag[k][j + 1] += d.y * x[k][j + 1];
          g[k][j] = __ldg(gamma + c + j) * d.x;
          g[k][j + 1] = __ldg(gamma + c + j + 1) * d.y;
        }
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) g[k][j] = 0.0f;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        s1 += g[k][j];
        s2 += g[k][j] * x[k][j];
      }
    }
    const float m1 = group_sum<G>(s1) / (float)N, m2 = group_sum<G>(s2) / (float)N;
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
      const int c = 8 * (lane + G * k);
      if (live && c < N) {
        uint4 o;
        __half2* h = reinterpret_cast<__half2*>(&o);
#pragma unroll
        for (int j = 0; j < 8; j += 2)
          h[j >> 1] = __floats2half2_rn(rstd * (g[k][j] - m1 - x[k][j] * m2),
                                        rstd * (g[k][j + 1] - m1 - x[k][j + 1] * m2));
        *reinterpret_cast<uint4*>(dz + row * ld_dz + c) = o;
      }
    }
  }
  // PASS columns per pass (those of chunk index k): every group parks its sums, one thread per column adds the groups
#pragma unroll
  for (int k = 0; k < NCH; ++k) {
#pragma unroll
    for (int which = 0; which < 2; ++which) {
#pragma unroll
      for (int j = 0; j < 8; ++j) red[grp][8 * lane + j] = which ? ab[k][j] : ag[k][j];
      __syncthreads();
      const int col = PASS * k + threadIdx.x;
      if (threadIdx.x < PASS && col < N) {
        float s = 0.0f;
#pragma unroll
        for (int q = 0; q < GROUPS; ++q) s += red[q][threadIdx.x];
        (which ? part_b : part_g)[(long long)blockIdx.x * N + col] = alpha * s;
      }
      __syncthreads();
    }
  }
}

static bool ln_shape_ok(int N, long long ld_a, long long ld_b, long long ld_c, const void* a, const void* b,
                        const void* c) {
  const uintptr_t p = reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c);
  return N >= 8 && N <= 1024 && N % 8 == 0 && ld_a % 8 == 0 && ld_b % 8 == 0 && ld_c % 8 == 0 && ld_a >= N &&
         ld_b >= N && ld_c >= N && (p & 15) == 0;
}

// (lanes per row, chunks per lane) instance for a row of N columns
#define LN_DISPATCH(N, KERNEL, GRID, ...)                                                           \
  do {                                                                                              \
    if ((N) <= 64) KERNEL<8, 1><<<(GRID)(8), 32 * LN_WARPS, 0, stream>>>(__VA_ARGS__);              \
    else if ((N) <= 256) KERNEL<32, 1><<<(GRID)(32), 32 * LN_WARPS, 0, stream>>>(__VA_ARGS__);      \
    else if ((N) <= 512) KERNEL<32, 2><<<(GRID)(32), 32 * LN_WARPS, 0, stream>>>(__VA_ARGS__);      \
    else KERNEL<32, 4><<<(GRID)(32), 32 * LN_WARPS, 0, stream>>>(__VA_ARGS__);                      \
  } while (0)

}  // namespace b200rl

using namespace b200rl;

extern "C" int b200rl_ln_fwd(const float* z, long long ld_z, const float* gamma, const float* beta, void* y,
                             long long ld_y, long long rows, int N, int act, float eps, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(z && gamma && beta && y && rows > 0 && act >= 0 && act <= 2, "ln_fwd: bad args");
  B200RL_REQUIRE(ln_shape_ok(N, ld_z, ld_y, ld_y, z, y, y),
                 "ln_fwd: N a multiple of 8 in [8, 1024], row pitches multiples of 8 and >= N, 16-byte aligned rows");
  auto grid = [rows](int G) { return (int)ceil_div_ll(rows, LN_WARPS * (32 / G)); };
  LN_DISPATCH(N, ln_fwd_kernel, grid, z, ld_z, gamma, beta, reinterpret_cast<__half*>(y), ld_y, rows, N, act, eps);
  return check_launch("ln_fwd_kernel");
}

extern "C" int b200rl_ln_bwd(const void* du, long long ld_du, const float* z, long long ld_z, const float* gamma,
                             void* dz, long long ld_dz, float* dgamma, float* dbeta, long long rows, int N, float alpha,
                             float eps, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(du && z && gamma && dz && dgamma && dbeta && rows > 0, "ln_bwd: bad args");
  B200RL_REQUIRE(ln_shape_ok(N, ld_du, ld_z, ld_dz, du, z, dz),
                 "ln_bwd: N a multiple of 8 in [8, 1024], row pitches multiples of 8 and >= N, 16-byte aligned rows");
  const int parts = (int)ceil_div_ll(rows, LN_BWD_ROWS);
  float* pg = det_workspace((size_t)parts * N * 2, stream);
  if (!pg) return B200RL_ERR_CUDA;
  float* pb = pg + (size_t)parts * N;
  auto grid = [parts](int) { return parts; };
  LN_DISPATCH(N, ln_bwd_kernel, grid, reinterpret_cast<const __half*>(du), ld_du, z, ld_z, gamma,
              reinterpret_cast<__half*>(dz), ld_dz, pg, pb, rows, N, alpha, eps);
  int rc = check_launch("ln_bwd_kernel");
  if (rc == B200RL_OK) rc = sum_partials(pg, parts, 1, N, dgamma, N, stream);
  if (rc == B200RL_OK) rc = sum_partials(pb, parts, 1, N, dbeta, N, stream);
  return rc;
}
