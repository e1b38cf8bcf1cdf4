// Observation encoding for vector observations (replaces common/input.py:43-63 encode_observation, the optional
// clip((x - mean) / std) of common/policies.py:182-185 and the arr[mbinds] row gather of ppo2/ppo2.py:165).
//
// The reference keeps observations in float32 end to end (tf.to_float, no narrowing).  The tensor cores take fp16
// operands, so every encoded value v is emitted as an fp16 PAIR
//     hi = fp16(v),  lo = fp16(v - hi)          (v - hi is exact in fp32)
// whose sum hi + lo differs from v by at most 2^-22 |v| while lo is an fp16 normal (|v| >= 2^-3 roughly) and by at most
// 2^-25 (half of lo's subnormal spacing 2^-24) below that.  fp16 ends at 65504: an encoded |v| >= 65520 rounds hi to
// +-inf (and lo to -+inf), which the first GEMM turns into NaN.  Such values set *overflow (when given); the host
// raises at its next synchronisation (common/policies.py PolicyNet.check_obs_range) instead of acting on NaN.  Values
// below the limit are encoded exactly as without the flag.
// laid out side by side as one operand row [hi(0..in_pad) | lo(0..in_pad)].  The first GEMM runs over K = 2*in_pad
// against the weight matrix stacked twice ([W ; W]), i.e. x.W = hi.W + lo.W accumulated in fp32: the observation
// itself is no longer quantised to 11 bits.  Discrete observations become exact one-hot rows (lo = 0); a MultiDiscrete
// observation (k integers) becomes the concatenation of k one-hot blocks [seg_off[s], seg_off[s+1]) (input.py:58-61),
// of which Discrete(n) is the single block [0, n).
#include "common.cuh"

namespace b200rl {

struct ObsEncodeParams {
  const float* x;            // [*, raw_dim] float32 rows (Discrete: raw_dim = 1, the integer stored as float)
  const long long* src_idx;  // optional row gather
  long long B;
  int raw_dim, in_dim, in_pad;
  const float* mean;         // optional [raw_dim]
  const float* inv_std;      // optional [raw_dim]
  float clip_lo, clip_hi;    // applied when mean != nullptr
  int onehot_n;              // > 0: Discrete(n) / MultiDiscrete observation, one-hot row width (= in_dim)
  const int* seg_off;        // optional [nseg + 1] one-hot block offsets (MultiDiscrete); null: one block [0, onehot_n)
  int nseg;
  __half* out;               // [B, 2 * in_pad]
  int* overflow;             // optional: set to 1 when an encoded value has |v| >= 65520 (beyond fp16)
};

__global__ void __launch_bounds__(256) obs_encode_kernel(const ObsEncodeParams p) {
  const int groups = p.in_pad >> 3;                                  // 8 columns (one 16-byte store each for hi / lo)
  const long long total = p.B * groups;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long b = i / groups;
    const int c0 = (int)(i - b * groups) << 3;
    const long long r = p.src_idx ? p.src_idx[b] : b;
    const float* src = p.x + r * p.raw_dim;
    float v[8];
    if (p.onehot_n > 0 && p.seg_off == nullptr) {
      const int k = (int)src[0];
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = (c0 + j == k) ? 1.0f : 0.0f;
    } else if (p.onehot_n > 0) {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = 0.0f;
      for (int s = 0; s < p.nseg; ++s) {           // the hot column of every block that reaches into this group
        const int lo = p.seg_off[s], hi = p.seg_off[s + 1];
        if (hi <= c0 || lo >= c0 + 8) continue;
        const int k = (int)src[s];
        const int c = lo + k;
        if (k >= 0 && c < hi && c >= c0 && c < c0 + 8) {
#pragma unroll
          for (int j = 0; j < 8; ++j)
            if (c0 + j == c) v[j] = 1.0f;
        }
      }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = c0 + j;
        float t = 0.0f;
        if (c < p.in_dim) {
          t = src[c];
          if (p.mean) t = fminf(fmaxf((t - p.mean[c]) * p.inv_std[c], p.clip_lo), p.clip_hi);
        }
        v[j] = t;
      }
      if (p.overflow && f16_overflow8(v)) *p.overflow = 1;
    }
    store_split_f16x8(p.out + b * (2LL * p.in_pad) + c0, p.in_pad, v);
  }
}

}  // namespace b200rl

using namespace b200rl;

extern "C" int b200rl_obs_encode(const float* x, const long long* src_idx, long long B, int raw_dim, int in_dim,
                                 int in_pad, const float* mean, const float* inv_std, float clip_lo, float clip_hi,
                                 int onehot_n, const int* seg_off, int nseg, void* out, int* overflow, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(x && out && B > 0, "obs_encode: null operand");
  B200RL_REQUIRE(in_pad % 8 == 0 && in_pad >= in_dim && in_dim > 0, "obs_encode: in_pad must be a multiple of 8 >= in_dim");
  B200RL_REQUIRE((reinterpret_cast<uintptr_t>(out) & 15) == 0, "obs_encode: output must be 16-byte aligned");
  B200RL_REQUIRE((mean == nullptr) == (inv_std == nullptr), "obs_encode: mean and inv_std come together");
  if (onehot_n > 0 && seg_off)
    B200RL_REQUIRE(nseg >= 1 && raw_dim == nseg && in_dim == onehot_n && mean == nullptr,
                   "obs_encode: MultiDiscrete one-hot needs raw_dim = nseg, in_dim = sum(nvec)");
  else if (onehot_n > 0)
    B200RL_REQUIRE(raw_dim == 1 && in_dim == onehot_n && mean == nullptr, "obs_encode: one-hot needs raw_dim 1, in_dim n");
  else
    B200RL_REQUIRE(raw_dim == in_dim, "obs_encode: raw_dim != in_dim");
  ObsEncodeParams p{x, src_idx, B, raw_dim, in_dim, in_pad, mean, inv_std, clip_lo, clip_hi, onehot_n,
                    onehot_n > 0 ? seg_off : nullptr, nseg, reinterpret_cast<__half*>(out), overflow};
  obs_encode_kernel<<<grid_blocks(B * (in_pad / 8), 256, 16), 256, 0, stream>>>(p);
  return check_launch("obs_encode_kernel");
}
