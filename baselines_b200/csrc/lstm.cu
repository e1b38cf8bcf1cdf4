// LSTM sequence kernels: the recurrence of baselines/a2c/utils.py lstm() (the cell of the `lstm` / `cnn_lstm` networks,
// common/models.py) over T steps, and its backward.  Everything that is not sequential runs on the wgmma GEMM: the
// input projection xg = x.Wx + b over all T*B rows before the forward, and dWx, dWh, db, dx from the dz this backward
// writes.
//
// Row ownership: a CTA owns LSTM_ROWS rows (environments) for all T steps.  Rows are independent, so the recurrence needs
// no cross-CTA synchronisation; Wh (forward) or Wh^T (backward) is loaded once into shared memory as fp16 and stays
// there.  A thread owns two adjacent hidden units j, j+1 of LSTM_RPT rows and all four gates of them, so the gate math
// runs from registers, and c (forward) / dc and the dh carry (backward) stay in fp32 registers for the whole sequence.
// The recurrent product is fp32 FMA over the fp16 weights and the fp32 h (forward) or dz (backward) held in shared
// memory, summed over k in a fixed order, so a row's result does not depend on T, on B or on which CTA runs it: T chained
// T = 1 passes give the same bits as one T-step pass.
//
// Layout.  Rows are time-major: row t*B + b is environment b at step t.  Gate columns are the reference's [i | f | o | u]
// blocks of H.  The state is [B, 2H] = [c | h] (utils.py:96 concat([c, h], axis=1)).  mask(t, b) is "done before step
// t": c and h are multiplied by 1 - mask before step t (utils.py:87-88).
#include "common.cuh"

namespace b200rl {

constexpr int LSTM_ROWS = 8;   // rows per CTA
constexpr int LSTM_RPT = 4;    // rows per thread (LSTM_ROWS / LSTM_RPT row groups of H / 2 threads)

struct LstmFwdParams {
  const float* xg;            // [T*B, ldxg] x.Wx + b
  long long ldxg;
  const __half* wh;           // [H, 4H]
  const uint8_t* masks;       // mask of row r at masks[mask_idx ? mask_idx[r] : r]
  const long long* mask_idx;  // optional [T*B]
  const float* state_in;      // [*, 2H]; environment b reads row state_idx ? state_idx[b] : b
  const long long* state_idx; // optional [B]
  float* state_out;           // optional [B, 2H] final (c, h); may alias state_in when state_idx is null
  __half* h_out;              // [T*B, ldh] h_t
  long long ldh;
  __half* hprev_out;          // optional [T*B, H] masked h_{t-1}: the A operand of dWh
  float* gates_out;           // optional [T*B, 4H] sigma(i), sigma(f), sigma(o), tanh(u); may alias xg (ldxg = 4H)
  float* c_out;               // optional [T*B, H] c_t
  int T, B;
};

struct LstmBwdParams {
  const __half* dh;           // [T*B, lddh] d loss / d h_t from the heads
  long long lddh;
  const float* gates;         // [T*B, 4H] as written by the forward
  const float* c;             // [T*B, H]
  const uint8_t* masks;
  const long long* mask_idx;
  const float* state_in;      // the forward's start state (c_{-1})
  const long long* state_idx;
  const __half* whT;          // [4H, H]
  __half* dz;                 // [T*B, lddz] d loss / d z_t (pre-activation gates)
  long long lddz;
  int T, B;
};

__device__ __forceinline__ float lstm_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

__device__ __forceinline__ float lstm_keep(const uint8_t* masks, const long long* idx, long long r) {
  return masks[idx ? idx[r] : r] ? 0.0f : 1.0f;
}

template <int H>
__global__ void __launch_bounds__(H) lstm_seq_fwd_kernel(const LstmFwdParams p) {
  extern __shared__ __align__(16) unsigned char lstm_smem[];
  __half* wh = reinterpret_cast<__half*>(lstm_smem);                          // [H][4H]
  float* hs = reinterpret_cast<float*>(lstm_smem + (size_t)H * 4 * H * 2);    // [2][LSTM_ROWS][H] masked h_{t-1}
  const int tid = threadIdx.x;
  const int j = 2 * (tid % (H / 2));
  const int rg = tid / (H / 2);
  const long long B = p.B;
  {
    const uint4* src = reinterpret_cast<const uint4*>(p.wh);
    uint4* dst = reinterpret_cast<uint4*>(wh);
    for (int i = tid; i < H * 4 * H / 8; i += H) dst[i] = src[i];
  }
  long long b[LSTM_RPT];
  bool ok[LSTM_RPT];
  float c[LSTM_RPT][2];
#pragma unroll
  for (int r = 0; r < LSTM_RPT; ++r) {
    const int lr = rg * LSTM_RPT + r;
    b[r] = (long long)blockIdx.x * LSTM_ROWS + lr;
    ok[r] = b[r] < B;
    float2 cs = make_float2(0.f, 0.f), hh = make_float2(0.f, 0.f);
    float keep = 0.f;
    if (ok[r]) {
      const float* s = p.state_in + (p.state_idx ? p.state_idx[b[r]] : b[r]) * (2LL * H);
      cs = *reinterpret_cast<const float2*>(s + j);
      hh = *reinterpret_cast<const float2*>(s + H + j);
      keep = lstm_keep(p.masks, p.mask_idx, b[r]);
    }
    c[r][0] = cs.x * keep;
    c[r][1] = cs.y * keep;
    const float2 hm = make_float2(hh.x * keep, hh.y * keep);
    *reinterpret_cast<float2*>(hs + lr * H + j) = hm;
    if (ok[r] && p.hprev_out)
      *reinterpret_cast<__half2*>(p.hprev_out + b[r] * H + j) = __floats2half2_rn(hm.x, hm.y);
  }
  __syncthreads();
  for (int t = 0; t < p.T; ++t) {
    const int cur = t & 1;
    float acc[LSTM_RPT][4][2];
#pragma unroll
    for (int r = 0; r < LSTM_RPT; ++r) {
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        float2 v = make_float2(0.f, 0.f);
        if (ok[r]) v = *reinterpret_cast<const float2*>(p.xg + (t * B + b[r]) * p.ldxg + g * H + j);
        acc[r][g][0] = v.x;
        acc[r][g][1] = v.y;
      }
    }
    const float* hcur = hs + (cur * LSTM_ROWS + rg * LSTM_RPT) * H;
#pragma unroll 2
    for (int k = 0; k < H; k += 4) {
      float4 hv[LSTM_RPT];
#pragma unroll
      for (int r = 0; r < LSTM_RPT; ++r) hv[r] = *reinterpret_cast<const float4*>(hcur + r * H + k);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const __half2* wrow = reinterpret_cast<const __half2*>(wh + (k + kk) * 4 * H + j);
        float2 w[4];
#pragma unroll
        for (int g = 0; g < 4; ++g) w[g] = __half22float2(wrow[g * (H / 2)]);
#pragma unroll
        for (int r = 0; r < LSTM_RPT; ++r) {
          const float hk = kk == 0 ? hv[r].x : kk == 1 ? hv[r].y : kk == 2 ? hv[r].z : hv[r].w;
#pragma unroll
          for (int g = 0; g < 4; ++g) {
            acc[r][g][0] = fmaf(hk, w[g].x, acc[r][g][0]);
            acc[r][g][1] = fmaf(hk, w[g].y, acc[r][g][1]);
          }
        }
      }
    }
    const bool last = t + 1 == p.T;
#pragma unroll
    for (int r = 0; r < LSTM_RPT; ++r) {
      const int lr = rg * LSTM_RPT + r;
      float gv[4][2], hn[2];
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const float i = lstm_sigmoid(acc[r][0][q]), f = lstm_sigmoid(acc[r][1][q]);
        const float o = lstm_sigmoid(acc[r][2][q]), u = tanhf(acc[r][3][q]);
        c[r][q] = f * c[r][q] + i * u;
        hn[q] = o * tanhf(c[r][q]);
        gv[0][q] = i; gv[1][q] = f; gv[2][q] = o; gv[3][q] = u;
      }
      float keepn = 1.f;
      if (ok[r]) {
        const long long row = t * B + b[r];
        *reinterpret_cast<__half2*>(p.h_out + row * p.ldh + j) = __floats2half2_rn(hn[0], hn[1]);
        if (p.gates_out) {
#pragma unroll
          for (int g = 0; g < 4; ++g)
            *reinterpret_cast<float2*>(p.gates_out + row * (4LL * H) + g * H + j) = make_float2(gv[g][0], gv[g][1]);
        }
        if (p.c_out) *reinterpret_cast<float2*>(p.c_out + row * H + j) = make_float2(c[r][0], c[r][1]);
        if (last) {
          if (p.state_out) {
            float* s = p.state_out + b[r] * (2LL * H);
            *reinterpret_cast<float2*>(s + j) = make_float2(c[r][0], c[r][1]);
            *reinterpret_cast<float2*>(s + H + j) = make_float2(hn[0], hn[1]);
          }
        } else {
          keepn = lstm_keep(p.masks, p.mask_idx, row + B);
          if (p.hprev_out)
            *reinterpret_cast<__half2*>(p.hprev_out + (row + B) * H + j) = __floats2half2_rn(hn[0] * keepn, hn[1] * keepn);
        }
      }
      if (!last) {
        c[r][0] *= keepn;
        c[r][1] *= keepn;
        *reinterpret_cast<float2*>(hs + ((cur ^ 1) * LSTM_ROWS + lr) * H + j) = make_float2(hn[0] * keepn, hn[1] * keepn);
      }
    }
    __syncthreads();
  }
}

template <int H>
__global__ void __launch_bounds__(H) lstm_seq_bwd_kernel(const LstmBwdParams p) {
  extern __shared__ __align__(16) unsigned char lstm_smem[];
  __half* whT = reinterpret_cast<__half*>(lstm_smem);                         // [4H][H]
  float* dzs = reinterpret_cast<float*>(lstm_smem + (size_t)H * 4 * H * 2);   // [2][LSTM_ROWS][4H]
  const int tid = threadIdx.x;
  const int j = 2 * (tid % (H / 2));
  const int rg = tid / (H / 2);
  const long long B = p.B;
  {
    const uint4* src = reinterpret_cast<const uint4*>(p.whT);
    uint4* dst = reinterpret_cast<uint4*>(whT);
    for (int i = tid; i < H * 4 * H / 8; i += H) dst[i] = src[i];
  }
  long long b[LSTM_RPT];
  bool ok[LSTM_RPT];
  float dc[LSTM_RPT][2], carry[LSTM_RPT][2];
#pragma unroll
  for (int r = 0; r < LSTM_RPT; ++r) {
    b[r] = (long long)blockIdx.x * LSTM_ROWS + rg * LSTM_RPT + r;
    ok[r] = b[r] < B;
    dc[r][0] = dc[r][1] = carry[r][0] = carry[r][1] = 0.f;
  }
  __syncthreads();
  for (int t = p.T - 1; t >= 0; --t) {
    const int cur = t & 1;
    float keep[LSTM_RPT];
#pragma unroll
    for (int r = 0; r < LSTM_RPT; ++r) {
      const int lr = rg * LSTM_RPT + r;
      float dz[4][2] = {{0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}};
      keep[r] = 0.f;
      if (ok[r]) {
        const long long row = t * B + b[r];
        keep[r] = lstm_keep(p.masks, p.mask_idx, row);
        const float* gr = p.gates + row * (4LL * H);
        const float2 gi = *reinterpret_cast<const float2*>(gr + j);
        const float2 gf = *reinterpret_cast<const float2*>(gr + H + j);
        const float2 go = *reinterpret_cast<const float2*>(gr + 2 * H + j);
        const float2 gu = *reinterpret_cast<const float2*>(gr + 3 * H + j);
        const float2 ct = *reinterpret_cast<const float2*>(p.c + row * H + j);
        const float* cprow = t > 0 ? p.c + (row - B) * H
                                   : p.state_in + (p.state_idx ? p.state_idx[b[r]] : b[r]) * (2LL * H);
        const float2 cp = *reinterpret_cast<const float2*>(cprow + j);
        const float2 dhh = __half22float2(*reinterpret_cast<const __half2*>(p.dh + row * p.lddh + j));
        const float iv[2] = {gi.x, gi.y}, fv[2] = {gf.x, gf.y}, ov[2] = {go.x, go.y}, uv[2] = {gu.x, gu.y};
        const float cv[2] = {ct.x, ct.y}, cpv[2] = {cp.x * keep[r], cp.y * keep[r]}, dhv[2] = {dhh.x, dhh.y};
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const float dh = dhv[q] + carry[r][q];
          const float tc = tanhf(cv[q]);
          const float dcq = dc[r][q] + dh * ov[q] * (1.f - tc * tc);
          dz[0][q] = dcq * uv[q] * iv[q] * (1.f - iv[q]);
          dz[1][q] = dcq * cpv[q] * fv[q] * (1.f - fv[q]);
          dz[2][q] = dh * tc * ov[q] * (1.f - ov[q]);
          dz[3][q] = dcq * iv[q] * (1.f - uv[q] * uv[q]);
          dc[r][q] = dcq * fv[q] * keep[r];
        }
#pragma unroll
        for (int g = 0; g < 4; ++g)
          *reinterpret_cast<__half2*>(p.dz + row * p.lddz + g * H + j) = __floats2half2_rn(dz[g][0], dz[g][1]);
      }
#pragma unroll
      for (int g = 0; g < 4; ++g)
        *reinterpret_cast<float2*>(dzs + (cur * LSTM_ROWS + lr) * 4 * H + g * H + j) = make_float2(dz[g][0], dz[g][1]);
    }
    __syncthreads();
    if (t == 0) break;
    // dh_{t-1} = (dz_t . Wh^T) * (1 - mask_t)
    float s[LSTM_RPT][2];
#pragma unroll
    for (int r = 0; r < LSTM_RPT; ++r) s[r][0] = s[r][1] = 0.f;
    const float* dzr = dzs + (cur * LSTM_ROWS + rg * LSTM_RPT) * 4 * H;
#pragma unroll 2
    for (int n = 0; n < 4 * H; n += 4) {
      float4 dv[LSTM_RPT];
#pragma unroll
      for (int r = 0; r < LSTM_RPT; ++r) dv[r] = *reinterpret_cast<const float4*>(dzr + r * 4 * H + n);
#pragma unroll
      for (int nn = 0; nn < 4; ++nn) {
        const float2 w = __half22float2(*reinterpret_cast<const __half2*>(whT + (n + nn) * H + j));
#pragma unroll
        for (int r = 0; r < LSTM_RPT; ++r) {
          const float d = nn == 0 ? dv[r].x : nn == 1 ? dv[r].y : nn == 2 ? dv[r].z : dv[r].w;
          s[r][0] = fmaf(d, w.x, s[r][0]);
          s[r][1] = fmaf(d, w.y, s[r][1]);
        }
      }
    }
#pragma unroll
    for (int r = 0; r < LSTM_RPT; ++r) {
      carry[r][0] = s[r][0] * keep[r];
      carry[r][1] = s[r][1] * keep[r];
    }
  }
}

static bool lstm_aligned(const void* ptr, int bytes) { return (reinterpret_cast<uintptr_t>(ptr) & (bytes - 1)) == 0; }

template <int H>
static int lstm_fwd_launch(const LstmFwdParams& p, cudaStream_t stream) {
  const int smem = H * 4 * H * 2 + 2 * LSTM_ROWS * H * 4;
  auto kern = lstm_seq_fwd_kernel<H>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) {
    set_last_error("lstm_seq_fwd: cudaFuncSetAttribute(smem=%d): %s", smem, cudaGetErrorString(e));
    return B200RL_ERR_CUDA;
  }
  kern<<<ceil_div(p.B, LSTM_ROWS), H, smem, stream>>>(p);
  return check_launch("lstm_seq_fwd_kernel");
}

template <int H>
static int lstm_bwd_launch(const LstmBwdParams& p, cudaStream_t stream) {
  const int smem = H * 4 * H * 2 + 2 * LSTM_ROWS * 4 * H * 4;
  auto kern = lstm_seq_bwd_kernel<H>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) {
    set_last_error("lstm_seq_bwd: cudaFuncSetAttribute(smem=%d): %s", smem, cudaGetErrorString(e));
    return B200RL_ERR_CUDA;
  }
  kern<<<ceil_div(p.B, LSTM_ROWS), H, smem, stream>>>(p);
  return check_launch("lstm_seq_bwd_kernel");
}

}  // namespace b200rl

using namespace b200rl;

extern "C" int b200rl_lstm_seq_fwd(const float* xg, long long ldxg, const void* wh, const uint8_t* masks,
                                   const long long* mask_idx, const float* state_in, const long long* state_idx,
                                   float* state_out, void* h_out, long long ldh, void* hprev_out, float* gates_out,
                                   float* c_out, int T, int B, int H, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(xg && wh && masks && state_in && h_out, "lstm_seq_fwd: null operand");
  B200RL_REQUIRE(H == 64 || H == 128, "lstm_seq_fwd: H = %d (instances: 64, 128)", H);
  B200RL_REQUIRE(T >= 1 && B >= 1, "lstm_seq_fwd: T = %d, B = %d", T, B);
  B200RL_REQUIRE(ldxg >= 4LL * H && ldxg % 2 == 0 && ldh >= H && ldh % 2 == 0, "lstm_seq_fwd: bad row pitch");
  B200RL_REQUIRE(lstm_aligned(xg, 8) && lstm_aligned(wh, 16) && lstm_aligned(state_in, 8) && lstm_aligned(h_out, 4) &&
                 (!state_out || lstm_aligned(state_out, 8)) && (!hprev_out || lstm_aligned(hprev_out, 4)) &&
                 (!gates_out || lstm_aligned(gates_out, 8)) && (!c_out || lstm_aligned(c_out, 8)),
                 "lstm_seq_fwd: misaligned operand");
  B200RL_REQUIRE(!state_out || state_out != state_in || !state_idx, "lstm_seq_fwd: in-place state needs state_idx = null");
  B200RL_REQUIRE(!gates_out || reinterpret_cast<const float*>(gates_out) != xg || ldxg == 4LL * H,
                 "lstm_seq_fwd: gates_out may alias xg only with ldxg = 4H");
  LstmFwdParams p{xg, ldxg, reinterpret_cast<const __half*>(wh), masks, mask_idx, state_in, state_idx, state_out,
                  reinterpret_cast<__half*>(h_out), ldh, reinterpret_cast<__half*>(hprev_out), gates_out, c_out, T, B};
  return H == 64 ? lstm_fwd_launch<64>(p, stream) : lstm_fwd_launch<128>(p, stream);
}

extern "C" int b200rl_lstm_seq_bwd(const void* dh, long long lddh, const float* gates, const float* c,
                                   const uint8_t* masks, const long long* mask_idx, const float* state_in,
                                   const long long* state_idx, const void* whT, void* dz, long long lddz, int T, int B,
                                   int H, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(dh && gates && c && masks && state_in && whT && dz, "lstm_seq_bwd: null operand");
  B200RL_REQUIRE(H == 64 || H == 128, "lstm_seq_bwd: H = %d (instances: 64, 128)", H);
  B200RL_REQUIRE(T >= 1 && B >= 1, "lstm_seq_bwd: T = %d, B = %d", T, B);
  B200RL_REQUIRE(lddh >= H && lddh % 2 == 0 && lddz >= 4LL * H && lddz % 2 == 0, "lstm_seq_bwd: bad row pitch");
  B200RL_REQUIRE(lstm_aligned(dh, 4) && lstm_aligned(gates, 8) && lstm_aligned(c, 8) && lstm_aligned(state_in, 8) &&
                 lstm_aligned(whT, 16) && lstm_aligned(dz, 4), "lstm_seq_bwd: misaligned operand");
  LstmBwdParams p{reinterpret_cast<const __half*>(dh), lddh, gates, c, masks, mask_idx, state_in, state_idx,
                  reinterpret_cast<const __half*>(whT), reinterpret_cast<__half*>(dz), lddz, T, B};
  return H == 64 ? lstm_bwd_launch<64>(p, stream) : lstm_bwd_launch<128>(p, stream);
}
