// Lowering of NHWC convolutions (tf.nn.conv2d, a2c/utils.py:56 of the reference) onto the wgmma GEMM:
//   im2col  : patches -> cols[B*OH*OW, rf*rf*C] fp16, K ordered (ky, kx, c) = HWIO weight flatten order
//             - uint8 source: the uint8->fp16 cast of models.py:19 is fused into this first load (the /255
//               is folded into the fp16 copy of the c1 weights), and the minibatch gather of
//               ppo2/ppo2.py:165 is fused too (src_idx picks samples straight out of the rollout buffer)
//   col2im  : dcols -> dx (gather form: every input element sums the taps that touched it), fused with
//             the activation derivative of the layer below
//   colsum  : bias gradients
// All HBM-bound: 16-byte vector accesses, consecutive lanes on consecutive 16 B chunks.
#include "common.cuh"

namespace b200rl {

struct ConvGeom {
  int H, W, C, rf, stride, OH, OW, pad_t, pad_l;   // pad_* = 0 for VALID
};

// one thread = one 16 B output chunk (8 fp16) of cols
template <typename SrcT>
__global__ void __launch_bounds__(256)
im2col_kernel(const SrcT* __restrict__ x, const long long* __restrict__ src_idx, __half* __restrict__ cols,
              long long B, ConvGeom g) {
  const int seg = g.rf * g.C;                 // contiguous elements per (pixel, ky)
  const int chunks_per_seg = seg / 8;
  const long long K = (long long)g.rf * seg;
  const long long total = B * g.OH * g.OW * g.rf * chunks_per_seg;
  for (long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x; id < total;
       id += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(id % chunks_per_seg);
    long long t = id / chunks_per_seg;
    const int ky = (int)(t % g.rf);
    t /= g.rf;                                 // t = output pixel row of cols
    const int ox = (int)(t % g.OW);
    long long t2 = t / g.OW;
    const int oy = (int)(t2 % g.OH);
    const long long b = t2 / g.OH;
    const long long sb = src_idx ? src_idx[b] : b;
    const int y = oy * g.stride + ky - g.pad_t;
    const int e0 = j * 8;                      // first element of this chunk inside the segment
    const int x_first = ox * g.stride - g.pad_l;
    __half out[8];
    const bool row_ok = (y >= 0 && y < g.H);
    const int kx0 = e0 / g.C, kx1 = (e0 + 7) / g.C;
    const bool all_in = row_ok && (x_first + kx0 >= 0) && (x_first + kx1 < g.W);
    const SrcT* src = x + ((sb * g.H + y) * g.W + x_first) * (long long)g.C + e0;
    const bool vec_ok = (sizeof(SrcT) != 1) || ((reinterpret_cast<uintptr_t>(src) & 7) == 0);
    if (all_in && vec_ok) {
      if (sizeof(SrcT) == 1) {
        const uint2 q = *reinterpret_cast<const uint2*>(src);
        const uint8_t* bp = reinterpret_cast<const uint8_t*>(&q);
#pragma unroll
        for (int i = 0; i < 8; ++i) out[i] = __ushort2half_rn((unsigned short)bp[i]);
      } else {
        *reinterpret_cast<uint4*>(out) = *reinterpret_cast<const uint4*>(src);
      }
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int el = e0 + i;
        const int xx = x_first + el / g.C;
        float v = 0.0f;
        if (row_ok && xx >= 0 && xx < g.W) {
          const SrcT s = x[((sb * g.H + y) * g.W + xx) * (long long)g.C + (el % g.C)];
          v = (sizeof(SrcT) == 1) ? (float)(*reinterpret_cast<const uint8_t*>(&s))
                                  : __half2float(*reinterpret_cast<const __half*>(&s));
        }
        out[i] = __float2half_rn(v);
      }
    }
    *reinterpret_cast<uint4*>(cols + t * K + (long long)ky * seg + e0) = *reinterpret_cast<const uint4*>(out);
  }
}

// one thread = 8 channels of one input pixel; dx = act'(saved) * sum over taps
__global__ void __launch_bounds__(256)
col2im_kernel(const __half* __restrict__ dcols, const __half* __restrict__ saved, __half* __restrict__ dx,
              long long B, ConvGeom g, int act) {
  const int cg = g.C / 8;
  const long long K = (long long)g.rf * g.rf * g.C;
  const long long total = B * g.H * g.W * cg;
  for (long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x; id < total;
       id += (long long)gridDim.x * blockDim.x) {
    const int c0 = (int)(id % cg) * 8;
    long long t = id / cg;
    const int xx = (int)(t % g.W);
    long long t2 = t / g.W;
    const int y = (int)(t2 % g.H);
    const long long b = t2 / g.H;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.0f;
    for (int ky = 0; ky < g.rf; ++ky) {
      const int yy = y + g.pad_t - ky;
      if (yy < 0 || (yy % g.stride) != 0) continue;
      const int oy = yy / g.stride;
      if (oy >= g.OH) continue;
      for (int kx = 0; kx < g.rf; ++kx) {
        const int xs = xx + g.pad_l - kx;
        if (xs < 0 || (xs % g.stride) != 0) continue;
        const int ox = xs / g.stride;
        if (ox >= g.OW) continue;
        const __half* src = dcols + ((b * g.OH + oy) * g.OW + ox) * K + ((long long)ky * g.rf + kx) * g.C + c0;
        const uint4 q = *reinterpret_cast<const uint4*>(src);
        const __half2* h = reinterpret_cast<const __half2*>(&q);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 f = __half22float2(h[i]);
          acc[2 * i] += f.x;
          acc[2 * i + 1] += f.y;
        }
      }
    }
    const long long o = ((b * g.H + y) * g.W + xx) * (long long)g.C + c0;
    if (saved != nullptr && act != 0) {
      const uint4 q = *reinterpret_cast<const uint4*>(saved + o);
      const __half* h = reinterpret_cast<const __half*>(&q);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float s = __half2float(h[i]);
        acc[i] *= (act == 1) ? (s > 0.0f ? 1.0f : 0.0f) : (1.0f - s * s);
      }
    }
    __half out[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) out[i] = __float2half_rn(acc[i]);
    *reinterpret_cast<uint4*>(dx + o) = *reinterpret_cast<const uint4*>(out);
  }
}

// Fused minibatch gather + uint8->fp16 cast + space-to-depth for the first conv layer:
//   out[b, Y, X, (dy*s + dx)*C + c] = x[src_idx[b], s*Y + dy, s*X + dx, c]
// A stride-s conv with filter rf = k*s over x becomes a stride-1 conv with filter k over `out`, whose
// s*s*C channels give TMA im2col full 128-byte rows.  One thread = 8 consecutive elements of one (dy) segment.
template <int EPT>   // elements per thread: 16 (one 16 B load, two 16 B stores) or 8
__global__ void __launch_bounds__(256)
s2d_gather_kernel(const uint8_t* __restrict__ x, const long long* __restrict__ src_idx, __half* __restrict__ out,
                  long long B, int H, int W, int C, int s) {
  const int seg = s * C;                   // contiguous elements per (Y, X, dy)
  const int cps = seg / EPT;
  const int HY = H / s, WX = W / s;
  const long long total = B * HY * WX * s * cps;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long id0 = (long long)blockIdx.x * blockDim.x + threadIdx.x; id0 < total; id0 += 4 * stride) {
    uint4 q[4];
    __half* dst[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {          // 4 independent loads in flight per thread
      const long long id = id0 + u * stride;
      dst[u] = nullptr;
      if (id < total) {
        const int j = (int)(id % cps);
        long long t = id / cps;
        const int dy = (int)(t % s);
        t /= s;
        const int X = (int)(t % WX);
        t /= WX;
        const int Y = (int)(t % HY);
        const long long b = t / HY;
        const long long sb = src_idx ? src_idx[b] : b;
        const uint8_t* src = x + ((sb * H + (long long)s * Y + dy) * W + (long long)s * X) * C + j * EPT;
        if (EPT == 16) q[u] = __ldg(reinterpret_cast<const uint4*>(src));
        else { const uint2 h = __ldg(reinterpret_cast<const uint2*>(src)); q[u] = make_uint4(h.x, h.y, 0, 0); }
        dst[u] = out + (((b * HY + Y) * WX + X) * (long long)s + dy) * seg + j * EPT;
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (dst[u]) {
        const uint32_t w[4] = {q[u].x, q[u].y, q[u].z, q[u].w};
        uint4 o[2];
        uint32_t* ow = reinterpret_cast<uint32_t*>(o);
#pragma unroll
        for (int i = 0; i < EPT / 4; ++i) {
          const __half2 lo = __floats2half2_rn((float)(w[i] & 0xffu), (float)((w[i] >> 8) & 0xffu));
          const __half2 hi = __floats2half2_rn((float)((w[i] >> 16) & 0xffu), (float)(w[i] >> 24));
          ow[2 * i] = *reinterpret_cast<const uint32_t*>(&lo);
          ow[2 * i + 1] = *reinterpret_cast<const uint32_t*>(&hi);
        }
        __stcs(reinterpret_cast<uint4*>(dst[u]), o[0]);
        if (EPT == 16) __stcs(reinterpret_cast<uint4*>(dst[u]) + 1, o[1]);
      }
    }
  }
}

// part[block, c] = alpha * sum over the block's rows of dz[row, c]  (b200rl_colsum adds the blocks' parts in order)
__global__ void __launch_bounds__(256)
colsum_kernel(const __half* __restrict__ dz, float* __restrict__ part, long long rows, int C, long long ld, float alpha,
              int rows_per_block) {
  __shared__ float red[256];
  const int cw = C < 256 ? C : 256;
  const int groups = 256 / cw;
  const int tid = threadIdx.x;
  const int grp = tid / cw;
  const int lc = tid % cw;
  const long long r0 = (long long)blockIdx.x * rows_per_block;
  const long long r1 = min(rows, r0 + rows_per_block);
  for (int cbase = 0; cbase < C; cbase += cw) {
    const int c = cbase + lc;
    float acc = 0.0f;
    if (grp < groups && c < C) {
      for (long long r = r0 + grp; r < r1; r += groups) acc += __half2float(dz[r * ld + c]);
    }
    red[tid] = acc;
    __syncthreads();
    if (tid < cw && cbase + tid < C) {
      float s = 0.0f;
      for (int gI = 0; gI < groups; ++gI) s += red[gI * cw + tid];
      part[(long long)blockIdx.x * C + cbase + tid] = s * alpha;
    }
    __syncthreads();
  }
}

// same sum with 16-byte loads: thread = (row group, 8-column slice); C and ld multiples of 8, 16-byte aligned base
__global__ void __launch_bounds__(256)
colsum_vec_kernel(const __half* __restrict__ dz, float* __restrict__ part, long long rows, int C, long long ld, float alpha,
                  int rows_per_block) {
  __shared__ float red[256][9];
  const int slices = C >> 3;                         // 8-column slices per row (<= 32)
  const int tid = threadIdx.x;
  const int sl = tid % slices, grp = tid / slices;
  const int groups = 256 / slices;
  const long long r0 = (long long)blockIdx.x * rows_per_block;
  const long long r1 = min(rows, r0 + rows_per_block);
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (grp < groups) {
    for (long long r = r0 + grp; r < r1; r += groups) {
      const uint4 q = *reinterpret_cast<const uint4*>(dz + r * ld + 8 * sl);
      const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
        acc[2 * i] += f.x;
        acc[2 * i + 1] += f.y;
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) red[tid][i] = acc[i];
  __syncthreads();
  if (tid < C) {
    const int s2 = tid >> 3, i = tid & 7;
    float s = 0.0f;
    for (int gI = 0; gI < groups; ++gI) s += red[gI * slices + s2][i];
    part[(long long)blockIdx.x * C + tid] = s * alpha;
  }
}

static int fill_geom(ConvGeom& g, int H, int W, int C, int rf, int stride, int same_pad) {
  g.H = H; g.W = W; g.C = C; g.rf = rf; g.stride = stride;
  if (same_pad) {
    g.OH = (H + stride - 1) / stride;
    g.OW = (W + stride - 1) / stride;
    int ph = (g.OH - 1) * stride + rf - H; if (ph < 0) ph = 0;
    int pw = (g.OW - 1) * stride + rf - W; if (pw < 0) pw = 0;
    g.pad_t = ph / 2; g.pad_l = pw / 2;      // TF 'SAME': extra pixel goes bottom/right
  } else {
    g.OH = (H - rf) / stride + 1;
    g.OW = (W - rf) / stride + 1;
    g.pad_t = g.pad_l = 0;
  }
  return (g.OH > 0 && g.OW > 0) ? 0 : -1;
}

// ------------------------------------------------------------------------------------------------ frame stack
// Device half of VecFrameStack (reference common/vec_env/vec_frame_stack.py:17-25): out = roll(prev, -1, axis=-1)
// (ONE channel, the reference's literal shift: a whole frame only when c == 1); out[news] = 0; out[..., -c:] = frame.
// Pixel p of env n holds K = nstack*c bytes.
template <int VEC>
__global__ void __launch_bounds__(256)
frame_stack_k4_kernel(const uint32_t* __restrict__ prev, const uint8_t* __restrict__ frame,
                      const uint8_t* __restrict__ news, uint32_t* __restrict__ out, long long pixels_per_env,
                      long long total_pixels) {
  // K = 4, c = 1: one 32-bit word per pixel; out = (prev >> 8) | frame << 24 (little endian: byte 3 = newest frame)
  const long long stride = (long long)gridDim.x * blockDim.x * VEC;
  for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * VEC; i < total_pixels; i += stride) {
    const bool fresh = news[i / pixels_per_env] != 0;       // VEC divides pixels_per_env: one env per vector
    if (VEC == 4) {
      const uint4 pv = fresh ? make_uint4(0, 0, 0, 0) : *reinterpret_cast<const uint4*>(prev + i);
      const uint32_t f = *reinterpret_cast<const uint32_t*>(frame + i);
      uint4 o;
      o.x = (pv.x >> 8) | ((f & 0xffu) << 24);
      o.y = (pv.y >> 8) | (((f >> 8) & 0xffu) << 24);
      o.z = (pv.z >> 8) | (((f >> 16) & 0xffu) << 24);
      o.w = (pv.w >> 8) | ((f >> 24) << 24);
      *reinterpret_cast<uint4*>(out + i) = o;
    } else {
      const uint32_t pv = fresh ? 0u : prev[i];
      out[i] = (pv >> 8) | ((uint32_t)frame[i] << 24);
    }
  }
}

__global__ void __launch_bounds__(256)
frame_stack_generic_kernel(const uint8_t* __restrict__ prev, const uint8_t* __restrict__ frame,
                           const uint8_t* __restrict__ news, uint8_t* __restrict__ out, long long pixels_per_env,
                           long long total_pixels, int K, int c) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total_pixels; i += stride) {
    const bool fresh = news[i / pixels_per_env] != 0;
    for (int k = 0; k < K - c; ++k) out[i * K + k] = fresh ? (uint8_t)0 : prev[i * K + k + 1];   // np.roll(.., -1)
    for (int k = 0; k < c; ++k) out[i * K + K - c + k] = frame[i * c + k];
  }
}

}  // namespace b200rl

using namespace b200rl;

extern "C" int b200rl_im2col(const void* x, int src_is_u8, const long long* src_idx, void* cols, long long B, int H,
                             int W, int C, int rf, int stride, int same_pad, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(x && cols && B > 0, "im2col: bad args");
  ConvGeom g;
  B200RL_REQUIRE(fill_geom(g, H, W, C, rf, stride, same_pad) == 0, "im2col: empty output");
  B200RL_REQUIRE((rf * C) % 8 == 0, "im2col: rf*C must be a multiple of 8 (got %d)", rf * C);
  if (src_is_u8)
    B200RL_REQUIRE((stride * C) % 8 == 0 && (W * C) % 8 == 0 && (reinterpret_cast<uintptr_t>(x) & 7) == 0,
                   "im2col(u8): stride*C and W*C must be multiples of 8");
  else
    B200RL_REQUIRE(C % 8 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0, "im2col(f16): C must be a multiple of 8");
  const long long total = B * g.OH * g.OW * rf * ((rf * C) / 8);
  const int grid = grid_blocks(total, 256, 32);
  if (src_is_u8)
    im2col_kernel<uint8_t><<<grid, 256, 0, stream>>>(reinterpret_cast<const uint8_t*>(x), src_idx,
                                                     reinterpret_cast<__half*>(cols), B, g);
  else
    im2col_kernel<__half><<<grid, 256, 0, stream>>>(reinterpret_cast<const __half*>(x), src_idx,
                                                    reinterpret_cast<__half*>(cols), B, g);
  return check_launch("im2col_kernel");
}

extern "C" int b200rl_frame_stack(const void* prev, const void* frame, const void* news, void* out, long long N,
                                  long long pixels, int nstack, int c, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(prev && frame && news && out && N > 0 && pixels > 0 && nstack >= 1 && c >= 1, "frame_stack: bad args");
  B200RL_REQUIRE(prev != out, "frame_stack: in-place update is not supported (pixels are shifted across threads' words)");
  const long long total = N * pixels;
  const int K = nstack * c;
  const bool al16 = ((reinterpret_cast<uintptr_t>(prev) | reinterpret_cast<uintptr_t>(out)) & 15) == 0 &&
                    (reinterpret_cast<uintptr_t>(frame) & 3) == 0;
  if (K == 4 && c == 1) {
    if (al16 && pixels % 4 == 0) {
      const int grid = grid_blocks(total / 4, 256, 16);
      frame_stack_k4_kernel<4><<<grid, 256, 0, stream>>>(reinterpret_cast<const uint32_t*>(prev),
                                                        reinterpret_cast<const uint8_t*>(frame),
                                                        reinterpret_cast<const uint8_t*>(news),
                                                        reinterpret_cast<uint32_t*>(out), pixels, total);
    } else {
      B200RL_REQUIRE(((reinterpret_cast<uintptr_t>(prev) | reinterpret_cast<uintptr_t>(out)) & 3) == 0,
                     "frame_stack: stacked buffers must be 4-byte aligned");
      const int grid = grid_blocks(total, 256, 16);
      frame_stack_k4_kernel<1><<<grid, 256, 0, stream>>>(reinterpret_cast<const uint32_t*>(prev),
                                                        reinterpret_cast<const uint8_t*>(frame),
                                                        reinterpret_cast<const uint8_t*>(news),
                                                        reinterpret_cast<uint32_t*>(out), pixels, total);
    }
  } else {
    const int grid = grid_blocks(total, 256, 16);
    frame_stack_generic_kernel<<<grid, 256, 0, stream>>>(reinterpret_cast<const uint8_t*>(prev),
                                                        reinterpret_cast<const uint8_t*>(frame),
                                                        reinterpret_cast<const uint8_t*>(news),
                                                        reinterpret_cast<uint8_t*>(out), pixels, total, K, c);
  }
  return check_launch("frame_stack_kernel");
}

extern "C" int b200rl_s2d_gather(const void* x, const long long* src_idx, void* out, long long B, int H, int W, int C,
                                 int s, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(x && out && B > 0 && s > 0, "s2d_gather: bad args");
  B200RL_REQUIRE(H % s == 0 && W % s == 0 && (s * C) % 8 == 0 && (reinterpret_cast<uintptr_t>(x) & 7) == 0 &&
                     (W * C) % 8 == 0,
                 "s2d_gather: need H,W multiples of s and s*C, W*C multiples of 8");
  const bool wide = ((s * C) % 16 == 0) && ((W * C) % 16 == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0);
  const long long total = B * (H / s) * (W / s) * s * ((s * C) / (wide ? 16 : 8));
  const int grid = grid_blocks((total + 3) / 4, 256, 32);
  if (wide)
    s2d_gather_kernel<16><<<grid, 256, 0, stream>>>(reinterpret_cast<const uint8_t*>(x), src_idx,
                                                    reinterpret_cast<__half*>(out), B, H, W, C, s);
  else
    s2d_gather_kernel<8><<<grid, 256, 0, stream>>>(reinterpret_cast<const uint8_t*>(x), src_idx,
                                                   reinterpret_cast<__half*>(out), B, H, W, C, s);
  return check_launch("s2d_gather_kernel");
}

extern "C" int b200rl_col2im(const void* dcols, const void* saved, void* dx, long long B, int H, int W, int C, int rf,
                             int stride, int same_pad, int act, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(dcols && dx && B > 0, "col2im: bad args");
  ConvGeom g;
  B200RL_REQUIRE(fill_geom(g, H, W, C, rf, stride, same_pad) == 0, "col2im: empty output");
  B200RL_REQUIRE(C % 8 == 0, "col2im: C must be a multiple of 8");
  const long long total = B * H * W * (C / 8);
  col2im_kernel<<<grid_blocks(total, 256, 32), 256, 0, stream>>>(reinterpret_cast<const __half*>(dcols),
                                                                  reinterpret_cast<const __half*>(saved),
                                                                  reinterpret_cast<__half*>(dx), B, g, act);
  return check_launch("col2im_kernel");
}

extern "C" int b200rl_colsum(const void* dz, float* db, long long rows, int C, long long ld, float alpha,
                             void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(dz && db && rows > 0 && C > 0, "colsum: bad args");
  long long rpb = (rows + (long long)device_num_sms() * 8 - 1) / ((long long)device_num_sms() * 8);
  if (rpb < 64) rpb = 64;
  const int grid = (int)((rows + rpb - 1) / rpb);
  float* part = det_workspace((size_t)grid * C, stream);
  if (!part) return B200RL_ERR_CUDA;
  int rc;
  if ((C & 7) == 0 && C <= 256 && (ld & 7) == 0 && (reinterpret_cast<uintptr_t>(dz) & 15) == 0) {
    colsum_vec_kernel<<<grid, 256, 0, stream>>>(reinterpret_cast<const __half*>(dz), part, rows, C, ld, alpha, (int)rpb);
    rc = check_launch("colsum_vec_kernel");
  } else {
    colsum_kernel<<<grid, 256, 0, stream>>>(reinterpret_cast<const __half*>(dz), part, rows, C, ld, alpha, (int)rpb);
    rc = check_launch("colsum_kernel");
  }
  if (rc == B200RL_OK) rc = sum_partials(part, grid, 1, C, db, C, stream);
  return rc;
}
