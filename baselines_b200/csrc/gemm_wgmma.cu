// Persistent warp-specialised wgmma GEMM / implicit-GEMM convolution for sm_90a
// (fp16 operands, fp32 accumulate in registers).
//
//   warps 0..7 : two consumer warpgroups; warpgroup g owns rows [64g, 64g+64) of the 128-row tile: it issues
//                wgmma.mma_async m64nBNk16 from the swizzled smem ring, frees each stage once its MMAs retired,
//                and runs the fused epilogue (bias / activation / mask / split-K parts / pixel-shuffle scatter) straight
//                from the accumulator registers
//   warp 8     : TMA producer (tiled or IM2COL-mode cp.async.bulk.tensor -> swizzled smem ring, mbarrier tx)
//
// K-major plain GEMMs with the f16 / f32-store epilogue (forward and data gradient of fc layers) instead stage their
// epilogue as conv_shift.cu does: the bias of a tile is read once into shared memory, each warp's fp16 fragment leaves
// through a per-warp swizzled scratch (stmatrix) as 16-byte row pieces, the column remap is computed once per 16-column
// chunk, a ReLU bit mask is staged by the producer warp with the tile's last k-block, and the fp16 saved activation is
// read as 16-byte pieces (ldmatrix hands it back in the accumulator layout).  Where the accumulators fit (BN <= 128,
// not the fp32 store at 128) they run the ping-pong schedule: each warpgroup takes whole tiles, even / odd, as two
// m64 accumulators, and named barriers order the groups' MMA issue, so one group's epilogue overlaps the other's MMAs.
//
// The reduction dimension is processed in stages of 64 elements made of 64/CPT "taps" of CPT elements
// (CPT = 64, 32 or 16 -> 128 B / 64 B / 32 B swizzled smem rows):
//   plain GEMM      : a tap is a 64-wide K chunk                                 (CPT = 64)
//   implicit conv   : a tap is one filter position (r, s) x CPT input channels, fetched straight from the NHWC
//                     activation by TMA im2col mode -- the im2col matrix is never materialised
// Operand layouts:
//   K-major  : A[M,K] rows = output pixels, B[N,K] = weights          C = A * B^T     (forward, dgrad)
//   MN-major : A[K,M], B[K,N] with K = batch pixels                    C += A^T * B    (wgrad, split-K)
//
// Replaces tf.matmul (a2c/utils.py:63), tf.nn.conv2d (a2c/utils.py:56) and their gradients
// (tf.gradients via ppo2/model.py:102) of the reference.
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>

#include <map>
#include <type_traits>
#include <mutex>

#include "common.cuh"
#include "tc_common.cuh"

namespace b200rl {

static constexpr int BM = 128;
static constexpr int BK = 64;          // elements of the reduction dimension per pipeline stage
static constexpr int MMA_K = 16;
static constexpr int CONSUMER_WARPS = 8;
static constexpr int NUM_THREADS = CONSUMER_WARPS * 32 + 32;


struct ConvCoords {       // im2col traversal of the A operand (all zero for plain GEMMs)
  int OW, OH;             // grid of base pixels per image (GEMM rows = n*OH*OW + p*OW + q)
  int stride_w, stride_h; // traversal strides (input pixels per base-pixel step)
  int lower_w, lower_h;   // coordinate of base pixel 0 (= -padding)
  int S, taps;            // filter width (taps per filter row) and total number of taps R*S
};

struct ShuffleOut {       // MODE_F16_SHUFFLE: GEMM row (n,i,j), col (py,px,c) -> dx[n, s*i+py, s*j+px, c]
  int H, W, C, s;
};

struct GemmParams {
  int M, N, K;
  int m_tiles, n_tiles, splits, kb_per_split, kb_total;
  void* C;
  long long ldc;
  const float* bias;
  const __half* saved;     // saved activation for MODE_F16_DACT / SHUFFLE masks
  const uint16_t* saved_bits;   // MODE_F16_DACT alternative: 1 bit per element (activation > 0), word (row*ld_saved + col)/16
  long long ld_saved;
  float alpha;
  int mode, act;
  ConvCoords cv;
  ShuffleOut sh;
  bool vec32;               // f16 outputs: rows / columns aligned so that a column pair is one 4-byte store
  bool vec16;               // staged epilogue: C and ldc allow 16-byte row pieces (8 fp16 / 4 fp32 columns)
  bool saved16;             // staged epilogue: `saved` and ld_saved allow 16-byte row pieces
  int rm_C, rm_OW, rm_Wg;   // rm_C > 0: output column (pix*rm_C + c) is stored at ((pix/rm_OW)*rm_Wg + pix%rm_OW)*rm_C + c
  float* ws;                // MODE_F32_ATOMIC with splits > 1: split s stores its partial [M, N] at ws + s*M*N
};

template <int BN>
struct Cfg {
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES_RAW = (196 * 1024) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_RAW > 8 ? 8 : STAGES_RAW;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
};

// Staged epilogue of the K-major plain instances (TMODE = MODE_F16_ACT, MODE_F16_DACT or MODE_F32_STORE), after the
// barrier block: the ReLU bit mask of each stage (DACT: 128 rows x BN bits, filled with a tile's last k-block), then one
// 16-row x 32-column fp16 transpose scratch per consumer warp (as in conv_shift.cu).
__host__ __device__ constexpr bool staged_epi(bool mn_major, bool im2col, int tmode) {
  return !mn_major && !im2col && (tmode == MODE_F16_ACT || tmode == MODE_F16_DACT || tmode == MODE_F32_STORE);
}
static constexpr int EPI_WARP_BYTES = 16 * 64;
__host__ __device__ constexpr int staged_mask_bytes(int BN, int tmode) { return tmode == MODE_F16_DACT ? BM * BN / 8 : 0; }
template <int BN, int TMODE>
__host__ __device__ constexpr int staged_smem_bytes() {
  return Cfg<BN>::STAGES * staged_mask_bytes(BN, TMODE) + CONSUMER_WARPS * EPI_WARP_BYTES;
}
// Ping-pong (each consumer warpgroup takes whole 128 x BN tiles, two m64 accumulators) where BN/2 * 2 accumulator
// registers fit under the 168-register cap of 9 warps next to the epilogue's: BN = 256, and the fp32 store at BN = 128
// (which would spill), keep the cooperative schedule (each group 64 rows of every tile).
__host__ __device__ constexpr bool gemm_pingpong(int BN, int tmode) {
  return BN <= 64 || (BN == 128 && tmode != MODE_F32_STORE);
}

// CPT: channels per tap (64 / 32 / 16); MN_MAJOR: wgrad layout; IM2COL: A operand through TMA im2col mode
// BRES (K-major implicit conv only): the whole weight matrix (taps x [BN x CPT]) is loaded ONCE per CTA and
// stays resident in shared memory; the ring then carries only the A (activation patch) tiles.
static constexpr int BRES_STAGES = 7;
static constexpr int BRES_B_BYTES = 80 * 1024;

// Read-only global loads as volatile asm: the compiler keeps them in program order next to the epilogue's stmatrix /
// ldmatrix instead of hoisting every chunk's load, whose registers the ping-pong accumulators cannot spare.
__device__ __forceinline__ uint4 ld_nc_v4(const void* p) {
  uint4 v;
  asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ unsigned short ld_nc_u16(const void* p) {
  unsigned short v;
  asm volatile("ld.global.nc.u16 %0, [%1];" : "=h"(v) : "l"(p));
  return v;
}

// Epilogue of one accumulator column pair (col, col + 1) of one row; `two`: col + 1 < N.
__device__ __forceinline__ void gemm_epi_pair(const GemmParams& p, int mode, int split, int row, int col, float v0,
                                              float v1, bool two) {
  if (mode == MODE_F32_ATOMIC) {
    if (p.ws) {                                // split-K: this split's partial, summed in split order afterwards
      float* w = p.ws + ((long long)split * p.M + row) * p.N + col;
      w[0] = v0;
      if (two) w[1] = v1;
      return;
    }
    float* out = reinterpret_cast<float*>(p.C) + (long long)row * p.ldc + col;
    atomicAdd(out, v0);
    if (two) atomicAdd(out + 1, v1);
    return;
  }
  if (mode == MODE_F32_STORE) {
    float* out = reinterpret_cast<float*>(p.C) + (long long)row * p.ldc + col;
    out[0] = v0 + (p.bias ? p.bias[col] : 0.0f);
    if (two) out[1] = v1 + (p.bias ? p.bias[col + 1] : 0.0f);
    return;
  }
  __half* C = reinterpret_cast<__half*>(p.C);
  if (mode == MODE_F16_SHUFFLE) {
    // dgrad of a strided conv: column (py, px, c) of GEMM row (n, i, j); C % 16 == 0 keeps the pair in one class
    const int cls = col / p.sh.C, c = col % p.sh.C;
    const int j = row % p.cv.OW, t3 = row / p.cv.OW;
    const int i = t3 % p.cv.OH, n = t3 / p.cv.OH;
    const int y = p.sh.s * i + cls / p.sh.s, x = p.sh.s * j + cls % p.sh.s;
    if (y < p.sh.H && x < p.sh.W) {
      const long long o = (((long long)n * p.sh.H + y) * p.sh.W + x) * p.sh.C + c;
      if (p.saved) {
        v0 *= act_grad_from_saved(__half2float(p.saved[o]), p.act);
        v1 *= act_grad_from_saved(__half2float(p.saved[o + 1]), p.act);
      }
      *reinterpret_cast<__half2*>(C + o) = __floats2half2_rn(v0, v1);
    }
    return;
  }
  if (mode == MODE_F16_ACT) {
    if (p.bias) {
      v0 += __ldg(p.bias + col);
      if (two) v1 += __ldg(p.bias + col + 1);
    }
    v0 = apply_act(v0, p.act);
    v1 = apply_act(v1, p.act);
  } else {  // MODE_F16_DACT: dX = (dY W^T) * act'(saved activation)
    const long long so = (long long)row * p.ld_saved + col;
    if (p.saved_bits != nullptr) {             // 1 bit per element: relu'(h) = (h > 0)
      const uint32_t w = __ldg(p.saved_bits + (so >> 4));
      const int b = (int)(so & 15);
      v0 = ((w >> b) & 1u) ? v0 : 0.0f;
      v1 = ((w >> (b + 1)) & 1u) ? v1 : 0.0f;
    } else {
      v0 *= act_grad_from_saved(__half2float(p.saved[so]), p.act);
      if (two) v1 *= act_grad_from_saved(__half2float(p.saved[so + 1]), p.act);
    }
  }
  int ocol = col;
  if (p.rm_C > 0) {
    const int pix = col / p.rm_C;
    ocol = ((pix / p.rm_OW) * p.rm_Wg + pix % p.rm_OW) * p.rm_C + col % p.rm_C;
  }
  __half* out = C + (long long)row * p.ldc + ocol;
  if (two && p.vec32) {
    *reinterpret_cast<__half2*>(out) = __floats2half2_rn(v0, v1);
  } else {
    out[0] = __float2half_rn(v0);
    if (two) out[1] = __float2half_rn(v1);
  }
}

// TMODE >= 0 fixes the epilogue mode at compile time (plain GEMMs): the multi-mode epilogue is several times larger.
template <int BN, int CPT, bool MN_MAJOR, bool IM2COL, bool BRES, int TMODE>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const GemmParams p) {
  using C_ = Cfg<BN>;
  static_assert(!BRES || (IM2COL && !MN_MAJOR), "resident weights: K-major implicit conv only");
  constexpr int STAGES = BRES ? BRES_STAGES : C_::STAGES;
  constexpr int STAGE_BYTES = BRES ? C_::A_BYTES : C_::STAGE_BYTES;
  constexpr int BROWB = MN_MAJOR ? (BN >= 64 ? 128 : BN * 2) : 0;     // MN-major B: bytes per pixel row
  constexpr uint32_t LAYOUT_B = sdesc_layout(BROWB);
  constexpr int BCHUNKS = (BN >= 64) ? BN / 64 : 1;
  constexpr int TPS = BK / CPT;                     // taps per stage
  constexpr int ROWB = CPT * 2;                     // bytes per smem row of a K-major / A-MN sub-tile
  constexpr uint32_t LAYOUT_A = sdesc_layout(ROWB);
  constexpr int A_SUB = BM * ROWB;                  // K-major: one tap of 128 rows
  constexpr int B_SUB = BN * ROWB;                  // K-major: one tap of BN weight rows
  constexpr int A_CHUNK = BK * ROWB;                // MN-major: 64 pixel rows x CPT channels (one tap)
  constexpr int MCH = BM / CPT;                     // MN-major: taps (M chunks) per M tile
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* bres = smem + STAGES * STAGE_BYTES;            // resident weights (BRES only)
  // K-major implicit conv: a zero weight tile, read by the tap slots of the last stage that hold no tap
  constexpr int ZT_BYTES = (IM2COL && !MN_MAJOR) ? B_SUB : 0;
  uint8_t* zero_tile = bres + (BRES ? BRES_B_BYTES : 0);
  uint64_t* bars = reinterpret_cast<uint64_t*>(zero_tile + ZT_BYTES);
  uint64_t* full_bar = bars;                  // [STAGES]
  uint64_t* empty_bar = bars + STAGES;        // [STAGES]
  uint64_t* bres_bar = bars + 2 * STAGES;     // [1]
  constexpr bool STAGED = staged_epi(MN_MAJOR, IM2COL, TMODE);
  constexpr bool PINGPONG = STAGED && gemm_pingpong(BN, TMODE);
  constexpr int MASK_STAGE = STAGED ? staged_mask_bytes(BN, TMODE) : 0;
  uint8_t* smask = reinterpret_cast<uint8_t*>(bars) + 256;      // STAGED DACT: the mask rows of stage s's tile
  uint8_t* sepi = smask + STAGES * MASK_STAGE;                  // STAGED: epilogue scratch, one per consumer warp
  __shared__ float s_bias[2][STAGED ? BN : 1];                  // STAGED: each group's copy of its tile's bias

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int total_work = p.m_tiles * p.n_tiles * p.splits;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      // a stage is released by the warps that read it: one group's 4 under ping-pong, both groups' 8 otherwise
      mbar_init(&empty_bar[s], PINGPONG ? 4 : CONSUMER_WARPS);
    }
    mbar_init(bres_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == CONSUMER_WARPS) {
    // ------------------------------------------------------------------ TMA producer
    if (elect_one()) {
      tma_prefetch_desc(&tmA);
      tma_prefetch_desc(&tmB);
      if (BRES) {
        mbar_arrive_expect_tx(bres_bar, (uint32_t)p.cv.taps * B_SUB);
        for (int g = 0; g < p.cv.taps; ++g) tma_load_2d(bres + g * B_SUB, &tmB, bres_bar, g * CPT, 0);
      }
    }
    __syncwarp();
    int s = 0;
    uint32_t ph = 0;
    for (int work = blockIdx.x; work < total_work; work += gridDim.x) {
      const int n_tile = work % p.n_tiles;
      const int t2 = work / p.n_tiles;
      const int m_tile = t2 % p.m_tiles;
      const int split = t2 / p.m_tiles;
      const int kb0 = split * p.kb_per_split;
      const int kb1 = min(kb0 + p.kb_per_split, p.kb_total);
      int cw = 0, ch = 0, cn = 0;
      if (IM2COL && !MN_MAJOR) {                 // base pixel of this 128-row tile
        const int m0 = m_tile * BM;
        const int q = m0 % p.cv.OW, t3 = m0 / p.cv.OW;
        cw = q * p.cv.stride_w + p.cv.lower_w;
        ch = (t3 % p.cv.OH) * p.cv.stride_h + p.cv.lower_h;
        cn = t3 / p.cv.OH;
      }
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&empty_bar[s], ph ^ 1);
        // STAGED DACT with the bit mask: the tile's mask rows travel with its last k-block (see below)
        const bool mstage = MASK_STAGE > 0 && p.saved_bits != nullptr && kb + 1 == kb1;
        if (elect_one()) {
          uint8_t* sa = smem + s * STAGE_BYTES;
          uint8_t* sb = sa + C_::A_BYTES;
          if (!MN_MAJOR) {
            const int ntap = IM2COL ? min(TPS, p.cv.taps - kb * TPS) : TPS;
            const uint32_t tx = (uint32_t)ntap * (A_SUB + (BRES ? 0 : B_SUB));
            if (mstage) mbar_expect_tx(&full_bar[s], tx);
            else mbar_arrive_expect_tx(&full_bar[s], tx);
#pragma unroll
            for (int t = 0; t < TPS; ++t) {
              if (t < ntap) {
                const int g = kb * TPS + t;
                if (IM2COL)
                  tma_load_im2col_4d(sa + t * A_SUB, &tmA, &full_bar[s], 0, cw, ch, cn, (uint16_t)(g % p.cv.S),
                                     (uint16_t)(g / p.cv.S));
                else
                  tma_load_2d(sa + t * A_SUB, &tmA, &full_bar[s], g * CPT, m_tile * BM);
                if (!BRES) tma_load_2d(sb + t * B_SUB, &tmB, &full_bar[s], g * CPT, n_tile * BN);
              }
            }
          } else {
            int nch = MCH;
            if (IM2COL) {
              nch = min(MCH, p.cv.taps - m_tile * MCH);
              const int k0 = kb * BK;              // first pixel row of this K block
              const int q = k0 % p.cv.OW, t3 = k0 / p.cv.OW;
              cw = q * p.cv.stride_w + p.cv.lower_w;
              ch = (t3 % p.cv.OH) * p.cv.stride_h + p.cv.lower_h;
              cn = t3 / p.cv.OH;
            }
            mbar_arrive_expect_tx(&full_bar[s], (uint32_t)nch * A_CHUNK + C_::B_BYTES);
#pragma unroll
            for (int j = 0; j < MCH; ++j) {
              if (j < nch) {
                if (IM2COL) {
                  const int g = m_tile * MCH + j;
                  tma_load_im2col_4d(sa + j * A_CHUNK, &tmA, &full_bar[s], 0, cw, ch, cn, (uint16_t)(g % p.cv.S),
                                     (uint16_t)(g / p.cv.S));
                } else {
                  tma_load_2d(sa + j * A_CHUNK, &tmA, &full_bar[s], m_tile * BM + j * CPT, kb * BK);
                }
              }
            }
#pragma unroll
            for (int j = 0; j < BCHUNKS; ++j)
              tma_load_2d(sb + j * (BK * BROWB), &tmB, &full_bar[s], n_tile * BN + j * 64, kb * BK);
          }
        }
        __syncwarp();
        if (mstage) {
          // 128 rows x BN/16 words at row pitch ld_saved/16 words.  That pitch is a multiple of 2 bytes only (fc1 of
          // NatureCNN: 392 B), which no tensor map or bulk copy takes, so the warp copies the words itself after issuing
          // the stage's TMA loads, and arrives once they are in shared memory.  Rows >= M and words >= N/16 read 0.
          constexpr int WPR = BN / 16;
          uint16_t* dst = reinterpret_cast<uint16_t*>(smask + s * MASK_STAGE);
          const int m0 = m_tile * BM, w0 = n_tile * WPR, nw = p.N >> 4;
          const long long pitch = p.ld_saved >> 4;
#pragma unroll 4
          for (int i = lane; i < BM * WPR; i += 32) {
            const int r = i / WPR, j = i % WPR;
            dst[i] = (m0 + r < p.M && w0 + j < nw) ? __ldg(p.saved_bits + (long long)(m0 + r) * pitch + w0 + j)
                                                   : (uint16_t)0;
          }
          __threadfence_block();
          __syncwarp();
          if (lane == 0) mbar_arrive(&full_bar[s]);
        }
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
    }
  } else if constexpr (STAGED) {
    // ------------------------------------------------------------------ consumer warpgroups, staged epilogue
    // Ping-pong: group wg takes the CTA's tiles i = wg, wg + 2, ... whole, as two m64 accumulators (tile rows [0, 64)
    // and [64, 128)), and issues a tile's MMAs only after the other group has issued the previous tile's (order_wait /
    // order_pass), so each group's epilogue runs while the tensor cores work on the other group's tile.  Cooperative:
    // both groups take every tile, rows [64*wg, 64*wg + 64).  Thread t holds rows r0 and r0 + 8 of each accumulator.
    constexpr int MH = PINGPONG ? 2 : 1;
    const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0), t = threadIdx.x & 127;
    const int row0 = PINGPONG ? 0 : wg * 64;
    const int kbt = p.kb_total;                                      // one split: every tile runs all k-blocks
    const int tile_count =
        (int)blockIdx.x < total_work ? (total_work - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
    // After the transpose lane l holds columns 8 * (l >> 4) .. + 7 of each 16-column chunk of row er = l & 15 of the
    // warp's 16 rows; that is also the row and piece whose address lane l hands to stmatrix / ldmatrix.
    const int er = lane & 15, ep = lane >> 4;
    const int erow = row0 + 16 * (warp & 3) + er;                    // tile row of accumulator 0 after the transpose
    uint32_t epi_addr[2];
#pragma unroll
    for (int jj = 0; jj < 2; ++jj)
      epi_addr[jj] = smem_u32(sepi + warp * EPI_WARP_BYTES) + er * 64 + (((2 * jj + ep) ^ ((er >> 1) & 3)) << 4);
    const bool masked = TMODE == MODE_F16_DACT && p.saved_bits != nullptr;
    const bool has_bias = TMODE != MODE_F16_DACT && p.bias != nullptr;
    __half* Ch = reinterpret_cast<__half*>(p.C);
    float acc[MH][BN / 2];
    auto release = [&](int st) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[st]);
    };
    for (int i = PINGPONG ? wg : 0; i < tile_count; i += PINGPONG ? 2 : 1) {
      const int work = (int)blockIdx.x + i * (int)gridDim.x;
      const int n_tile = work % p.n_tiles, m_tile = work / p.n_tiles;
      const int col0 = n_tile * BN;
      if (has_bias) {                                                // the bias of the tile's columns, read once
        asm volatile("bar.sync %0, 128;" ::"r"(4 + wg) : "memory");  // the group's previous epilogue is done with it
        for (int c = t; c < BN; c += 128) s_bias[wg][c] = col0 + c < p.N ? __ldg(p.bias + col0 + c) : 0.0f;
        asm volatile("bar.sync %0, 128;" ::"r"(4 + wg) : "memory");
      }
      const long long q0 = (long long)i * kbt;                       // stage sequence number of the tile's first k-block
      int s = (int)(q0 % STAGES);
      uint32_t ph = (uint32_t)(q0 / STAGES) & 1u;
      if (PINGPONG && i > 0) order_wait(wg);                         // the other group has issued tile i - 1
      int prev = -1;
      for (int kb = 0; kb < kbt; ++kb) {
        mbar_wait(&full_bar[s], ph);
        const uint32_t st = smem_u32(smem + s * STAGE_BYTES);
        wgmma_fence();
#pragma unroll
        for (int tp = 0; tp < TPS; ++tp) {
#pragma unroll
          for (int k = 0; k < CPT / MMA_K; ++k) {
            const uint64_t bdesc = make_sdesc(st + C_::A_BYTES + tp * B_SUB + k * (MMA_K * 2), 16, 8 * ROWB, LAYOUT_A);
#pragma unroll
            for (int mh = 0; mh < MH; ++mh) {
              const uint64_t adesc =
                  make_sdesc(st + tp * A_SUB + (row0 + mh * 64) * ROWB + k * (MMA_K * 2), 16, 8 * ROWB, LAYOUT_A);
              wgmma_f16<BN, 0, 0>(acc[mh], adesc, bdesc, (kb > 0 || tp > 0 || k > 0) ? 1u : 0u);
            }
          }
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0) release(prev);
        prev = s;
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
      if (PINGPONG && i + 1 < tile_count) order_pass(wg);           // the other group may issue tile i + 1
      wgmma_wait<0>();
      if constexpr (TMODE == MODE_F32_STORE) {
        release(prev);
#pragma unroll
        for (int mh = 0; mh < MH; ++mh) {
          // fp32: lanes q and q ^ 1 of a row quad swap pairs, so that each holds 4 consecutive columns of one row
          const int q = t & 3;
          const bool odd = q & 1;
          const int orow = m_tile * BM + row0 + mh * 64 + 16 * (warp & 3) + (lane >> 2) + (odd ? 8 : 0);
          float* Cf = reinterpret_cast<float*>(p.C) + (long long)orow * p.ldc;
#pragma unroll
          for (int b = 0; b < BN / 8; ++b) {
            const int c = 8 * b + 2 * q;
            const float b0 = has_bias ? s_bias[wg][c] : 0.0f, b1 = has_bias ? s_bias[wg][c + 1] : 0.0f;
            const float f0 = fmaf(acc[mh][4 * b], p.alpha, b0), f1 = fmaf(acc[mh][4 * b + 1], p.alpha, b1);
            const float f2 = fmaf(acc[mh][4 * b + 2], p.alpha, b0), f3 = fmaf(acc[mh][4 * b + 3], p.alpha, b1);
            const float s0 = __shfl_xor_sync(0xffffffffu, odd ? f0 : f2, 1);
            const float s1 = __shfl_xor_sync(0xffffffffu, odd ? f1 : f3, 1);
            const float o[4] = {odd ? s0 : f0, odd ? s1 : f1, odd ? f2 : s0, odd ? f3 : s1};
            const int oc = col0 + 8 * b + 2 * (q & ~1);
            if (orow < p.M && oc < p.N) {
              if (p.vec16 && oc + 4 <= p.N) {
                st_global_v4(Cf + oc, make_uint4(__float_as_uint(o[0]), __float_as_uint(o[1]), __float_as_uint(o[2]),
                                                 __float_as_uint(o[3])));
              } else {
#pragma unroll
                for (int k = 0; k < 4; ++k)
                  if (oc + k < p.N) Cf[oc + k] = o[k];
              }
            }
          }
        }
      } else {
        // fp16 epilogue; the DACT mask and saved-activation variants are separate instantiations (MASKED), so that the
        // registers of one are not live in the other
        auto epi16 = [&](auto masked_c) {
        constexpr bool MASKED = decltype(masked_c)::value;
        // DACT with the bit mask: this lane's mask rows, staged with the last k-block.  The fence makes the loads
        // complete before the stage is released (an arrive alone does not wait for another lane's shared-memory load
        // in flight).
        uint32_t mrow[MH][MASKED ? (BN + 31) / 32 : 1];
        if constexpr (MASKED) {
#pragma unroll
          for (int mh = 0; mh < MH; ++mh) {
            const uint32_t r = smem_u32(smask + prev * MASK_STAGE) + (uint32_t)((erow + mh * 64) * (BN / 8));
#pragma unroll
            for (int w = 0; w < BN / 32; ++w)
              asm volatile("ld.shared.b32 %0, [%1];" : "=r"(mrow[mh][w]) : "r"(r + 4 * w));
          }
          __threadfence_block();
        }
        release(prev);
#pragma unroll
        for (int mh = 0; mh < MH; ++mh) {
          const int grow = m_tile * BM + erow + mh * 64;             // this lane's output row after the transpose
          const bool rok = grow < p.M;
#pragma unroll
          for (int ps = 0; ps < BN / 32; ++ps) {                     // passes of 32 columns = two 16-column chunks
#pragma unroll
            for (int jj = 0; jj < 2; ++jj) {
              // chunk 2 * ps + jj = 8-column blocks b, b + 1; stmatrix matrices (b, row t/4), (b, + 8), (b + 1, ...)
              const int b = 2 * (2 * ps + jj);
              // DACT with the fp16 saved activation: each lane reads its 16-byte piece of the chunk into the scratch,
              // and ldmatrix hands every thread the values of its accumulator columns
              uint32_t hs[4];
              if constexpr (TMODE == MODE_F16_DACT && !MASKED) {
                const int gc = col0 + 16 * (2 * ps + jj) + 8 * ep;
                uint4 sv = make_uint4(0u, 0u, 0u, 0u);
                if (rok && gc < p.N) {
                  const __half* sp = p.saved + (long long)grow * p.ld_saved + gc;
                  if (p.saved16 && gc + 8 <= p.N) {
                    sv = ld_nc_v4(sp);
                  } else {
                    uint32_t w[4] = {0u, 0u, 0u, 0u};
#pragma unroll
                    for (int k = 0; k < 8; ++k)
                      if (gc + k < p.N) w[k >> 1] |= (uint32_t)ld_nc_u16(sp + k) << (16 * (k & 1));
                    sv = make_uint4(w[0], w[1], w[2], w[3]);
                  }
                }
                st_shared_v4(epi_addr[jj], sv);
                __syncwarp();
                ldmatrix_x4(epi_addr[jj], hs);
                __syncwarp();
              }
              uint32_t r[4];
#pragma unroll
              for (int k = 0; k < 4; ++k) {
                const int e = 4 * (b + (k >> 1)) + 2 * (k & 1);
                const int c = 8 * (b + (k >> 1)) + 2 * (t & 3);
                // per element and in the order of the unstaged epilogue: product with alpha, then bias and activation
                // (ACT) or the activation's derivative (DACT), then one rounding to fp16
                float v0 = __fmul_rn(acc[mh][e], p.alpha), v1 = __fmul_rn(acc[mh][e + 1], p.alpha);
                if (TMODE == MODE_F16_ACT) {
                  if (has_bias) {
                    v0 = __fadd_rn(v0, s_bias[wg][c]);
                    v1 = __fadd_rn(v1, s_bias[wg][c + 1]);
                  }
                  v0 = apply_act(v0, p.act);
                  v1 = apply_act(v1, p.act);
                } else if constexpr (!MASKED) {
                  const __half2 h = *reinterpret_cast<const __half2*>(&hs[k]);
                  v0 = __fmul_rn(v0, act_grad_from_saved(__low2float(h), p.act));
                  v1 = __fmul_rn(v1, act_grad_from_saved(__high2float(h), p.act));
                }
                r[k] = h2_bits(__floats2half2_rn(v0, v1));
              }
              stmatrix_x4(epi_addr[jj], r);
            }
            __syncwarp();
#pragma unroll
            for (int jj = 0; jj < 2; ++jj) {
              const int j = 2 * ps + jj;
              uint4 v = ld_shared_v4(epi_addr[jj]);                 // columns 16 * j + 8 * ep .. + 7 of row er
              if constexpr (MASKED) {                                // zeroing the rounded value gives what rounding
                const uint32_t b8 = (mrow[mh][j >> 1] >> (16 * (j & 1) + 8 * ep)) & 0xffu;   // 0.0f gives: +0
                v.x &= mask_pair(b8, 0);
                v.y &= mask_pair(b8, 1);
                v.z &= mask_pair(b8, 2);
                v.w &= mask_pair(b8, 3);
              }
              const int gc = col0 + 16 * j + 8 * ep;
              if (rok && gc < p.N) {
                long long oc = gc;
                if (p.rm_C > 0) {              // rm_C % 16 == 0: the chunk's 16 columns lie in one pixel, in order
                  const int c16 = col0 + 16 * j, pix = c16 / p.rm_C;
                  oc = (long long)((pix / p.rm_OW) * p.rm_Wg + pix % p.rm_OW) * p.rm_C + (c16 - pix * p.rm_C) + 8 * ep;
                }
                __half* out = Ch + (long long)grow * p.ldc + oc;
                if (p.vec16 && gc + 8 <= p.N) {
                  st_global_v4(out, v);
                } else {
                  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                  for (int k = 0; k < 8; ++k)
                    if (gc + k < p.N) out[k] = __ushort_as_half((unsigned short)(w[k >> 1] >> (16 * (k & 1))));
                }
              }
            }
            __syncwarp();                                            // the scratch is rewritten by the next pass
          }
        }
        };
        if (TMODE == MODE_F16_DACT && masked) epi16(std::integral_constant<bool, TMODE == MODE_F16_DACT>{});
        else epi16(std::false_type{});
      }
    }
  } else {
    // ------------------------------------------------------------------ consumer warpgroups
    // Rows of this warpgroup in the tile: [64*wg, 64*wg + 64).  Tiles in M chunks that were not loaded (the last
    // MN-major conv tile) compute garbage rows >= M, which the epilogue drops.
    const int wg = warp >> 2;
    const int t = threadIdx.x & 127;
    const int mode = (TMODE >= 0) ? TMODE : p.mode;
    float acc[BN / 2];
    int s = 0;
    uint32_t ph = 0;
    if (ZT_BYTES > 0) {
      for (int i = threadIdx.x; i < ZT_BYTES / 16; i += CONSUMER_WARPS * 32)
        reinterpret_cast<uint4*>(zero_tile)[i] = make_uint4(0u, 0u, 0u, 0u);
      fence_proxy_async_smem();                              // generic-proxy writes -> visible to wgmma
      asm volatile("bar.sync 1, %0;" ::"n"(CONSUMER_WARPS * 32) : "memory");
    }
    if (BRES) mbar_wait(bres_bar, 0);
    for (int work = blockIdx.x; work < total_work; work += gridDim.x) {
      const int n_tile = work % p.n_tiles;
      const int t2 = work / p.n_tiles;
      const int m_tile = t2 % p.m_tiles;
      const int split = t2 / p.m_tiles;
      const int kb0 = split * p.kb_per_split;
      const int kb1 = min(kb0 + p.kb_per_split, p.kb_total);
      int prev = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[s], ph);
        const uint32_t st = smem_u32(smem + s * STAGE_BYTES);
        const uint32_t b_addr = BRES ? smem_u32(bres) + (uint32_t)(kb * TPS) * B_SUB : st + C_::A_BYTES;
        wgmma_fence();
        if (!MN_MAJOR) {
          const uint32_t a_addr = st + wg * 64 * ROWB;
          // The last stage of an implicit conv may hold fewer taps.  Its empty tap slots multiply tap 0's A tile by
          // the zero tile (adding exact zeros) instead of skipping their MMAs: a wgmma under a branch makes the
          // compiler serialise every wgmma of the kernel.
          const int ntap = IM2COL ? min(TPS, p.cv.taps - kb * TPS) : TPS;
#pragma unroll
          for (int tp = 0; tp < TPS; ++tp) {
            const bool live = tp < ntap;
            const uint32_t at = a_addr + (live ? tp * A_SUB : 0);
            const uint32_t bt = live ? b_addr + tp * B_SUB : smem_u32(zero_tile);
#pragma unroll
            for (int k = 0; k < CPT / MMA_K; ++k) {
              const uint64_t adesc = make_sdesc(at + k * (MMA_K * 2), 16, 8 * ROWB, LAYOUT_A);
              const uint64_t bdesc = make_sdesc(bt + k * (MMA_K * 2), 16, 8 * ROWB, LAYOUT_A);
              wgmma_f16<BN, 0, 0>(acc, adesc, bdesc, (kb > kb0 || tp > 0 || k > 0) ? 1u : 0u);
            }
          }
        } else {
          const uint32_t a_addr = st + wg * (64 / CPT) * A_CHUNK;
#pragma unroll
          for (int k = 0; k < BK / MMA_K; ++k) {
            const uint64_t adesc = make_sdesc(a_addr + k * (MMA_K * ROWB), A_CHUNK, 8 * ROWB, LAYOUT_A);
            const uint64_t bdesc = make_sdesc(b_addr + k * (MMA_K * BROWB), BK * BROWB, 8 * BROWB, LAYOUT_B);
            wgmma_f16<BN, 1, 1>(acc, adesc, bdesc, (kb > kb0 || k > 0) ? 1u : 0u);
          }
        }
        wgmma_commit();
        // the stage before this one is free once its MMAs retired; this stage's MMAs keep running meanwhile
        wgmma_wait<1>();
        if (prev >= 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[prev]);
        }
        prev = s;
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[prev]);

      const int row0 = m_tile * BM + wg * 64;
      const int col0 = n_tile * BN;
#pragma unroll
      for (int e = 0; e < BN / 2; e += 2) {
        const int row = row0 + acc_row(t, e), col = col0 + acc_col(t, e);
        if (row < p.M && col < p.N)
          gemm_epi_pair(p, mode, split, row, col, acc[e] * p.alpha, acc[e + 1] * p.alpha, col + 1 < p.N);
      }
    }
  }
}

// ---------------------------------------------------------------------------------- host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
typedef CUresult (*PFN_encodeIm2col)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                     const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t,
                                     const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                     CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static void* driver_fn(const char* name) {
  void* ptr = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint(name, &ptr, cudaEnableDefault, &qres);
  return (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) ? ptr : nullptr;
}

static CUtensorMapSwizzle swizzle_for(int row_bytes) {
  return row_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : row_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                                                          : CU_TENSOR_MAP_SWIZZLE_32B;
}

// 2-D fp16 tensor [rows, cols] with row pitch ld (elements); box = {box_cols (inner), box_rows}
static int make_tmap(CUtensorMap* tm, const void* ptr, long long rows, long long cols, long long ld, int box_cols,
                     int box_rows) {
  static PFN_encodeTiled enc = reinterpret_cast<PFN_encodeTiled>(driver_fn("cuTensorMapEncodeTiled"));
  if (!enc) {
    set_last_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    return B200RL_ERR_DRIVER;
  }
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstr[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), gdim, gstr, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_for(box_cols * 2), CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed (%d): rows=%lld cols=%lld ld=%lld box=%dx%d ptr=%p", (int)r, rows,
                   cols, ld, box_cols, box_rows, ptr);
    return B200RL_ERR_DRIVER;
  }
  return B200RL_OK;
}

// NHWC fp16 activation [B, H, W, C] read in im2col mode: `pixels` base pixels x C channels per load
static int make_tmap_im2col(CUtensorMap* tm, const void* ptr, long long B, int H, int W, int C, int lower_w,
                            int lower_h, int upper_w, int upper_h, int stride_w, int stride_h, int pixels) {
  static PFN_encodeIm2col enc = reinterpret_cast<PFN_encodeIm2col>(driver_fn("cuTensorMapEncodeIm2col"));
  if (!enc) {
    set_last_error("cuTensorMapEncodeIm2col entry point unavailable");
    return B200RL_ERR_DRIVER;
  }
  cuuint64_t gdim[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t gstr[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  int lo[2] = {lower_w, lower_h};
  int hi[2] = {upper_w, upper_h};
  cuuint32_t estr[4] = {1, (cuuint32_t)stride_w, (cuuint32_t)stride_h, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(ptr), gdim, gstr, lo, hi, (cuuint32_t)C,
                   (cuuint32_t)pixels, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_for(C * 2),
                   CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeIm2col failed (%d): B=%lld H=%d W=%d C=%d lo=(%d,%d) hi=(%d,%d) st=(%d,%d) px=%d",
                   (int)r, B, H, W, C, lower_w, lower_h, upper_w, upper_h, stride_w, stride_h, pixels);
    return B200RL_ERR_DRIVER;
  }
  return B200RL_OK;
}

int make_tmap_2d_f16(CUtensorMap* tm, const void* ptr, long long rows, long long cols, long long ld, int box_cols,
                     int box_rows) {
  return make_tmap(tm, ptr, rows, cols, ld, box_cols, box_rows);
}

static int g_num_sms = 0;
int device_num_sms();
static int num_sms() { return device_num_sms(); }
int device_num_sms() {
  if (g_num_sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_num_sms <= 0) g_num_sms = 132;
  }
  return g_num_sms;
}

// One buffer per device.  It is not keyed by stream: a CUDA-graph capture runs on a side stream of its own and must
// reuse the buffer its eager first pass sized (it cannot allocate).  Uses stay ordered because every reduction is issued
// on the caller's current stream and the training path keeps one stream (graph replays run on it too).
struct DetBuf {
  float* ptr;
  size_t floats;
};
static std::map<int, DetBuf> g_det_ws;
static std::mutex g_det_mu;

float* det_workspace(size_t floats, cudaStream_t stream) {
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> lock(g_det_mu);
  DetBuf& b = g_det_ws[dev];
  if (b.ptr && b.floats >= floats) return b.ptr;
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(stream, &cap);
  if (cap != cudaStreamCaptureStatusNone) {
    set_last_error("det_workspace: %zu floats needed while capturing a graph (run the sequence eagerly once first)",
                   floats);
    return nullptr;
  }
  const size_t grow = floats + floats / 4 + (1u << 18);
  float* buf = nullptr;
  cudaError_t e = cudaMalloc(&buf, grow * sizeof(float));
  if (e != cudaSuccess) {
    set_last_error("det_workspace: cudaMalloc(%zu B): %s", grow * sizeof(float), cudaGetErrorString(e));
    return nullptr;
  }
  b.ptr = buf;                         // the previous buffer stays allocated: captured graphs may still use it
  b.floats = grow;
  return buf;
}

// 32 consecutive elements per block; warp w sums parts w, w + 8, ... in order, then lane sums the 8 warp totals in
// order: a fixed association for any number of parts, with 8 loads in flight per element
__global__ void __launch_bounds__(256)
sum_partials_kernel(const float* __restrict__ ws, int parts, long long rows, int cols, float* __restrict__ out,
                    long long ldo) {
  __shared__ float red[8][32];
  const long long n = rows * cols;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (long long i0 = (long long)blockIdx.x * 32; i0 < n; i0 += (long long)gridDim.x * 32) {
    const long long i = i0 + lane;
    float s = 0.0f;
    if (i < n)
      for (int q = w; q < parts; q += 8) s += ws[(long long)q * n + i];
    red[w][lane] = s;
    __syncthreads();
    if (w == 0 && i < n) {
      float t = 0.0f;
#pragma unroll
      for (int k = 0; k < 8; ++k) t += red[k][lane];
      const long long r = i / cols;
      out[r * ldo + (i - r * cols)] += t;
    }
    __syncthreads();
  }
}

int sum_partials(const float* ws, int parts, long long rows, int cols, float* out, long long ldo, cudaStream_t stream) {
  const long long n = rows * cols;
  long long blocks = (n + 31) / 32;
  if (blocks > 16LL * num_sms()) blocks = 16LL * num_sms();
  sum_partials_kernel<<<(int)blocks, 256, 0, stream>>>(ws, parts, rows, cols, out, ldo);
  return check_launch("sum_partials_kernel");
}

template <int BN, int CPT, bool MN, bool IM2COL, bool BRES = false, int TMODE = -1>
static int launch(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, int max_ctas,
                  cudaStream_t stream) {
  using C_ = Cfg<BN>;
  constexpr int ZT = (IM2COL && !MN) ? BN * CPT * 2 : 0;    // zero weight tile of the implicit conv
  constexpr int SMEM = (BRES ? (BRES_STAGES * C_::A_BYTES + BRES_B_BYTES + 1024 + 256) : C_::SMEM_BYTES) + ZT +
                       (staged_epi(MN, IM2COL, TMODE) ? staged_smem_bytes<BN, TMODE>() : 0);
  static_assert(SMEM <= 227 * 1024, "gemm: shared memory budget");
  static bool attr_set = false;
  auto kern = gemm_wgmma_kernel<BN, CPT, MN, IM2COL, BRES, TMODE>;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    if (e != cudaSuccess) {
      set_last_error("cudaFuncSetAttribute(smem=%d): %s", SMEM, cudaGetErrorString(e));
      return B200RL_ERR_CUDA;
    }
    attr_set = true;
  }
  const int total = p.m_tiles * p.n_tiles * p.splits;
  int grid = total < num_sms() ? total : num_sms();
  if (max_ctas > 0 && grid > max_ctas) grid = max_ctas;
  kern<<<grid, NUM_THREADS, SMEM, stream>>>(tmA, tmB, p);
  return check_launch("gemm_wgmma_kernel");
}

static void fill_splits(GemmParams& p, int split_k) {
  int splits = split_k < 1 ? 1 : split_k;
  if (splits > p.kb_total) splits = p.kb_total;
  p.kb_per_split = ceil_div(p.kb_total, splits);
  p.splits = ceil_div(p.kb_total, p.kb_per_split);
}

static int gemm_dispatch(int BN, int mn_major, int mode, const CUtensorMap& tmA, const CUtensorMap& tmB,
                         const GemmParams& p, int max_ctas, cudaStream_t stream) {
  if (mn_major) {
    B200RL_REQUIRE(mode == MODE_F32_ATOMIC, "gemm: the MN-major (wgrad) layout uses the fp32 atomic epilogue");
    if (BN == 64) return launch<64, 64, true, false, false, MODE_F32_ATOMIC>(tmA, tmB, p, max_ctas, stream);
    if (BN == 256) return launch<256, 64, true, false, false, MODE_F32_ATOMIC>(tmA, tmB, p, max_ctas, stream);
    return launch<128, 64, true, false, false, MODE_F32_ATOMIC>(tmA, tmB, p, max_ctas, stream);
  }
#define GEMM_KMAJOR(bn)                                                                                         \
  switch (mode) {                                                                                               \
    case MODE_F16_ACT: return launch<bn, 64, false, false, false, MODE_F16_ACT>(tmA, tmB, p, max_ctas, stream);   \
    case MODE_F32_STORE: return launch<bn, 64, false, false, false, MODE_F32_STORE>(tmA, tmB, p, max_ctas, stream); \
    case MODE_F16_DACT: return launch<bn, 64, false, false, false, MODE_F16_DACT>(tmA, tmB, p, max_ctas, stream);  \
    default: return launch<bn, 64, false, false, false, MODE_F32_ATOMIC>(tmA, tmB, p, max_ctas, stream);          \
  }
  switch (BN) {
    case 32: GEMM_KMAJOR(32)
    case 64: GEMM_KMAJOR(64)
    case 128: GEMM_KMAJOR(128)
    default: GEMM_KMAJOR(256)
  }
#undef GEMM_KMAJOR
}

template <int CPT, bool MN>
static int launch_conv(int BN, bool bres, const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p,
                       cudaStream_t st) {
  if (MN) {
    switch (BN) {
      case 32: return launch<32, CPT, MN, true>(tmA, tmB, p, 0, st);
      case 64: return launch<64, CPT, MN, true>(tmA, tmB, p, 0, st);
      case 128: return launch<128, CPT, MN, true>(tmA, tmB, p, 0, st);
      default: break;
    }
  } else if (bres) {
    switch (BN) {
      case 32: return launch<32, CPT, false, true, !MN>(tmA, tmB, p, 0, st);
      case 64: return launch<64, CPT, false, true, !MN>(tmA, tmB, p, 0, st);
      case 128: return launch<128, CPT, false, true, !MN>(tmA, tmB, p, 0, st);
      default: break;
    }
  } else {
    switch (BN) {
      case 32: return launch<32, CPT, false, true>(tmA, tmB, p, 0, st);
      case 64: return launch<64, CPT, false, true>(tmA, tmB, p, 0, st);
      case 128: return launch<128, CPT, false, true>(tmA, tmB, p, 0, st);
      default: break;
    }
  }
  set_last_error("conv_gemm: unsupported tile N=%d", BN);
  return B200RL_ERR_UNSUPPORTED;
}

}  // namespace b200rl

using namespace b200rl;

extern "C" int b200rl_gemm_f16(const void* A, const void* B, void* C, const float* bias, const void* saved, int M,
                               int N, int K, long long lda, long long ldb, long long ldc, long long ld_saved,
                               int mn_major, int mode, int act, float alpha, int split_k, int max_ctas, int rm_C,
                               int rm_OW, int rm_Wg, const void* saved_bits, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(A && B && C, "gemm: null operand");
  B200RL_REQUIRE(rm_C == 0 || (rm_C % 16 == 0 && rm_OW > 0 && rm_Wg >= rm_OW && (mode == MODE_F16_ACT || mode == MODE_F16_DACT)),
                 "gemm: bad column remap");
  B200RL_REQUIRE(M > 0 && N > 0 && K > 0, "gemm: bad shape M=%d N=%d K=%d", M, N, K);
  B200RL_REQUIRE((lda % 8) == 0 && (ldb % 8) == 0, "gemm: lda/ldb must be multiples of 8 fp16 (16 B): %lld %lld", lda,
                 ldb);
  B200RL_REQUIRE((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(B) & 15) == 0,
                 "gemm: operands must be 16-byte aligned");
  B200RL_REQUIRE(mode >= 0 && mode <= 3, "gemm: bad mode %d", mode);
  B200RL_REQUIRE(mode != MODE_F16_DACT || saved != nullptr || saved_bits != nullptr,
                 "gemm: MODE_F16_DACT needs the saved activation (or its bit mask)");
  B200RL_REQUIRE(saved_bits == nullptr || (mode == MODE_F16_DACT && act == ACT_RELU && (ld_saved % 16) == 0 && (N % 16) == 0),
                 "gemm: saved_bits is a ReLU mask for MODE_F16_DACT with ld_saved and N multiples of 16");

  int BN;
  // a 256-wide N tile stages each A tile once per 256 output columns instead of per 128
  if (mn_major) BN = (N > 128 && N % 256 == 0) ? 256 : (N > 64) ? 128 : 64;
  else BN = (N > 128 && (N % 256 == 0)) ? 256 : (N > 64) ? 128 : (N > 32) ? 64 : 32;

  GemmParams p = {};
  p.M = M; p.N = N; p.K = K;
  p.m_tiles = ceil_div(M, BM);
  p.n_tiles = ceil_div(N, BN);
  p.kb_total = ceil_div(K, BK);
  B200RL_REQUIRE(split_k <= 1 || mode == MODE_F32_ATOMIC, "gemm: split_k needs the fp32 atomic epilogue");
  fill_splits(p, split_k);
  p.C = C; p.ldc = ldc; p.bias = bias; p.saved = reinterpret_cast<const __half*>(saved); p.ld_saved = ld_saved;
  p.saved_bits = reinterpret_cast<const uint16_t*>(saved_bits);
  p.alpha = alpha; p.mode = mode; p.act = act;
  p.rm_C = rm_C; p.rm_OW = rm_OW; p.rm_Wg = rm_Wg;
  p.vec32 = ((ldc & 15) == 0) && ((reinterpret_cast<uintptr_t>(C) & 31) == 0) && (rm_C == 0 || (rm_C & 15) == 0) &&
            (!saved || (((ld_saved & 15) == 0) && ((reinterpret_cast<uintptr_t>(saved) & 31) == 0)));
  B200RL_REQUIRE(saved_bits == nullptr || p.vec32, "gemm: saved_bits needs 32-byte aligned 16-column output chunks");
  p.vec16 = ((reinterpret_cast<uintptr_t>(C) & 15) == 0) && (ldc % (mode == MODE_F32_STORE ? 4 : 8)) == 0;
  p.saved16 = saved && ((reinterpret_cast<uintptr_t>(saved) & 15) == 0) && (ld_saved % 8) == 0;

  CUtensorMap tmA, tmB;
  int rc;
  if (!mn_major) {
    if ((rc = make_tmap(&tmA, A, M, K, lda, BK, BM)) != 0) return rc;
    if ((rc = make_tmap(&tmB, B, N, K, ldb, BK, BN)) != 0) return rc;
  } else {
    if ((rc = make_tmap(&tmA, A, K, M, lda, 64, BK)) != 0) return rc;
    if ((rc = make_tmap(&tmB, B, K, N, ldb, 64, BK)) != 0) return rc;
  }
  if (mode == MODE_F32_ATOMIC && p.splits > 1) {
    if ((p.ws = det_workspace((size_t)p.splits * M * N, stream)) == nullptr) return B200RL_ERR_CUDA;
  }
  rc = gemm_dispatch(BN, mn_major, mode, tmA, tmB, p, max_ctas, stream);
  if (rc == B200RL_OK && p.ws) rc = sum_partials(p.ws, p.splits, M, N, reinterpret_cast<float*>(C), ldc, stream);
  return rc;
}

// Implicit-GEMM convolution on an NHWC fp16 tensor x[B, H, W, C] whose filter window is described by
// (R x S taps, stride, lower padding).  kind: 0 = forward / dgrad-style (rows = base pixels, K = taps*C,
// Wt = [N, taps*C] K-major), 1 = wgrad (out[taps*C, N] += x_patches^T * dz, dz = [B*OH*OW, N]).
extern "C" int b200rl_conv_gemm(const void* x, long long B, int H, int W, int C, int R, int S, int stride_h,
                                int stride_w, int pad_h, int pad_w, int OH, int OW, const void* Wt_or_dz, long long ldb,
                                void* out, long long ldc, const float* bias, const void* saved, long long ld_saved,
                                int N, int kind, int mode, int act, float alpha, int split_k, int sh_H, int sh_W,
                                int sh_C, int sh_s, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE(x && Wt_or_dz && out && B > 0, "conv_gemm: null operand");
  B200RL_REQUIRE(C == 16 || C == 32 || C == 64, "conv_gemm: channels per tap must be 16, 32 or 64 (got %d)", C);
  B200RL_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (ldb % 8) == 0, "conv_gemm: alignment");
  B200RL_REQUIRE(kind == 0 || kind == 1, "conv_gemm: bad kind");
  const int taps = R * S;
  const long long rows = B * OH * OW;
  B200RL_REQUIRE(rows < (1LL << 31), "conv_gemm: too many rows");
  // bounding box of base pixels: lower = -pad, upper chosen so that exactly OW x OH base pixels exist:
  //   OW = (W + upper_w - lower_w - 1) / stride_w + 1   (cute::make_im2col_tma_copy_desc convention)
  const int lower_w = -pad_w, lower_h = -pad_h;
  const int upper_w = (OW - 1) * stride_w + 1 + lower_w - W;
  const int upper_h = (OH - 1) * stride_h + 1 + lower_h - H;

  GemmParams p = {};
  p.C = out; p.ldc = ldc; p.bias = bias; p.saved = reinterpret_cast<const __half*>(saved); p.ld_saved = ld_saved;
  p.alpha = alpha; p.mode = mode; p.act = act;
  p.cv.OW = OW; p.cv.OH = OH; p.cv.stride_w = stride_w; p.cv.stride_h = stride_h;
  p.cv.lower_w = lower_w; p.cv.lower_h = lower_h; p.cv.S = S; p.cv.taps = taps;
  p.sh.H = sh_H; p.sh.W = sh_W; p.sh.C = sh_C; p.sh.s = sh_s;
  p.vec32 = ((ldc & 15) == 0) && ((reinterpret_cast<uintptr_t>(out) & 31) == 0) &&
            (!saved || (((ld_saved & 15) == 0) && ((reinterpret_cast<uintptr_t>(saved) & 31) == 0)));
  if (mode == MODE_F16_SHUFFLE)
    B200RL_REQUIRE((sh_C & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 31) == 0 &&
                       (!saved || (reinterpret_cast<uintptr_t>(saved) & 31) == 0),
                   "conv_gemm: shuffle epilogue needs C %% 16 == 0 and 32-byte aligned tensors");
  CUtensorMap tmA, tmB;
  int rc;
  if (kind == 0) {
    B200RL_REQUIRE(mode == MODE_F16_ACT || mode == MODE_F16_DACT || mode == MODE_F16_SHUFFLE, "conv_gemm: bad mode");
    B200RL_REQUIRE(mode != MODE_F16_SHUFFLE || (sh_C % 16 == 0 && sh_s >= 1 && N == sh_s * sh_s * sh_C),
                   "conv_gemm: shuffle epilogue needs N == s*s*C and C %% 16 == 0");
    const int BN = (N > 64) ? 128 : (N > 32) ? 64 : 32;
    p.M = (int)rows; p.N = N; p.K = taps * C;
    p.m_tiles = ceil_div(p.M, BM);
    p.n_tiles = ceil_div(N, BN);
    p.kb_total = ceil_div(taps, BK / C);
    fill_splits(p, 1);
    if ((rc = make_tmap_im2col(&tmA, x, B, H, W, C, lower_w, lower_h, upper_w, upper_h, stride_w, stride_h, BM)) != 0)
      return rc;
    if ((rc = make_tmap(&tmB, Wt_or_dz, N, (long long)taps * C, ldb, C, BN)) != 0) return rc;
    // weights resident in smem when the whole [N, taps*C] matrix fits next to the A ring
    const bool bres = (p.n_tiles == 1) && ((long long)taps * BN * C * 2 <= BRES_B_BYTES) && (split_k != -1);
    if (C == 64) return launch_conv<64, false>(BN, bres, tmA, tmB, p, stream);
    if (C == 32) return launch_conv<32, false>(BN, bres, tmA, tmB, p, stream);
    return launch_conv<16, false>(BN, bres, tmA, tmB, p, stream);
  }
  B200RL_REQUIRE(mode == MODE_F32_ATOMIC, "conv_gemm: wgrad needs the fp32 atomic epilogue");
  const int BN = (N > 64) ? 128 : (N > 32) ? 64 : 32;
  p.M = taps * C; p.N = N; p.K = (int)rows;
  p.m_tiles = ceil_div(p.M, BM);
  p.n_tiles = ceil_div(N, BN);
  p.kb_total = ceil_div(p.K, BK);
  fill_splits(p, split_k);
  if ((rc = make_tmap_im2col(&tmA, x, B, H, W, C, lower_w, lower_h, upper_w, upper_h, stride_w, stride_h, BK)) != 0)
    return rc;
  if ((rc = make_tmap(&tmB, Wt_or_dz, rows, N, ldb, BN < 64 ? BN : 64, BK)) != 0) return rc;
  if (p.splits > 1) {
    if ((p.ws = det_workspace((size_t)p.splits * p.M * p.N, stream)) == nullptr) return B200RL_ERR_CUDA;
  }
  rc = (C == 64) ? launch_conv<64, true>(BN, false, tmA, tmB, p, stream)
     : (C == 32) ? launch_conv<32, true>(BN, false, tmA, tmB, p, stream)
                 : launch_conv<16, true>(BN, false, tmA, tmB, p, stream);
  if (rc == B200RL_OK && p.ws) rc = sum_partials(p.ws, p.splits, p.M, p.N, reinterpret_cast<float*>(out), ldc, stream);
  return rc;
}
