// "Shift-GEMM" convolutions for sm_90a: stride-1 convolutions over an NHWC fp16 activation viewed as a plain
// 2-D matrix X[rows = (n, y, x) grid positions, C] (strided convs are brought to this form by space-to-depth).
//
// Every input row is loaded into shared memory ONCE per tile by a tiled 2-D TMA; each filter tap (r, s) is then
// just the same smem buffer read through a wgmma descriptor whose start address is shifted by (r*Wg + s) rows
// (a SWIZZLE_128B descriptor may start at any 128-byte row: the swizzle is a function of the smem address).
// This removes the R*S-fold duplication of an im2col operand on the L2->SM path.
//
//   conv_shift_fwd_kernel   (K-major):  OUT[m, :] = act( sum_t X[m + sh_t, :] * W_t^T + b )          forward
//                                       and, with negative shifts over a zero-bordered dY, the data gradient
//                                       dX[m, :] = ( sum_t dY[m - sh_t, :] * W_t ) * (saved activation > 0)
//   conv_shift_wgrad_kernel (MN-major): G[t, c, n] += alpha * sum_m X[m + sh_t, c] * dY[m, n]         wgrad
//                                       (G's 64-row chunks, tap x 64 channels, are dealt evenly to the warpgroups of
//                                        a row range, at most QW each, and accumulate in registers; where clusters
//                                        tile the SMs, the CTAs of one row range form a cluster and share each X / dY
//                                        stage by TMA multicast)
//
// Warp roles: warps 0-7 are two consumer warpgroups (they issue the wgmma.mma_async chains, and run the epilogue --
// or, in the wgrad, the fused bias-gradient sums -- from their own registers) | warp 8 TMA loads | uint8-fed first
// layer only: warps 9-16 are uint8 producers that cast raw frames into a rolling A ring instead of the TMA.  The
// forward epilogue can also write 1 bit per output element (act > 0); the dgrad of the next layer reads that as its
// ReLU mask, which the TMA warp stages with each A tile (one bulk copy of the tile's 128 mask rows on the stage's full
// barrier), so the epilogue reads it from shared memory.
//
// Epilogue: bias / ReLU / alpha (or the mask) are applied to the fp32 accumulators and rounded to fp16 in registers;
// each warp then moves its 16-row fragment through a small shared scratch (stmatrix) so that every lane holds 8
// consecutive columns of one row, and the tile leaves as 16-byte stores (the ReLU bits as one 16-bit word per two lanes).
//
// "Ping-pong" schedule of the forward / dgrad: the two consumer warpgroups take whole 128-row tiles (even / odd) and
// turns on the tensor cores.  Named barriers 2 and 3 order their MMA issue: a group issues its next tile only after
// the other group has issued the previous one.  The tiles' MMAs therefore retire in order, and each group's epilogue
// runs while the tensor cores work on the other group's tile.  (Cooperative schedule, where ping-pong does not pay:
// each group takes 64 rows of every tile.)
//
// Outputs at grid positions that are not valid conv outputs are computed from wrapped rows and discarded (fwd),
// or multiply a zero of the zero-bordered dY (wgrad / dgrad) -- so dY tensors live on the conv's INPUT grid.
// Replaces tf.nn.conv2d (a2c/utils.py:56) and its gradients (ppo2/model.py:102) of the reference.
#include <stdlib.h>

#include <type_traits>

#include "common.cuh"
#include "tc_common.cuh"

namespace b200rl {

static constexpr int SH_BM = 128;
static constexpr int SH_CONSUMER_WARPS = 8;        // two warpgroups, 64 tile rows each
static constexpr int SH_TMA_WARP = SH_CONSUMER_WARPS;
__host__ __device__ constexpr int sh_threads(bool u8) { return (SH_CONSUMER_WARPS + 1) * 32 + (u8 ? 256 : 0); }
static constexpr int SH_MAX_TAPS = 16;
// rows of one TMA-fed A stage: 128 + the largest shift span.  64-channel inputs: span <= 32.  128-channel inputs (two
// halves per stage): span <= 16, so that four stages fit beside the weights.
__host__ __device__ constexpr int sh_arows(int KH) { return KH == 1 ? 160 : 144; }
__host__ __device__ constexpr int sh_stages(int KH) { return KH == 1 ? 6 : 4; }
// uint8-fed first layer: its weights (N = 32, <= 4 taps) need 16 KB, so the rolling ring takes 12 tiles.  Both consumer
// groups hold a tile (+ the next tile's head unit) under ping-pong; the deeper ring keeps the producer warps' loads
// running ahead of them.
static constexpr int SH_U8_STAGES = 12;
static constexpr int SH_U8_WRES_BYTES = 16 * 1024;
__host__ __device__ constexpr int sh_wgrad_krows(bool u8) { return u8 ? 128 : 64; }   // wgrad: reduction rows per stage
// resident-weight region of the forward kernel (all taps): 80 KB beside 64-channel stages, 64 KB beside 128-channel
// ones, 16 KB beside the uint8 ring
__host__ __device__ constexpr int sh_wres_bytes(int KH, bool u8) {
  return u8 ? SH_U8_WRES_BYTES : KH == 1 ? 80 * 1024 : 64 * 1024;
}
static constexpr int SH_BAR_BYTES = 512;             // forward kernel: mbarrier block after the weights
// forward / dgrad kernel, after the barriers: the staged ReLU mask of each A stage (DACT: 128 rows x BN bits), then one
// 16-row x 32-column fp16 epilogue scratch per consumer warp
__host__ __device__ constexpr int sh_mask_stage_bytes(int BN, bool DACT) { return DACT ? SH_BM * BN / 8 : 0; }
static constexpr int SH_EPI_WARP_BYTES = 16 * 64;
static constexpr int SH_EPI_BYTES = SH_CONSUMER_WARPS * SH_EPI_WARP_BYTES;
static constexpr int SH_WROWS_K = 96;                // wgrad: 64 + max shift span (<= 32)
static constexpr int SH_WABYTES = SH_WROWS_K * 128;
// wgrad: at most QW 64-channel accumulator chunks per consumer warpgroup (QW * N/2 accumulator registers per thread).
// N = 64 over 64 channels: QW = 3, so that a 3x3 conv's 9 chunks fit one 2-CTA cluster and X / dY are read once.
__host__ __device__ constexpr int sh_wgrad_qw(int BN, int KH, bool u8) { return u8 ? 2 : BN == 32 ? 4 : KH == 1 ? 3 : 2; }

// address map of an output / saved tensor: grid position (n, y, x) + column -> element offset
struct AddrMap {
  int mode;              // 0: n*sN + y*sY + x*sX + col
                         // 1: depth->space: cls = col/Cq: (s*y + cls/s, s*x + cls%s, col%Cq)
                         // 2: space->depth: (y/s, x/s, ((y%s)*s + x%s)*Cq + col)
  long long sN, sY, sX;
  int Cq, s;             // powers of two for modes 1 / 2
  int Cq_log2, s_log2;
};

// part of the address that does not depend on the column
__device__ __forceinline__ long long map_rowbase(const AddrMap& a, int n, int y, int x) {
  if (a.mode == 2) {
    const int sm = a.s - 1;
    return (long long)n * a.sN + (long long)(y >> a.s_log2) * a.sY + (long long)(x >> a.s_log2) * a.sX +
           ((((y & sm) << a.s_log2) + (x & sm)) << a.Cq_log2);
  }
  if (a.mode == 1) return (long long)n * a.sN + ((long long)y << a.s_log2) * a.sY + ((long long)x << a.s_log2) * a.sX;
  return (long long)n * a.sN + (long long)y * a.sY + (long long)x * a.sX;
}
// column-dependent part (col is a multiple of 16, so a 16-column chunk never straddles a class)
__device__ __forceinline__ long long map_coloff(const AddrMap& a, int col) {
  if (a.mode == 1) {
    const int cls = col >> a.Cq_log2;
    return (long long)(cls >> a.s_log2) * a.sY + (long long)(cls & (a.s - 1)) * a.sX + (col & (a.Cq - 1));
  }
  return col;
}

// Optional fused source for the FIRST conv layer: uint8 NHWC images gathered through src_idx.  Producer warps
// build the space-to-depth fp16 A tile directly in shared memory (tf.cast of models.py:19 and arr[mbinds] of
// ppo2.py:165 fused into the first load): grid row (n, Y, X) = 64 channels (dy, dx, c) = s segments of s*C bytes.
// n / d for n < 2^31, d >= 2 without the ~25-instruction runtime division: q = umulhi(n, mul) >> sh with
// mul = floor(2^(31+s) / d) + 1, s = ceil(log2 d), sh = s - 1 (error term n*e / (d*2^(31+s)) < 1/d since e <= d <= 2^s).
struct FastDiv {
  uint32_t mul, sh, d;
  __device__ __forceinline__ uint32_t div(uint32_t n) const { return __umulhi(n, mul) >> sh; }
};
static FastDiv make_fastdiv(uint32_t d) {
  FastDiv f;
  f.d = d;
  uint32_t s = 0;
  while ((1ull << s) < d) ++s;
  if (s == 0) s = 1;                                   // d == 1: mul = 2^31 + 1 does not fit; callers require d >= 2
  f.mul = (uint32_t)(((1ull << (31 + s)) / d) + 1);
  f.sh = s - 1;
  return f;
}

struct U8Src {
  const uint8_t* x;        // nullptr: A tiles come from the fp16 matrix through TMA
  const long long* idx;    // sample gather (may be null)
  long long sample_bytes;  // H*W*C
  int row_bytes;           // W*C: distance between the s segments (dy) of one grid row
  int y_bytes, x_bytes;    // s*W*C, s*C
  FastDiv per, wg;         // grid rows per sample (Hg*Wg), Wg
};

static constexpr int U8_WARPS = 8;

// 16 uint8 -> 16 fp16 (exact): bytes are spliced into 0x64xx (= 1024 + b) and 1024 is subtracted
__device__ __forceinline__ void u8x16_to_f16(const uint4& q, uint4& lo, uint4& hi) {
  const uint32_t w[4] = {q.x, q.y, q.z, q.w};
  uint32_t o[8];
  const __half2 k1024 = __floats2half2_rn(1024.0f, 1024.0f);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint32_t a = __byte_perm(w[i], 0x64646464u, 0x5140);
    const uint32_t b = __byte_perm(w[i], 0x64646464u, 0x5342);
    const __half2 ha = __hsub2(*reinterpret_cast<const __half2*>(&a), k1024);
    const __half2 hb = __hsub2(*reinterpret_cast<const __half2*>(&b), k1024);
    o[2 * i] = *reinterpret_cast<const uint32_t*>(&ha);
    o[2 * i + 1] = *reinterpret_cast<const uint32_t*>(&hb);
  }
  lo = make_uint4(o[0], o[1], o[2], o[3]);
  hi = make_uint4(o[4], o[5], o[6], o[7]);
}

// Rolling A ring of the uint8-fed kernels.  A CTA's tiles are CONSECUTIVE in grid rows, so the rows tile i reads
// through its shifted descriptors past its own TR rows are simply the first rows of tile i+1: the producer warps cast
// every input row exactly once into a circular buffer of STAGES tiles (TR rows of 128 B each, 128B-swizzled by
// absolute shared-memory address) instead of re-building a halo per tile.  The buffer ends with one extra 32-row
// unit that mirrors the first unit of stage 0, so the tile in the last stage can read past the end.
//
// The raw bytes go global -> registers -> cast -> one swizzled store: no staging copy in shared memory (the port is
// shared with the tensor core's operand fetch), and no 25-50 % of halo rows cast twice.
//
// Work unit = 32 consecutive grid rows (one warp, lane = row); unit u of the CTA covers rows row_start + 32u ...,
// belongs to tile u / UPT, and the units are dealt round-robin to the U8_WARPS producer warps.  Each warp keeps
// D units of loads in flight in registers (the sample index of the gather is looked up one round earlier).
// Barriers per stage: full (UPT unit arrivals [+ the TMA of the other operand]), head (the first unit alone: the
// tile in the PREVIOUS stage waits for it), empty (8 consumer warp arrivals: a stage may be refilled only once its own
// tile AND the tile of the previous stage, which read its first unit, have retired -- see the kernels).

__device__ __forceinline__ uint4 ldg_stream_v4(const void* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}

template <int TR, int STAGES>
struct U8Ring {
  static constexpr int UPT = TR / 32;                    // units per tile
  static constexpr int ROWS = STAGES * TR + 32;          // + the mirror unit
  static constexpr int BYTES = ROWS * 128;
  static_assert(TR % 32 == 0 && BYTES % 1024 == 0, "ring keeps the 1024 B swizzle atoms aligned");
};

// sample slot of this lane's row of `unit` (-1: outside the matrix -> zeros)
__device__ __forceinline__ long long u8_lookup(const U8Src& u, long long row_start, int unit, int total, long long M,
                                               int lane) {
  const long long m = row_start + (long long)unit * 32 + lane;
  if (unit >= total || m < 0 || m >= M) return -1;
  const uint32_t n = u.per.div((uint32_t)m);
  return u.idx ? __ldg(u.idx + n) : (long long)n;
}
// the s segments (dy) of s*C = 16 bytes of this lane's grid row
__device__ __forceinline__ void u8_load(const U8Src& u, long long row_start, int unit, long long sb, int lane,
                                        uint4 (&q)[4]) {
  if (sb >= 0) {
    const uint32_t mm = (uint32_t)(row_start + (long long)unit * 32 + lane);
    const uint32_t rem = mm - u.per.div(mm) * u.per.d;
    const uint32_t Y = u.wg.div(rem), X = rem - Y * u.wg.d;
    const uint8_t* src = u.x + sb * u.sample_bytes + (long long)(Y * (uint32_t)u.y_bytes + X * (uint32_t)u.x_bytes);
#pragma unroll
    for (int dy = 0; dy < 4; ++dy) q[dy] = ldg_stream_v4(src + (long long)dy * u.row_bytes);
  } else {
#pragma unroll
    for (int dy = 0; dy < 4; ++dy) q[dy] = make_uint4(0u, 0u, 0u, 0u);
  }
}

template <int TR, int STAGES, int D>
__device__ __forceinline__ void u8_ring_producer(const U8Src& u, long long M, long long row_start, int ntiles,
                                                 uint8_t* ring, uint64_t* full_bar, uint64_t* head_bar,
                                                 uint64_t* empty_bar, int pw, int lane) {
  using R = U8Ring<TR, STAGES>;
  constexpr int UPT = R::UPT, RND = U8_WARPS * D;
  if (ntiles <= 0) return;
  const int total = ntiles * UPT + 1;                    // + the head unit the last tile reads into
  // row_sw = address of this lane's row of unit 0 of stage 0, + ((lane & 7) << 4): chunk c of a row lives at row_sw ^ (c << 4)
  const uint32_t ring0 = smem_u32(ring) + lane * 128 + ((lane & 7) << 4);
  uint4 q[D][4];
  long long sb[D];
#pragma unroll
  for (int d = 0; d < D; ++d) sb[d] = u8_lookup(u, row_start, pw + U8_WARPS * d, total, M, lane);
#pragma unroll
  for (int d = 0; d < D; ++d) {
    u8_load(u, row_start, pw + U8_WARPS * d, sb[d], lane, q[d]);
    sb[d] = u8_lookup(u, row_start, pw + U8_WARPS * d + RND, total, M, lane);
  }
  for (int base = pw; base < total; base += RND) {
#pragma unroll
    for (int d = 0; d < D; ++d) {
      const int uc = base + U8_WARPS * d;
      if (uc < total) {                                  // warp-uniform
        const int tile = uc / UPT, ub = uc - tile * UPT;
        const int s = tile % STAGES;
        const uint32_t fill = (uint32_t)(tile / STAGES);
        mbar_wait(&empty_bar[s], (fill & 1u) ^ 1u);
        const uint32_t dst = ring0 + (uint32_t)(s * TR + ub * 32) * 128u;
        const bool mirror = (s == 0) && (ub == 0);
#pragma unroll
        for (int dy = 0; dy < 4; ++dy) {
          uint4 lo, hi;
          u8x16_to_f16(q[d][dy], lo, hi);
          st_shared_v4(dst ^ (uint32_t)((2 * dy) << 4), lo);
          st_shared_v4(dst ^ (uint32_t)((2 * dy + 1) << 4), hi);
          if (mirror) {
            st_shared_v4((dst + (uint32_t)(STAGES * TR) * 128u) ^ (uint32_t)((2 * dy) << 4), lo);
            st_shared_v4((dst + (uint32_t)(STAGES * TR) * 128u) ^ (uint32_t)((2 * dy + 1) << 4), hi);
          }
        }
        fence_proxy_async_smem();                        // generic-proxy writes -> visible to wgmma
        __syncwarp();
        if (lane == 0) {
          if (tile < ntiles) mbar_arrive(&full_bar[s]);
          if (ub == 0) mbar_arrive(&head_bar[s]);
        }
        u8_load(u, row_start, uc + RND, sb[d], lane, q[d]);
        sb[d] = u8_lookup(u, row_start, uc + 2 * RND, total, M, lane);
      }
    }
  }
}

struct ShiftParams {
  U8Src u8;
  FastDiv fwg, fhg;        // epilogue row -> (n, y, x)
  long long M;             // grid rows = B*Hg*Wg
  int Hg, Wg;              // grid
  int N;                   // output channels of the conv
  int taps;
  int shift[SH_MAX_TAPS];  // row shift of tap t, relative to min_shift (>= 0)
  int min_shift;           // smallest absolute shift (negative for dgrad)
  int vy, vx;              // rows with y < vy && x < vx produce an output
  __half* out;
  AddrMap omap;
  uint16_t* bits_out;           // optional (forward): bit k of word e/16 = (out element e + k) > 0, e = element offset
  const uint16_t* saved_bits;   // optional (DACT): the same bit array of the saved activation (ReLU mask), rows of
                                // N bits at m * N (row-contiguous), 16-byte aligned
  const float* bias;
  int act, dact;           // dact = 1: multiply by the saved_bits mask (if any) instead of applying act
  float alpha;
  int num_tiles;
};

// ------------------------------------------------------------------------------------------------ forward / dgrad
// Weights: [BN rows, taps*KH*64 columns (t, h, c)], all resident in shared memory as (t, h) sub-tiles of BN rows x 128 B.
template <int BN, int KH, bool DACT, bool U8>
__global__ void __launch_bounds__(sh_threads(U8), 1)
conv_shift_fwd_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW,
                      const __grid_constant__ ShiftParams p) {
  constexpr int SH_ABYTES = sh_arows(KH) * 128;      // one 64-channel half of an A stage
  constexpr int STAGE_BYTES = KH * SH_ABYTES;
  constexpr int STAGES = U8 ? SH_U8_STAGES : sh_stages(KH);
  using Ring = U8Ring<SH_BM, STAGES>;                // uint8-fed first layer: rolling ring instead of per-tile stages
  // Ping-pong (whole tiles per group) or cooperative schedule (both groups on every tile, 64 rows each).  Ping-pong
  // needs 2 * BN/2 accumulator registers per thread.  The 9 warps get at most 168 registers each (3 warps share one
  // SM sub-partition's register file), and BN = 128 with the bias / bit-mask epilogue would spill: that instance
  // keeps the cooperative schedule.
  constexpr bool PINGPONG = !(BN == 128 && !DACT);
  constexpr int MH = PINGPONG ? 2 : 1;               // m64 accumulators per thread
  static_assert(PINGPONG || !U8, "the uint8 ring's release rule assumes ping-pong");
  constexpr int A_PITCH = U8 ? SH_BM * 128 : STAGE_BYTES;
  constexpr int A_TOTAL = U8 ? Ring::BYTES : STAGES * STAGE_BYTES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* wres = smem + A_TOTAL;                    // resident weights: taps*KH sub-tiles
  uint64_t* bars = reinterpret_cast<uint64_t*>(wres + sh_wres_bytes(KH, U8));
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;
  uint64_t* w_bar = bars + 2 * STAGES;
  uint64_t* head_bar = bars + 2 * STAGES + 1;        // U8: first unit of the stage's tile is in place
  static_assert((3 * STAGES + 1) * 8 <= SH_BAR_BYTES, "barrier block");
  constexpr int MASK_STAGE = sh_mask_stage_bytes(BN, DACT);
  uint8_t* smask = reinterpret_cast<uint8_t*>(bars) + SH_BAR_BYTES;   // DACT: the mask rows of stage s's tile
  uint8_t* sepi = smask + STAGES * MASK_STAGE;                         // epilogue scratch, one per consumer warp

  __shared__ float s_bias[BN];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int w_sub = BN * 128;                    // one (t, h) weight sub-tile
  if (threadIdx.x < BN) s_bias[threadIdx.x] = (p.bias && (int)threadIdx.x < p.N) ? p.bias[threadIdx.x] : 0.0f;
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], U8 ? Ring::UPT : 1);
      // TMA-fed: a stage holds its own halo rows and is released by the 4 warps of the group that owns its tile (both
      // groups' 8 warps without ping-pong).  Ring: a tile also reads the first unit of the next stage, and the two
      // tiles belong to different groups, so a stage is released by 8 arrivals: 4 from its own tile and 4 from the
      // tile of the previous stage
      mbar_init(&empty_bar[s], (U8 || !PINGPONG) ? SH_CONSUMER_WARPS : 4);
      if (U8) mbar_init(&head_bar[s], 1);
    }
    mbar_init(w_bar, 1);
    // the CTA's first tile has no predecessor to release the first fill of stage 0 as a head reader: arrive for it
    if (U8)
      for (int w = 0; w < 4; ++w) mbar_arrive(&empty_bar[0]);
    fence_barrier_init();
  }
  __syncthreads();

  // Tiles of this CTA: tile(i) = tile_first + i * tile_stride, i < tile_count.  TMA-fed layers interleave the CTAs
  // (neighbouring CTAs share L2 lines of the halo rows); the uint8-fed layer gives every CTA one consecutive run.
  int tile_first, tile_stride, tile_count;
  if (U8) {
    const int q = p.num_tiles / (int)gridDim.x, r = p.num_tiles % (int)gridDim.x, b = (int)blockIdx.x;
    tile_first = b * q + min(b, r);
    tile_stride = 1;
    tile_count = q + (b < r ? 1 : 0);
  } else {
    tile_first = (int)blockIdx.x;
    tile_stride = (int)gridDim.x;
    tile_count = tile_first < p.num_tiles ? (p.num_tiles - tile_first + tile_stride - 1) / tile_stride : 0;
  }

  if (warp == SH_TMA_WARP) {
    if (elect_one()) {
      tma_prefetch_desc(&tmX);
      tma_prefetch_desc(&tmW);
      mbar_arrive_expect_tx(w_bar, (uint32_t)(p.taps * KH) * w_sub);
      for (int q = 0; q < p.taps * KH; ++q) tma_load_2d(wres + q * w_sub, &tmW, w_bar, q * 64, 0);
    }
    __syncwarp();
    int s = 0;
    uint32_t ph = 0;
    if (!U8) {
      for (int i = 0; i < tile_count; ++i) {
        const int tile = tile_first + i * tile_stride;
        mbar_wait(&empty_bar[s], ph ^ 1);
        if (elect_one()) {
          uint8_t* sa = smem + s * STAGE_BYTES;
          // DACT: the tile's mask words are one contiguous run (rows of BN bits), clamped to M; the bulk copy takes
          // whole 16-byte pieces and this thread copies the last 4- or 8-byte rows of a short tail itself (before its
          // arrive, which releases them to the consumers)
          uint32_t mbytes = 0;
          const uint8_t* msrc = nullptr;
          if (DACT && p.saved_bits != nullptr) {
            const long long left = p.M - (long long)tile * SH_BM;
            mbytes = (uint32_t)(left < SH_BM ? left : SH_BM) * (BN / 8);
            msrc = reinterpret_cast<const uint8_t*>(p.saved_bits) + (long long)tile * MASK_STAGE;
#pragma unroll 1
            for (uint32_t b = mbytes & ~15u; b < mbytes; b += 4)
              *reinterpret_cast<uint32_t*>(smask + s * MASK_STAGE + b) = __ldg(reinterpret_cast<const uint32_t*>(msrc + b));
            if (mbytes & 15u) __threadfence_block();          // the tail stores are performed before the arrive
          }
          mbar_arrive_expect_tx(&full_bar[s], (uint32_t)STAGE_BYTES + (mbytes & ~15u));
          const int row0 = tile * SH_BM + p.min_shift;                  // may be negative: TMA zero-fills
#pragma unroll
          for (int h = 0; h < KH; ++h) tma_load_2d(sa + h * SH_ABYTES, &tmX, &full_bar[s], h * 64, row0);
          if (mbytes >= 16) bulk_load_1d(smask + s * MASK_STAGE, msrc, mbytes & ~15u, &full_bar[s]);
        }
        __syncwarp();
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
    }
  } else if (U8 && warp > SH_TMA_WARP) {
    // uint8 producer warps (2 units of loads in flight each)
    u8_ring_producer<SH_BM, STAGES, 2>(p.u8, p.M, (long long)tile_first * SH_BM + p.min_shift, tile_count, smem,
                                       full_bar, head_bar, empty_bar, warp - (SH_TMA_WARP + 1), lane);
  } else {
    // consumer warpgroup wg: ping-pong: the CTA's tiles i = wg, wg + 2, ... whole, as two m64 accumulators (tile rows
    // [0, 64) and [64, 128)); cooperative: rows [64*wg, 64*wg + 64) of every tile.  Thread t holds rows r0 and r0 + 8
    // of each accumulator.  (wg is broadcast: the compiler then knows the tile loop is warp-uniform and keeps the
    // wgmma chain asynchronous.)
    const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0), t = threadIdx.x & 127;
    const int row0 = PINGPONG ? 0 : wg * 64;
    const uint32_t w_base = smem_u32(wres);
    const float lo = (p.act == ACT_RELU) ? 0.0f : -INFINITY;
    const __half2 lo2 = __floats2half2_rn(lo, lo);
    const __half2 zero2 = __floats2half2_rn(0.0f, 0.0f);
    // Epilogue: after the transpose, lane l holds columns 8 * (l >> 4) .. + 7 of each 16-column chunk of row
    // er = l & 15 of the warp's 16 rows (rows 16 * (warp % 4) + er of each m64 accumulator).  That is also the row
    // and piece whose address lane l hands to stmatrix for the chunk, so one scratch address per chunk parity.
    const int er = lane & 15, ep = lane >> 4;
    const int erow = row0 + 16 * (warp & 3) + er;                 // tile row of accumulator 0
    uint32_t epi_addr[2];
#pragma unroll
    for (int jj = 0; jj < 2; ++jj)
      epi_addr[jj] = smem_u32(sepi + warp * SH_EPI_WARP_BYTES) + er * 64 + (((2 * jj + ep) ^ ((er >> 1) & 3)) << 4);
    const bool masked = DACT && p.saved_bits != nullptr;
    float acc[MH][BN / 2];
    mbar_wait(w_bar, 0);
    for (int i = PINGPONG ? wg : 0; i < tile_count; i += PINGPONG ? 2 : 1) {
      const int tile = tile_first + i * tile_stride;
      const int s = i % STAGES, s1 = (s + 1 == STAGES) ? 0 : s + 1;
      const uint32_t ph = (uint32_t)(i / STAGES) & 1u;
      mbar_wait(&full_bar[s], ph);
      if (U8) mbar_wait(&head_bar[s1], s1 == 0 ? ph ^ 1 : ph);   // the shifted taps read into the next tile's first unit
      if (PINGPONG && i > 0) order_wait(wg);                      // the other group has issued tile i - 1
      const uint32_t a_base = smem_u32(smem + s * A_PITCH) + (uint32_t)(row0 * 128);
      wgmma_fence();
      // tap 0 overwrites the accumulators with its first MMA; the others accumulate
#pragma unroll 1
      for (int a = 0; a < p.taps; ++a) {
        const uint32_t at = a_base + (uint32_t)p.shift[a] * 128u;
        const uint32_t wt = w_base + (uint32_t)(a * KH * w_sub);
#pragma unroll
        for (int h = 0; h < KH; ++h) {
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const uint64_t bdesc = make_sdesc(wt + h * w_sub + k * 32, 16, 1024, 1);
#pragma unroll
            for (int mh = 0; mh < MH; ++mh) {
              const uint64_t adesc = make_sdesc(at + mh * 64 * 128 + h * SH_ABYTES + k * 32, 16, 1024, 1);
              wgmma_f16<BN, 0, 0>(acc[mh], adesc, bdesc, (a | h | k) ? 1u : 0u);
            }
          }
        }
      }
      wgmma_commit();
      if (PINGPONG && i + 1 < tile_count) order_pass(wg);         // the other group may issue tile i + 1
      wgmma_wait<0>();
      auto release = [&]() {
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(&empty_bar[s]);
          if (U8) mbar_arrive(&empty_bar[s1]);                    // the head unit this tile read
        }
      };
      // DACT: this lane's mask rows (BN bits each).  The stage is released only after the epilogue has used them: an
      // arrive does not wait for a shared-memory load still in flight, and while the other group's MMAs stream their
      // operands from shared memory such a load can still be pending when the TMA warp refills the stage.
      uint32_t mrow[MH][BN / 32];
      if (masked) {
#pragma unroll
        for (int mh = 0; mh < MH; ++mh) {
          const uint32_t r = smem_u32(smask + s * MASK_STAGE) + (uint32_t)((erow + mh * 64) * (BN / 8));
#pragma unroll
          for (int i = 0; i < BN / 32; ++i) asm volatile("ld.shared.b32 %0, [%1];" : "=r"(mrow[mh][i]) : "r"(r + 4 * i));
        }
      } else {
        release();
      }

#pragma unroll
      for (int mh = 0; mh < MH; ++mh) {
        const uint32_t m = (uint32_t)tile * SH_BM + mh * 64 + erow;    // M < 2^31 (checked on the host)
        const uint32_t t2 = p.fwg.div(m);
        const int x = (int)(m - t2 * (uint32_t)p.Wg);
        const int n = (int)p.fhg.div(t2);
        const int y = (int)(t2 - (uint32_t)n * (uint32_t)p.Hg);
        const bool ok = ((long long)m < p.M) && (y < p.vy) && (x < p.vx);
        const long long obase = map_rowbase(p.omap, n, y, x);
#pragma unroll
        for (int ps = 0; ps < BN / 32; ++ps) {               // passes of 32 columns = two 16-column chunks
#pragma unroll
          for (int jj = 0; jj < 2; ++jj) {
            // chunk 2 * ps + jj = 8-column blocks b, b + 1; stmatrix matrices (b, row t/4), (b, + 8), (b + 1, ...)
            const int b = 2 * (2 * ps + jj);
            uint32_t r[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const int e = 4 * (b + (k >> 1)) + 2 * (k & 1);
              const int c = 8 * (b + (k >> 1)) + 2 * (t & 3);
              __half2 o;
              if (DACT) {                                     // the mask is applied to the fp16 words below
                o = __floats2half2_rn(acc[mh][e] * p.alpha, acc[mh][e + 1] * p.alpha);
              } else {                                        // relu after the rounding: same result, one packed max
                o = __hmax2(__floats2half2_rn(fmaf(acc[mh][e], p.alpha, s_bias[c]),
                                              fmaf(acc[mh][e + 1], p.alpha, s_bias[c + 1])),
                            lo2);
              }
              r[k] = h2_bits(o);
            }
            stmatrix_x4(epi_addr[jj], r);
          }
          __syncwarp();
#pragma unroll
          for (int jj = 0; jj < 2; ++jj) {
            const int j = 2 * ps + jj;
            uint4 v = ld_shared_v4(epi_addr[jj]);            // columns 16 * j + 8 * ep .. + 7 of row er
            // a 16-column chunk never straddles a class of the map: column 16 * j + cc lies at coloff(16 * j) + cc
            const long long ocol = map_coloff(p.omap, 16 * j);
            if (masked) {
              // zeroing the rounded value gives what rounding 0.0f gives: +0
              const uint32_t b8 = (mrow[mh][j >> 1] >> (16 * (j & 1) + 8 * ep)) & 0xffu;
              v.x &= mask_pair(b8, 0);
              v.y &= mask_pair(b8, 1);
              v.z &= mask_pair(b8, 2);
              v.w &= mask_pair(b8, 3);
            }
            if (ok) st_global_v4(p.out + obase + ocol + 8 * ep, v);
            if (!DACT && p.bits_out != nullptr) {             // the two lanes of a row assemble the chunk's 16 bits
              const uint32_t w[4] = {v.x, v.y, v.z, v.w};
              uint32_t bits = 0;
#pragma unroll
              for (int k = 0; k < 4; ++k) {
                const uint32_t gt = __hgt2_mask(*reinterpret_cast<const __half2*>(&w[k]), zero2);
                bits |= ((gt & 1u) | ((gt >> 15) & 2u)) << (2 * k);
              }
              bits <<= 8 * ep;
              bits |= __shfl_xor_sync(0xffffffffu, bits, 16);
              if (ok && ep == 0) p.bits_out[(obase + ocol) >> 4] = (uint16_t)bits;
            }
          }
          __syncwarp();                                       // the scratch is rewritten by the next pass
        }
      }
      if (masked) release();
    }
  }
}

// ------------------------------------------------------------------------------------------------ wgrad
struct ShiftWgradParams {
  U8Src u8;
  float* gbias;            // optional: gbias[n] += alpha_b * sum_m dY[m, n]  (fused bias gradient)
  float alpha_b;
  long long M;             // reduction rows = B*Hg*Wg
  int N;                   // dY channels
  int taps;                // filter rows (kx > 1) or taps (kx == 1)
  int kx;                  // taps per filter row: tap (a, b) reads X shifted by shift[a] + b
  int shift[SH_MAX_TAPS];  // >= 0
  float* G;                // [taps*kx*KH*64, N] fp32, row pitch ldg; row ((a*kx + b)*KH + h)*64 + c
  long long ldg;
  float alpha;
  int kb_total, kb_per_cta;
  // CTA x stores its partial G at ws_g + x*grows*N and its partial bias gradient at ws_b + x*N (summed in x order
  // afterwards, so the result does not depend on which CTA finishes first)
  float* ws_g;
  float* ws_b;
  long long grows;         // rows of G = taps*kx*KH*64
};

// blockIdx.x: a run of k-blocks (reduction rows); blockIdx.y: a group of 2*QW 64-row accumulator chunks
// q = (tap, h) of G.  Both operands are MN-major: X[rows, 64 channels] (shifted per tap) and dY[rows, N].
//
// TMA-fed instances may run as clusters of (1, g, 1) CTAs: g chunk groups of the same row range, so the same k-blocks
// (every CTA of a cluster has the same blockIdx.x, hence the same kb0..kb1).  A stage is then loaded once per cluster:
// its TMA boxes (the KH X halves, then the dY tile) are dealt round-robin to the cluster's producers, each box
// multicast into every CTA.  Each CTA's full barrier still expects the whole stage's bytes; its empty barrier counts the
// 8 consumer warps of every CTA (8*g arrivals), since a producer's boxes overwrite the stage in all of them.  The
// cluster synchronises after the barriers are initialised (peers arrive on them and multicast into them) and before
// exit (a peer's consumers may still arrive on this CTA's empty barriers).
template <int BN, int KH, bool U8>
__global__ void __launch_bounds__(sh_threads(U8), 1)
conv_shift_wgrad_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmD,
                        const __grid_constant__ ShiftWgradParams p) {
  constexpr int BROWB = (BN >= 64) ? 128 : BN * 2;            // dY row bytes in smem
  constexpr uint32_t LAYOUT_B = sdesc_layout(BROWB);
  constexpr int KR = sh_wgrad_krows(U8);                      // reduction rows per pipeline stage ("k-block")
  constexpr int B_BYTES = KR * BROWB;
  constexpr int B_REGION = (B_BYTES + 1023) & ~1023;
  constexpr int STAGES = (KH == 1) ? 8 : 6;
  constexpr int QW = sh_wgrad_qw(BN, KH, U8);
  static_assert(!U8 || KH == 1, "the uint8-fed layer has 64 space-to-depth channels");
  // TMA-fed: stage = [A halves | B], 1024 B aligned.  uint8-fed: [rolling A ring (KR-row blocks) | B stages]
  using Ring = U8Ring<KR, STAGES>;
  constexpr int A_PITCH = U8 ? KR * 128 : KH * SH_WABYTES + B_REGION;
  constexpr int B_PITCH = U8 ? B_REGION : KH * SH_WABYTES + B_REGION;
  constexpr int B_BASE = U8 ? Ring::BYTES : KH * SH_WABYTES;
  constexpr int SMEM_TILES = U8 ? Ring::BYTES + STAGES * B_REGION : STAGES * (KH * SH_WABYTES + B_REGION);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + SMEM_TILES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;
  uint64_t* head_bar = bars + 2 * STAGES;                     // U8: first unit of the stage's k-block is in place

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kb0 = blockIdx.x * p.kb_per_cta;
  const int kb1 = min(kb0 + p.kb_per_cta, p.kb_total);
  const int nchunks = p.taps * p.kx * KH;
  const uint32_t ncta = U8 ? 1u : cluster_nctarank();        // the uint8-fed instance never runs as a cluster

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], U8 ? 1 + Ring::UPT : 1);
      // ring: a k-block also reads the first unit of the next stage; both groups finish k-blocks in order, so the
      // next stage's own k-block releasing it implies this one is done too
      mbar_init(&empty_bar[s], SH_CONSUMER_WARPS * ncta);
      if (U8) mbar_init(&head_bar[s], 1);
    }
    fence_barrier_init();
  }
  if (ncta > 1) cluster_sync();
  else __syncthreads();

  if (warp == SH_TMA_WARP) {
    if (elect_one()) {
      tma_prefetch_desc(&tmX);
      tma_prefetch_desc(&tmD);
    }
    __syncwarp();
    const uint32_t rank = U8 ? 0u : cluster_ctarank();
    const uint16_t mask = (uint16_t)((1u << ncta) - 1u);
    int s = 0;
    uint32_t ph = 0;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(&empty_bar[s], ph ^ 1);
      if (elect_one()) {
        uint8_t* sa = smem + s * A_PITCH;
        uint8_t* sb = smem + B_BASE + s * B_PITCH;
        mbar_arrive_expect_tx(&full_bar[s], (uint32_t)((U8 ? 0 : KH * SH_WABYTES) + B_BYTES));
        if (U8) {
          tma_load_2d(sb, &tmD, &full_bar[s], 0, kb * KR);
        } else {
          // box b < KH: X half b; box KH: the dY tile.  This CTA loads boxes rank, rank + ncta, ...
          for (int b = (int)rank; b <= KH; b += (int)ncta) {
            void* dst = b < KH ? (void*)(sa + b * SH_WABYTES) : (void*)sb;
            const CUtensorMap* tm = b < KH ? &tmX : &tmD;
            if (ncta == 1) tma_load_2d(dst, tm, &full_bar[s], b < KH ? b * 64 : 0, kb * KR);
            else tma_load_2d_multicast(dst, tm, &full_bar[s], b < KH ? b * 64 : 0, kb * KR, mask);
          }
        }
      }
      __syncwarp();
      if (++s == STAGES) { s = 0; ph ^= 1; }
    }
  } else if (U8 && warp > SH_TMA_WARP) {
    u8_ring_producer<KR, STAGES, 3>(p.u8, p.M, (long long)kb0 * KR, kb1 - kb0, smem, full_bar, head_bar, empty_bar,
                                    warp - (SH_TMA_WARP + 1), lane);
  } else {
    const int wg = warp >> 2, t = threadIdx.x & 127;
    // The chunks are dealt to the 2 * gridDim.y warpgroups of the grid in contiguous runs whose lengths differ by at
    // most one (c3's 9 chunks: 3 + 2 | 2 + 2), so no warpgroup issues MMAs for a chunk it does not own.
    const int nwg = 2 * (int)gridDim.y, w = 2 * (int)blockIdx.y + wg;
    const int q0 = w * (nchunks / nwg) + min(w, nchunks % nwg);     // this warpgroup's first accumulator chunk
    const int nq = nchunks / nwg + (w < nchunks % nwg ? 1 : 0);     // its chunk count, 0 .. QW (warpgroup-uniform)
    // A descriptor start of chunk q relative to the stage: half h, rows shifted by the tap's shift
    int a_rel[QW];
#pragma unroll
    for (int i = 0; i < QW; ++i) {
      const int q = min(q0 + i, nchunks - 1);
      const int tap = q / KH, h = q - tap * KH;
      a_rel[i] = h * SH_WABYTES + (p.shift[tap / p.kx] + tap % p.kx) * 128;
    }
    // fused bias gradient (first chunk group only): column sums of the dY tile while it sits in shared memory
    // (swizzle undone by hand); LPR lanes cover one row with 8-byte loads (4 columns per lane)
    const bool do_bias = p.gbias != nullptr && blockIdx.y == 0;
    constexpr int LPR = BROWB / 8;
    constexpr int RG = 32 / LPR;                               // row groups per warp
    const int cq = lane % LPR, rg = lane / LPR;
    const int chunk = (cq * 8) >> 4, within = (cq * 8) & 15;
    float bsum[4] = {0.f, 0.f, 0.f, 0.f};
    auto bias_sums = [&](int st) {
      const uint8_t* sb = smem + B_BASE + st * B_PITCH;
#pragma unroll 4
      for (int r = warp * RG + rg; r < KR; r += SH_CONSUMER_WARPS * RG) {
        const int sw = (BROWB == 128) ? (r & 7) : ((r >> 1) & 3);
        const uint2 v = *reinterpret_cast<const uint2*>(sb + r * BROWB + ((chunk ^ sw) << 4) + within);
        bsum[0] += __half2float(__ushort_as_half((unsigned short)(v.x & 0xffffu)));
        bsum[1] += __half2float(__ushort_as_half((unsigned short)(v.x >> 16)));
        bsum[2] += __half2float(__ushort_as_half((unsigned short)(v.y & 0xffffu)));
        bsum[3] += __half2float(__ushort_as_half((unsigned short)(v.y >> 16)));
      }
    };
    auto release = [&](int st) {
      __syncwarp();
      if (U8 || ncta == 1) {
        if (lane == 0) mbar_arrive(&empty_bar[st]);
      } else if (lane < (int)ncta) {
        mbar_arrive_cluster(&empty_bar[st], (uint32_t)lane);   // lane r releases the stage in CTA r of the cluster
      }
    };
    // Each (k-block, chunk) MMA group starts a fresh accumulator (part) that is then added to acc in fp32 registers: a
    // CTA reduces ~10^4 rows, and one chain of that many tensor-core accumulations loses ~1e-5 relative against an fp32
    // sum.  With NP = 2 part buffers the chunks of a k-block alternate between them, so chunk i's acc += part runs while
    // chunk i+1's MMAs execute (wgmma_wait<1>).  QW = 3 leaves registers for one buffer only (288 threads cap the kernel
    // at 168 registers): each chunk then waits for its own MMAs, and the other warpgroup's MMAs fill the tensor pipe.
    constexpr int NP = (QW + 2) * (BN / 2) <= 128 ? 2 : 1;
    float acc[QW][BN / 2], part[NP][BN / 2];
#pragma unroll
    for (int i = 0; i < QW; ++i)
#pragma unroll
      for (int e = 0; e < BN / 2; ++e) acc[i][e] = 0.0f;
    auto add_part = [&](float(&a)[BN / 2], const float(&pt)[BN / 2]) {
#pragma unroll
      for (int e = 0; e < BN / 2; ++e) a[e] += pt[e];
    };
    // the warpgroup's k-block loop for NQ chunks (a compile-time count, so that every register index is static)
    auto consume = [&](auto nq_c) {
      constexpr int NQ = decltype(nq_c)::value;
      int s = 0;
      uint32_t ph = 0;
      for (int kb = kb0; kb < kb1; ++kb) {
        const int s1 = (s + 1 == STAGES) ? 0 : s + 1;
        mbar_wait(&full_bar[s], ph);
        if (U8) mbar_wait(&head_bar[s1], s1 == 0 ? ph ^ 1 : ph);   // the shifted taps read into the next block's first unit
        const uint32_t a_base = smem_u32(smem + s * A_PITCH);
        const uint32_t b_base = smem_u32(smem + B_BASE + s * B_PITCH);
        if (NQ == 0 && do_bias) bias_sums(s);
#pragma unroll
        for (int i = 0; i < NQ; ++i) {
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < KR / 16; ++k) {
            const uint64_t adesc = make_sdesc(a_base + a_rel[i] + k * 16 * 128, 8 * 1024, 1024, 1);
            const uint64_t bdesc = make_sdesc(b_base + k * 16 * BROWB, 8 * 8 * BROWB, 8 * BROWB, LAYOUT_B);
            wgmma_f16<BN, 1, 1>(part[i % NP], adesc, bdesc, k > 0 ? 1u : 0u);
          }
          wgmma_commit();
          if (i == 0 && do_bias) bias_sums(s);
          wgmma_wait<NP - 1>();                                    // chunk i - (NP - 1) has retired
          if (i >= NP - 1) add_part(acc[i - (NP - 1)], part[(i - (NP - 1)) % NP]);
        }
        if constexpr (NP == 2 && NQ > 0) {
          wgmma_wait<0>();
          add_part(acc[NQ - 1], part[(NQ - 1) % NP]);
        }
        release(s);
        s = s1;
        if (s == 0) ph ^= 1;
      }
    };
    static_assert(QW >= 2 && QW <= 4, "conv_shift_wgrad: 2..4 chunks per warpgroup");
    switch (nq) {                                              // warpgroup-uniform
      case 0: consume(std::integral_constant<int, 0>{}); break;
      case 1: consume(std::integral_constant<int, 1>{}); break;
      case 2: consume(std::integral_constant<int, 2>{}); break;
      default:
        if constexpr (QW >= 3) if (nq == 3) consume(std::integral_constant<int, 3>{});
        if constexpr (QW >= 4) if (nq == 4) consume(std::integral_constant<int, 4>{});
    }
    if (do_bias) {
      __shared__ float s_bsum[SH_CONSUMER_WARPS][64];
#pragma unroll
      for (int o = LPR; o < 32; o <<= 1)                       // fold the row groups together
#pragma unroll
        for (int i = 0; i < 4; ++i) bsum[i] += __shfl_xor_sync(0xffffffffu, bsum[i], o);
      if (rg == 0) {
#pragma unroll
        for (int i = 0; i < 4; ++i) s_bsum[warp][4 * cq + i] = bsum[i];
      }
      asm volatile("bar.sync 1, %0;" ::"n"(SH_CONSUMER_WARPS * 32) : "memory");   // consumer warps only
      if ((int)threadIdx.x < p.N) {
        float b = 0.0f;
#pragma unroll
        for (int w = 0; w < SH_CONSUMER_WARPS; ++w) b += s_bsum[w][threadIdx.x];
        p.ws_b[(long long)blockIdx.x * p.N + threadIdx.x] = b * p.alpha_b;
      }
    }
    if (kb1 > kb0) {
#pragma unroll
      for (int i = 0; i < QW; ++i) {
        if (i < nq) {
#pragma unroll
          for (int e = 0; e < BN / 2; ++e) {
            const int cn = acc_col(t, e);
            const long long grow = (long long)(q0 + i) * 64 + acc_row(t, e);
            if (cn < p.N) p.ws_g[((long long)blockIdx.x * p.grows + grow) * p.N + cn] = acc[i][e] * p.alpha;
          }
        }
      }
    }
  }
  if (ncta > 1) cluster_sync();
}

// ------------------------------------------------------------------------------------------------ host
static U8Src make_u8src(const void* x, const long long* idx, int H, int W, int C, int s) {
  U8Src u{};
  u.x = reinterpret_cast<const uint8_t*>(x);
  if (!x) return u;
  u.idx = idx;
  u.sample_bytes = (long long)H * W * C;
  u.row_bytes = W * C;
  u.y_bytes = s * W * C;
  u.x_bytes = s * C;
  u.per = make_fastdiv((uint32_t)((H / s) * (W / s)));
  u.wg = make_fastdiv((uint32_t)(W / s));
  return u;
}

template <int BN, int KH, bool DACT, bool U8 = false>
static int launch_fwd(const CUtensorMap& tmX, const CUtensorMap& tmW, const ShiftParams& p, cudaStream_t st) {
  constexpr int STAGES = U8 ? SH_U8_STAGES : sh_stages(KH);
  constexpr int SMEM = (U8 ? U8Ring<SH_BM, STAGES>::BYTES : STAGES * KH * sh_arows(KH) * 128) + sh_wres_bytes(KH, U8) +
                       1024 + SH_BAR_BYTES + STAGES * sh_mask_stage_bytes(BN, DACT) + SH_EPI_BYTES;
  static_assert(SMEM + 1024 <= 227 * 1024, "conv_shift_fwd: shared memory budget (+ static bias array)");
  static bool attr = false;
  auto kern = conv_shift_fwd_kernel<BN, KH, DACT, U8>;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    if (e != cudaSuccess) {
      set_last_error("conv_shift_fwd: smem attr %d: %s", SMEM, cudaGetErrorString(e));
      return B200RL_ERR_CUDA;
    }
    attr = true;
  }
  const int grid = p.num_tiles < device_num_sms() ? p.num_tiles : device_num_sms();
  kern<<<grid, sh_threads(U8), SMEM, st>>>(tmX, tmW, p);
  return check_launch("conv_shift_fwd_kernel");
}

// CTAs per cluster of the weight gradient: the largest divisor of the chunk-group count (grid.y) up to the portable
// cluster size 8
static int wgrad_cluster(int groups) {
  int g = groups < 8 ? groups : 8;
  while (groups % g) --g;
  return g;
}

// grid.x: row ranges (k-block runs); grid.y: chunk groups.  The chunk groups of a row range run as one cluster when
// clusters of that size tile the SMs.  Otherwise they do not cluster: a cluster's CTAs share one GPC, so clusters of 3
// fit only 117 of an H100's 132 SMs at this kernel's shared memory, and the SMs left idle cost more than the operand
// reads a cluster saves (measured: c3 of cfg-2 slower as clusters of 3).
template <int BN, int KH, bool U8 = false>
static int launch_wgrad(const CUtensorMap& tmX, const CUtensorMap& tmD, const ShiftWgradParams& p, dim3 grid,
                        cudaStream_t st) {
  constexpr int STAGES = (KH == 1) ? 8 : 6;
  constexpr int KR = sh_wgrad_krows(U8);
  constexpr int BROWB = (BN >= 64) ? 128 : BN * 2;
  constexpr int B_REGION = (KR * BROWB + 1023) & ~1023;
  constexpr int SMEM =
      (U8 ? U8Ring<KR, STAGES>::BYTES + STAGES * B_REGION : STAGES * (KH * SH_WABYTES + B_REGION)) + 1024 + 512;
  static_assert(SMEM <= 227 * 1024, "conv_shift_wgrad: shared memory budget");
  static bool attr = false;
  static int co_resident[9] = {};                 // clusters of g CTAs that fit on the device at once, per g
  auto kern = conv_shift_wgrad_kernel<BN, KH, U8>;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    if (e != cudaSuccess) {
      set_last_error("conv_shift_wgrad: smem attr %d: %s", SMEM, cudaGetErrorString(e));
      return B200RL_ERR_CUDA;
    }
    attr = true;
  }
  int g = U8 ? 1 : wgrad_cluster((int)grid.y);
  cudaLaunchAttribute cl;
  cl.id = cudaLaunchAttributeClusterDimension;
  cl.val.clusterDim.x = 1;
  cl.val.clusterDim.y = (unsigned)g;
  cl.val.clusterDim.z = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(sh_threads(U8));
  cfg.dynamicSmemBytes = SMEM;
  cfg.stream = st;
  cfg.attrs = &cl;
  cfg.numAttrs = 1;
  if (g > 1) {
    if (co_resident[g] == 0) {
      cudaError_t e = cudaOccupancyMaxActiveClusters(&co_resident[g], kern, &cfg);
      if (e != cudaSuccess) {
        set_last_error("conv_shift_wgrad: cluster occupancy (%d CTAs): %s", g, cudaGetErrorString(e));
        co_resident[g] = 0;
        return B200RL_ERR_CUDA;
      }
    }
    if (co_resident[g] * g < device_num_sms()) g = 1;
  }
  cfg.numAttrs = g > 1 ? 1 : 0;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kern, tmX, tmD, p);
  const int rc = check_launch("conv_shift_wgrad_kernel");
  if (rc == B200RL_OK && e != cudaSuccess) {
    set_last_error("conv_shift_wgrad_kernel: %s", cudaGetErrorString(e));
    return B200RL_ERR_CUDA;
  }
  return rc;
}

static int ilog2(int v) { int l = 0; while ((1 << l) < v) ++l; return l; }
static bool fill_map(AddrMap& a, const long long* m) {       // {mode, sN, sY, sX, Cq, s}
  a.mode = (int)m[0]; a.sN = m[1]; a.sY = m[2]; a.sX = m[3]; a.Cq = (int)m[4]; a.s = (int)m[5];
  a.Cq_log2 = a.s_log2 = 0;
  if (a.mode == 0) return true;
  if (a.Cq < 16 || (a.Cq & (a.Cq - 1)) || a.s < 1 || (a.s & (a.s - 1))) return false;
  a.Cq_log2 = ilog2(a.Cq); a.s_log2 = ilog2(a.s);
  return true;
}

}  // namespace b200rl

using namespace b200rl;

// X: [B*Hg*Wg, C] fp16 (C = 64 or 128, row pitch C); W: [N, taps*C] fp16 (row pitch ldw), K order (tap, channel);
// shifts[taps]: absolute row shifts (all >= 0 for forward, all <= 0 for the data gradient).
extern "C" int b200rl_conv_shift_fwd(const void* X, long long B, int Hg, int Wg, int C, const void* W, long long ldw,
                                     int N, int taps, const int* shifts, int vy, int vx, void* out,
                                     const long long* omap, const long long* smap, const float* bias, int act, int dact,
                                     float alpha, const void* u8_x, const long long* u8_idx, int u8_H, int u8_W,
                                     int u8_C, int u8_s, void* bits_out, const void* saved_bits, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE((X || u8_x) && W && out && omap && B > 0, "conv_shift_fwd: null operand");
  B200RL_REQUIRE(!(bits_out && dact) && !(saved_bits && !(dact && smap)), "conv_shift_fwd: bits_out is a forward output, saved_bits a dact input (with smap)");
  if (u8_x) {
    B200RL_REQUIRE(C == 64 && u8_s * u8_C == 16 && u8_s == 4 && u8_H == Hg * u8_s && u8_W == Wg * u8_s && !dact &&
                       N == 32 && (reinterpret_cast<uintptr_t>(u8_x) & 15) == 0 && (u8_W * u8_C) % 16 == 0,
                   "conv_shift_fwd: fused uint8 source needs s=4, s*C=16, N=32, 16 B aligned rows");
  }
  B200RL_REQUIRE(C == 64 || C == 128, "conv_shift_fwd: C must be 64 or 128 (got %d)", C);
  B200RL_REQUIRE(N == 32 || N == 64 || N == 128, "conv_shift_fwd: N must be 32, 64 or 128 (got %d)", N);
  B200RL_REQUIRE(taps >= 1 && taps <= SH_MAX_TAPS, "conv_shift_fwd: 1..%d taps", SH_MAX_TAPS);
  B200RL_REQUIRE((C == 64 || C == 128) && (long long)taps * (C / 64) * N * 128 <= sh_wres_bytes(C / 64, u8_x != nullptr),
                 "conv_shift_fwd: weights do not fit in smem");
  ShiftParams p = {};
  int lo = shifts[0], hi = shifts[0];
  for (int t = 1; t < taps; ++t) { lo = shifts[t] < lo ? shifts[t] : lo; hi = shifts[t] > hi ? shifts[t] : hi; }
  B200RL_REQUIRE(hi - lo <= sh_arows(C / 64) - SH_BM, "conv_shift_fwd: shift span %d too large for C = %d", hi - lo,
                 C);
  B200RL_REQUIRE(B * Hg * Wg < (1LL << 31) - 4096, "conv_shift_fwd: too many rows");
  p.M = B * Hg * Wg; p.Hg = Hg; p.Wg = Wg; p.N = N; p.taps = taps; p.min_shift = lo;
  for (int t = 0; t < taps; ++t) p.shift[t] = shifts[t] - lo;
  p.vy = vy; p.vx = vx; p.out = reinterpret_cast<__half*>(out);
  B200RL_REQUIRE(fill_map(p.omap, omap), "conv_shift_fwd: output map needs power-of-two Cq >= 16 and s");
  p.bits_out = reinterpret_cast<uint16_t*>(bits_out);
  p.saved_bits = reinterpret_cast<const uint16_t*>(saved_bits);
  // the epilogue stores 8-column pieces as 16-byte words and writes the activation bits per 16-column chunk
  B200RL_REQUIRE(((omap[1] | omap[2] | omap[3]) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 31) == 0,
                 "conv_shift_fwd: output strides must be multiples of 16 elements, base 32-byte aligned");
  // a tile's mask is staged with its A tile as one contiguous run: the saved activation must be row-contiguous on
  // the output grid, N elements per grid row
  if (saved_bits)
    B200RL_REQUIRE(smap[0] == 0 && smap[3] == N && smap[2] == (long long)Wg * N && smap[1] == (long long)Hg * Wg * N &&
                       (reinterpret_cast<uintptr_t>(saved_bits) & 15) == 0,
                   "conv_shift_fwd: saved_bits needs the row-contiguous map (0, Hg*Wg*N, Wg*N, N) and a 16-byte aligned "
                   "base");
  p.bias = bias; p.act = act; p.dact = dact; p.alpha = alpha;
  p.num_tiles = (int)((p.M + SH_BM - 1) / SH_BM);
  p.u8 = make_u8src(u8_x, u8_idx, u8_H, u8_W, u8_C, u8_s);
  B200RL_REQUIRE(Hg >= 2 && Wg >= 2, "conv_shift_fwd: grid must be at least 2x2");
  p.fwg = make_fastdiv((uint32_t)Wg);
  p.fhg = make_fastdiv((uint32_t)Hg);
  CUtensorMap tmX, tmW;
  int rc;
  B200RL_REQUIRE(act == ACT_NONE || act == ACT_RELU, "conv_shift_fwd: activation must be none or relu");
  if ((rc = make_tmap_2d_f16(&tmW, W, N, (long long)taps * C, ldw, 64, N)) != 0) return rc;
  if (u8_x) {                                                          // tmX unused: A tiles come from the producers
    B200RL_REQUIRE(hi - lo <= 32, "conv_shift_fwd: uint8-fed shift span %d exceeds one 32-row unit", hi - lo);
    return launch_fwd<32, 1, false, true>(tmW, tmW, p, stream);
  }
  if ((rc = make_tmap_2d_f16(&tmX, X, p.M, C, C, 64, sh_arows(C / 64))) != 0) return rc;
  const int KH = C / 64;
#define SHIFT_FWD_CASE(bn)                                                                                    \
  if (N == bn) {                                                                                              \
    if (dact) return KH == 1 ? launch_fwd<bn, 1, true>(tmX, tmW, p, stream) : launch_fwd<bn, 2, true>(tmX, tmW, p, stream); \
    return KH == 1 ? launch_fwd<bn, 1, false>(tmX, tmW, p, stream) : launch_fwd<bn, 2, false>(tmX, tmW, p, stream);        \
  }
  SHIFT_FWD_CASE(32)
  SHIFT_FWD_CASE(64)
  SHIFT_FWD_CASE(128)
#undef SHIFT_FWD_CASE
  return B200RL_ERR_UNSUPPORTED;
}

// G[taps*C, N] (fp32, row pitch ldg) += alpha * sum_m X[m + shift_t, c] * dY[m, n]
extern "C" int b200rl_conv_shift_wgrad(const void* X, long long rows, int C, const void* dY, int N, int taps,
                                       const int* shifts, float* G, long long ldg, float alpha, float* gbias,
                                       float alpha_b, int max_ctas, const void* u8_x, const long long* u8_idx, int u8_H,
                                       int u8_W, int u8_C, int u8_s, int kx, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  B200RL_REQUIRE((X || u8_x) && dY && G && rows > 0, "conv_shift_wgrad: null operand");
  if (kx < 1) kx = 1;
  B200RL_REQUIRE(kx <= 3, "conv_shift_wgrad: kx must be 1..3");
  if (u8_x)
    B200RL_REQUIRE(C == 64 && u8_s == 4 && u8_s * u8_C == 16 && N == 32 && u8_H % 4 == 0 && u8_W % 4 == 0 &&
                       (reinterpret_cast<uintptr_t>(u8_x) & 15) == 0,
                   "conv_shift_wgrad: fused uint8 source needs s=4, s*C=16, N=32");
  B200RL_REQUIRE(C == 64 || C == 128, "conv_shift_wgrad: C must be 64 or 128");
  B200RL_REQUIRE(N == 32 || N == 64, "conv_shift_wgrad: N must be 32 or 64 (got %d)", N);
  B200RL_REQUIRE(taps >= 1 && taps <= SH_MAX_TAPS, "conv_shift_wgrad: 1..%d taps", SH_MAX_TAPS);
  const int KH = C / 64;
  ShiftWgradParams p = {};
  for (int t = 0; t < taps; ++t) {
    B200RL_REQUIRE(shifts[t] >= 0 && shifts[t] + kx - 1 <= SH_WROWS_K - 64, "conv_shift_wgrad: shift %d out of range",
                   shifts[t]);
    p.shift[t] = shifts[t];
  }
  p.M = rows; p.N = N; p.taps = taps; p.kx = kx; p.G = G; p.ldg = ldg; p.alpha = alpha;
  p.gbias = gbias; p.alpha_b = alpha_b;
  const int KR = sh_wgrad_krows(u8_x != nullptr);
  p.kb_total = (int)((rows + KR - 1) / KR);
  int ctas = device_num_sms();
  if (max_ctas > 0 && max_ctas < ctas) ctas = max_ctas;
  if (ctas > p.kb_total) ctas = p.kb_total;
  p.kb_per_cta = (p.kb_total + ctas - 1) / ctas;
  const int qw = sh_wgrad_qw(N, KH, u8_x != nullptr);
  const dim3 grid((p.kb_total + p.kb_per_cta - 1) / p.kb_per_cta, (taps * kx * KH + 2 * qw - 1) / (2 * qw));
  p.u8 = make_u8src(u8_x, u8_idx, u8_H, u8_W, u8_C, u8_s);
  p.grows = (long long)taps * kx * KH * 64;
  const size_t g_floats = (size_t)grid.x * p.grows * N;
  float* ws = det_workspace(g_floats + (size_t)grid.x * N, stream);
  if (!ws) return B200RL_ERR_CUDA;
  p.ws_g = ws;
  p.ws_b = ws + g_floats;
  CUtensorMap tmX, tmD;
  int rc;
  if ((rc = make_tmap_2d_f16(&tmD, dY, rows, N, N, N < 64 ? N : 64, KR)) != 0) return rc;
  if (u8_x) {
    rc = launch_wgrad<32, 1, true>(tmD, tmD, p, grid, stream);
  } else {
    if ((rc = make_tmap_2d_f16(&tmX, X, rows, C, C, 64, SH_WROWS_K)) != 0) return rc;
    if (N == 32) rc = KH == 1 ? launch_wgrad<32, 1>(tmX, tmD, p, grid, stream) : launch_wgrad<32, 2>(tmX, tmD, p, grid, stream);
    else rc = KH == 1 ? launch_wgrad<64, 1>(tmX, tmD, p, grid, stream) : launch_wgrad<64, 2>(tmX, tmD, p, grid, stream);
  }
  if (rc == B200RL_OK) rc = sum_partials(p.ws_g, (int)grid.x, p.grows, N, G, ldg, stream);
  if (rc == B200RL_OK && gbias) rc = sum_partials(p.ws_b, (int)grid.x, 1, N, gbias, N, stream);
  return rc;
}
