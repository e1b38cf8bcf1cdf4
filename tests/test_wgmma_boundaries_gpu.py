"""Exact-arithmetic sweep of the wgmma GEMM and convolution kernels at their tile, stage, split and ring boundaries.

Operands are small integers (|v| <= 2, mostly zero) and every alpha is a power of two.  Before each launch the test
asserts max(|A| @ |B|) <= 2048 over the actual reduction (tests/_refs.py): every partial sum is then an integer (or a
dyadic fraction) that fp32 -- and any accumulator with >= 12 significant bits -- holds exactly in any summation order,
and every fp16 output is exact.  So each result is compared with torch.equal against a float64 reference: a dropped,
duplicated or misplaced row, tap, column, chunk, split or CTA part changes some output by at least 1.

Where a reduction runs over many rows (wgrad, split-K, column sums) the sparse operand is nonzero mainly at probe rows:
the first / last row of every 128-row tile, the last row of every k-block and of every CTA's k-range, the rows a
shifted tap reads past a tile's end, the last row, and a few random rows.

Regions a kernel must not read are NaN (pitch padding between K and lda / ldb, rows past M in a larger allocation);
regions it must not write hold a sentinel (ldc padding, rows past M, the border of dY grids, invalid grid positions
of the shift-conv forward).  Each case id names the boundary it is for.
"""
import math

import pytest
import torch

import _refs as R

pytestmark = pytest.mark.gpu

DEV = "cuda"
NAN16 = float("nan")
SENT = 1234.0                      # sentinel: exact in fp16 and fp32, larger than any exact result here


@pytest.fixture(scope="module")
def ops():
    from baselines_b200 import ops as _ops
    return _ops


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _ints(shape, density, gen, lo=-2, hi=2):
    return R.small_ints(shape, density, gen, device=DEV, lo=lo, hi=hi)


def _pad8(n):
    return (n + 7) // 8 * 8


def _cdiv(a, b):
    return -(-a // b)


def _padded16(rows, cols, ld, fill, extra_rows=0, dtype=torch.float16):
    """[rows + extra_rows, ld] tensor filled with `fill` (the caller writes [:rows, :cols])."""
    return torch.full((rows + extra_rows, ld), fill, dtype=dtype, device=DEV)


def _density(K, target=150.0):
    """Density p of both operands so that K * p^2 * E|a||b| (= 2.25) stays near `target`."""
    return min(0.8, math.sqrt(target / (2.25 * K)))


# ------------------------------------------------------------------------------ python model of the host launch logic
def gemm_bn(N, mn_major):
    """N tile b200rl_gemm_f16 picks (csrc/gemm_wgmma.cu)."""
    if mn_major:
        return 256 if (N > 128 and N % 256 == 0) else 128 if N > 64 else 64
    return 256 if (N > 128 and N % 256 == 0) else 128 if N > 64 else 64 if N > 32 else 32


def gemm_stages(BN):
    return min(8, (196 * 1024) // (128 * 64 * 2 + BN * 64 * 2))


def fill_splits(kb_total, split_k):
    s = min(max(split_k, 1), kb_total)
    per = _cdiv(kb_total, s)
    return per, _cdiv(kb_total, per)


def gemm_kblocks_per_cta(work, kb_per_work, grid):
    return _cdiv(work, grid) * kb_per_work


def _sms():
    from baselines_b200 import ops
    return ops.num_sms()


# ------------------------------------------------------------------------------------------ ops.gemm, K-major
KMAJOR = ([(f"N{n}_BN{gemm_bn(n, False)}", 129, n, 72) for n in
           (1, 8, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 384, 512)] +
          [(f"M{m}_tiles", m, 64, 64) for m in (1, 63, 64, 65, 127, 128)] +
          [(f"K{k}_tail", 200, 96, k) for k in (8, 16, 24, 56)] +
          [("M4097_K3136_N512_BN256", 4097, 512, 3136)])


@pytest.mark.parametrize("name,M,N,K", KMAJOR, ids=[c[0] for c in KMAJOR])
def test_gemm_kmajor_exact(ops, name, M, N, K):
    """Every epilogue mode at N / M / K tile edges: f16 (none, no bias, scalar stores), f16 relu + bias (vec32
    stores where ldc allows), f32 store + bias, f16 dact with the saved activation and with its bit mask."""
    gen = _gen(M * 7 + N * 3 + K)
    p = _density(K)
    lda = _pad8(K) + 8                                       # pitch padding between K and lda: NaN, never read
    A = _padded16(M, K, lda, NAN16, extra_rows=5)            # rows past M: NaN
    B = _padded16(N, K, lda, NAN16, extra_rows=5)
    A64, B64 = _ints((M, K), p, gen), _ints((N, K), p, gen)
    A[:M, :K], B[:N, :K] = A64.half(), B64.half()
    bias = _ints((N,), 0.7, gen, -3, 3).float()
    ref = R.gemm(A64, B64)
    absprod = A64.abs() @ B64.abs().t()
    R.assert_exact_ok(absprod, what=name)
    assert float((0.5 * absprod).max()) + 3 <= 1024                     # half-integers below 1024: exact in fp16
    n16 = (N + 15) // 16 * 16

    def run_f16(mode, act, ldc, alpha, **kw):
        C = _padded16(M, N, ldc, SENT, extra_rows=3)
        ops.gemm(A, B, C, M=M, N=N, K=K, lda=lda, ldb=lda, ldc=ldc, mode=mode, act=act, alpha=alpha, **kw)
        torch.cuda.synchronize()
        assert torch.all(C[:M, N:] == SENT) and torch.all(C[M:] == SENT), (name, "write outside [M, N]")
        return C[:M, :N].double()

    # f16, no activation, no bias; ldc = N + 3 -> scalar stores
    got = run_f16(ops.MODE_F16_ACT, ops.ACT_NONE, N + 3, 0.5)
    assert torch.equal(got, 0.5 * ref), (name, "f16 none", float((got - 0.5 * ref).abs().max()))
    # f16 relu + bias; ldc multiple of 16 -> vec32 stores
    got = run_f16(ops.MODE_F16_ACT, ops.ACT_RELU, n16, 0.5, bias=bias)
    assert torch.equal(got, torch.relu(0.5 * ref + bias.double())), (name, "f16 relu+bias")
    # f32 store + bias
    C = _padded16(M, N, N + 5, SENT, extra_rows=3, dtype=torch.float32)
    ops.gemm(A, B, C, M=M, N=N, K=K, lda=lda, ldb=lda, ldc=N + 5, bias=bias, mode=ops.MODE_F32_STORE, alpha=0.25)
    torch.cuda.synchronize()
    assert torch.equal(C[:M, :N].double(), 0.25 * ref + bias.double()), (name, "f32 store")
    assert torch.all(C[:M, N:] == SENT) and torch.all(C[M:] == SENT), (name, "f32 write outside [M, N]")
    # f16 dact: relu mask from the saved fp16 activation (and from its bit mask where the layout allows)
    saved = torch.relu(_ints((M, n16), 0.6, gen)).half()
    want = 0.5 * ref * (saved[:, :N].double() > 0)
    got = run_f16(ops.MODE_F16_DACT, ops.ACT_RELU, n16, 0.5, saved=saved, ld_saved=n16)
    assert torch.equal(got, want), (name, "dact saved")
    if N % 16 == 0:
        got = run_f16(ops.MODE_F16_DACT, ops.ACT_RELU, n16, 0.5, saved_bits=R.relu_bits(saved), ld_saved=n16)
        assert torch.equal(got, want), (name, "dact saved_bits")


def test_gemm_column_remap_exact(ops):
    """Column remap (pix*C + c -> grid position) with a partial last N tile (N = 400 = 3*128 + 16), f16 act and dact
    with the bit mask; the grid border the remap skips keeps its sentinel."""
    gen = _gen(11)
    M, K, rmC, OWr, Wg = 300, 136, 16, 5, 7
    N = 5 * OWr * rmC                                       # 5 x 5 pixels of 16 channels
    ldc = 5 * Wg * rmC
    A64, B64 = _ints((M, K), 0.5, gen), _ints((N, K), 0.5, gen)
    A, B = A64.half().contiguous(), B64.half().contiguous()
    ref = R.gemm(A64, B64)
    R.assert_exact_ok(A64.abs() @ B64.abs().t(), what="remap")
    saved = torch.relu(_ints((M, N), 0.6, gen)).half()
    for mode, kw, want in ((ops.MODE_F16_ACT, {}, ref),
                           (ops.MODE_F16_DACT, dict(saved_bits=R.relu_bits(saved), ld_saved=N), ref * (saved.double() > 0))):
        out = torch.full((M, ldc), SENT, dtype=torch.float16, device=DEV)
        ops.gemm(A, B, out, M=M, N=N, K=K, lda=K, ldb=K, ldc=ldc, mode=mode, act=ops.ACT_RELU if kw else ops.ACT_NONE,
                 remap=(rmC, OWr, Wg), **kw)
        torch.cuda.synchronize()
        grid = out.double().view(M, 5, Wg, rmC)
        assert torch.equal(grid[:, :, :OWr].reshape(M, N), want), ("remap", mode)
        assert torch.all(grid[:, :, OWr:] == SENT), ("remap border", mode)


@pytest.mark.parametrize("max_ctas", [1, 2, 3])
def test_gemm_kmajor_ring_wraps(ops, max_ctas):
    """max_ctas = 1 / 2 / 3: each persistent CTA walks dozens of (M, N) tiles x 49 k-blocks, so the 4-stage mbarrier
    ring of the 256-wide N tile wraps hundreds of times; bit-identical to the exact reference at every CTA count."""
    gen = _gen(5)
    M, N, K = 2049, 512, 3136
    BN = gemm_bn(N, False)
    kb = _cdiv(K, 64)
    per_cta = gemm_kblocks_per_cta(_cdiv(M, 128) * _cdiv(N, BN), kb, max_ctas)
    assert BN == 256 and per_cta > 2 * gemm_stages(BN) * 10, per_cta
    p = _density(K)
    A64, B64 = _ints((M, K), p, gen), _ints((N, K), p, gen)
    ref = R.gemm(A64, B64)
    R.assert_exact_ok(A64.abs() @ B64.abs().t(), what="ring")
    A, B = A64.half().contiguous(), B64.half().contiguous()
    C = torch.full((M, N), SENT, dtype=torch.float32, device=DEV)
    ops.gemm(A, B, C, M=M, N=N, K=K, lda=K, ldb=K, ldc=N, mode=ops.MODE_F32_STORE, max_ctas=max_ctas)
    torch.cuda.synchronize()
    assert torch.equal(C.double(), ref)


# ------------------------------------------------------------------------------------------ ops.gemm, MN-major split-K
MNMAJOR = [("BN64_N33", 100, 33), ("BN128_N100", 70, 100), ("BN256_N256", 130, 256)]


@pytest.mark.parametrize("Kred", [1, 63, 65, 20000])
@pytest.mark.parametrize("name,M,N", MNMAJOR, ids=[c[0] for c in MNMAJOR])
def test_gemm_mnmajor_splitk_exact(ops, name, M, N, Kred):
    """C += alpha A^T B over Kred reduction rows with split_k in {1, 2, 3, kb_total, kb_total + 5} (the last clamps to
    kb_total), accumulating into a non-zero C; all splits bit-identical to the exact reference.  At Kred = 20000 also
    max_ctas = 1 / 2 / 3 (hundreds of k-blocks per CTA: the ring wraps)."""
    gen = _gen(M + N + Kred)
    kb_total = _cdiv(Kred, 64)
    splits = sorted({1, 2, 3, kb_total, kb_total + 5})
    ends = [Kred]
    for sk in splits:
        per, ns = fill_splits(kb_total, sk)
        ends += [min((i + 1) * per * 64, Kred) for i in range(ns)]
    rows = R.probe_rows(Kred, tile=128, kblock=64, ends=ends, n_random=32, seed=Kred)
    lda, ldb = _pad8(M) + 8, _pad8(N) + 8
    A64 = R.rows_only(_ints((Kred, M), 0.5, gen), rows)
    B64 = _ints((Kred, N), 0.5, gen)
    A = _padded16(Kred, M, lda, NAN16, extra_rows=7)
    B = _padded16(Kred, N, ldb, NAN16, extra_rows=7)
    A[:Kred, :M], B[:Kred, :N] = A64.half(), B64.half()
    R.assert_exact_ok(A64.abs().t() @ B64.abs(), what=name)
    C0 = _ints((M, N), 0.7, gen, -5, 5)
    want = C0 + 0.25 * (A64.t() @ B64)
    runs = [(sk, 0) for sk in splits] + ([(1, mc) for mc in (1, 2, 3)] if Kred == 20000 else [])
    first = None
    for sk, mc in runs:
        if mc:
            per_cta = gemm_kblocks_per_cta(_cdiv(M, 128) * _cdiv(N, gemm_bn(N, True)), kb_total, mc)
            assert per_cta > 2 * gemm_stages(gemm_bn(N, True)), per_cta
        C = torch.full((M + 2, N + 3), SENT, dtype=torch.float32, device=DEV)
        C[:M, :N] = C0.float()
        ops.gemm(A, B, C, M=M, N=N, K=Kred, lda=lda, ldb=ldb, ldc=N + 3, mn_major=True, mode=ops.MODE_F32_ATOMIC,
                 alpha=0.25, split_k=sk, max_ctas=mc)
        torch.cuda.synchronize()
        got = C[:M, :N].double()
        assert torch.equal(got, want), (name, Kred, sk, mc, float((got - want).abs().max()))
        assert torch.all(C[:M, N:] == SENT) and torch.all(C[M:] == SENT), (name, "write outside")
        first = got if first is None else first
        assert torch.equal(got, first)                       # every split / CTA count gives the same bits


# ------------------------------------------------------------------------------------------ ops.conv_gemm forward
CONV_FWD = [
    # name, B, H, W, C, R, S, sh, sw, ph, pw, N
    ("c16_3x3_s1_pad1_zero_tile", 3, 13, 11, 16, 3, 3, 1, 1, 1, 1, 32),
    ("c16_5x5_s2_pad2_zero_tile", 2, 21, 19, 16, 5, 5, 2, 2, 2, 2, 64),
    ("c32_3x3_s2_pad1_zero_tile", 3, 15, 17, 32, 3, 3, 2, 2, 1, 1, 64),
    ("c64_4x4_s2_pad1", 4, 21, 21, 64, 4, 4, 2, 2, 1, 1, 64),
    ("c64_1x1_s1_N128", 2, 9, 7, 64, 1, 1, 1, 1, 0, 0, 128),
    ("c16_8x2_s4x1_superpixel", 5, 84, 21, 16, 8, 2, 4, 1, 0, 0, 32),
    ("c32_4x4_s4_N100_partial_cols", 3, 23, 23, 32, 4, 4, 4, 4, 0, 0, 100),
    ("c64_3x3_s1_N192_two_ntiles", 2, 11, 9, 64, 3, 3, 1, 1, 1, 1, 192),
    ("c16_3x3_s1_ring_wraps", 60, 41, 41, 16, 3, 3, 1, 1, 1, 1, 32),
]


@pytest.mark.parametrize("name,B,H,W,C,Rr,S,sh,sw,ph,pw,N", CONV_FWD, ids=[c[0] for c in CONV_FWD])
def test_conv_gemm_forward_exact(ops, name, B, H, W, C, Rr, S, sh, sw, ph, pw, N):
    """Implicit TMA-im2col convolution, relu + bias epilogue: resident weights (when they fit) and streamed weights
    (split_k = -1) both equal the float64 convolution; taps*C % 64 != 0 reaches the zero weight tile of the partial
    last stage; odd H / W and SAME-style lower padding.  The image past B is NaN and never read."""
    gen = _gen(B * H + C * N)
    OH, OW = (H + 2 * ph - Rr) // sh + 1, (W + 2 * pw - S) // sw + 1
    taps, K = Rr * S, Rr * S * C
    x64 = _ints((B, H, W, C), 0.5, gen)
    x = torch.full((B + 1, H, W, C), NAN16, dtype=torch.float16, device=DEV)
    x[:B] = x64.half()
    ldb = _pad8(K) + 8
    w64 = _ints((N, K), 0.5, gen)
    wt = _padded16(N, K, ldb, NAN16)
    wt[:, :K] = w64.half()
    bias = _ints((N,), 0.7, gen, -3, 3).float()
    P = R.patches(x64, Rr, S, sh, sw, ph, pw, OH, OW)
    ref = torch.relu(0.5 * (P @ w64.t()) + bias.double())
    R.assert_exact_ok(P.abs() @ w64.abs().t(), what=name)
    rows = B * OH * OW
    BN = 128 if N > 64 else 64 if N > 32 else 32
    resident = _cdiv(N, BN) == 1 and taps * BN * C * 2 <= 80 * 1024
    kb = _cdiv(taps, 64 // C)
    if name.endswith("ring_wraps"):
        per_cta = _cdiv(_cdiv(rows, 128), min(_cdiv(rows, 128), _sms())) * kb
        assert per_cta > 2 * 8, per_cta                     # > 2 x the stages of either weight path
    for split in ((1, -1) if resident else (-1,)):
        out = torch.full((rows + 2, N), SENT, dtype=torch.float16, device=DEV)
        ops.conv_gemm(x, B, H, W, C, Rr, S, sh, sw, ph, pw, OH, OW, wt, ldb, out, N, N, 0, ops.MODE_F16_ACT,
                      act=ops.ACT_RELU, alpha=0.5, bias=bias, split_k=split)
        torch.cuda.synchronize()
        got = out[:rows].double()
        assert torch.equal(got, ref), (name, "resident" if split == 1 else "streamed", float((got - ref).abs().max()))
        assert torch.all(out[rows:] == SENT), (name, "rows past M")


# ------------------------------------------------------------------------------------------ ops.conv_gemm wgrad
CONV_WGRAD = [
    # name, B, H, W, C, R, S, sh, sw, ph, pw, N   (last M tile: taps*C % 128 rows = fewer than 128/C taps)
    ("c64_3x3_last_tile_1of2_taps", 6, 11, 9, 64, 3, 3, 1, 1, 1, 1, 64),
    ("c32_3x3_s2_last_tile_1of4_taps", 5, 15, 13, 32, 3, 3, 2, 2, 0, 0, 32),
    ("c16_5x5_last_tile_1of8_taps_N100", 4, 13, 13, 16, 5, 5, 1, 1, 2, 2, 100),
]


@pytest.mark.parametrize("name,B,H,W,C,Rr,S,sh,sw,ph,pw,N", CONV_WGRAD, ids=[c[0] for c in CONV_WGRAD])
def test_conv_gemm_wgrad_exact(ops, name, B, H, W, C, Rr, S, sh, sw, ph, pw, N):
    """out[taps*C, N] += alpha patches^T dz with split_k in {1, 3, kb_total, kb_total + 5}, into a non-zero output;
    dz nonzero at probe rows; its pitch padding is NaN."""
    gen = _gen(B * 31 + N)
    OH, OW = (H + 2 * ph - Rr) // sh + 1, (W + 2 * pw - S) // sw + 1
    K, rows = Rr * S * C, B * OH * OW
    kb_total = _cdiv(rows, 64)
    splits = sorted({1, 3, kb_total, kb_total + 5})
    ends = []
    for sk in splits:
        per, ns = fill_splits(kb_total, sk)
        ends += [min((i + 1) * per * 64, rows) for i in range(ns)]
    x64 = _ints((B, H, W, C), 0.5, gen)
    x = x64.half().contiguous()
    ld = _pad8(N) + 8
    dz64 = R.rows_only(_ints((rows, N), 0.5, gen), R.probe_rows(rows, tile=128, kblock=64, ends=ends, seed=N))
    dz = _padded16(rows, N, ld, NAN16, extra_rows=3)
    dz[:rows, :N] = dz64.half()
    P = R.patches(x64, Rr, S, sh, sw, ph, pw, OH, OW)
    R.assert_exact_ok(P.abs().t() @ dz64.abs(), what=name)
    G0 = _ints((K, N), 0.7, gen, -5, 5)
    want = G0 + 0.25 * (P.t() @ dz64)
    assert K % 128 and (K % 128) < 128, "the last M tile is partial"
    for sk in splits:
        G = torch.full((K + 1, N), SENT, dtype=torch.float32, device=DEV)
        G[:K] = G0.float()
        ops.conv_gemm(x, B, H, W, C, Rr, S, sh, sw, ph, pw, OH, OW, dz, ld, G, N, N, 1, ops.MODE_F32_ATOMIC, alpha=0.25,
                      split_k=sk)
        torch.cuda.synchronize()
        assert torch.equal(G[:K].double(), want), (name, sk, float((G[:K].double() - want).abs().max()))
        assert torch.all(G[K:] == SENT), (name, "rows past taps*C")


def test_conv_gemm_pixel_shuffle_dgrad_exact(ops):
    """dx = conv_transpose(dz, W) * relu'(h_in) through the pixel-shuffle epilogue with H, W not multiples of the
    stride (21 x 19, 3x3 filter, stride 2): the GEMM rows of the last grid row / column scatter partly outside the
    image and must be dropped.  The image past B keeps its sentinel."""
    gen = _gen(21)
    B, H, W, Cin, Cout, rf, s = 3, 21, 19, 16, 32, 3, 2
    OHc, OWc = (H - rf) // s + 1, (W - rf) // s + 1
    w64 = _ints((rf, rf, Cin, Cout), 0.6, gen)
    dz64 = _ints((B, OHc, OWc, Cout), 0.6, gen)
    h_in = _ints((B, H, W, Cin), 0.7, gen).half()
    An = -(-rf // s)
    ldw = An * An * Cout
    wdg = torch.zeros(s * s * Cin, ldw, dtype=torch.float16, device=DEV)
    ops.dgrad_weights(w64.float().contiguous(), wdg, rf, rf, Cin, Cout, s, ldw)
    dx = torch.full((B + 1, H, W, Cin), SENT, dtype=torch.float16, device=DEV)
    ops.conv_gemm(dz64.half().contiguous(), B, OHc, OWc, Cout, An, An, 1, 1, An - 1, An - 1, -(-H // s), -(-W // s), wdg,
                  ldw, dx, 0, s * s * Cin, 0, ops.MODE_F16_SHUFFLE, act=ops.ACT_RELU, saved=h_in, shuffle=(H, W, Cin, s))
    torch.cuda.synchronize()
    R.assert_exact_ok(R.conv2d_dgrad(dz64.abs(), w64.abs(), H, W, (s, s), (0, 0)), what="shuffle")
    want = R.conv2d_dgrad(dz64, w64, H, W, (s, s), (0, 0)) * (h_in.double() > 0)
    assert torch.equal(dx[:B].double(), want), float((dx[:B].double() - want).abs().max())
    assert torch.all(dx[B:] == SENT)


# ------------------------------------------------------------------------------------------ ops.conv_shift_fwd
def _shift_taps(k, Wg, kx):
    """Row shifts of a k x k filter over a grid of width Wg: all k*k taps, or (kx = k) one per filter row."""
    return [a * Wg for a in range(k)] if kx > 1 else [a * Wg + b for a in range(k) for b in range(k)]


SHIFT_FWD = [
    # name, B, Hg, Wg, C, N, k, omap ("compact" / "grid" / "s2d"), bits
    ("c64_n32_span32_limit", 3, 9, 31, 64, 32, 2, "grid", False),
    ("c64_n64_3x3_bits", 5, 11, 11, 64, 64, 3, "compact", True),
    ("c64_n128_2x2", 4, 9, 13, 64, 128, 2, "compact", True),
    ("c128_n32_span16_limit", 3, 11, 15, 128, 32, 2, "grid", False),
    ("c128_n64_2x2_bits", 4, 10, 10, 128, 64, 2, "compact", True),
    ("c64_n32_s2d_out", 3, 21, 21, 64, 32, 2, "s2d", True),
    ("c64_n32_many_tiles_per_cta", 400, 17, 31, 64, 32, 2, "compact", True),
    ("c128_n128_1x1_bits", 3, 10, 10, 128, 128, 1, "compact", True),
    ("c64_n32_16taps_limit", 4, 9, 9, 64, 32, 4, "compact", True),
    ("c128_n32_s2d_out", 3, 15, 15, 128, 32, 2, "s2d", True),
]


@pytest.mark.parametrize("name,B,Hg,Wg,C,N,k,omode,bits", SHIFT_FWD, ids=[c[0] for c in SHIFT_FWD])
def test_conv_shift_fwd_exact(ops, name, B, Hg, Wg, C, N, k, omode, bits):
    """Shift-GEMM forward (relu + bias, alpha 0.5) == the float64 k x k VALID convolution: shift spans at the limit
    (32 rows for C = 64, 16 for C = 128), 16 taps, every (C, N) instance, M not a multiple of 128, compact /
    full-grid / space-to-depth output maps and the 1-bit ReLU mask.  Grid positions that are not conv outputs keep their sentinel."""
    gen = _gen(B * Hg * Wg + N)
    OH, OW = Hg - k + 1, Wg - k + 1
    M = B * Hg * Wg
    assert M % 128
    shifts = _shift_taps(k, Wg, 1)
    span = max(shifts) - min(shifts)
    assert span <= (32 if C == 64 else 16)
    K = k * k * C
    x64 = _ints((M, C), 0.5, gen)
    X = torch.full((M + 200, C), NAN16, dtype=torch.float16, device=DEV)
    X[:M] = x64.half()
    w64 = _ints((N, K), 0.5, gen)
    ldw = K + 8
    W = torch.full((N, ldw), NAN16, dtype=torch.float16, device=DEV)
    W[:, :K] = w64.half()
    bias = _ints((N,), 0.7, gen, -3, 3).float()
    full = R.shift_conv(x64, shifts, w64).view(B, Hg, Wg, N)
    R.assert_exact_ok(R.shift_conv(x64.abs(), shifts, w64.abs()), what=name)
    ref = torch.relu(0.5 * full[:, :OH, :OW] + bias.double())
    if name.endswith("many_tiles_per_cta"):
        tiles = _cdiv(M, 128)
        assert _cdiv(tiles, min(tiles, _sms())) > 2 * 6, "tiles per CTA"
    if omode == "compact":
        out = torch.full((B, OH, OW, N), SENT, dtype=torch.float16, device=DEV)
        omap, want = (0, OH * OW * N, OW * N, N, 0, 0), ref
    elif omode == "grid":                                     # full input grid: invalid positions keep the sentinel
        out = torch.full((B, Hg, Wg, N), SENT, dtype=torch.float16, device=DEV)
        omap = (0, Hg * Wg * N, Wg * N, N, 0, 0)
        want = torch.full((B, Hg, Wg, N), SENT, dtype=torch.float64, device=DEV)
        want[:, :OH, :OW] = ref
    else:                                                     # space-to-depth for a following stride-2 layer
        assert OH % 2 == 0 and OW % 2 == 0
        out = torch.full((B, OH // 2, OW // 2, 4 * N), SENT, dtype=torch.float16, device=DEV)
        omap, want = (2, (OH // 2) * (OW // 2) * 4 * N, (OW // 2) * 4 * N, 4 * N, N, 2), R.space_to_depth(ref, 2)
    bo = torch.full((out.numel() // 16,), 0x5A5A, dtype=torch.int16, device=DEV) if bits else None
    ops.conv_shift_fwd(X, B, Hg, Wg, C, W, ldw, N, shifts, OH, OW, out, omap, bias=bias, act=ops.ACT_RELU, alpha=0.5,
                       bits_out=bo)
    torch.cuda.synchronize()
    assert torch.equal(out.double(), want), (name, float((out.double() - want).abs().max()))
    if bits:
        assert torch.equal(bo, R.relu_bits(out)), (name, "bits")


@pytest.mark.parametrize("k,mode,mask", [(3, "grid", "none"), (3, "grid", "bits"), (2, "d2s", "none"), (2, "d2s", "bits")])
def test_conv_shift_dgrad_exact(ops, k, mode, mask):
    """Data gradient: negative shifts (min_shift < 0, so the first tile's TMA zero-fills), masked by the bit array of
    the saved activation's ReLU (smap) or unmasked, mode 0 output on the input grid or mode 1 depth->space into a
    larger grid whose border keeps its sentinel."""
    bits = mask == "bits"
    gen = _gen(k * 10 + bits)
    if mode == "grid":
        B, Hg, Wg, Cdz, Cout = 7, 9, 9, 64, 64
    else:
        B, Hg, Wg, Cdz, Cout = 5, 10, 10, 64, 128
    OH, OW = Hg - k + 1, Wg - k + 1
    M = B * Hg * Wg
    taps = k * k
    shifts = [a * Wg + b for a in range(k) for b in range(k)]
    dY64 = torch.zeros(B, Hg, Wg, Cdz, dtype=torch.float64, device=DEV)
    dY64[:, :OH, :OW] = _ints((B, OH, OW, Cdz), 0.5, gen)
    dY = dY64.half().reshape(M, Cdz)
    wd64 = _ints((Cout, taps * Cdz), 0.5, gen)                # [c_in, (t, c_out)]
    saved = torch.relu(_ints((B, Hg, Wg, Cout), 0.6, gen)).half()
    smap = (0, Hg * Wg * Cout, Wg * Cout, Cout, 0, 0)
    full = R.shift_conv(dY64.reshape(M, Cdz), [-s for s in shifts], wd64).view(B, Hg, Wg, Cout)
    R.assert_exact_ok(R.shift_conv(dY64.reshape(M, Cdz).abs(), [-s for s in shifts], wd64.abs()), what="dgrad")
    dx = 0.5 * full * (saved.double() > 0) if bits else 0.5 * full
    if mode == "grid":
        out = torch.full((B, Hg, Wg, Cout), SENT, dtype=torch.float16, device=DEV)
        omap, want = smap, dx
    else:                                                     # depth->space: (y, x, (dy, dx, c)) -> (2y+dy, 2x+dx, c)
        Cq = Cout // 4
        Ho = 2 * Hg + 1
        out = torch.full((B, Ho, Ho, Cq), SENT, dtype=torch.float16, device=DEV)
        omap = (1, Ho * Ho * Cq, Ho * Cq, Cq, Cq, 2)
        want = torch.full((B, Ho, Ho, Cq), SENT, dtype=torch.float64, device=DEV)
        want[:, :2 * Hg, :2 * Wg] = R.depth_to_space(dx, 2)
    kw = dict(saved_bits=R.relu_bits(saved)) if bits else {}
    ops.conv_shift_fwd(dY, B, Hg, Wg, Cdz, wd64.half().contiguous(), taps * Cdz, Cout, [-s for s in shifts], Hg, Wg,
                       out, omap, smap=smap, act=ops.ACT_RELU, dact=True, alpha=0.5, **kw)
    torch.cuda.synchronize()
    assert torch.equal(out.double(), want), (k, mode, mask, float((out.double() - want).abs().max()))


def _u8_frames(pool, H, W, C, gen):
    return torch.randint(0, 3, (pool, H, W, C), generator=gen, dtype=torch.uint8).to(DEV)      # 0..2: the bound holds


@pytest.mark.parametrize("B,gather", [(5, False), (300, True), (301, False)])
def test_conv_shift_uint8_forward_exact(ops, B, gather):
    """First layer straight from uint8 frames (gather + cast + space-to-depth in the producer warps): uneven CTA runs
    (num_tiles % grid != 0) and a last CTA whose head unit lies past M; equal to the float64 convolution of the
    space-to-depth'ed frames."""
    gen = _gen(B)
    H = Wd = 84
    C, s, Hg, Wg, N = 4, 4, 21, 21, 32
    M = B * Hg * Wg
    tiles = _cdiv(M, 128)
    grid = min(tiles, _sms())
    assert M % 128 and (B < 10 or tiles % grid), "uneven CTA runs"
    pool = 2 * B + 3
    frames = _u8_frames(pool, H, Wd, C, gen)
    idx = torch.randperm(pool, generator=gen)[:B].to(DEV) if gather else None
    imgs = (frames[idx] if gather else frames[:B]).double()
    x64 = R.space_to_depth(imgs, s).reshape(M, 64)
    shifts = [0, 1, Wg, Wg + 1]
    w64 = _ints((N, 256), 0.5, gen)
    bias = _ints((N,), 0.7, gen, -3, 3).float()
    R.assert_exact_ok(R.shift_conv(x64, shifts, w64.abs()), what="u8")
    ref = torch.relu(0.5 * R.shift_conv(x64, shifts, w64).view(B, Hg, Wg, N)[:, :20, :20] + bias.double())
    out = torch.full((B, 10, 10, 4 * N), SENT, dtype=torch.float16, device=DEV)
    bo = torch.zeros(out.numel() // 16, dtype=torch.int16, device=DEV)
    ops.conv_shift_fwd(None, B, Hg, Wg, 64, w64.half().contiguous(), 256, N, shifts, 20, 20, out,
                       (2, 100 * 4 * N, 10 * 4 * N, 4 * N, N, 2), bias=bias, act=ops.ACT_RELU, alpha=0.5,
                       u8=(frames, idx, H, Wd, C, s), bits_out=bo)
    torch.cuda.synchronize()
    want = R.space_to_depth(ref, 2)
    assert torch.equal(out.double(), want), float((out.double() - want).abs().max())
    assert torch.equal(bo, R.relu_bits(out))


# ------------------------------------------------------------------------------------------ ops.conv_shift_wgrad
SHIFT_WGRAD = [
    # name, B, Hg, Wg, C, N, k, kx, u8
    ("c64_n64_9taps_surplus_chunk", 40, 9, 9, 64, 64, 3, 1, False),
    ("c64_n32_kx3_surplus_chunk", 40, 9, 9, 64, 32, 3, 3, False),
    ("c64_n64_kx2", 37, 10, 12, 64, 64, 2, 2, False),
    ("c128_n32_3x3_surplus_chunks", 20, 11, 15, 128, 32, 3, 1, False),
    ("c128_n64_kx2", 30, 10, 10, 128, 64, 2, 2, False),
    ("u8_n32_4taps", 13, 21, 21, 64, 32, 2, 1, True),
    ("u8_n32_kx2", 13, 21, 21, 64, 32, 2, 2, True),
]


@pytest.mark.parametrize("name,B,Hg,Wg,C,N,k,kx,u8", SHIFT_WGRAD, ids=[c[0] for c in SHIFT_WGRAD])
def test_conv_shift_wgrad_exact(ops, name, B, Hg, Wg, C, N, k, kx, u8):
    """G[taps*C, N] += alpha sum_m X[m + shift_t] dY[m] and the fused bias gradient, over a zero-bordered dY that is
    nonzero at probe rows; rows not a multiple of the k-block, surplus accumulator chunks (taps*kx*KH not a multiple
    of 2*QW), kx = 2 / 3, the uint8 source, and max_ctas in {default, 1, 2, 7} -- all bit-identical."""
    gen = _gen(B * N + k + kx)
    OH, OW = Hg - k + 1, Wg - k + 1
    rows = B * Hg * Wg
    KR = 128 if u8 else 64
    stages = 8 if C == 64 else 6
    qw = 2 if (u8 or N == 64) else 4
    nchunks = k * k * (C // 64)
    assert rows % KR
    if "surplus" in name:
        assert nchunks % (2 * qw), "surplus accumulator chunks"
    kb_total = _cdiv(rows, KR)
    assert kb_total > 2 * stages                              # max_ctas = 1: the ring wraps
    shifts = _shift_taps(k, Wg, kx)
    all_shifts = [a * Wg + b for a in range(k) for b in range(k)]
    ends = []
    for mc in (_sms(), 1, 2, 7):
        per = _cdiv(kb_total, min(mc, kb_total))
        ends += [min((i + 1) * per * KR, rows) for i in range(_cdiv(kb_total, per))]
    pos = torch.arange(rows, device=DEV) % (Hg * Wg)
    valid = ((pos // Wg) < OH) & ((pos % Wg) < OW)
    probe = R.probe_rows(rows, tile=128, kblock=KR, ends=ends, shifts=all_shifts, n_random=64, seed=B, valid=valid)
    dY64 = R.rows_only(_ints((rows, N), 0.6, gen), probe)
    if u8:
        H, Wd = 4 * Hg, 4 * Wg
        frames = _u8_frames(2 * B + 1, H, Wd, 4, gen)
        idx = torch.randperm(2 * B + 1, generator=gen)[:B].to(DEV)
        x64 = R.space_to_depth(frames[idx].double(), 4).reshape(rows, 64)
        X, u8a = None, (frames, idx, H, Wd, 4, 4)
    else:
        x64 = _ints((rows, C), 0.5, gen)
        X, u8a = x64.half().contiguous(), None
    G_ref = R.shift_wgrad(x64, dY64, all_shifts)
    R.assert_exact_ok(R.shift_wgrad(x64.abs(), dY64.abs(), all_shifts), what=name)
    G0 = _ints((k * k * C, N), 0.7, gen, -5, 5)
    b0 = _ints((N,), 0.7, gen, -5, 5)
    wantG = G0 + 0.5 * G_ref
    wantb = b0 + 0.25 * dY64.sum(0)
    dY = dY64.half().contiguous()
    for mc in (0, 1, 2, 7):
        G = torch.full((k * k * C + 2, N), SENT, dtype=torch.float32, device=DEV)
        G[:k * k * C] = G0.float()
        gb = b0.float().clone()
        ops.conv_shift_wgrad(X, rows, C, dY, N, shifts, G, N, alpha=0.5, max_ctas=mc, gbias=gb, alpha_b=0.25, u8=u8a,
                             kx=kx)
        torch.cuda.synchronize()
        got = G[:k * k * C].double()
        assert torch.equal(got, wantG), (name, mc, float((got - wantG).abs().max()))
        assert torch.equal(gb.double(), wantb), (name, mc, "gbias")
        assert torch.all(G[k * k * C:] == SENT), (name, "rows past taps*C")


# ------------------------------------------------------------------------------------------ ops.colsum
@pytest.mark.parametrize("C", [7, 64, 300])
def test_colsum_exact(ops, C):
    """db += alpha * column sums of fp16 rows, at row counts around the per-block row count (64 rows, and where it
    grows past 64: num_sms * 8 * 64) and C not a multiple of 8 (scalar kernel) / above 256 (two column passes)."""
    gen = _gen(C)
    big = _sms() * 8 * 64
    for rows in (1, 63, 64, 65, 129, big - 1, big, big + 1, big + 77):
        ld = _pad8(C) + 8
        probe = R.probe_rows(rows, tile=64, kblock=max(64, _cdiv(rows, _sms() * 8)), n_random=32, seed=rows)
        d64 = R.rows_only(_ints((rows, C), 0.25, gen), probe)
        dz = _padded16(rows, C, ld, NAN16, extra_rows=3)
        dz[:rows, :C] = d64.half()
        R.assert_exact_ok(d64.abs().sum(0), what="colsum")
        b0 = _ints((C,), 0.7, gen, -5, 5)
        db = b0.float().clone()
        ops.colsum(dz, db, rows, C, ld, alpha=0.5)
        torch.cuda.synchronize()
        assert torch.equal(db.double(), b0 + 0.5 * d64.sum(0)), (rows, C)
