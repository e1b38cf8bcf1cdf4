"""Exact-arithmetic cases of the K-major plain wgmma GEMM's staged epilogue and ping-pong schedule (csrc/gemm_wgmma.cu).

As in test_wgmma_boundaries_gpu.py, operands are small integers with max(|A| @ |B|) <= 2048, so every fp32 partial sum
and every fp16 output is exact and results are compared with torch.equal against float64.  Cases cover the ping-pong
tile counts per CTA (through max_ctas), M off the 64 / 128 row grid, NatureCNN's fc1 data-gradient shape (column remap
into the zero-bordered grid, staged ReLU bit mask, the partial last N tile of 3136 = 24.5 x 128), head data gradients
with the fp16 saved activation (K = 7 and 16), and outputs that take the element-wise fallback store (an odd ldc, a
base that is not 16-byte aligned).  Regions the kernel must not write hold a sentinel.
"""
import pytest
import torch

import _refs as R

pytestmark = pytest.mark.gpu

DEV = "cuda"
SENT = 1234.0


@pytest.fixture(scope="module")
def ops():
    from baselines_b200 import ops as _ops
    return _ops


def _ints(shape, density, gen, lo=-2, hi=2):
    return R.small_ints(shape, density, gen, device=DEV, lo=lo, hi=hi)


def _operands(M, N, K, seed, density=None):
    gen = torch.Generator().manual_seed(seed)
    p = density or min(0.8, (150.0 / (2.25 * K)) ** 0.5)
    A64, B64 = _ints((M, K), p, gen), _ints((N, K), p, gen)
    R.assert_exact_ok(A64.abs() @ B64.abs().t())
    return gen, A64, B64, A64.half().contiguous(), B64.half().contiguous(), R.gemm(A64, B64)


def _f16_out(M, ldc, offset=0, extra_rows=3):
    buf = torch.full(((M + extra_rows) * ldc + offset + 8,), SENT, dtype=torch.float16, device=DEV)
    return buf, buf[offset:offset + (M + extra_rows) * ldc].view(M + extra_rows, ldc)


def _check_f16(buf, C, M, N, want, what):
    torch.cuda.synchronize()
    assert torch.equal(C[:M, :N].double(), want), (what, float((C[:M, :N].double() - want).abs().max()))
    written = torch.zeros_like(buf, dtype=torch.bool)
    base = C.storage_offset() - buf.storage_offset()
    idx = base + torch.arange(M, device=DEV)[:, None] * C.stride(0) + torch.arange(N, device=DEV)[None, :]
    written[idx.reshape(-1)] = True
    assert torch.all(buf[~written] == SENT), (what, "write outside [M, N]")


@pytest.mark.parametrize("max_ctas", [1, 2, 3, 5, 0])
@pytest.mark.parametrize("N", [64, 128, 256])
def test_pingpong_tile_counts(ops, N, max_ctas):
    """5 M tiles x N/BN tiles over 1, 2, 3, 5 or all CTAs: per-CTA tile counts 1 .. 5 (odd, even, a CTA whose second
    group has none), for ReLU + bias, the saved fp16 mask, the bit mask and the fp32 store."""
    M, K = 5 * 128 - 3, 200
    gen, A64, B64, A, B, ref = _operands(M, N, K, seed=N + max_ctas)
    bias = _ints((N,), 0.7, gen, -3, 3).float()
    buf, C = _f16_out(M, N)
    ops.gemm(A, B, C, M=M, N=N, K=K, lda=K, ldb=K, ldc=N, bias=bias, mode=ops.MODE_F16_ACT, act=ops.ACT_RELU,
             alpha=0.5, max_ctas=max_ctas)
    _check_f16(buf, C, M, N, torch.relu(0.5 * ref + bias.double()), "relu+bias")
    saved = torch.relu(_ints((M, N), 0.6, gen)).half()
    want = 0.5 * ref * (saved.double() > 0)
    for kw in (dict(saved=saved), dict(saved_bits=R.relu_bits(saved))):
        buf, C = _f16_out(M, N)
        ops.gemm(A, B, C, M=M, N=N, K=K, lda=K, ldb=K, ldc=N, ld_saved=N, mode=ops.MODE_F16_DACT, act=ops.ACT_RELU,
                 alpha=0.5, max_ctas=max_ctas, **kw)
        _check_f16(buf, C, M, N, want, "dact " + next(iter(kw)))
    C32 = torch.full((M + 3, N + 4), SENT, dtype=torch.float32, device=DEV)
    ops.gemm(A, B, C32, M=M, N=N, K=K, lda=K, ldb=K, ldc=N + 4, bias=bias, mode=ops.MODE_F32_STORE, alpha=0.25,
             max_ctas=max_ctas)
    torch.cuda.synchronize()
    assert torch.equal(C32[:M, :N].double(), 0.25 * ref + bias.double())
    assert torch.all(C32[:M, N:] == SENT) and torch.all(C32[M:] == SENT)


@pytest.mark.parametrize("M", [1, 63, 65, 129, 200, 4095])
def test_rows_off_the_tile_grid(ops, M):
    """M not a multiple of 64 or 128: the rows past M of the last tile are computed and dropped."""
    N, K = 128, 96
    gen, A64, B64, A, B, ref = _operands(M, N, K, seed=M)
    saved = torch.relu(_ints((M, N), 0.6, gen)).half()
    buf, C = _f16_out(M, N)
    ops.gemm(A, B, C, M=M, N=N, K=K, lda=K, ldb=K, ldc=N, saved_bits=R.relu_bits(saved), ld_saved=N,
             mode=ops.MODE_F16_DACT, act=ops.ACT_RELU)
    _check_f16(buf, C, M, N, ref * (saved.double() > 0), "dact bits")
    buf, C = _f16_out(M, N)
    ops.gemm(A, B, C, M=M, N=N, K=K, lda=K, ldb=K, ldc=N, mode=ops.MODE_F16_ACT, act=ops.ACT_NONE)
    _check_f16(buf, C, M, N, ref, "none")


@pytest.mark.parametrize("M", [300, 4096])
def test_fc1_dgrad_shape(ops, M):
    """NatureCNN's fc1 data gradient: N = 3136 = 7 x 7 pixels x 64 channels (24.5 N tiles of 128), K = 512, stored
    into the zero-bordered 9 x 9 grid through the column remap, masked by c3's ReLU bits; the border keeps its
    sentinel."""
    N, K, rmC, OW, Wg = 3136, 512, 64, 7, 9
    gen, A64, B64, A, B, ref = _operands(M, N, K, seed=M)
    saved = torch.relu(_ints((M, N), 0.6, gen)).half()
    ldc = Wg * Wg * rmC
    out = torch.full((M, ldc), SENT, dtype=torch.float16, device=DEV)
    ops.gemm(A, B, out, M=M, N=N, K=K, lda=K, ldb=K, ldc=ldc, saved_bits=R.relu_bits(saved), ld_saved=N,
             mode=ops.MODE_F16_DACT, act=ops.ACT_RELU, alpha=0.5, remap=(rmC, OW, Wg))
    torch.cuda.synchronize()
    grid = out.double().view(M, Wg, Wg, rmC)
    assert torch.equal(grid[:, :OW, :OW].reshape(M, N), 0.5 * ref * (saved.double() > 0))
    assert torch.all(grid[:, OW:] == SENT) and torch.all(grid[:, :, OW:] == SENT)


@pytest.mark.parametrize("K", [7, 16])
def test_head_dgrad_saved(ops, K):
    """A head's data gradient into fc1: K = 7 or 16 (one k-block), N = 512 (BN = 256, cooperative), the fp16 saved
    activation read as 16-byte pieces; and a 7-wide output with an odd saved pitch (element-wise reads)."""
    M, N = 1000, 512
    gen, A64, B64, A, B, ref = _operands(M, N, K, seed=K, density=0.8)
    lda = (K + 7) // 8 * 8
    Ap = torch.zeros(M, lda, dtype=torch.float16, device=DEV)
    Bp = torch.zeros(N, lda, dtype=torch.float16, device=DEV)
    Ap[:, :K], Bp[:, :K] = A, B
    saved = torch.relu(_ints((M, N), 0.6, gen)).half()
    buf, C = _f16_out(M, N)
    ops.gemm(Ap, Bp, C, M=M, N=N, K=K, lda=lda, ldb=lda, ldc=N, saved=saved, ld_saved=N, mode=ops.MODE_F16_DACT,
             act=ops.ACT_RELU)
    _check_f16(buf, C, M, N, ref * (saved.double() > 0), "head dgrad")
    # N = 7 output, saved with pitch 9: neither 16-byte pieces of the output nor of the saved activation
    N7 = 7
    B7 = Bp[:N7].contiguous()
    saved7 = torch.relu(_ints((M, 9), 0.6, gen)).half()
    buf, C = _f16_out(M, 9)
    ops.gemm(Ap, B7, C, M=M, N=N7, K=K, lda=lda, ldb=lda, ldc=9, saved=saved7, ld_saved=9, mode=ops.MODE_F16_DACT,
             act=ops.ACT_RELU)
    _check_f16(buf, C, M, N7, ref[:, :N7] * (saved7[:, :N7].double() > 0), "N7 dact")


@pytest.mark.parametrize("offset,ldc", [(0, 131), (1, 136), (4, 136), (3, 133)])
def test_fallback_store(ops, offset, ldc):
    """Outputs whose rows are not 16-byte aligned (odd ldc, or a base 2 / 8 bytes past a 16-byte boundary): the
    element-wise store, for f16 ReLU + bias and the fp32 store."""
    M, N, K = 257, 130, 64
    gen, A64, B64, A, B, ref = _operands(M, N, K, seed=offset * 1000 + ldc)
    bias = _ints((N,), 0.7, gen, -3, 3).float()
    buf, C = _f16_out(M, ldc, offset=offset)
    ops.gemm(A, B, C, M=M, N=N, K=K, lda=K, ldb=K, ldc=ldc, bias=bias, mode=ops.MODE_F16_ACT, act=ops.ACT_RELU)
    _check_f16(buf, C, M, N, torch.relu(ref + bias.double()), "f16 fallback")
    buf32 = torch.full(((M + 3) * ldc + offset + 8,), SENT, dtype=torch.float32, device=DEV)
    C32 = buf32[offset:offset + (M + 3) * ldc].view(M + 3, ldc)
    ops.gemm(A, B, C32, M=M, N=N, K=K, lda=K, ldb=K, ldc=ldc, bias=bias, mode=ops.MODE_F32_STORE)
    _check_f16(buf32, C32, M, N, ref + bias.double(), "f32 fallback")
