"""Exact tests of the shift-GEMM forward / data-gradient epilogue (csrc/conv_shift.cu, conv_shift_fwd_kernel): the
accumulators leave through a per-warp shared-memory transpose as 16-byte row pieces, and a data gradient's ReLU mask
is staged with its A tile.

Operands are small integers and alpha is 0.5, so every output is exact in fp16 and is compared with torch.equal
against a float64 reference (see test_wgmma_boundaries_gpu.py).  The reference output is scattered through a Python
model of the kernel's address maps into a sentinel-filled buffer, so a misplaced 16-byte piece, row or chunk, and any
write outside the mapped elements, changes some element.  The bit array (bits_out) starts from a sentinel pattern too.
"""
import pytest
import torch

import _refs as R

pytestmark = pytest.mark.gpu

DEV = "cuda"
SENT = 1234.0
SENT_BITS = 0x5A5A


@pytest.fixture(scope="module")
def ops():
    from baselines_b200 import ops as _ops
    return _ops


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _ints(shape, density, gen, lo=-2, hi=2):
    return R.small_ints(shape, density, gen, device=DEV, lo=lo, hi=hi)


def _b_for_tail(Hg, Wg, tail):
    """Smallest batch whose B*Hg*Wg grid rows leave `tail` rows in the last 128-row tile."""
    return next(b for b in range(1, 4096) if (b * Hg * Wg) % 128 == tail)


def _omap(mode, B, vy, vx, N, s):
    """Output map (mode, sN, sY, sX, Cq, s) of mode 0 (a padded NHWC grid with a wider row pitch), 1 (depth->space with
    stride s, Cq = N / s^2, into a grid one larger than s*vy x s*vx) or 2 (space->depth with stride 2)."""
    if mode == 0:
        pitch = N + 16
        return (0, (vy + 1) * vx * pitch, vx * pitch, pitch, 0, 0)
    if mode == 1:
        Cq = N // (s * s)
        Ho, Wo = s * vy + 1, s * vx + 1
        return (1, Ho * Wo * Cq, Wo * Cq, Cq, Cq, s)
    ho, wo = -(-vy // 2), -(-vx // 2)
    return (2, ho * wo * 4 * N, wo * 4 * N, 4 * N, N, 2)


def _offsets(omap, n, y, x, N):
    """Element offsets [rows, N] of output columns 0..N-1 of grid positions (n, y, x) -- the kernel's AddrMap."""
    mode, sN, sY, sX, Cq, s = omap
    col = torch.arange(N, device=DEV)
    if mode == 0:
        return (n * sN + y * sY + x * sX)[:, None] + col
    if mode == 1:
        cls = col // Cq
        return (n * sN + y * s * sY + x * s * sX)[:, None] + ((cls // s) * sY + (cls % s) * sX + col % Cq)[None]
    return (n * sN + (y // s) * sY + (x // s) * sX + ((y % s) * s + x % s) * Cq)[:, None] + col


def _scatter(omap, full, B, Hg, Wg, vy, vx, N):
    """Sentinel buffer holding `full` [B*Hg*Wg, N] at the mapped offsets of the valid positions; also the written mask."""
    m = torch.arange(B * Hg * Wg, device=DEV)
    n, y, x = m // (Hg * Wg), (m // Wg) % Hg, m % Wg
    keep = (y < vy) & (x < vx)
    offs = _offsets(omap, n[keep], y[keep], x[keep], N)
    assert offs.unique().numel() == offs.numel(), "the map must be one-to-one"
    size = (int(offs.max()) + 1 + 64 + 15) // 16 * 16                   # + a tail the kernel must not touch
    want = torch.full((size,), SENT, dtype=torch.float64, device=DEV)
    want[offs.reshape(-1)] = full[keep].reshape(-1)
    written = torch.zeros(size, dtype=torch.bool, device=DEV)
    written[offs.reshape(-1)] = True
    return want, written


def _run(ops, kind, B, Hg, Wg, C, N, shifts, vy, vx, omap, seed):
    """kind: fwd (bias + relu, with bits_out), dgrad_mask (saved_bits of a row-contiguous saved activation), dgrad."""
    gen = _gen(seed)
    M = B * Hg * Wg
    taps = len(shifts)
    X64 = _ints((M, C), 0.5, gen)
    if kind != "fwd":                                        # dY lives on the grid: rows it does not cover are zero
        X64 = X64 * (torch.rand(M, 1, generator=gen).to(DEV) < 0.8)
    W64 = _ints((N, taps * C), 0.5, gen)
    R.assert_exact_ok(R.shift_conv(X64.abs(), shifts, W64.abs()), what=kind)
    full = 0.5 * R.shift_conv(X64, shifts, W64)
    kw = {}
    if kind == "fwd":
        bias = _ints((N,), 0.7, gen, -3, 3).float()
        full = torch.relu(full + bias.double())
        kw = dict(bias=bias, act=ops.ACT_RELU)
    else:
        kw = dict(smap=(0, Hg * Wg * N, Wg * N, N, 0, 0), act=ops.ACT_RELU, dact=True)
        if kind == "dgrad_mask":
            saved = torch.relu(_ints((M, N), 0.6, gen)).half()
            full = full * (saved.double() > 0)
            kw["saved_bits"] = R.relu_bits(saved)
    want, written = _scatter(omap, full, B, Hg, Wg, vy, vx, N)
    out = torch.full(want.shape, SENT, dtype=torch.float16, device=DEV)
    bo = None
    if kind == "fwd":
        bo = torch.full((out.numel() // 16,), SENT_BITS, dtype=torch.int16, device=DEV)
        kw["bits_out"] = bo
    ops.conv_shift_fwd(X64.half().contiguous(), B, Hg, Wg, C, W64.half().contiguous(), taps * C, N, shifts, vy, vx,
                       out, omap, alpha=0.5, **kw)
    torch.cuda.synchronize()
    assert torch.equal(out.double(), want), (kind, float((out.double() - want).abs().nan_to_num(1e9).max()))
    if bo is not None:
        wrote = written.view(-1, 16).all(1)
        assert torch.equal(written.view(-1, 16).any(1), wrote), "16-element words are written whole"
        want_bits = torch.where(wrote, R.relu_bits(want), torch.full_like(bo, SENT_BITS))
        assert torch.equal(bo, want_bits), (kind, "bits")


EPILOGUE = [
    # name, kind, B (or (Hg, Wg, tail) -> the batch leaving `tail` rows in the last tile), Hg, Wg, C, N, k, mode, s
    ("fwd_n32_mode0", "fwd", 3, 11, 11, 64, 32, 2, 0, 1),
    ("fwd_n32_mode1", "fwd", 3, 11, 11, 64, 32, 2, 1, 1),
    ("fwd_n32_mode2", "fwd", 3, 11, 11, 128, 32, 2, 2, 2),
    ("fwd_n64_mode0", "fwd", 4, 10, 13, 128, 64, 2, 0, 1),
    ("fwd_n64_mode1", "fwd", 4, 11, 11, 64, 64, 2, 1, 2),
    ("fwd_n64_mode2", "fwd", 4, 11, 11, 64, 64, 3, 2, 2),
    ("fwd_n128_mode0_cooperative", "fwd", 3, 9, 13, 64, 128, 2, 0, 1),
    ("fwd_n128_mode1_cooperative", "fwd", 3, 11, 11, 64, 128, 2, 1, 2),
    ("fwd_n128_mode2_cooperative_c128", "fwd", 3, 11, 11, 128, 128, 1, 2, 2),
    ("fwd_n64_last_tile_1_row", "fwd", (9, 9, 1), 9, 9, 64, 64, 3, 0, 1),
    ("dgrad_mask_n32_last_tile_1_row", "dgrad_mask", (9, 9, 1), 9, 9, 64, 32, 3, 0, 1),
    ("dgrad_mask_n32_mode1_tail_rows", "dgrad_mask", (9, 9, 37), 9, 9, 64, 32, 2, 1, 1),
    ("dgrad_mask_n64_last_tile_1_row", "dgrad_mask", (9, 9, 1), 9, 9, 64, 64, 3, 1, 1),
    ("dgrad_mask_n64_mode2_tail_rows", "dgrad_mask", (9, 9, 3), 9, 9, 128, 64, 2, 2, 2),
    ("dgrad_mask_n128_mode1", "dgrad_mask", (11, 11, 5), 11, 11, 64, 128, 2, 1, 2),
    ("dgrad_mask_n128_mode0_c128", "dgrad_mask", (9, 9, 1), 9, 9, 128, 128, 1, 0, 1),
    ("dgrad_mask_n128_mode2", "dgrad_mask", 6, 10, 10, 64, 128, 2, 2, 2),
    ("dgrad_nomask_n32_mode2", "dgrad", 3, 10, 10, 64, 32, 2, 2, 2),
    ("dgrad_nomask_n64_mode0_c128", "dgrad", (9, 9, 1), 9, 9, 128, 64, 2, 0, 1),
    ("dgrad_nomask_n128_mode1", "dgrad", 5, 10, 10, 64, 128, 2, 1, 2),
]


@pytest.mark.parametrize("name,kind,B,Hg,Wg,C,N,k,mode,s", EPILOGUE, ids=[c[0] for c in EPILOGUE])
def test_conv_shift_epilogue_exact(ops, name, kind, B, Hg, Wg, C, N, k, mode, s):
    """Every (BN, KH, DACT) instance through omap modes 0 / 1 / 2: forwards with bias, ReLU and bits_out, data
    gradients with the staged mask (a last tile of 1 row, tails of 4- and 8-byte mask rows) and without it.  Every
    grid has Hg*Wg rows per sample, not a multiple of 128, so tiles cross sample boundaries."""
    if isinstance(B, tuple):
        B = _b_for_tail(*B)
    M = B * Hg * Wg
    assert M % 128, "M not a multiple of 128"
    fwd = kind == "fwd"
    shifts = [a * Wg + b for a in range(k) for b in range(k)]
    if not fwd:
        shifts = [-t for t in shifts]
    vy, vx = (Hg - k + 1, Wg - k + 1) if fwd else (Hg, Wg)
    _run(ops, kind, B, Hg, Wg, C, N, shifts, vy, vx, _omap(mode, B, vy, vx, N, s), seed=M + N + mode)


@pytest.mark.parametrize("layer,B", [("c2", 512), ("c2", 345), ("c3", 512), ("c3", 345)])
def test_conv_shift_dgrad_cfg2_shapes(ops, layer, B):
    """NatureCNN's two data gradients as nn.Tower issues them: c2 (dY 10x10x64 -> 128 = 2x2x32 channels, 4 taps,
    depth->space into c1's 21x21x32 grid) and c3 (dY 9x9x64 -> 64 channels, 9 taps, into c2's 10x10x64 grid), masked
    by the saved activation's bits.  B = 512 (a partial last wave of tiles) and B = 345 (a partial wave and a partial
    last tile)."""
    if layer == "c2":
        Hg = Wg = 10
        N, k, s, Hp = 128, 2, 2, 21
    else:
        Hg = Wg = 9
        N, k, s, Hp = 64, 3, 1, 10
    Cq = N // (s * s)
    omap = (1, Hp * Hp * Cq, Hp * Cq, Cq, Cq, s)
    shifts = [-(a * Wg + b) for a in range(k) for b in range(k)]
    _run(ops, "dgrad_mask", B, Hg, Wg, 64, N, shifts, Hg, Wg, omap, seed=B + N)


def test_conv_shift_saved_bits_need_row_contiguous_map(ops):
    """The mask is staged as one contiguous run per tile: saved_bits with any other saved map is refused."""
    B, Hg, Wg, C, N = 2, 9, 9, 64, 64
    M = B * Hg * Wg
    dY = torch.zeros(M, C, dtype=torch.float16, device=DEV)
    W = torch.zeros(N, C, dtype=torch.float16, device=DEV)
    out = torch.zeros(M, N + 16, dtype=torch.float16, device=DEV)
    omap = (0, Hg * Wg * (N + 16), Wg * (N + 16), N + 16, 0, 0)
    bits = torch.zeros(M * (N + 16) // 16 + 8, dtype=torch.int16, device=DEV)
    for smap in [omap, (1, Hg * Wg * N, Wg * N, N, N, 1), (0, Hg * Wg * N, Wg * N + 16, N, 0, 0)]:
        with pytest.raises(RuntimeError, match="row-contiguous"):
            ops.conv_shift_fwd(dY, B, Hg, Wg, C, W, C, N, [0], Hg, Wg, out, omap, smap=smap, act=ops.ACT_RELU,
                               dact=True, saved_bits=bits)
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        ops.conv_shift_fwd(dY, B, Hg, Wg, C, W, C, N, [0], Hg, Wg, out, omap, smap=(0, Hg * Wg * N, Wg * N, N, 0, 0),
                           act=ops.ACT_RELU, dact=True, saved_bits=bits[1:])
    # the same call with the row-contiguous map runs
    ops.conv_shift_fwd(dY, B, Hg, Wg, C, W, C, N, [0], Hg, Wg, out, omap, smap=(0, Hg * Wg * N, Wg * N, N, 0, 0),
                       act=ops.ACT_RELU, dact=True, saved_bits=bits)
    torch.cuda.synchronize()
    assert float(out.abs().max()) == 0.0
