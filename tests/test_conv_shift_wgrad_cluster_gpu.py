"""The shift-GEMM weight gradient (csrc/conv_shift.cu conv_shift_wgrad_kernel) at its thread-block-cluster boundaries.

A CTA holds the accumulators of 2*QW 64-row chunks of G; taps*kx*KH chunks need `groups` CTAs per row range.  The
CTAs of one row range may form a cluster of g CTAs (the largest divisor of `groups` up to 8) that loads every X / dY
stage once and multicasts it to all of them: a stage is refilled only after the consumers of every CTA of the cluster
have released it.  They do so when clusters of g tile the SMs (on an H100 at this kernel's shared memory: g = 2;
clusters of 3, 4, 5 or 8 leave SMs idle and the groups run unclustered).  These tests cover group counts of 1, 2, 3,
4, 5, 8 and 9 (three clusters of 3 per row range, were they to tile); per-CTA
k-block counts of 1, fewer than the ring's stages, exactly the stages, and several ring wraps; reduction rows that are
not a multiple of the 64-row k-block; max_ctas in {default, 1, 2, 7}; surplus chunk slots; the fused bias gradient,
which only chunk group 0 adds; and cfg-2's c2 and c3 instances at batches whose last wave of clusters is partial.

Operands are small integers, as in test_wgmma_boundaries_gpu.py: each result is exact and is compared with
torch.equal against float64, so a stage read before it is complete, or overwritten while a peer still reads it, or a
chunk group that drops or repeats rows, changes some output by at least 1.
"""
import pytest
import torch

import _refs as R

pytestmark = pytest.mark.gpu

DEV = "cuda"
SENT = 1234.0
KR = 64                                   # reduction rows per k-block (TMA-fed instances)


@pytest.fixture(scope="module")
def ops():
    from baselines_b200 import ops as _ops
    return _ops


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _ints(shape, density, gen, lo=-2, hi=2):
    return R.small_ints(shape, density, gen, device=DEV, lo=lo, hi=hi)


def _cdiv(a, b):
    return -(-a // b)


def _sms():
    from baselines_b200 import ops
    return ops.num_sms()


def _groups(C, N, shifts, kx):
    """Chunk groups (grid.y) and CTAs per cluster that b200rl_conv_shift_wgrad chooses."""
    qw = 2 if N == 64 else 4
    groups = _cdiv(len(shifts) * kx * (C // 64), 2 * qw)
    g = min(groups, 8)
    while groups % g:
        g -= 1
    return groups, g


def _check(ops, rows, C, N, shifts, kx, gen, valid=None, max_ctas=(0, 1, 2, 7), what=""):
    """G (+ a preset G0) and the fused bias gradient of every max_ctas equal float64, bit for bit."""
    all_shifts = [s + b for s in shifts for b in range(kx)]
    kb_total = _cdiv(rows, KR)
    ends = []
    for mc in max_ctas:
        per = _cdiv(kb_total, min(mc if mc > 0 else _sms(), kb_total))
        ends += [min((i + 1) * per * KR, rows) for i in range(_cdiv(kb_total, per))]
    # probes at every k-block (its first and last row, and the rows whose largest shift reads across its end); every
    # shift's probes would push |X|^T |dY| past the exact bound at 16-36 shifts
    probe = R.probe_rows(rows, tile=KR, kblock=KR, ends=ends, shifts=[max(all_shifts)], n_random=64, seed=rows,
                         valid=valid)
    dY64 = R.rows_only(_ints((rows, N), 0.5, gen), probe)
    x64 = _ints((rows, C), 0.5, gen)
    G_ref = R.shift_wgrad(x64, dY64, all_shifts)
    R.assert_exact_ok(R.shift_wgrad(x64.abs(), dY64.abs(), all_shifts), what=what)
    K = len(all_shifts) * C
    G0 = _ints((K, N), 0.7, gen, -5, 5)
    b0 = _ints((N,), 0.7, gen, -5, 5)
    wantG = G0 + 0.5 * G_ref
    wantb = b0 + 0.25 * dY64.sum(0)
    X, dY = x64.half().contiguous(), dY64.half().contiguous()
    for mc in max_ctas:
        G = torch.full((K + 2, N), SENT, dtype=torch.float32, device=DEV)
        G[:K] = G0.float()
        gb = b0.float().clone()
        ops.conv_shift_wgrad(X, rows, C, dY, N, shifts, G, N, alpha=0.5, max_ctas=mc, gbias=gb, alpha_b=0.25, kx=kx)
        torch.cuda.synchronize()
        got = G[:K].double()
        assert torch.equal(got, wantG), (what, mc, float((got - wantG).abs().max()))
        assert torch.equal(gb.double(), wantb), (what, mc, "gbias: chunk group 0 alone adds it")
        assert torch.all(G[K:] == SENT), (what, mc, "rows past taps*C")


def _square(k, Wg, kx):
    return [a * Wg for a in range(k)] if kx > 1 else [a * Wg + b for a in range(k) for b in range(k)]


# name, C (X channels), N (dY channels), shifts (filter rows when kx > 1), kx, groups, CTAs per cluster
CLUSTERS = [
    ("cluster1_c64_n64_2x2_kx2", 64, 64, _square(2, 10, 2), 2, 1, 1),
    ("cluster2_c128_n64_2x2_kx2", 128, 64, _square(2, 10, 2), 2, 2, 2),               # cfg-2's c2
    ("cluster3_c64_n64_3x3_kx3_surplus", 64, 64, _square(3, 9, 3), 3, 3, 3),          # cfg-2's c3: 9 of 12 slots
    ("cluster3_c128_n32_3x3_surplus", 128, 32, _square(3, 11, 1), 1, 3, 3),           # 18 of 24 slots
    ("cluster4_c64_n64_4x4", 64, 64, _square(4, 9, 1), 1, 4, 4),
    ("cluster5_c128_n64_3x3_surplus", 128, 64, _square(3, 11, 1), 1, 5, 5),           # 18 of 20 slots
    ("cluster8_c128_n64_4x4", 128, 64, _square(4, 9, 1), 1, 8, 8),
    ("three_clusters3_c64_n64_12rows_kx3", 64, 64, [0, 2, 5, 7, 10, 12, 15, 17, 20, 22, 25, 30], 3, 9, 3),
]


@pytest.mark.parametrize("per_cta", [1, 3, "stages", "wraps"])
@pytest.mark.parametrize("name,C,N,shifts,kx,groups,g", CLUSTERS, ids=[c[0] for c in CLUSTERS])
def test_wgrad_cluster_kblocks_per_cta_exact(ops, name, C, N, shifts, kx, groups, g, per_cta):
    """With max_ctas = 7 every CTA but the last runs `per_cta` k-blocks (1, 3, the ring's stages, or 3 wraps of the
    ring + 2) and the last one fewer; max_ctas = 1 / 2 / default give one long, two, and many row ranges."""
    assert _groups(C, N, shifts, kx) == (groups, g), _groups(C, N, shifts, kx)
    stages = 8 if C == 64 else 6
    per = {"stages": stages, "wraps": 3 * stages + 2}.get(per_cta, per_cta)
    kb_total = 7 if per == 1 else 7 * per - 1
    rows = kb_total * KR - 17                                 # not a multiple of the k-block
    assert _cdiv(kb_total, 7) == per
    gen = _gen(groups * 1000 + C + N + per)
    _check(ops, rows, C, N, shifts, kx, gen, what=f"{name} per_cta={per}")


# cfg-2's weight-gradient instances on their grids (NatureCNN on 84x84): c2 = 4x4 s2 over the 10x10 space-to-depth
# grid of 128 channels (kx = 2), c3 = 3x3 over 9x9 of 64 (kx = 3); dY is zero outside the valid outputs
CFG2 = [
    # name, Hg, Wg, C, k
    ("c2", 10, 10, 128, 2),
    ("c3", 9, 9, 64, 3),
]


@pytest.mark.parametrize("per_range", [2, 4])
@pytest.mark.parametrize("name,Hg,Wg,C,k", CFG2, ids=[c[0] for c in CFG2])
def test_wgrad_cluster_cfg2_partial_last_wave_exact(ops, name, Hg, Wg, C, k, per_range):
    """B gives kb_total = 1 + (per_range - 1) * SMs k-blocks.  Over one row range per SM (2-CTA clusters that tile
    the SMs, as c2's do on an H100) the row ranges hold 2 or 4 k-blocks, and there are 67 or 100 of them on 132 SMs:
    the last wave holds 1 or 34 of the 66 clusters.  Where clusters do not tile the SMs, one wave of the co-resident
    clusters takes longer row ranges, and a small B leaves part of that wave empty."""
    N = 64
    target = 1 + (per_range - 1) * _sms()
    B = _cdiv((target - 1) * KR + 1, Hg * Wg)
    rows = B * Hg * Wg
    assert _cdiv(rows, KR) == target and rows % KR, (B, rows)
    OH, OW = Hg - k + 1, Wg - k + 1
    pos = torch.arange(rows, device=DEV) % (Hg * Wg)
    valid = ((pos // Wg) < OH) & ((pos % Wg) < OW)
    assert _cdiv(target, _sms()) == per_range
    gen = _gen(B + k)
    _check(ops, rows, C, N, _square(k, Wg, k), k, gen, valid=valid, max_ctas=(0, 7), what=f"{name} B={B}")
