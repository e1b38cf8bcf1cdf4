"""The shift-GEMM weight gradient (csrc/conv_shift.cu conv_shift_wgrad_kernel) at every chunk count a warpgroup runs.

G's taps*kx*KH 64-row chunks are dealt to the 2 * groups warpgroups of a row range (groups = chunk count over 2*QW,
QW = 4 for N = 32, 3 for N = 64 over 64 channels, 2 for N = 64 over 128) in contiguous runs whose lengths differ by
at most one, so a warpgroup runs 0 .. QW chunks: c3's 9 chunks split 3 + 2 | 2 + 2 over one 2-CTA cluster.  Each
count has its own MMA loop (with two alternating accumulator buffers where registers allow, one for QW = 3).

These tests cover chunk counts 1-9 over 64 channels (N = 64 and 32) and 2-10 over 128, so every per-warpgroup count
0 .. QW, one and two chunk groups, clustered and unclustered launches; per-CTA k-block counts of 1, fewer than the
ring's stages, exactly the stages and several ring wraps; reduction rows that are not a multiple of the k-block;
max_ctas in {default, 1, 2, 7}; the fused bias gradient; and cfg-2's c2 / c3 at batches whose last wave is partial,
and at the DQN trunk's B = 512.

Operands are small integers (test_conv_shift_wgrad_cluster_gpu._check): every result is exact and compared with
torch.equal against float64, so a chunk computed twice, dropped, or given to the wrong G rows changes an output.
"""
import pytest
import torch

from test_conv_shift_wgrad_cluster_gpu import KR, _cdiv, _check, _gen, _square

pytestmark = pytest.mark.gpu

DEV = "cuda"
SHIFTS = [0, 1, 2, 5, 9, 10, 11, 20, 32]      # single taps (kx = 1), all within the 32-row shift span


@pytest.fixture(scope="module")
def ops():
    from baselines_b200 import ops as _ops
    return _ops


def _sms():
    from baselines_b200 import ops
    return ops.num_sms()


def _plan(C, N, nchunks):
    """Chunk groups and the per-warpgroup chunk counts b200rl_conv_shift_wgrad and the kernel choose."""
    qw = 4 if N == 32 else (3 if C == 64 else 2)
    groups = _cdiv(nchunks, 2 * qw)
    nwg = 2 * groups
    return groups, [nchunks // nwg + (w < nchunks % nwg) for w in range(nwg)]


# name, C, N, taps (kx = 1), per-warpgroup chunk counts
CHUNKS = [(f"c{C}_n{N}_{t}chunks", C, N, t, _plan(C, N, t * C // 64)[1])
          for C, N, taps in ((64, 64, range(1, 10)), (64, 32, (1, 3, 8, 9)), (128, 64, (1, 2, 3, 5)))
          for t in taps]


def test_wgrad_chunk_plan():
    """The plan these tests rely on: every count 0 .. QW occurs, and c3's 9 chunks split 5 + 4 over 2 CTAs."""
    seen = {}
    for _, C, N, _, counts in CHUNKS:
        seen.setdefault((C, N), set()).update(counts)
    assert seen[(64, 64)] == {0, 1, 2, 3} and seen[(64, 32)] == {0, 1, 2, 3, 4} and seen[(128, 64)] == {1, 2}
    assert _plan(64, 64, 9) == (2, [3, 2, 2, 2])
    assert _plan(128, 64, 8) == (2, [2, 2, 2, 2])                # cfg-2's c2 keeps its grouping


@pytest.mark.parametrize("per_cta", [1, 3, "stages", "wraps"])
@pytest.mark.parametrize("name,C,N,taps,counts", CHUNKS, ids=[c[0] for c in CHUNKS])
def test_wgrad_chunk_counts_exact(ops, name, C, N, taps, counts, per_cta):
    """With max_ctas = 7 every CTA but the last runs `per_cta` k-blocks and the last one fewer; max_ctas = 1 / 2 /
    default give one long, two, and many row ranges."""
    stages = 8 if C == 64 else 6
    per = {"stages": stages, "wraps": 3 * stages + 2}.get(per_cta, per_cta)
    kb_total = 7 if per == 1 else 7 * per - 1
    rows = kb_total * KR - 17
    gen = _gen(taps * 100 + C + N + per)
    _check(ops, rows, C, N, SHIFTS[:taps], 1, gen, what=f"{name} counts={counts} per_cta={per}")


# cfg-2's weight-gradient instances (NatureCNN on 84x84): c2 = 4x4 s2 over the 10x10 space-to-depth grid of 128
# channels (kx = 2), c3 = 3x3 over 9x9 of 64 (kx = 3); dY is zero outside the valid outputs
NATURE = [("c2", 10, 10, 128, 2), ("c3", 9, 9, 64, 3)]


def _nature(ops, name, Hg, Wg, C, k, B, max_ctas):
    rows = B * Hg * Wg
    pos = torch.arange(rows, device=DEV) % (Hg * Wg)
    valid = ((pos // Wg) < Hg - k + 1) & ((pos % Wg) < Wg - k + 1)
    _check(ops, rows, C, 64, _square(k, Wg, k), k, _gen(B + k), valid=valid, max_ctas=max_ctas, what=f"{name} B={B}")


@pytest.mark.parametrize("per_range", [1, 3])
@pytest.mark.parametrize("name,Hg,Wg,C,k", NATURE, ids=[c[0] for c in NATURE])
def test_wgrad_nature_partial_last_wave_exact(ops, name, Hg, Wg, C, k, per_range):
    """kb_total = 1 + (per_range - 1) * SMs + 2 k-blocks: with one row range per SM, a last wave of 2-CTA clusters
    that holds a few of them (per_range 1: fewer k-blocks than SMs, so some row ranges are empty of work)."""
    target = 3 + (per_range - 1) * _sms()
    B = _cdiv((target - 1) * KR + 1, Hg * Wg)
    _nature(ops, name, Hg, Wg, C, k, B, (0, 7))


@pytest.mark.parametrize("name,Hg,Wg,C,k", NATURE, ids=[c[0] for c in NATURE])
def test_wgrad_nature_dqn_batch_exact(ops, name, Hg, Wg, C, k):
    """The DQN trunk's train batch (B = 512) runs the same instances as cfg-2's PPO2 update."""
    _nature(ops, name, Hg, Wg, C, k, 512, (0, 1, 2, 7))
