"""The ping-pong schedule of the shift-GEMM convolution kernels (csrc/conv_shift.cu) at its turn-taking boundaries.

In the forward / data-gradient kernel the two consumer warpgroups take turns issuing MMAs: group 0 takes a CTA's
even tiles and group 1 its odd ones, so a CTA with 1, 2, 3 or an odd number of tiles ends on a group that has no
further tile.  The uint8-fed first layer's rolling A ring releases a stage only after its own tile and the tile before
it (the other group) have retired.

Operands are small integers, as in test_wgmma_boundaries_gpu.py: each result is exact and is compared with
torch.equal against float64.  Tiles per CTA are set through B (the CTA count is the SM count).
"""
import math

import numpy as np
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


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _ints(shape, density, gen, lo=-2, hi=2):
    return R.small_ints(shape, density, gen, device=DEV, lo=lo, hi=hi)


def _cdiv(a, b):
    return -(-a // b)


def _sms():
    from baselines_b200 import ops
    return ops.num_sms()


def _batch_for_tiles_per_cta(per_cta, rows_per_sample):
    """B such that the interleaved TMA-fed tiles give some CTAs `per_cta` tiles and the others per_cta - 1 (per_cta =
    1: every CTA one tile and some SMs idle)."""
    sms = _sms()
    tiles = sms // 2 if per_cta == 1 else (per_cta - 1) * sms + sms // 2 + 1
    return _cdiv(tiles * 128, rows_per_sample)


def _tiles_per_cta(M):
    tiles = _cdiv(M, 128)
    grid = min(tiles, _sms())
    return {_cdiv(tiles - b, grid) for b in range(grid)}


# ------------------------------------------------------------------------------------------ forward / data gradient
# cfg-2's shift-conv forward and data-gradient instances (NatureCNN on 84x84: c2 = 4x4 s2 over a 10x10 space-to-depth
# grid of 128 channels, c3 = 3x3 s1 over 9x9 of 64) and the BN = 128 forward, which keeps the cooperative schedule
# (the tile-count boundaries are the same for both schedules)
FWD = [
    # name, dgrad, Hg, Wg, C (input channels), N (output channels), k
    ("fwd_c2_bn64_kh2", False, 10, 10, 128, 64, 2),
    ("fwd_c3_bn64_kh1", False, 9, 9, 64, 64, 3),
    ("fwd_bn128_cooperative", False, 9, 9, 64, 128, 2),
    ("dgrad_c3_bn64", True, 9, 9, 64, 64, 3),
    ("dgrad_c2_bn128", True, 10, 10, 64, 128, 2),
]


@pytest.mark.parametrize("per_cta", [1, 2, 3, 7, 20])
@pytest.mark.parametrize("name,dgrad,Hg,Wg,C,N,k", FWD, ids=[c[0] for c in FWD])
def test_shift_fwd_dgrad_tiles_per_cta_exact(ops, name, dgrad, Hg, Wg, C, N, k, per_cta):
    """Every CTA ends on either group, with 1 .. per_cta tiles: the forward (relu + bias + bit mask) and the data
    gradient (negative shifts, the relu mask from the bit array) equal float64."""
    B = _batch_for_tiles_per_cta(per_cta, Hg * Wg)
    M = B * Hg * Wg
    counts = _tiles_per_cta(M)
    assert max(counts) == per_cta and (per_cta == 1 or per_cta - 1 in counts), counts
    gen = _gen(per_cta * 100 + C + N + k)
    OH, OW = Hg - k + 1, Wg - k + 1
    taps = k * k
    shifts = [a * Wg + b for a in range(k) for b in range(k)]
    if not dgrad:
        x64 = _ints((M, C), 0.5, gen)
        w64 = _ints((N, taps * C), 0.5, gen)
        bias = _ints((N,), 0.7, gen, -3, 3).float()
        full = R.shift_conv(x64, shifts, w64)
        R.assert_exact_ok(R.shift_conv(x64.abs(), shifts, w64.abs()), what=name)
        want = torch.relu(0.5 * full.view(B, Hg, Wg, N)[:, :OH, :OW] + bias.double())
        out = torch.full((B, OH, OW, N), SENT, dtype=torch.float16, device=DEV)
        bo = torch.full((out.numel() // 16,), 0x5A5A, dtype=torch.int16, device=DEV)
        ops.conv_shift_fwd(x64.half(), B, Hg, Wg, C, w64.half(), taps * C, N, shifts, OH, OW, out,
                           (0, OH * OW * N, OW * N, N, 0, 0), bias=bias, act=ops.ACT_RELU, alpha=0.5, bits_out=bo)
        torch.cuda.synchronize()
        assert torch.equal(out.double(), want), (name, B, float((out.double() - want).abs().max()))
        assert torch.equal(bo, R.relu_bits(out)), (name, B, "bits")
        return
    dY64 = torch.zeros(B, Hg, Wg, C, dtype=torch.float64, device=DEV)
    dY64[:, :OH, :OW] = _ints((B, OH, OW, C), 0.5, gen)
    dY64 = dY64.reshape(M, C)
    wd64 = _ints((N, taps * C), 0.5, gen)
    saved = torch.relu(_ints((B, Hg, Wg, N), 0.6, gen)).half()
    smap = (0, Hg * Wg * N, Wg * N, N, 0, 0)
    neg = [-s for s in shifts]
    R.assert_exact_ok(R.shift_conv(dY64.abs(), neg, wd64.abs()), what=name)
    dx = 0.5 * R.shift_conv(dY64, neg, wd64).view(B, Hg, Wg, N) * (saved.double() > 0)
    if N == 128:                                              # c2: depth->space into the c1 output grid (Cq = 32, s = 2)
        Cq, Ho = N // 4, 2 * Hg
        out = torch.full((B, Ho, Ho, Cq), SENT, dtype=torch.float16, device=DEV)
        omap, want = (1, Ho * Ho * Cq, Ho * Cq, Cq, Cq, 2), R.depth_to_space(dx, 2)
    else:
        out = torch.full((B, Hg, Wg, N), SENT, dtype=torch.float16, device=DEV)
        omap, want = smap, dx
    ops.conv_shift_fwd(dY64.half(), B, Hg, Wg, C, wd64.half(), taps * C, N, neg, Hg, Wg, out, omap, smap=smap,
                       act=ops.ACT_RELU, dact=True, alpha=0.5, saved_bits=R.relu_bits(saved))
    torch.cuda.synchronize()
    assert torch.equal(out.double(), want), (name, B, float((out.double() - want).abs().max()))


# ------------------------------------------------------------------------------------------ uint8-fed first layer
U8_STAGES = 12


@pytest.mark.parametrize("B", [5, 60, 100, 230, 460, 1000])
def test_shift_fwd_uint8_ring_exact(ops, B):
    """c1 straight from uint8 frames.  Each CTA takes a consecutive run of q or q + 1 tiles (q = tiles // CTAs):
    B = 5: one tile per CTA; 60: 1 / 2; 100: 2 / 3; 230: 6 / 7; 460: 12 / 13 (a multiple of the 12 ring stages
    and not); 1000: 26 / 27 (the ring wraps twice).  The tile in the last stage reads the mirror unit, under either
    group."""
    gen = _gen(B + 7)
    H = Wd = 84
    C, s, Hg, Wg, N = 4, 4, 21, 21, 32
    M = B * Hg * Wg
    tiles = _cdiv(M, 128)
    grid = min(tiles, _sms())
    q, r = divmod(tiles, grid)
    if B == 460:
        assert q % U8_STAGES == 0 and r > 0, (q, r)
    if B == 1000:
        assert q > 2 * U8_STAGES, (q, r)
    pool = B + 3
    frames = torch.randint(0, 3, (pool, H, Wd, C), generator=gen, dtype=torch.uint8).to(DEV)
    idx = torch.randperm(pool, generator=gen)[:B].to(DEV)
    x64 = R.space_to_depth(frames[idx].double(), s).reshape(M, 64)
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
    assert torch.equal(out.double(), want), (B, float((out.double() - want).abs().max()))
    assert torch.equal(bo, R.relu_bits(out))


# ------------------------------------------------------------------------------------------ full cfg-2 minibatch
def test_cfg2_minibatch_train_step_repeats_bit_for_bit():
    """Two models from the same seed take one train step on the same cfg-2-sized minibatch (131072 NatureCNN samples:
    every shift-conv forward, data gradient and weight gradient at full size): identical parameters afterwards."""
    from baselines_b200.common import spaces
    from baselines_b200.common.policies import build_policy
    from baselines_b200.ppo2.model import Model

    class E:
        observation_space = spaces.Box(0, 255, (84, 84, 4), np.uint8)
        action_space = spaces.Discrete(6)
        num_envs = 16

    M = 131072
    rng = np.random.RandomState(3)
    obs = rng.randint(0, 256, (M, 84, 84, 4), dtype=np.uint8)
    actions = rng.randint(0, 6, M)
    values = rng.randn(M).astype(np.float32)
    returns = (values + rng.randn(M)).astype(np.float32)
    nlp = np.full(M, math.log(6), np.float32)
    params = []
    for _ in range(2):
        np.random.seed(0)
        model = Model(policy=build_policy(E, "cnn"), ob_space=E.observation_space, ac_space=E.action_space,
                      nbatch_act=16, nbatch_train=M, nsteps=1, ent_coef=0.01, vf_coef=0.5, max_grad_norm=0.5,
                      comm=False)
        model.train(2.5e-4, 0.1, obs, returns, None, actions, values, nlp)
        params.append(model.get_params())
        del model
        torch.cuda.empty_cache()
    assert params[0].keys() == params[1].keys()
    for key in params[0]:
        assert np.array_equal(params[0][key], params[1][key]), key
