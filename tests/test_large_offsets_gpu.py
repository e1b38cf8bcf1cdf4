"""Every minibatch gather at the buffer sizes the benchmark trains from: sample offsets past 2^31 and 2^32.

The learners gather their minibatches through int64 indices out of device buffers far larger than 2^31 bytes: cfg2's
rollout [128, 4096, 84, 84, 4] uint8 (14.8 GB, read by c1 through src_idx), cfg3's [512, 16384, 376] float32
(3.15e9 elements, 12.6 GB, read by obs_encode) and cfg4's replay storage [2^20, 84, 84, 4] uint8 (29.6 GB per array).
Every other test gathers from buffers of a few hundred MB, so an offset product narrowed to 32 bits would pass them all
while the benchmark trained, at full speed, on the wrong samples.

Kernel level: one device buffer just past the boundaries (uint8 images: more than 2^32 + 2 samples' bytes; float32
rows: more than 2^31 + 2 rows' elements), filled on the device.  The indices hold the samples that straddle byte
offsets 2^31 and 2^32 (and, for float rows, element 2^31), the first samples wholly past them, the last sample, sample
0, a repeated index and random ones.  The kernel gathers them from the big buffer and, through the identity gather,
from the compact copy big.index_select(0, idx) (torch's 64-bit indexing): the outputs are bit-identical.  The pure
data-movement kernels (s2d_gather, im2col, obs_encode) also equal an exact host reference of the gathered rows.  The
tests show they can fail: every boundary sample holds other data than a wrapped address (offset mod 2^32, mod 2^31)
reads, and the compact launch with one row replaced by its wrapped bytes gives a different output.

Learner level: two models from one seed, one training from the bench-shaped buffer through indices, the other from a
compact copy of the same samples through consecutive indices (the same graph-captured path).  After two minibatches
every parameter and both Adam slots are bit-identical, and so are DQN's TD errors; the PPO2 loss statistics, float64
atomic sums, agree to their summation order.  The float64 update tests (test_update_composition*_gpu.py) tie the
compact run to float64.

Each big allocation first checks torch.cuda.mem_get_info() and skips, naming the bytes it needs, when the device does
not have them; every test releases its buffers when it ends, whether it passes or fails.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
G29, G30, G31, G32 = 1 << 29, 1 << 30, 1 << 31, 1 << 32
HEADROOM = 3 << 30                 # models, compact copies and outputs next to the big buffers
U8_MARKS = (G31, G32)              # byte offsets
F32_MARKS = (G29, G30, G31)        # element offsets of float32 rows: bytes 2^31 and 2^32, element 2^31
# a uint8 image buffer > 2^32 + 2 samples for every sample size used here (the largest: 84 x 84 x 16)
U8_BYTES = G32 + 4 * 84 * 84 * 16
# float32 rows of 376 (cfg3's observation): > 2^31 + 2 rows of elements
F32_ROWS = G31 // 376 + 3
BATCHES = [37, 300]                # a small odd batch and one that gives every persistent CTA several tiles


@pytest.fixture
def big():
    """alloc(shape, dtype, fill) -> a device tensor filled in place by fill(t); released when the test ends."""
    held = []

    def alloc(shape, dtype, fill):
        nbytes = math.prod(shape) * torch.empty((), dtype=dtype).element_size()
        free, _ = torch.cuda.mem_get_info()
        if free < nbytes + HEADROOM:
            pytest.skip(f"needs {nbytes} bytes ({nbytes / 1e9:.1f} GB) of free device memory plus "
                        f"{HEADROOM / 1e9:.1f} GB headroom; {free / 1e9:.1f} GB free")
        t = torch.empty(shape, dtype=dtype, device=DEV)
        fill(t)
        held.append(t)
        return t

    yield alloc
    for t in held:                 # frees the memory even where a failure's traceback still holds a view of it
        t.untyped_storage().resize_(0)
    held.clear()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _u8_fill(seed):
    return lambda t: t.random_(0, 256, generator=_gen(seed))


def _randn_fill(seed, scale=3.0):
    return lambda t: t.normal_(0.0, scale, generator=_gen(seed))


def _boundaries(n, per, marks):
    """Samples of `per` units: for every mark K the one that straddles it (when no sample starts at K) and the first
    one wholly at or past K; then sample 0 and the last sample."""
    out = []
    for K in marks:
        out += ([K // per] if K % per else []) + [-(-K // per)]
    out += [0, n - 1]
    assert max(out) < n and -(-marks[-1] // per) < n - 1, "the buffer does not reach past the last mark"
    return sorted(set(out))


def _indices(n, per, marks, B, seed):
    """B indices: the boundary samples, the first sample past the last mark once more, random ones; shuffled."""
    bnd = _boundaries(n, per, marks)
    g = torch.Generator().manual_seed(seed)
    rest = torch.randint(0, n, (B - len(bnd) - 1,), generator=g).tolist()
    idx = torch.tensor(bnd + [-(-marks[-1] // per)] + rest, dtype=torch.int64)
    return idx[torch.randperm(B, generator=g)].to(DEV), bnd


def _wrapped(flat, s, per, M):
    """The units a read of sample s would see with its address taken mod M."""
    span = torch.arange(s * per, (s + 1) * per, device=DEV)
    return flat[span % M]


def _assert_wraps_differ(flat, samples, per, moduli):
    """Every boundary sample past a modulus holds other data than the address mod that modulus: a kernel that wrapped
    there would read different values, so the bit-for-bit comparisons below would see it."""
    for s in samples:
        if s == 0:
            continue
        mine = flat[s * per:(s + 1) * per]
        checked = [M for M in moduli if (s + 1) * per > M]
        assert checked, f"sample {s} ends below every modulus"
        for M in checked:
            assert not torch.equal(_wrapped(flat, s, per, M), mine), \
                f"sample {s} ({per} units at {s * per}) holds the same data as its address mod {M}"


def _bits(t):
    return t.detach().contiguous().reshape(-1).view(torch.uint8)


def _assert_same(got, want, what):
    for k in want:
        assert torch.equal(_bits(got[k]), _bits(want[k])), f"{what}: {k} differs between the big and the compact gather"


def _differs(a, b):
    return any(not torch.equal(_bits(a[k]), _bits(b[k])) for k in b)


def _images(flat, shape):
    sb = math.prod(shape)
    S = flat.numel() // sb
    return flat[:S * sb].view((S,) + tuple(shape)), S, sb


def _gather_case(flat, shape, B, seed, run, ref=None, what=""):
    """run(images, idx) -> dict of output tensors.  Big buffer through idx == compact copy through arange, bit for bit
    (== ref(compact images on the host) when given); the compact launch with the first sample past 2^32 replaced by
    the bytes its address mod 2^32 holds gives a different output."""
    pool, S, sb = _images(flat, shape)
    idx, bnd = _indices(S, sb, U8_MARKS, B, seed)
    _assert_wraps_differ(pool.view(-1), bnd, sb, U8_MARKS)
    x_c = pool.index_select(0, idx)
    ident = torch.arange(B, device=DEV)
    got = run(pool, idx)
    want = run(x_c, ident)
    _assert_same(got, want, what)
    if ref is not None:
        expect = ref(x_c.cpu())
        for k, v in expect.items():
            assert torch.equal(_bits(got[k].cpu()), _bits(v)), f"{what}: {k} differs from the host reference"
    past = -(-G32 // sb)
    k = int((idx == past).nonzero()[0, 0])
    x_w = x_c.clone()
    x_w[k] = _wrapped(pool.view(-1), past, sb, G32).view(shape)
    assert _differs(run(x_w, ident), want), f"{what}: a row read at its address mod 2^32 does not change the output"


# ------------------------------------------------------------------------------------------------ conv stacks
# planner paths of the conv stack (test_conv_paths_gpu.CONFIGS) and the gather each one's first layer makes
CONV_CASES = {
    "default": "conv_shift_fwd / conv_shift_wgrad with the fused uint8 source (cfg2, cfg4)",
    "shift_unfused_60x60x8": "s2d_gather<16> into the shift-GEMM stack",
    "implicit_s2d_64x64x4": "s2d_gather<16> into the implicit GEMM",
    "implicit_superpixel_85x84x4": "im2col gather_cast (H = W = 1) into the implicit GEMM",
    "implicit_merged_84x84x16": "im2col gather_cast (H = W = 1) into the implicit GEMM",
    "explicit_c1_84x84x6": "im2col of c1 (explicit GEMM)",
    "dqn_conv_only": "im2col of c1, SAME padding (DQN conv_only)",
}


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("name", list(CONV_CASES))
def test_conv_stack_gathers_past_4gib(name, B, big):
    """A whole conv tower forward and backward from the big buffer: the gathered fp16 input (unfused paths), every
    conv activation, the shift-GEMM ReLU bit masks, every fc activation and every weight and bias gradient (c1's G and
    bias gradient included) equal the compact run's."""
    from test_conv_paths_gpu import CONFIGS, _build
    shape = CONFIGS[name][0]
    print(f"  {name}: {CONV_CASES[name]}")
    tower, store, _ = _build(name, B)                  # asserts the planned path
    L, ldd = tower.latent_dim, tower.ld_dlatent
    dlat = (torch.randn(B, L, device=DEV, generator=_gen(5)) * 0.1).half()

    def run(x, idx):
        h, ldh = tower.forward(x, B, idx)
        tower.dlatent.reshape(-1)[:B * ldd].view(B, ldd)[:, :L].copy_(dlat)
        store.grads.zero_()
        tower.backward(B, 1.0 / B)
        torch.cuda.synchronize()
        out = {"latent": h.reshape(-1)[:B * ldh].clone(), "grads": store.grads.clone()}
        if getattr(tower, "x16", None) is not None:                  # s2d_gather / gather_cast output
            out["x16"] = tower.x16.clone()
        if getattr(tower, "cols", None) and tower.cols[0] is not None:  # c1's im2col output
            out["cols0"] = tower.cols[0].clone()
        out.update({f"act{i}": a.clone() for i, a in enumerate(tower.hconv)})
        out.update({f"fc{i}": a.clone() for i, a in enumerate(tower.hfc)})
        if tower.shift_mode:
            out.update({f"bits{i}": b.clone() for i, b in enumerate(tower.hbits)})
        return out

    flat = big((U8_BYTES,), torch.uint8, _u8_fill(1))
    _gather_case(flat, shape, B, 100 + B, run, what=f"{name} B={B}")


# ------------------------------------------------------------------------------------------------ s2d_gather
S2D_CASES = {                      # name: (sample shape, stride, elements per thread of the instance it takes)
    "shift_unfused_60x60x8": ((60, 60, 8), 4, 16),
    "implicit_s2d_64x64x4": ((64, 64, 4), 4, 16),
    "implicit_s2d_84x84x2": ((84, 84, 2), 4, 8),    # s*C = 8
}


def _s2d_ref(x, s):
    B, H, W, C = x.shape
    return x.view(B, H // s, s, W // s, s, C).permute(0, 1, 3, 2, 4, 5).reshape(B, -1).half()


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("name", list(S2D_CASES))
def test_s2d_gather_past_4gib(name, B, big):
    from baselines_b200 import nn as bnn
    from baselines_b200 import ops
    (H, W, C), s, ept = S2D_CASES[name]
    assert ((s * C) % 16 == 0) == (ept == 16)          # b200rl_s2d_gather's choice of instance (16-byte aligned x)
    if name.startswith("implicit"):
        lp = bnn.plan_conv_stack((H, W, C), bnn.NATURE_CONVS, False, True)
        assert not lp.shift and lp.layers[0].s2d
    out = torch.empty(B, H * W * C, dtype=torch.float16, device=DEV)

    def run(x, idx):
        ops.s2d_gather(x, out, B, H, W, C, s, src_idx=idx)
        torch.cuda.synchronize()
        return {"out": out.clone()}

    flat = big((U8_BYTES,), torch.uint8, _u8_fill(2))
    _gather_case(flat, (H, W, C), B, 200 + B, run, ref=lambda x: {"out": _s2d_ref(x, s)}, what=f"s2d {name} B={B}")


# ------------------------------------------------------------------------------------------------ im2col
IM2COL_CASES = {                   # name: (sample shape, (H, W, C, rf, stride) the kernel sees, SAME padding)
    "explicit_c1_84x84x6": ((84, 84, 6), (84, 84, 6, 8, 4), False),
    "gather_cast_85x84x4": ((85, 84, 4), (1, 1, 85 * 84 * 4, 1, 1), False),
    "gather_cast_84x84x16": ((84, 84, 16), (1, 1, 84 * 84 * 16, 1, 1), False),
    "dqn_conv_only_same_84x84x4": ((84, 84, 4), (84, 84, 4, 8, 4), True),
}


def _im2col_ref(x, H, W, C, rf, st, same):
    from baselines_b200 import ops
    B = x.shape[0]
    x = x.view(B, H, W, C)
    OH, OW = ops._conv_out(H, W, rf, st, same)
    ph = max((OH - 1) * st + rf - H, 0) if same else 0
    pw = max((OW - 1) * st + rf - W, 0) if same else 0
    xp = F.pad(x.permute(0, 3, 1, 2).float(), (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2))
    u = F.unfold(xp, rf, stride=st)                    # [B, C * rf * rf, OH * OW], K ordered (c, ky, kx)
    return u.view(B, C, rf, rf, OH * OW).permute(0, 4, 2, 3, 1).reshape(B * OH * OW, rf * rf * C).half()


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("name", list(IM2COL_CASES))
def test_im2col_uint8_gather_past_4gib(name, B, big):
    from baselines_b200 import ops
    shape, (H, W, C, rf, st), same = IM2COL_CASES[name]
    OH, OW = ops._conv_out(H, W, rf, st, same)
    cols = torch.empty(B * OH * OW, rf * rf * C, dtype=torch.float16, device=DEV)

    def run(x, idx):
        ops.im2col(x, cols, B, H, W, C, rf, st, same, src_idx=idx)
        torch.cuda.synchronize()
        return {"cols": cols.clone()}

    flat = big((U8_BYTES,), torch.uint8, _u8_fill(3))
    _gather_case(flat, shape, B, 300 + B, run, ref=lambda x: {"cols": _im2col_ref(x, H, W, C, rf, st, same)},
                 what=f"im2col {name} B={B}")


# ------------------------------------------------------------------------------------------------ obs_encode
def _encode_ref(x, in_dim, in_pad, norm=None, onehot_n=0):
    """Exact: v (normalised and clipped in float32 like the kernel), hi = fp16(v), lo = fp16(v - hi)."""
    B = x.shape[0]
    if onehot_n:
        v = torch.zeros(B, in_pad)
        v[torch.arange(B), x[:, 0].long()] = 1.0
    else:
        v = x.clone()
        if norm is not None:
            mean, inv_std, lo, hi = norm
            v = torch.clamp((v - mean) * inv_std, lo, hi)
        v = F.pad(v, (0, in_pad - in_dim))
    h = v.half()
    return torch.cat([h, (v - h.float()).half()], 1)


def _encode_case(x2d, B, seed, in_dim, in_pad, norm=None, onehot_n=0, what=""):
    """obs_encode from float32 rows x2d [R, raw_dim] through indices at the element boundaries F32_MARKS, against
    the compact copy and the host reference; the first row past element 2^31 read at its byte offset mod 2^32 (element
    offset mod 2^30) changes the output."""
    from baselines_b200 import ops
    R, raw = x2d.shape
    flat = x2d.view(-1)
    idx, bnd = _indices(R, raw, F32_MARKS, B, seed)
    _assert_wraps_differ(flat, bnd, raw, F32_MARKS)
    out = torch.empty(B, 2 * in_pad, dtype=torch.float16, device=DEV)
    over = torch.zeros(1, dtype=torch.int32, device=DEV)
    mean, inv_std, lo, hi = norm if norm is not None else (None, None, 0.0, 0.0)

    def run(x, i):
        out.fill_(float("nan"))
        ops.obs_encode(x, out, B, raw, in_dim, in_pad, src_idx=i, mean=mean, inv_std=inv_std, clip=(lo, hi),
                       onehot_n=onehot_n, overflow=over)
        torch.cuda.synchronize()
        return {"out": out.clone(), "overflow": over.clone()}

    x_c = x2d.index_select(0, idx)
    ident = torch.arange(B, device=DEV)
    got, want = run(x2d, idx), run(x_c, ident)
    _assert_same(got, want, what)
    assert int(got["overflow"]) == 0
    hn = None if norm is None else (mean.cpu(), inv_std.cpu(), lo, hi)
    assert torch.equal(_bits(got["out"].cpu()), _bits(_encode_ref(x_c.cpu(), in_dim, in_pad, hn, onehot_n))), \
        f"{what}: differs from the host reference"
    past = -(-G31 // raw)
    k = int((idx == past).nonzero()[0, 0])
    x_w = x_c.clone()
    x_w[k] = _wrapped(flat, past, raw, G30)
    assert _differs(run(x_w, ident), want), f"{what}: a row read at its byte offset mod 2^32 does not change the output"


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("in_pad", [376, 384], ids=["in_pad_376", "in_pad_384"])
@pytest.mark.parametrize("norm", [False, True], ids=["raw", "mean_inv_std_clip"])
def test_obs_encode_gather_past_2pow31_elements(norm, in_pad, B, big):
    """cfg3's rows (raw_dim 376) from a buffer of more than 2^31 + 2 rows' elements: hi / lo pairs bit for bit."""
    x = big((F32_ROWS, 376), torch.float32, _randn_fill(4))
    nm = None
    if norm:
        g = _gen(40)
        mean = torch.randn(376, device=DEV, generator=g)
        inv_std = torch.rand(376, device=DEV, generator=g) * 3.0 + 0.25
        nm = (mean, inv_std, -5.0, 5.0)
        assert bool(((x[:64] - mean) * inv_std).abs().gt(5.0).any()), "the clip is not active"
    _encode_case(x, B, 400 + B, 376, in_pad, nm, what=f"obs_encode raw_dim 376 in_pad {in_pad} norm {norm} B={B}")


@pytest.mark.parametrize("B", BATCHES)
def test_obs_encode_discrete_rows_past_2pow31(B, big):
    """The same allocation as raw_dim = 1 Discrete(18) rows: the row indices themselves exceed 2^31.  Boundary rows
    that happen to equal a wrapped row's integer are set to another one, so a wrapped read changes the one-hot row."""
    n = 18
    x = big((F32_ROWS * 376, 1), torch.float32, lambda t: t.random_(0, n, generator=_gen(6)))
    flat = x.view(-1)
    for r in _boundaries(x.shape[0], 1, F32_MARKS):
        seen = {int(flat[r % M]) for M in F32_MARKS if r + 1 > M}
        if int(flat[r]) in seen:
            flat[r] = float(next(v for v in range(n) if v not in seen))
    _encode_case(x, B, 500 + B, n, 24, onehot_n=n, what=f"obs_encode Discrete({n}) B={B}")


# ------------------------------------------------------------------------------------------------ learners
def _cfg(key):
    from bench import CFGS
    return CFGS[key]


def _ppo_models(ob, ac, network, M, nsteps, cfg, **kw):
    """Two PPO2 models from one seed with cfg's loss coefficients, a minibatch of M and one chunk per minibatch."""
    from baselines_b200.common.policies import PolicyBuilder
    from baselines_b200.ppo2.model import Model
    models = []
    for _ in range(2):
        np.random.seed(0)
        pol = PolicyBuilder(ob, ac, network, **kw)
        models.append(Model(policy=pol, ob_space=ob, ac_space=ac, nbatch_act=8, nbatch_train=M, nsteps=nsteps,
                            ent_coef=cfg["ent_coef"], vf_coef=cfg["vf_coef"], max_grad_norm=cfg["max_grad_norm"],
                            comm=False))
    return models


def _assert_stats(got, want, what):
    """The loss statistics are float64 atomic sums over the minibatch (DESIGN.md §6), whose order varies from run to
    run, so they may differ in the last bits (observed: one unit in the last place).  A single sample read from the
    wrong place moves a mean over M = 1536 samples by order 1e-4; the bound is six orders of magnitude below that."""
    err = float(((got - want).abs() / (1.0 + want.abs())).max())
    assert err <= 1e-10, f"{what}: loss statistics differ by {err:.3e} (relative to 1 + |value|)"


def _assert_same_state(a, b, start, what):
    for k in ("params", "m", "v"):
        assert torch.equal(_bits(getattr(a, k)), _bits(getattr(b, k))), f"{what}: {k} differ"
    assert not torch.equal(a.params, start), f"{what}: the updates changed nothing"


def _rollout_arrays(n, ac, seed):
    g = _gen(seed)
    if ac == "cat":
        acts = torch.randint(0, 6, (n,), device=DEV, generator=g)
    else:
        acts = torch.randn(n, ac, device=DEV, generator=g)
    vals = torch.randn(n, device=DEV, generator=g)
    rets = vals + torch.randn(n, device=DEV, generator=g)
    nlp = torch.rand(n, device=DEV, generator=g) * 2.0 + 0.5
    return [acts, rets, vals, nlp]


def _ppo_pair_run(key, obs, ob, ac, network, marks, per, arrays, seed, **kw):
    """Two minibatches of ~1.5 k samples (boundary samples, the last one, random ones; shuffled) from the flat rollout
    obs [n, ...] through indices, and from a compact copy of them through consecutive indices."""
    cfg = _cfg(key)
    n, M = obs.shape[0], 1536
    big_m, comp_m = _ppo_models(ob, ac, network, M, 1, cfg, **kw)
    start = big_m.net.store.params.clone()
    idx = [_indices(n, per, marks, M, seed + k)[0] for k in range(2)]
    allidx = torch.cat(idx)
    obs_c = obs.index_select(0, allidx)
    arr_c = [a.index_select(0, allidx) for a in arrays]
    for k in range(2):
        st_b = big_m.train_rollout(cfg["lr"], cfg["cliprange"], obs, *arrays, idx[k]).clone()
        st_c = comp_m.train_rollout(cfg["lr"], cfg["cliprange"], obs_c, *arr_c,
                                    torch.arange(k * M, (k + 1) * M, device=DEV)).clone()
        _assert_stats(st_b, st_c, f"{key} minibatch {k}")
    torch.cuda.synchronize()
    _assert_same_state(big_m.net.store, comp_m.net.store, start, key)


def test_ppo2_cfg2_rollout_past_2pow32_bytes(big):
    """cfg2: NatureCNN (the fused uint8 shift-GEMM c1) trained from the exact [128, 4096, 84, 84, 4] rollout."""
    from baselines_b200.common import spaces
    T, N, shape = 128, 4096, (84, 84, 4)
    obs = big((T, N) + shape, torch.uint8, _u8_fill(7)).view((T * N,) + shape)
    arrays = _rollout_arrays(T * N, "cat", 70)
    _ppo_pair_run("cfg2", obs, spaces.Box(0, 255, shape, np.uint8), spaces.Discrete(6), "cnn", U8_MARKS,
                  math.prod(shape), arrays, 700)


def test_ppo2_cfg3_rollout_past_2pow31_elements(big):
    """cfg3: mlp, 17-d Gaussian, value_network='copy', trained from the exact [512, 16384, 376] float32 rollout."""
    from baselines_b200.common import spaces
    T, N = 512, 16384
    obs = big((T, N, 376), torch.float32, _randn_fill(8)).view(T * N, 376)
    arrays = _rollout_arrays(T * N, 17, 80)
    _ppo_pair_run("cfg3", obs, spaces.Box(-10, 10, (376,), np.float32), spaces.Box(-1, 1, (17,), np.float32), "mlp",
                  F32_MARKS, 376, arrays, 800, value_network="copy")


def test_dqn_cfg4_replay_past_2pow32_bytes(big):
    """cfg4's network (NatureCNN + dueling, hiddens 256) trained through train_device from replay storage of capacity
    2^18 (7.4 GB per array): TD errors of both steps, parameters and Adam slots equal the compact run's."""
    from baselines_b200.common import spaces
    from baselines_b200.deepq.build_graph import DQNModel
    cfg = _cfg("cfg4")
    cap, shape, B = 1 << 18, cfg["ob_shape"], cfg["batch"]
    o_t = big((cap,) + shape, torch.uint8, _u8_fill(9))
    o_1 = big((cap,) + shape, torch.uint8, _u8_fill(10))
    g = _gen(90)
    acts = torch.randint(0, cfg["n_actions"], (cap,), device=DEV, generator=g)
    rew = torch.randn(cap, device=DEV, generator=g)
    done = (torch.rand(cap, device=DEV, generator=g) < 0.1).float()
    models = []
    for _ in range(2):
        np.random.seed(0)
        models.append(DQNModel(spaces.Box(0, 255, shape, np.uint8), cfg["n_actions"], "cnn", lr=cfg["lr"],
                               gamma=cfg["gamma"], grad_norm_clipping=10, batch_cap=B, seed=0, hiddens=(256,),
                               dueling=True))
    big_m, comp_m = models
    start = big_m.q.store.params.clone()
    idx = [_indices(cap, math.prod(shape), U8_MARKS, B, 900 + k)[0] for k in range(2)]
    allidx = torch.cat(idx)
    sel = lambda t: t.index_select(0, allidx)
    comp = [sel(t) for t in (o_t, o_1, acts, rew, done)]
    for k in range(2):
        w = torch.rand(B, device=DEV, generator=g) * 0.9 + 0.1
        td_b = big_m.train_device(o_t, o_1, acts, rew, done, w, idx[k], B).clone()
        td_c = comp_m.train_device(*comp, w, torch.arange(k * B, (k + 1) * B, device=DEV), B).clone()
        assert torch.equal(_bits(td_b), _bits(td_c)), f"DQN step {k}: TD errors differ"
    torch.cuda.synchronize()
    _assert_same_state(big_m.q.store, comp_m.q.store, start, "DQN")


def test_ppo2_cnn_lstm_rollout_past_2pow32_bytes(big):
    """cnn_lstm through train_rollout_seq from a [128, 1200, 84, 84, 4] rollout (4.3 GB): whole environments whose
    sequences hold the boundary samples; the observations, the LSTM's masks (mask_idx) and start states (state_idx)
    are gathered through the rows.  The compact copy holds the same environments as a rollout of its own."""
    from baselines_b200.common import spaces
    T, N, shape = 128, 1200, (84, 84, 4)
    n, E = T * N, 12
    cfg = _cfg("cfg2")
    obs = big((T, N) + shape, torch.uint8, _u8_fill(11)).view((n,) + shape)
    arrays = _rollout_arrays(n, "cat", 110)
    g = _gen(111)
    dones = (torch.rand(n, device=DEV, generator=g) < 0.05).to(torch.uint8)
    big_m, comp_m = _ppo_models(spaces.Box(0, 255, shape, np.uint8), spaces.Discrete(6), "cnn_lstm", E * T, T, cfg)
    H = big_m.net.nlstm
    states0 = torch.randn(N, 2 * H, device=DEV, generator=g) * 0.5
    start = big_m.net.store.params.clone()
    sb = math.prod(shape)
    bnd_envs = sorted({s % N for s in _boundaries(n, sb, U8_MARKS)})
    assert len(bnd_envs) < E
    rng = np.random.RandomState(112)
    others = rng.permutation([e for e in range(N) if e not in bnd_envs])
    envs = [rng.permutation(bnd_envs + list(others[k * E:(k + 1) * E - len(bnd_envs)])) for k in range(2)]
    # compact rollout: minibatch k's environments are its environments k*E .. k*E + E - 1, buffer row k*E*T + t*E + e'
    order = np.concatenate([(np.arange(T)[:, None] * N + np.asarray(ev)[None, :]).reshape(-1) for ev in envs])
    oi = torch.as_tensor(order).to(DEV)
    obs_c = obs.index_select(0, oi)
    arr_c = [a.index_select(0, oi) for a in arrays]
    dones_c = dones.index_select(0, oi)
    states0_c = states0.index_select(0, torch.as_tensor(np.concatenate(envs)).to(DEV))
    for k in range(2):
        rows = np.arange(T)[None, :] * N + np.asarray(envs[k])[:, None]            # [E, T] buffer offsets
        rows_c = k * E * T + np.arange(T)[None, :] * E + np.arange(E)[:, None]
        st_b = big_m.train_rollout_seq(cfg["lr"], cfg["cliprange"], obs, *arrays, dones, states0, rows,
                                       np.asarray(envs[k])).clone()
        st_c = comp_m.train_rollout_seq(cfg["lr"], cfg["cliprange"], obs_c, *arr_c, dones_c, states0_c, rows_c,
                                        k * E + np.arange(E)).clone()
        _assert_stats(st_b, st_c, f"cnn_lstm minibatch {k}")
    torch.cuda.synchronize()
    _assert_same_state(big_m.net.store, comp_m.net.store, start, "cnn_lstm")
