"""GPU: every kernel between the last GEMM of an update and the parameter write, against float64.

Loss heads (Gaussian at every DMAX instance, Discrete categorical around the 8-column store group), the PPO2 branches
deliberately populated, the advantage moments, the optimiser kernels (sumsq, seg_sumsq, clip_adam, clip_accumulate)
and the DQN TD step.  References are tests/_loss_refs.py; every tolerance goes through _refs.assert_within, which also
asserts that the bound rejects references built with a plausible kernel mistake (the mutants named in each call).

Bounds:
  * fp16 gradients: |got - ref| <= 2^-11 |ref| + 1e-6 (one fp16 rounding of an fp32 value; test_action_spaces_gpu.py).
    For a Gaussian row the fp32 neglogp (a sum over d dimensions) moves the ratio, and with it the row's gradient, by
    up to G_NLP times the row's absolute neglogp terms; that term is added for the Gaussian head.
  * fp32 reductions (dL/dlogstd, the five loss statistics): g * S with S the sum of the absolute per-row terms.
  * G_DLOGSTD, G_STATS and G_NLP are 3.5x the largest value observed on an H100 (80 GB); the mutants show each bound
    still rejects a one-row mistake.
  * fp64 reductions (adv_stats, sumsq, seg_sumsq): the recursive-summation bound gamma_k of the kernel's summation
    depth k, derived in each test.
"""
import math

import numpy as np
import pytest
import torch

import _loss_refs as lr
from _refs import R_F16, assert_within

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
G_DLOGSTD = 1.3e-6           # dL/dlogstd: fp32 warp sums, 8 warp slots, block partials added in order (3.6e-7 seen)
G_STATS = 1.7e-7             # the five PPO statistics: fp32 per-row values, fp64 atomics (4.6e-8 seen)
G_NLP = 7.5e-8               # fp32 neglogp of a Gaussian row: ratio error per unit of its absolute terms (2.1e-8 seen)


def _dev(a, dt=None):
    t = torch.as_tensor(np.ascontiguousarray(a))
    return (t if dt is None else t.to(dt)).cuda()


def _t(x):
    return torch.as_tensor(np.asarray(x, dtype=np.float64))


def _within_f16(got, ref, mutants, what, nscale=None):
    """The fp16 gradient bound, with its mutants.  nscale [rows]: the absolute terms of each row's fp32 neglogp; the
    ratio exp(old - neglogp) then carries a relative error up to G_NLP * nscale, and so does the row's gradient."""
    ref = _t(ref)
    scale = torch.ones_like(ref)
    if nscale is not None:
        ns = _t(nscale).reshape(-1, *([1] * (ref.dim() - 1)))
        scale = scale + (G_NLP / lr.F16_G) * ref.abs() * ns
        e = ((_t(got) - ref).abs() - R_F16 * ref.abs() - lr.F16_G).clamp_min(0) / (ref.abs() * ns).clamp_min(1e-30)
        _report(what + " (neglogp term)", float(e.max()), G_NLP)
    return assert_within(_t(got), ref, scale, lr.F16_G, R_F16, {k: _t(v) for k, v in mutants.items()}, what)


def _gauss_nscale(acts, head, logstd, oldnlp):
    """Sum of the absolute terms of a Gaussian row's neglogp, and of the old neglogp it is compared with."""
    t = (np.asarray(acts, np.float64) - head) / np.exp(np.asarray(logstd, np.float64))
    return (0.5 * t * t + np.abs(logstd) + 0.92).sum(1) + np.abs(oldnlp)


def _report(what, g_seen, g):
    print(f"[observed] {what}: g = {g_seen:.3e} (allowed {g:.3e})")


# ================================================================================================ shared PPO inputs
def _ppo_inputs(rng, pd, head, v32, B, Bbuf, src, d_or_nA, logstd=None, nvec=None, ratio_sd=0.15):
    """Rollout buffers of Bbuf rows (rows src[b] belong to minibatch row b): actions, old neglogp near the current one,
    old values near the head's value, returns."""
    if pd == "gauss":
        acts_buf = rng.randn(Bbuf, d_or_nA).astype(np.float32)
        acts_buf[src] = (head + np.exp(logstd) * rng.randn(B, d_or_nA)).astype(np.float32)
    else:
        acts_buf = rng.randint(0, d_or_nA, Bbuf).astype(np.int64)
    acts = acts_buf[src]
    z = np.zeros(B)
    nlp_cur = lr.ppo_ref(pd, head, v32, acts, z, z, z, z, 0.2, 0.0, 0.0, nvec=nvec, logstd=logstd).nlp
    oldnlp_buf = rng.randn(Bbuf).astype(np.float32)
    oldnlp_buf[src] = (nlp_cur + rng.randn(B) * ratio_sd).astype(np.float32)
    oldv_buf = rng.randn(Bbuf).astype(np.float32)
    oldv_buf[src] = (v32 + rng.randn(B) * 0.3).astype(np.float32)
    R_buf = (oldv_buf + rng.randn(Bbuf)).astype(np.float32)
    return acts_buf, acts, oldnlp_buf, oldv_buf, R_buf


def _stats_check(got, ref, pd, head, acts, oldnlp, adv, logstd, B, what):
    """The five statistics: pg / vf / entropy / approxkl within G_STATS * S, S the sum of |per-row term| plus, for the
    two terms that depend on the recomputed neglogp, its fp32 error scale; clipfrac may differ only by rows within
    rounding of the clip boundary.  Mutant: the rows of block 1 (256..511) missing, as a lost block sum would be."""
    if pd == "gauss":
        nscale = _gauss_nscale(acts, head, logstd, oldnlp)
    else:
        nscale = 2 * np.abs(head).max(1) + np.log(head.shape[1]) + 1.0 + np.abs(oldnlp)
    dn = np.abs(ref.nlp - oldnlp)
    S = np.abs(ref.rows5[:, :4]).sum(0)
    S[0] += (np.abs(adv * ref.ratio) * nscale).sum()
    S[3] += (dn * nscale).sum()
    blk = slice(256, min(512, B))
    seen = assert_within(_t(got[:4]), _t(ref.stats[:4]), _t(S), G_STATS, 0.0,
                         {"block 1 dropped": _t(ref.stats[:4] - ref.rows5[blk, :4].sum(0))}, what + " statistics")
    assert abs(got[4] - ref.stats[4]) <= ref.near.sum(), (what, got[4], ref.stats[4])
    return seen


# ================================================================================================ 1. Gaussian head
GAUSS_D = [1, 3, 7, 8, 9, 17, 24, 25, 40]          # both sides of DMAX = 8 / 24 / generic and of the 8-column groups


@pytest.mark.parametrize("layout", lr.LAYOUTS)
@pytest.mark.parametrize("gather", [False, True], ids=["direct", "src_idx"])
@pytest.mark.parametrize("B", [300, 2 * 256 + 1])
@pytest.mark.parametrize("d", GAUSS_D)
def test_gauss_loss_every_instance_and_layout(d, B, gather, layout):
    from baselines_b200 import ops
    rng = np.random.RandomState(d * 1009 + B)
    hb = lr.head_bufs(d, B, layout, rows=B + 3)
    mean32 = rng.randn(B, d).astype(np.float32)
    v32 = rng.randn(B).astype(np.float32)
    ls32 = (0.3 * rng.randn(d)).astype(np.float32)
    hb.ho[:, :d] = _dev(mean32)
    hb.vo[:, 0] = _dev(v32)
    Bbuf = B + 41 if gather else B
    src = rng.permutation(Bbuf)[:B] if gather else np.arange(B)
    acts_buf, acts, oldnlp_buf, oldv_buf, R_buf = _ppo_inputs(rng, "gauss", mean32, v32, B, Bbuf, src, d, logstd=ls32)
    clip, ent, vfc, inv_M = 0.2, 0.03, 0.5, 1.0 / B
    idx = _dev(src.astype(np.int64)) if gather else None
    adv_st = torch.zeros(2, dtype=torch.float64, device="cuda")
    ops.adv_stats(_dev(R_buf), _dev(oldv_buf), idx, B, adv_st)
    prefill = (rng.rand(d) + 0.5).astype(np.float32)         # dL/dlogstd is ACCUMULATED into the buffer
    runs = []
    for _ in range(3):
        dls = _dev(prefill)
        stats = torch.zeros(5, dtype=torch.float64, device="cuda")
        ops.gauss_loss(hb.ho, hb.ld, _dev(ls32), d, hb.vo, hb.ldv, _dev(acts_buf), idx, _dev(R_buf), _dev(oldv_buf),
                       _dev(oldnlp_buf), adv_st, clip, ent, vfc, hb.g, hb.ld_g, hb.dv, hb.ld_dv, dls, inv_M, stats, B)
        torch.cuda.synchronize()
        runs.append((dls.cpu(), stats.cpu().numpy()))
    for dls, _ in runs[1:]:
        assert torch.equal(dls, runs[0][0]), "dL/dlogstd changed between identical calls"
    mean, std = adv_st.cpu().numpy()
    R, oldv, oldnlp = R_buf[src], oldv_buf[src], oldnlp_buf[src]
    adv = lr.adv_normalise(R, oldv, mean, std)
    args = ("gauss", mean32, v32, acts, R, oldv, oldnlp, adv, clip, ent, vfc)
    ref = lr.ppo_ref(*args, logstd=ls32)
    mut = lambda m: lr.ppo_ref(*args, logstd=ls32, mutant=m)
    nb = lr.ppo_ref("gauss", mean32, v32, np.roll(acts, 1, 0), R, oldv, oldnlp, adv, clip, ent, vfc, logstd=ls32)
    ok = ~ref.near
    assert ok.mean() > 0.97
    got = hb.g[:B, :d].float().cpu().numpy()
    _within_f16(got[ok], ref.dhead[ok], {"clipped surrogate passing gradient": mut("pg_clip_passes").dhead[ok],
                                         "actions of the neighbouring row": nb.dhead[ok]}, f"dmean d={d}",
                _gauss_nscale(acts, mean32, ls32, oldnlp)[ok])
    _within_f16(hb.dv[:B, 0].float().cpu().numpy()[ok], ref.dv[ok],
                {"value clip passing gradient": mut("vf_clip_passes").dv[ok],
                 "value gradient of the wrong branch": mut("vf_wrong_branch").dv[ok]}, "dv")
    lr.check_untouched(hb, B, d)
    # dL/dlogstd: sum over rows (fp32), times inv_M, ADDED to the prefill
    rows = ref.dlogstd_rows * inv_M
    want = rows.sum(0)
    delta = runs[0][0].double().numpy() - prefill.astype(np.float64)
    S = np.abs(rows).sum(0) + np.abs(prefill) + np.abs(want)
    seen = assert_within(_t(delta), _t(want), _t(S), G_DLOGSTD, 0.0, {
        "last row of the partial block dropped": _t(want - rows[B - 1]),
        "row 0 of block 1 dropped": _t(want - rows[256]),
        "-ent_coef term dropped": _t(mut("no_entropy").dlogstd_rows.sum(0) * inv_M),
        "overwritten instead of accumulated": _t(want - prefill)}, f"dlogstd d={d}")
    _report(f"gauss dlogstd d={d} B={B} {layout}", seen, G_DLOGSTD)
    for _, st in runs:
        s = _stats_check(st, ref, "gauss", mean32, acts, oldnlp, adv, ls32, B, f"gauss d={d}")
    _report(f"gauss stats d={d} B={B}", s, G_STATS)


@pytest.mark.parametrize("d", GAUSS_D)
def test_gauss_step_injected_normals_vs_float64(d):
    from baselines_b200 import ops
    rng = np.random.RandomState(d)
    B = 300
    hb = lr.head_bufs(d, B, "fused")
    mu = rng.randn(B, d).astype(np.float32)
    v32 = rng.randn(B).astype(np.float32)
    ls = (0.3 + 0.2 * rng.randn(d)).astype(np.float32)
    n = rng.randn(B, d).astype(np.float32)
    hb.ho[:, :d] = _dev(mu)
    hb.vo[:, 0] = _dev(v32)
    a = torch.zeros(B, d, device="cuda")
    val, nlp = torch.zeros(B, device="cuda"), torch.zeros(B, device="cuda")
    ops.gauss_step(hb.ho, hb.ld, _dev(ls), d, hb.vo, hb.ldv, a, val, nlp, B, normals=_dev(n))
    torch.cuda.synchronize()
    assert np.array_equal(val.cpu().numpy(), v32)
    mu64, sd64, n64 = mu.astype(np.float64), np.exp(ls.astype(np.float64)), n.astype(np.float64)
    x = mu64 + sd64 * n64
    got_a = a.cpu().numpy()
    seen = assert_within(_t(got_a), _t(x), _t(np.abs(mu64) + sd64 * np.abs(n64)), 8 * U32, 0.0,
                         {"logstd used as the std": _t(mu64 + ls * n64),
                          "normal of the next row": _t(mu64 + sd64 * np.roll(n64, 1, 0))}, "gauss_step actions")
    _report(f"gauss_step actions d={d}", seen, 8 * U32)
    _check_gauss_nlp(got_a, mu64, ls, nlp.cpu().numpy(), f"gauss_step neglogp d={d}")


def _check_gauss_nlp(got_a, mu64, ls, got_nlp, what):
    """neglogp of the drawn actions against float64 (distributions.py:238-241), within 16 fp32 roundings of the sum of
    its absolute terms."""
    t = (got_a.astype(np.float64) - mu64) / np.exp(ls.astype(np.float64))
    d = t.shape[1]
    want = 0.5 * (t * t).sum(1) + 0.5 * math.log(2 * math.pi) * d + ls.astype(np.float64).sum()
    S = (0.5 * t * t + np.abs(ls) + 0.92).sum(1)
    seen = assert_within(_t(got_nlp), _t(want), _t(S), 16 * U32, 0.0,
                         {"one dimension's log(2 pi) / 2 missing": _t(want - 0.5 * math.log(2 * math.pi)),
                          "sum(logstd) counted twice": _t(want + ls.astype(np.float64).sum())}, what)
    _report(what, seen, 16 * U32)


def test_gauss_step_philox_stream_statistics():
    """d = 25 (odd: the last Box-Muller pair is half used), B = 2^17, fixed seed: the standardised actions have mean 0
    and variance 1 per column, the two members of each pair are uncorrelated (each within 6 sigma), neglogp agrees with
    float64, and offset_dev gives the bits of the equal offset argument."""
    from baselines_b200 import ops
    d, B = 25, 1 << 17
    rng = np.random.RandomState(25)
    mu = rng.randn(d).astype(np.float32)
    ls = (0.2 * rng.randn(d)).astype(np.float32)
    head = torch.zeros(B, 32, device="cuda")
    head[:, :d] = _dev(mu)
    head[:, d] = 0.25
    outs = []
    for kw in (dict(offset=7), dict(offset=0, offset_dev=torch.tensor([7], dtype=torch.int64, device="cuda"))):
        a = torch.zeros(B, d, device="cuda")
        val, nlp = torch.zeros(B, device="cuda"), torch.zeros(B, device="cuda")
        ops.gauss_step(head, 32, _dev(ls), d, head[:, d:], 32, a, val, nlp, B, seed=2024, **kw)
        torch.cuda.synchronize()
        outs.append((a.cpu(), nlp.cpu()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    got_a = outs[0][0].numpy()
    z = (got_a.astype(np.float64) - mu) / np.exp(ls.astype(np.float64))
    assert np.all(np.abs(z.mean(0)) < 6 / math.sqrt(B)), np.abs(z.mean(0)).max()
    assert np.all(np.abs(z.var(0) - 1) < 6 * math.sqrt(2.0 / B)), np.abs(z.var(0) - 1).max()
    corr = (z[:, 0:24:2] * z[:, 1:24:2]).mean(0)
    assert np.all(np.abs(corr) < 6 / math.sqrt(B)), np.abs(corr).max()
    _check_gauss_nlp(got_a, np.broadcast_to(mu.astype(np.float64), (B, d)), ls, outs[0][1].numpy(),
                     "gauss_step Philox neglogp")


# ================================================================================================ 2. Discrete head
CAT_NA = [1, 2, 6, 7, 8, 9, 18]


@pytest.mark.parametrize("layout", lr.LAYOUTS)
@pytest.mark.parametrize("gather", [False, True], ids=["direct", "src_idx"])
@pytest.mark.parametrize("nA", CAT_NA)
def test_cat_step_and_loss_vs_float64(nA, gather, layout):
    from baselines_b200 import ops
    from oracle import nets
    rng = np.random.RandomState(nA * 31 + gather)
    B = 300
    hb = lr.head_bufs(nA, B, layout, rows=B + 3)
    l32 = (rng.randn(B, nA) * 1.5).astype(np.float32)
    v32 = rng.randn(B).astype(np.float32)
    hb.ho[:, :nA] = _dev(l32)
    hb.vo[:, 0] = _dev(v32)
    # ---- act with injected uniforms
    u = (rng.rand(B, nA) * 0.998 + 0.001).astype(np.float32)
    a = torch.zeros(B, dtype=torch.int64, device="cuda")
    val, nlp = torch.zeros(B, device="cuda"), torch.zeros(B, device="cuda")
    ops.cat_step(hb.ho, hb.ld, nA, hb.vo, hb.ldv, a, val, nlp, B, uniforms=_dev(u))
    torch.cuda.synchronize()
    got_a = a.cpu().numpy()
    l64 = torch.tensor(l32, dtype=torch.float64)
    want_a = nets.cat_sample(l64, torch.tensor(u, dtype=torch.float64)).numpy()
    clear = lr.gumbel_clear(l32, u, [nA])
    assert clear.mean() > 0.9 and np.array_equal(got_a[clear], want_a[clear])
    assert np.array_equal(val.cpu().numpy(), v32)
    nlp_ref = nets.cat_neglogp(l64, torch.as_tensor(got_a)).numpy()
    if nA == 1:
        assert float(nlp.abs().max()) == 0.0
    else:
        S = np.abs(l32).max(1) + math.log(nA) + np.abs(l32[np.arange(B), got_a]) + 1
        nxt = nets.cat_neglogp(l64, torch.as_tensor((got_a + 1) % nA)).numpy()
        assert_within(nlp.cpu(), _t(nlp_ref), _t(S), 8 * U32, 0.0, {"neglogp of the next action": _t(nxt)},
                      "cat_step neglogp")
    # ---- loss + gradient
    Bbuf = B + 37 if gather else B
    src = rng.permutation(Bbuf)[:B] if gather else np.arange(B)
    acts_buf, acts, oldnlp_buf, oldv_buf, R_buf = _ppo_inputs(rng, "cat", l32, v32, B, Bbuf, src, nA)
    clip, ent, vfc = 0.2, 0.3, 0.5
    idx = _dev(src.astype(np.int64)) if gather else None
    adv_st = torch.zeros(2, dtype=torch.float64, device="cuda")
    stats = torch.zeros(5, dtype=torch.float64, device="cuda")
    ops.adv_stats(_dev(R_buf), _dev(oldv_buf), idx, B, adv_st)
    ops.cat_loss(hb.ho, hb.ld, nA, hb.vo, hb.ldv, _dev(acts_buf), idx, _dev(R_buf), _dev(oldv_buf), _dev(oldnlp_buf),
                 adv_st, clip, ent, vfc, hb.g, hb.ld_g, hb.dv, hb.ld_dv, stats, B)
    torch.cuda.synchronize()
    mean, std = adv_st.cpu().numpy()
    R, oldv, oldnlp = R_buf[src], oldv_buf[src], oldnlp_buf[src]
    adv = lr.adv_normalise(R, oldv, mean, std)
    args = ("cat", l32, v32, acts, R, oldv, oldnlp, adv, clip, ent, vfc)
    ref = lr.ppo_ref(*args)
    mut = lambda m: lr.ppo_ref(*args, mutant=m)
    ok = ~ref.near
    assert ok.mean() > 0.97
    got = hb.g[:B, :nA].float().cpu().numpy()
    st = stats.cpu().numpy()
    if nA == 1:                                   # p = 1: entropy 0, gradient exactly 0
        assert float(np.abs(got).max()) == 0.0 and st[2] == 0.0
    else:
        nb = lr.ppo_ref("cat", l32, v32, np.roll(acts, 1), R, oldv, oldnlp, adv, clip, ent, vfc)
        _within_f16(got[ok], ref.dhead[ok], {"-ent_coef term dropped": mut("no_entropy").dhead[ok],
                                             "clipped surrogate passing gradient": mut("pg_clip_passes").dhead[ok],
                                             "actions of the neighbouring row": nb.dhead[ok]}, f"dlogits nA={nA}")
    _within_f16(hb.dv[:B, 0].float().cpu().numpy()[ok], ref.dv[ok],
                {"value clip passing gradient": mut("vf_clip_passes").dv[ok],
                 "value gradient of the wrong branch": mut("vf_wrong_branch").dv[ok]}, "dv")
    lr.check_untouched(hb, B, nA)
    s = _stats_check(st, ref, "cat", l32, acts, oldnlp, adv, None, B, f"cat nA={nA}")
    _report(f"cat stats nA={nA} {layout}", s, G_STATS)


def test_cat_step_philox_frequencies_full_atari_action_set():
    """nA = 18 spans five Philox counters; B = 2e5 draws of one logit row match the softmax within 6 sigma per column."""
    from baselines_b200 import ops
    nA, B = 18, 200000
    row = np.linspace(-1.5, 1.2, nA).astype(np.float32)[np.random.RandomState(18).permutation(nA)]
    head = torch.zeros(B, 24, device="cuda")
    head[:, :nA] = _dev(row)
    a = torch.zeros(B, dtype=torch.int64, device="cuda")
    ops.cat_step(head, 24, nA, head[:, nA:], 24, a, torch.zeros(B, device="cuda"), torch.zeros(B, device="cuda"), B,
                 seed=99, offset=3)
    freq = torch.bincount(a, minlength=nA).double().cpu().numpy() / B
    assert len(freq) == nA
    p = np.exp(row.astype(np.float64) - row.max())
    p /= p.sum()
    assert np.all(np.abs(freq - p) < 6 * np.sqrt(p * (1 - p) / B)), np.abs(freq - p) / np.sqrt(p * (1 - p) / B)


# ================================================================================================ 3. PPO branches
def _branch_rows(rng, B, clip):
    """Per row: adv sign and ratio zone (row % 6), value zone compatible with the sign ((row // 6) % 4).  Every quantity
    sits at least 0.05 away from its branch boundary.  Returns target ratio r, adv_raw = R - oldv, dv = v - oldv."""
    r = np.empty(B)
    A = np.empty(B)
    dv = np.empty(B)
    for i in range(B):
        sgn = 1.0 if (i % 6) < 3 else -1.0
        zone = i % 3
        r[i] = [rng.uniform(0.5, 1 - clip - 0.05), rng.uniform(1 - clip + 0.05, 1 + clip - 0.05),
                rng.uniform(1 + clip + 0.05, 1.6)][zone]
        A[i] = sgn * rng.uniform(1.0, 2.0)
        vz = (i // 6) % 4
        a = abs(A[i])
        if vz == 0:                                              # unclipped
            dv[i] = rng.uniform(-clip + 0.05, clip - 0.05)
        elif vz == 1:                                            # clipped away from R: l1 > l2
            dv[i] = -sgn * rng.uniform(clip + 0.05, 1.0)
        elif vz == 2:                                            # clipped towards R, overshooting: l1 >= l2
            dv[i] = sgn * (2 * a - clip + rng.uniform(0.2, 0.5))
        else:                                                    # clipped towards R, short of it: l1 < l2
            dv[i] = sgn * rng.uniform(clip + 0.1, 2 * a - clip - 0.2)
    return r, A, dv


@pytest.mark.parametrize("pd,n", [("cat", 6), ("gauss", 3), ("gauss", 17)])
def test_ppo_loss_branches_deliberately_populated(pd, n):
    from baselines_b200 import ops
    rng = np.random.RandomState(7 + n)
    B, clip, ent, vfc = 600, 0.2, 0.05, 0.5
    hb = lr.head_bufs(n, B, "fused", rows=B)
    head = rng.randn(B, n).astype(np.float32)
    ls = (0.2 * rng.randn(n)).astype(np.float32) if pd == "gauss" else None
    acts = (head + np.exp(ls) * rng.randn(B, n)).astype(np.float32) if pd == "gauss" else rng.randint(0, n, B)
    r, A, dvv = _branch_rows(rng, B, clip)
    z = np.zeros(B)
    nlp = lr.ppo_ref(pd, head, z, acts, z, z, z, z, clip, 0, 0, logstd=ls).nlp
    oldnlp = (nlp + np.log(r)).astype(np.float32)
    oldv = rng.randn(B).astype(np.float32)
    R = (oldv + A).astype(np.float32)
    v32 = (oldv + dvv).astype(np.float32)
    hb.ho[:, :n] = _dev(head)
    hb.vo[:, 0] = _dev(v32)
    adv_st = torch.zeros(2, dtype=torch.float64, device="cuda")
    stats = torch.zeros(5, dtype=torch.float64, device="cuda")
    ops.adv_stats(_dev(R), _dev(oldv), None, B, adv_st)
    dls = torch.zeros(n, device="cuda")
    if pd == "gauss":
        ops.gauss_loss(hb.ho, hb.ld, _dev(ls), n, hb.vo, hb.ldv, _dev(acts), None, _dev(R), _dev(oldv), _dev(oldnlp),
                       adv_st, clip, ent, vfc, hb.g, hb.ld_g, hb.dv, hb.ld_dv, dls, 1.0, stats, B)
    else:
        ops.cat_loss(hb.ho, hb.ld, n, hb.vo, hb.ldv, _dev(acts), None, _dev(R), _dev(oldv), _dev(oldnlp), adv_st, clip,
                     ent, vfc, hb.g, hb.ld_g, hb.dv, hb.ld_dv, stats, B)
    torch.cuda.synchronize()
    mean, std = adv_st.cpu().numpy()
    adv = lr.adv_normalise(R, oldv, mean, std)
    args = (pd, head, v32, acts, R, oldv, oldnlp, adv, clip, ent, vfc)
    ref = lr.ppo_ref(*args, logstd=ls)
    mut = lambda m: lr.ppo_ref(*args, logstd=ls, mutant=m)
    zn = ref.zones
    assert ref.near.sum() == 0
    counts = {f"{s}/{q}": int((zn[s] & zn[q]).sum()) for s in ("adv_pos", "adv_neg")
              for q in ("ratio_below", "ratio_inside", "ratio_above")}
    counts.update({"v_unclipped": int(zn["v_unclipped"].sum())})
    counts.update({f"{q}/{c}": int((zn[q] & zn[c]).sum()) for q in ("v_low", "v_high") for c in ("l1_ge_l2", "l1_lt_l2")})
    print(f"[branches {pd} n={n}] {counts}")
    assert min(counts.values()) >= 20, counts
    got = hb.g[:B, :n].float().cpu().numpy()
    _within_f16(got, ref.dhead, {"clipped surrogate passing gradient": mut("pg_clip_passes").dhead}, "dhead",
                _gauss_nscale(acts, head, ls, oldnlp) if pd == "gauss" else None)
    _within_f16(hb.dv[:B, 0].float().cpu().numpy(), ref.dv,
                {"value clip passing gradient": mut("vf_clip_passes").dv,
                 "value gradient of the wrong branch": mut("vf_wrong_branch").dv}, "dv")
    if pd == "gauss":
        rows = ref.dlogstd_rows
        assert_within(dls.cpu(), _t(rows.sum(0)), _t(np.abs(rows).sum(0)), G_DLOGSTD, 0.0,
                      {"clipped surrogate passing gradient": _t(mut("pg_clip_passes").dlogstd_rows.sum(0))}, "dlogstd")
    _stats_check(stats.cpu().numpy(), ref, pd, head, acts, oldnlp, adv, ls, B, f"branches {pd}")


@pytest.mark.parametrize("pd,n", [("cat", 6), ("cat", 18), ("gauss", 6), ("gauss", 17), ("gauss", 40)])
def test_first_minibatch_old_values_from_the_step_kernel(pd, n):
    """The first minibatch of every update: old neglogp and old values are the step kernel's own outputs on the same
    head values, so v - old_v is exactly 0 and the ratio is 1 (or within an ulp of it)."""
    from baselines_b200 import ops
    rng = np.random.RandomState(n)
    B, clip, ent, vfc = 300, 0.2, 0.01, 0.5
    hb = lr.head_bufs(n, B, "fused")
    head = rng.randn(B, n).astype(np.float32)
    v32 = rng.randn(B).astype(np.float32)
    hb.ho[:, :n] = _dev(head)
    hb.vo[:, 0] = _dev(v32)
    val, nlp = torch.zeros(B, device="cuda"), torch.zeros(B, device="cuda")
    ls = (0.2 * rng.randn(n)).astype(np.float32) if pd == "gauss" else None
    if pd == "gauss":
        a = torch.zeros(B, n, device="cuda")
        ops.gauss_step(hb.ho, hb.ld, _dev(ls), n, hb.vo, hb.ldv, a, val, nlp, B, seed=5, offset=1)
    else:
        a = torch.zeros(B, dtype=torch.int64, device="cuda")
        ops.cat_step(hb.ho, hb.ld, n, hb.vo, hb.ldv, a, val, nlp, B, seed=5, offset=1)
    R = (v32 + rng.randn(B)).astype(np.float32)
    adv_st = torch.zeros(2, dtype=torch.float64, device="cuda")
    stats = torch.zeros(5, dtype=torch.float64, device="cuda")
    ops.adv_stats(_dev(R), val, None, B, adv_st)
    dls = torch.zeros(n, device="cuda")
    if pd == "gauss":
        ops.gauss_loss(hb.ho, hb.ld, _dev(ls), n, hb.vo, hb.ldv, a, None, _dev(R), val, nlp, adv_st, clip, ent, vfc,
                       hb.g, hb.ld_g, hb.dv, hb.ld_dv, dls, 1.0, stats, B)
    else:
        ops.cat_loss(hb.ho, hb.ld, n, hb.vo, hb.ldv, a, None, _dev(R), val, nlp, adv_st, clip, ent, vfc, hb.g,
                     hb.ld_g, hb.dv, hb.ld_dv, stats, B)
    torch.cuda.synchronize()
    oldv, oldnlp, acts = val.cpu().numpy(), nlp.cpu().numpy(), a.cpu().numpy()
    assert np.array_equal(oldv, v32)
    st = stats.cpu().numpy()
    # approxkl sums 0.5 (nlp - old_nlp)^2 over rows: it is exactly 0 iff the loss kernel reproduced every row's
    # neglogp bit for bit, i.e. the ratio is exactly 1 in every row
    exact = st[3] == 0.0
    print(f"[first minibatch {pd} n={n}] ratio exactly 1 in {'all' if exact else 'not all'} {B} rows "
          f"(approxkl sum {st[3]:.3e}), clipfrac sum {st[4]}")
    assert st[3] <= B * 1e-10 and st[4] == 0.0
    mean, std = adv_st.cpu().numpy()
    adv = lr.adv_normalise(R, oldv, mean, std)
    args = (pd, head, v32, acts, R, oldv, oldnlp, adv, clip, ent, vfc)
    ref = lr.ppo_ref(*args, logstd=ls)
    mut = lambda m: lr.ppo_ref(*args, logstd=ls, mutant=m)
    assert not ref.near.any() and np.all(np.abs(ref.ratio - 1) < 1e-4)
    _within_f16(hb.g[:B, :n].float().cpu().numpy(), ref.dhead,
                {"-ent_coef term dropped": mut("no_entropy").dhead} if pd == "cat" else
                {"actions of the neighbouring row": lr.ppo_ref(pd, head, v32, np.roll(acts, 1, 0), R, oldv, oldnlp,
                                                               adv, clip, ent, vfc, logstd=ls).dhead}, "dhead",
                _gauss_nscale(acts, head, ls, oldnlp) if pd == "gauss" else None)
    _within_f16(hb.dv[:B, 0].float().cpu().numpy(), ref.dv, {"value gradient 0": np.zeros(B)}, "dv")
    assert np.allclose(ref.dv, vfc * (v32.astype(np.float64) - R))


# ================================================================================================ 4. adv_stats
def _adv_depth(M):
    """Longest chain of fp64 additions in adv_stats: 8 per 4096-element sweep of a thread, 5 warp-shuffle levels, the 16
    warp sums of a block, then the blocks' partials in order."""
    blocks = min((M + 4095) // 4096, 128)
    per = -(-M // blocks)
    return 8 * (-(-per // 4096)) + 5 + 16 + blocks, blocks, per


def _adv_bound(d, M):
    """One-pass fp64 bound.  S1 = sum d and S2 = sum d^2 (each d^2 exact in fp64) carry at most gamma_k of sum|d| and
    sum d^2; mean = S1/M and var = S2/M - mean^2 then give
        |mean - mean*| <= gamma_{k+1} E|d|,   |var - var*| <= 4 gamma_{k+3} E[d^2],
        |std - std*| <= 4 gamma_{k+3} E[d^2] / std* + 2u std*."""
    k = _adv_depth(M)[0]
    d = d.astype(np.float64)
    e1, e2 = np.abs(d).mean(), (d * d).mean()
    std = d.std()
    return np.array([lr.gamma_k(k + 1) * e1 + 1e-300,
                     4 * lr.gamma_k(k + 3) * e2 / max(std, 1e-300) + 2 * 2.0 ** -53 * std]), k


def _run_adv(R, V, idx, M, reps=3):
    from baselines_b200 import ops
    outs = []
    for _ in range(reps):
        out = torch.zeros(2, dtype=torch.float64, device="cuda")
        ops.adv_stats(R, V, idx, M, out)
        torch.cuda.synchronize()
        outs.append(out.cpu())
    for o in outs[1:]:
        assert torch.equal(o, outs[0]), "adv_stats changed between identical calls"
    return outs[0].numpy()


@pytest.mark.parametrize("gather", [False, True], ids=["direct", "src_idx"])
@pytest.mark.parametrize("M", [1, 4095, 4096, 4097, 128 * 4096, 128 * 4096 + 1, 3_000_000])
def test_adv_stats_vs_two_pass_float64(M, gather):
    gen = torch.Generator(device="cuda").manual_seed(M + gather)
    Mbuf = M + 13 if gather else M
    R = torch.randn(Mbuf, device="cuda", generator=gen) * 1.5 + 0.3
    V = torch.randn(Mbuf, device="cuda", generator=gen)
    src = torch.randperm(Mbuf, device="cuda", generator=gen)[:M] if gather else None
    got = _run_adv(R, V, src, M)
    s = src.cpu().numpy() if gather else np.arange(M)
    d = (R.cpu().numpy()[s] - V.cpu().numpy()[s])
    mean, std = lr.adv_moments(R.cpu().numpy()[s], V.cpu().numpy()[s])
    if M == 1:
        assert got[0] == d[0] and got[1] == 0.0
        return
    bound, k = _adv_bound(d, M)
    _, blocks, per = _adv_depth(M)

    def moments_without(keep):                 # what the kernel would report with the other elements' sums lost
        x = d[keep].astype(np.float64)
        m = x.sum() / M
        return _t([m, math.sqrt(max((x * x).sum() / M - m * m, 0.0))])

    mutants = {"last element dropped": moments_without(slice(0, M - 1))}
    if blocks > 1:
        mutants["last block's partial dropped"] = moments_without(slice(0, (blocks - 1) * per))
    else:
        mutants["the only block's partial dropped"] = _t([0.0, 0.0])
    seen = assert_within(_t(got), _t([mean, std]), _t(bound), 1.0, 0.0, mutants, f"adv_stats M={M}")
    print(f"[observed] adv_stats M={M} blocks={blocks} k={k}: {seen:.3e} of the one-pass bound")


def test_adv_stats_single_row_normalises_to_zero():
    """M = 1: std is exactly 0 and the normalised advantage (d - mean) / (std + 1e-8) is exactly 0, not NaN."""
    from baselines_b200 import ops
    hb = lr.head_bufs(6, 1, "fused")
    hb.ho[:, :7] = torch.tensor([[0.5, -1.0, 2.0, 0.0, 0.25, 1.0, 0.75]], device="cuda")
    R, V = torch.tensor([1.7], device="cuda"), torch.tensor([-0.4], device="cuda")
    adv_st = torch.zeros(2, dtype=torch.float64, device="cuda")
    ops.adv_stats(R, V, None, 1, adv_st)
    stats = torch.zeros(5, dtype=torch.float64, device="cuda")
    ops.cat_loss(hb.ho, hb.ld, 6, hb.vo, hb.ldv, torch.tensor([2], device="cuda"), None, R, V,
                 torch.tensor([1.0], device="cuda"), adv_st, 0.2, 0.0, 0.0, hb.g, hb.ld_g, hb.dv, hb.ld_dv, stats, 1)
    torch.cuda.synchronize()
    assert float(adv_st[1]) == 0.0 and float(adv_st[0]) == float(np.float32(1.7) - np.float32(-0.4))
    assert float(hb.g[0, :6].float().abs().max()) == 0.0                 # adv 0, no entropy or value term
    st = stats.cpu().numpy()
    assert np.all(np.isfinite(st)) and st[0] == 0.0


def test_adv_stats_large_mean_over_std():
    """|mean| / std = 1e4 stresses the E[d^2] - mean^2 form: its one-pass bound is 4 gamma_{k+3} (1 + 1e8) relative to
    the variance, under 1e-5 of std for M = 1e6 (k = 165); numpy's float32 np.std of the same array, which
    ppo2/model.py:138 uses, is no better.  The kernel must stay inside it."""
    M = 1_000_000
    gen = torch.Generator(device="cuda").manual_seed(4)
    R = 1e4 + torch.randn(M + 5, device="cuda", generator=gen)
    V = torch.randn(M + 5, device="cuda", generator=gen) * 0.1
    src = torch.randperm(M + 5, device="cuda", generator=gen)[:M]
    got = _run_adv(R, V, src, M)
    s = src.cpu().numpy()
    d = R.cpu().numpy()[s] - V.cpu().numpy()[s]
    mean, std = lr.adv_moments(R.cpu().numpy()[s], V.cpu().numpy()[s])
    assert 0.9e4 < abs(mean) / std < 1.1e4
    bound, k = _adv_bound(d, M)
    assert bound[1] / std < 2e-5
    x = d[:-1].astype(np.float64)
    seen = assert_within(_t(got), _t([mean, std]), _t(bound), 1.0, 0.0,
                         {"last element dropped": _t([x.sum() / M, std])}, "adv_stats |mean|/std = 1e4")
    print(f"[observed] adv_stats |mean|/std=1e4: std rel err {abs(got[1] - std) / std:.3e}, {seen:.3e} of the bound")


# ================================================================================================ 5. optimiser
def _sumsq_depth(n, sms):
    grid = max(1, min(-(-(n // 4 + 1) // 256), 4 * sms))
    per = -(-(n // 4) // (grid * 256)) if n >= 4 else 0
    return 4 * per + 1 + 5 + 8 + grid


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 1023, (1 << 20) + 3])
def test_sumsq_tail_carries_the_mass(n):
    """Relative bound gamma_k (all terms positive), k the summation depth: 4 adds per float4 per grid-stride sweep, the
    tail, 5 shuffle levels, 8 warp sums, then one add per block.  The n % 4 tail elements carry most of the mass."""
    from baselines_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(n)
    g = torch.randn(n, device="cuda", generator=gen) * 1e-3
    tail = n - n % 4
    g[tail:] = 1e3 * (1 + torch.rand(n - tail, device="cuda", generator=gen))
    g64 = g.double().cpu().numpy()
    ref = math.fsum(g64 * g64)
    outs = []
    for _ in range(3):
        ss = torch.zeros(1, dtype=torch.float64, device="cuda")
        ops.sumsq(g, ss)
        torch.cuda.synchronize()
        outs.append(ss.cpu())
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
    k = _sumsq_depth(n, ops.num_sms())
    mutants = {"last element dropped": _t([ref - g64[-1] ** 2])}
    if n % 4:
        mutants["tail dropped"] = _t([ref - math.fsum(g64[tail:] ** 2)])
    if n >= 4:
        mutants["first element dropped"] = _t([ref - g64[0] ** 2])
    seen = assert_within(outs[0], _t([ref]), _t([ref]), lr.gamma_k(k), 0.0, mutants, f"sumsq n={n}")
    print(f"[observed] sumsq n={n} k={k}: rel err {seen:.3e} (gamma_k {lr.gamma_k(k):.3e})")


def test_sumsq_refuses_an_unaligned_gradient():
    from baselines_b200 import ops
    buf = torch.ones(17, device="cuda")
    ss = torch.full((1,), -1.0, dtype=torch.float64, device="cuda")
    with pytest.raises(RuntimeError, match="16 B aligned"):
        ops.sumsq(buf[1:], ss)
    torch.cuda.synchronize()
    assert float(ss[0]) == -1.0


SEG_TABLES = {
    "empty_and_single": [0, 1, 5000, 0, 1, 3, 17, 0, 4096, 4097],
    "300_segments": list(np.random.RandomState(300).choice([0, 1, 2, 7, 33, 260], 300)),
}


def _check_seg_sumsq(g, off, what):
    """Per segment: relative gamma_k bound, k = ceil(len / 4096) + 5 + 8 + 16 (thread sweep, shuffles, warp sums,
    the 16 slice sums); empty segments are exactly 0 and length-1 segments exact."""
    from baselines_b200 import ops
    nseg = len(off) - 1
    outs = []
    for _ in range(3):
        out = torch.full((nseg,), float("nan"), dtype=torch.float64, device="cuda")
        ops.seg_sumsq(g, _dev(off.astype(np.int64)), nseg, out)
        torch.cuda.synchronize()
        outs.append(out.cpu())
    for o in outs[1:]:
        assert torch.equal(o, outs[0]), f"{what}: seg_sumsq changed between identical calls"
    g64 = g.double().cpu().numpy()
    sq = g64 * g64
    lens = np.diff(off)
    ref = np.array([math.fsum(sq[off[s]:off[s + 1]]) for s in range(nseg)])
    k = np.ceil(lens / 4096) + 5 + 8 + 16
    bound = np.array([lr.gamma_k(int(x)) for x in k]) * ref
    got = outs[0].numpy()
    assert np.all(got[lens == 0] == 0.0) and np.array_equal(got[lens == 1], ref[lens == 1])
    last = np.array([sq[off[s + 1] - 1] if lens[s] else 0.0 for s in range(nseg)])
    shifted = np.array([math.fsum(sq[off[s] + 1:off[s + 1] + 1]) if lens[s] else 0.0 for s in range(nseg)])
    seen = assert_within(outs[0], _t(ref), _t(bound), 1.0, 0.0,
                         {"each segment's last element dropped": _t(ref - last),
                          "segment bounds shifted by one": _t(shifted)}, what)
    print(f"[observed] {what}: {seen:.3e} of the gamma_k bound")
    return outs[0]


@pytest.mark.parametrize("table", list(SEG_TABLES))
def test_seg_sumsq_tables(table):
    sizes = np.asarray(SEG_TABLES[table], np.int64)
    off = np.concatenate([[0], np.cumsum(sizes)])
    n = int(off[-1]) + 1                                   # one element past the last segment: must not count
    gen = torch.Generator(device="cuda").manual_seed(len(sizes))
    scale = np.repeat(10.0 ** np.random.RandomState(1).uniform(-3, 1, len(sizes)), sizes)
    g = torch.randn(n, device="cuda", generator=gen)
    g[:-1] *= _dev(scale).float()
    g[_dev(off[1:][sizes > 0] - 1)] = 1.0                  # last element of every segment is visible
    _check_seg_sumsq(g, off, f"seg_sumsq {table}")


def test_seg_sumsq_dqn_store_table():
    """The per-variable table of a DQN network's parameter store (tf.clip_by_norm per variable)."""
    from baselines_b200.common import spaces
    from baselines_b200.deepq.build_graph import DQNModel
    model = DQNModel(spaces.Box(-5, 5, (8,), np.float32), 6, "mlp", lr=1e-4, gamma=0.99, grad_norm_clipping=10,
                     batch_cap=32, seed=0, hiddens=(256,), dueling=True)
    store = model.q.store
    off = store.segment_offsets()
    assert len(off) > 4 and off[-1] == store.numel
    gen = torch.Generator(device="cuda").manual_seed(0)
    store.grads.copy_(torch.randn(store.numel, device="cuda", generator=gen))
    store.grads[_dev(off[1:] - 1)] = 1.0
    _check_seg_sumsq(store.grads, off, "seg_sumsq DQN store")


def test_clip_adam_per_segment_factor_at_every_boundary():
    """beta1 = beta2 = 0 makes m the clipped gradient.  Neighbouring segments' norms differ by >= 2x (some above, some
    below clip, one segment empty, one of length 1); every element, including each segment's first and last, must
    carry its own segment's factor."""
    from baselines_b200 import ops
    sizes = [37, 0, 300, 1, 5000, 64, 129, 2]
    norms = [8.0, 1.0, 0.5, 4.0, 1.5, 16.0, 0.25, 3.0]
    clip = 1.0
    rng = np.random.RandomState(8)
    parts = []
    for s, nm in zip(sizes, norms):
        x = rng.randn(s)
        parts.append(x / np.linalg.norm(x) * nm if s else x)
    g64 = np.concatenate(parts).astype(np.float32).astype(np.float64)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    n = int(off[-1])
    g = _dev(g64.astype(np.float32))
    ss = torch.zeros(len(sizes), dtype=torch.float64, device="cuda")
    ops.seg_sumsq(g, _dev(off), len(sizes), ss)
    p, m, v = (torch.zeros(n, device="cuda") for _ in range(3))
    ops.clip_adam(p, g, m, v, 1.0, 0.0, 0.0, 1.0, clip, ss, seg_off=_dev(off), nseg=len(sizes))
    torch.cuda.synchronize()
    fac = np.array([lr.clip_scale(math.fsum(g64[off[s]:off[s + 1]] ** 2), clip) for s in range(len(sizes))])
    nonempty = [s for s in range(len(sizes)) if sizes[s]]
    for a, b in zip(nonempty, nonempty[1:]):
        assert max(fac[a], fac[b]) >= 2 * min(fac[a], fac[b]), (a, b, fac)
    seg_of = np.repeat(np.arange(len(sizes)), sizes)
    ref = g64 * fac[seg_of]
    first, last = off[:-1][np.array(sizes) > 0], off[1:][np.array(sizes) > 0] - 1
    prev_fac, next_fac = ref.copy(), ref.copy()
    prev_fac[first[1:]] = g64[first[1:]] * fac[seg_of[first[1:] - 1]]       # the previous segment's factor
    next_fac[last[:-1]] = g64[last[:-1]] * fac[seg_of[last[:-1] + 1]]       # the next segment's factor
    assert_within(m.cpu(), _t(ref), _t(np.abs(ref)), 4 * U32, 0.0,
                  {"first element scaled by the previous segment's factor": _t(prev_fac),
                   "last element scaled by the next segment's factor": _t(next_fac)}, "clip_adam per segment")


def test_clip_adam_global_norm_below_at_and_above_clip():
    """Small-integer gradient with ||g|| = 10 exactly: clip 20 (below) and 10 (equal) give a scale of exactly 1, clip 4
    gives fp32(4 / 10); clip <= 0 without a norm buffer does not clip.  m (beta1 = 0) is compared bit for bit."""
    from baselines_b200 import ops
    rng = np.random.RandomState(9)
    g32 = rng.choice([-1.0, 1.0], 100).astype(np.float32)               # sum of squares 100
    g = _dev(g32)
    ss = torch.zeros(1, dtype=torch.float64, device="cuda")
    ops.sumsq(g, ss)
    torch.cuda.synchronize()
    assert float(ss[0]) == 100.0
    for clip, want in ((20.0, g32), (10.0, g32), (4.0, g32 * (np.float32(4.0) / np.float32(10.0))),
                       (0.0, g32), (-1.0, g32)):
        p, m, v = (torch.zeros(100, device="cuda") for _ in range(3))
        ops.clip_adam(p, g, m, v, 1.0, 0.0, 0.0, 1.0, clip, ss if clip > 0 else None)
        torch.cuda.synchronize()
        assert np.array_equal(m.cpu().numpy(), want), clip


def _adam_case(n=10001, seed=10):
    rng = np.random.RandomState(seed)
    p0 = rng.randn(n).astype(np.float32)
    gs = [(rng.randn(n) * 1e-3 * s).astype(np.float32) for s in (1.0, 0.3, 0.2)]
    return p0, gs


def test_clip_adam_lr_t_dev_equals_host_lr_t():
    from baselines_b200 import ops
    p0, gs = _adam_case(seed=11)
    res = []
    for use_dev in (False, True):
        p, g = _dev(p0), _dev(gs[0])
        m, v = torch.zeros_like(p), torch.zeros_like(p)
        lr_t = 1e-3 * math.sqrt(1 - 0.999) / (1 - 0.9)
        dev_t = torch.tensor([lr_t], dtype=torch.float32, device="cuda") if use_dev else None
        ops.clip_adam(p, g, m, v, 123.0 if use_dev else lr_t, 0.9, 0.999, 1e-5, 0.0, None, lr_t_dev=dev_t)
        torch.cuda.synchronize()
        res.append(p.cpu())
    assert torch.equal(res[0], res[1]) and not torch.equal(res[0], torch.from_numpy(p0))


def test_clip_adam_three_step_trajectory_vs_float64_tf_adam():
    """Global clipping (step 1 above clip, steps 2-3 below) + TF-Adam in the order of mpi_adam.py:37-42, three steps,
    against float64 with the same fp32 hyper-parameters.  Bound: 16 fp32 roundings of a scale that is the same
    trajectory run on |g| (no cancellation); mutants: eps inside the bias correction (the Keras / paper order) and the
    first step unclipped."""
    from baselines_b200 import ops
    f = lambda x: float(np.float32(x))
    b1, b2, eps, base_lr, clip = f(0.9), f(0.999), f(1e-5), 1e-3, 0.05
    p0, gs = _adam_case()
    p, m, v = _dev(p0), torch.zeros(len(p0), device="cuda"), torch.zeros(len(p0), device="cuda")
    ss = torch.zeros(1, dtype=torch.float64, device="cuda")
    P = {k: p0.astype(np.float64) for k in ("ref", "keras", "noclip")}
    M = {k: np.zeros(len(p0)) for k in P}
    V = {k: np.zeros(len(p0)) for k in P}
    Sp, Sm = np.abs(p0).astype(np.float64), np.zeros(len(p0))
    norms = []
    for t, g32 in enumerate(gs, 1):
        gd = _dev(g32)
        ops.sumsq(gd, ss)
        lr_t = f(base_lr * math.sqrt(1 - b2 ** t) / (1 - b1 ** t))
        ops.clip_adam(p, gd, m, v, lr_t, b1, b2, eps, clip, ss)
        g64 = g32.astype(np.float64)
        sq = math.fsum(g64 * g64)
        norms.append(math.sqrt(sq))
        sc = lr.clip_scale(sq, clip)
        for k in P:
            gk = g64 * (1.0 if (k == "noclip" and t == 1) else sc)
            if k == "keras":
                M[k] = b1 * M[k] + (1 - b1) * gk
                V[k] = b2 * V[k] + (1 - b2) * gk * gk
                P[k] = P[k] - base_lr * (M[k] / (1 - b1 ** t)) / (np.sqrt(V[k] / (1 - b2 ** t)) + eps)
            else:
                P[k], M[k], V[k] = lr.adam_tf(P[k], gk, M[k], V[k], lr_t, b1, b2, eps)
        Sm = b1 * Sm + (1 - b1) * np.abs(g64 * sc)
        Sp = Sp + lr_t * Sm / (np.sqrt(V["ref"]) + eps)
    torch.cuda.synchronize()
    assert norms[0] > clip > max(norms[1:]), norms
    gb = 16 * U32
    assert_within(m.cpu(), _t(M["ref"]), _t(Sm), gb, 0.0, {"first step unclipped": _t(M["noclip"])}, "adam m")
    assert_within(v.cpu(), _t(V["ref"]), _t(V["ref"]), gb, 0.0, {"first step unclipped": _t(V["noclip"])}, "adam v")
    seen = assert_within(p.cpu(), _t(P["ref"]), _t(Sp), gb, 0.0,
                         {"eps inside the bias correction": _t(P["keras"]), "first step unclipped": _t(P["noclip"])},
                         "adam p")
    _report("adam p after 3 steps", seen, gb)


def test_clip_accumulate_microbatches_then_adam():
    """MicrobatchedModel: three microbatch gradients with norms 3, 0.5, 1.5 against clip 1 (clipped, not, clipped),
    each added with weight 1/3; the sum then goes through clip_adam with clip = 0 unchanged."""
    from baselines_b200 import ops
    rng = np.random.RandomState(12)
    n, clip, w = 4099, 1.0, 1.0 / 3
    gs = []
    for nm in (3.0, 0.5, 1.5):
        x = rng.randn(n)
        gs.append((x / np.linalg.norm(x) * nm).astype(np.float32))
    acc = torch.zeros(n, device="cuda")
    ss = torch.zeros(1, dtype=torch.float64, device="cuda")
    ref, S, unclipped, noweight = (np.zeros(n) for _ in range(4))
    for i, g32 in enumerate(gs):
        gd = _dev(g32)
        ops.sumsq(gd, ss)
        ops.clip_accumulate(gd, acc, clip, w, ss)
        g64 = g32.astype(np.float64)
        sc = lr.clip_scale(math.fsum(g64 * g64), clip)
        ref += g64 * sc * w
        S += np.abs(g64) * sc * w
        unclipped += g64 * (1.0 if i == 0 else sc) * w
        noweight += g64 * sc
    torch.cuda.synchronize()
    assert_within(acc.cpu(), _t(ref), _t(S), 8 * U32, 0.0,
                  {"first microbatch unclipped": _t(unclipped), "weight missing": _t(noweight)}, "clip_accumulate")
    p, m, v = (torch.zeros(n, device="cuda") for _ in range(3))
    ops.clip_adam(p, acc, m, v, 1.0, 0.0, 0.0, 1.0, 0.0, None)
    torch.cuda.synchronize()
    assert torch.equal(m, acc)


# ================================================================================================ 6. DQN TD step
def _run_dqn(heads, nA, dueling, idx, act, rew, done, w, gamma, double_q, B):
    from baselines_b200 import ops
    ht, hon, htg = (_dev(h) for h in heads)
    ld = heads[0].shape[1]
    sp = (lambda h: h[:, nA:]) if dueling else (lambda h: None)
    td = torch.zeros(B, device="cuda")
    d_a = torch.full((B, 32), float("nan"), dtype=torch.float16, device="cuda")
    d_s = torch.full((B, 8), float("nan"), dtype=torch.float16, device="cuda") if dueling else None
    loss = torch.zeros(1, dtype=torch.float64, device="cuda")
    ops.dqn_td(ht, ld, sp(ht), ld, hon, ld, sp(hon), ld, htg, ld, sp(htg), ld, nA, idx, _dev(act), _dev(rew),
               _dev(done), _dev(w), gamma, double_q, td, d_a, 32, d_s, 8, loss, B)
    torch.cuda.synchronize()
    assert bool(torch.isnan(d_a[:, nA:].float()).all()), "dqn_td wrote past nA"
    return (td.cpu().numpy(), d_a[:, :nA].float().cpu().numpy(),
            d_s[:, 0].float().cpu().numpy() if dueling else None, float(loss[0]))


def _dqn_ref(heads, nA, dueling, rows, act, rew, done, w, gamma, double_q, mutant=None):
    s = (lambda h: h[:, nA]) if dueling else (lambda h: None)
    ht, hon, htg = heads
    return lr.dqn_ref(ht[:, :nA], s(ht), hon[:, :nA], s(hon), htg[:, :nA], s(htg), act[rows], rew[rows], done[rows],
                      w, gamma, double_q, mutant=mutant)


@pytest.mark.parametrize("gather", [False, True], ids=["idx_none", "replay_idx"])
@pytest.mark.parametrize("nA", [1, 2, 6, 18])
@pytest.mark.parametrize("dueling", [True, False], ids=["dueling", "plain"])
@pytest.mark.parametrize("double_q", [True, False], ids=["double_q", "max"])
def test_dqn_td_vs_float64(double_q, dueling, nA, gather):
    rng = np.random.RandomState(nA * 7 + 2 * dueling + double_q)
    B, gamma = 300, 0.99
    Nbuf = 1000 if gather else B
    heads = []
    for _ in range(3):
        h = np.zeros((B, 24), np.float32)
        h[:, :nA + 1] = rng.randn(B, nA + 1) * 2
        heads.append(h)
    act = rng.randint(0, nA, Nbuf).astype(np.int64)
    rew = rng.randn(Nbuf).astype(np.float32)
    done = (rng.rand(Nbuf) < 0.1).astype(np.float32)
    w = (rng.rand(B) * 0.9 + 0.1).astype(np.float32)               # per batch row, never gathered
    rows = rng.permutation(Nbuf)[:B] if gather else np.arange(B)
    # where the online top-2 gap is inside fp32 rounding the kernel may pick either action: make those rows terminal
    gap = _dqn_ref(heads, nA, dueling, rows, act, rew, done, w, gamma, double_q).gap
    tie = gap < 1e-4
    assert tie.sum() <= 3
    done[rows[tie]] = 1.0
    idx = _dev(rows.astype(np.int64)) if gather else None
    td, d_a, d_s, loss = _run_dqn(heads, nA, dueling, idx, act, rew, done, w, gamma, double_q, B)
    ref = _dqn_ref(heads, nA, dueling, rows, act, rew, done, w, gamma, double_q)
    no_done = _dqn_ref(heads, nA, dueling, rows, act, rew, np.zeros_like(done), w, gamma, double_q)
    g2 = _dqn_ref(heads, nA, dueling, rows, act, rew, done, w, gamma * gamma, double_q)
    muts = {"dones ignored": no_done.td, "gamma squared": g2.td}
    if gather:
        muts["rewards read by batch row"] = ref.td - rew[rows] + rew[np.arange(B)]
    _within_f16(td, ref.td, muts, "td")
    clipped = np.clip(ref.td, -1, 1)
    ratio = np.where(clipped != 0, ref.td / np.where(clipped != 0, clipped, 1), 1.0)
    if dueling and nA == 1:
        assert float(np.abs(d_a).max()) == 0.0
    else:
        _within_f16(d_a, ref.d_a, {"Huber gradient not clipped": ref.d_a * ratio[:, None],
                                   "weights ignored": ref.d_a / w[:, None]}, "d_a")
    if dueling:
        _within_f16(d_s, ref.d_s, {"Huber gradient not clipped": ref.d_s * ratio, "weights ignored": ref.d_s / w},
                    "d_s")
    big = int(np.argmax(ref.rows_loss))
    assert_within(_t([loss]), _t([ref.loss]), _t([np.abs(ref.rows_loss).sum()]), 1e-6, 0.0,
                  {"largest row dropped": _t([ref.loss - ref.rows_loss[big]])}, "loss_sum")


@pytest.mark.parametrize("double_q", [True, False], ids=["double_q", "max"])
@pytest.mark.parametrize("dueling", [True, False], ids=["dueling", "plain"])
def test_dqn_td_exact_small_integer_cases(dueling, double_q):
    """Small integers, gamma = 0.5, dyadic weights, nA = 4 (the dueling mean is exact): every value is exact in fp32,
    fp16 and fp64, so the kernel must match float64 bit for bit.  Rows cycle through: an online argmax tie (the first
    index must win), a tie in the target max, |td| = 1 exactly, done = 1, and plain random rows."""
    rng = np.random.RandomState(13 + 2 * dueling + double_q)
    B, nA, gamma, Nbuf = 64, 4, 0.5, 200
    ints = lambda *s: rng.randint(-4, 5, s).astype(np.float32)
    heads = [np.zeros((B, 8), np.float32) for _ in range(3)]
    for h in heads:
        h[:, :nA + 1] = ints(B, nA + 1)
    rows = rng.permutation(Nbuf)[:B]
    act = rng.randint(0, nA, Nbuf).astype(np.int64)
    rew = ints(Nbuf)
    done = np.zeros(Nbuf, np.float32)
    w = rng.choice([0.25, 0.5, 1.0], B).astype(np.float32)
    kind = np.arange(B) % 5
    for b in np.where(kind == 0)[0]:
        heads[1][b, :nA] = [2, 5, 5, 1]
        heads[2][b, :nA] = [0, 1, 3, -2]
    for b in np.where(kind == 1)[0]:
        heads[2][b, :nA] = [4, 1, 4, 0]
    done[rows[kind == 3]] = 1.0
    # |td| = 1: set the selected q (or, dueling, the state score) so that q_sel - target = +-1
    r0 = _dqn_ref(heads, nA, dueling, rows, act, rew, done, w, gamma, double_q)
    for b in np.where(kind == 2)[0]:
        shift = (1.0 if b % 2 else -1.0) - r0.td[b]
        heads[0][b, nA if dueling else act[rows[b]]] += shift
    ref = _dqn_ref(heads, nA, dueling, rows, act, rew, done, w, gamma, double_q)
    assert np.array_equal(np.abs(ref.td[kind == 2]), np.ones((kind == 2).sum()))
    assert np.array_equal(ref.td, ref.td.astype(np.float32)), "a case is not exact in fp32"
    for x in (ref.d_a, ref.d_s if dueling else ref.d_a):
        assert np.array_equal(x, x.astype(np.float16).astype(np.float64)), "a case is not exact in fp16"
    td, d_a, d_s, loss = _run_dqn(heads, nA, dueling, _dev(rows.astype(np.int64)), act, rew, done, w, gamma,
                                  double_q, B)
    assert np.array_equal(td, ref.td) and np.array_equal(d_a, ref.d_a)
    if dueling:
        assert np.array_equal(d_s, ref.d_s)
    assert loss == ref.loss
    if double_q:                                          # the tie rows are what a last-max-wins kernel gets wrong
        last = _dqn_ref(heads, nA, dueling, rows, act, rew, done, w, gamma, double_q, mutant="last_max")
        assert not np.array_equal(td[kind == 0], last.td[kind == 0])


# ================================================================================================ determinism
def test_update_path_reductions_repeat_bit_for_bit():
    """dL/dlogstd (per-block partials added in order), adv_stats (the last block adds the block partials in order) and
    seg_sumsq (16 slices per segment added in order) give the same bits on every call, at sizes with many blocks."""
    from baselines_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(21)
    for d in (6, 17, 40):
        B = 3 * 4096 + 5
        mean = torch.randn(B, d + 1, device="cuda", generator=gen)
        acts = torch.randn(B, d, device="cuda", generator=gen)
        ls = torch.randn(d, device="cuda", generator=gen) * 0.2
        R, V = torch.randn(B, device="cuda", generator=gen), torch.randn(B, device="cuda", generator=gen)
        onlp = torch.randn(B, device="cuda", generator=gen) + d
        adv_st = torch.zeros(2, dtype=torch.float64, device="cuda")
        ops.adv_stats(R, V, None, B, adv_st)
        ld_dm = lr.pad(d, 8)
        dmean = torch.zeros(B, ld_dm, dtype=torch.float16, device="cuda")
        dv = torch.zeros(B, 8, dtype=torch.float16, device="cuda")
        stats = torch.zeros(5, dtype=torch.float64, device="cuda")
        outs = []
        for _ in range(3):
            dls = torch.zeros(d, device="cuda")
            ops.gauss_loss(mean, d + 1, ls, d, mean[:, d:], d + 1, acts, None, R, V, onlp, adv_st, 0.2, 0.01, 0.5,
                           dmean, ld_dm, dv, 8, dls, 1.0 / B, stats, B)
            outs.append(dls.cpu())
        assert all(torch.equal(o, outs[0]) for o in outs[1:]), d
    M = 3_000_000
    R, V = torch.randn(M, device="cuda", generator=gen), torch.randn(M, device="cuda", generator=gen)
    src = torch.randperm(M, device="cuda", generator=gen)
    _run_adv(R, V, src, M)                                     # asserts three identical results
    g = torch.randn(400000, device="cuda", generator=gen)
    off = np.concatenate([[0], np.cumsum(np.random.RandomState(2).randint(0, 3000, 133))])
    assert off[-1] <= g.numel()
    _check_seg_sumsq(g, off, "seg_sumsq repeat")
