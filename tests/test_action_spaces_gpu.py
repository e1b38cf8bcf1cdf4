"""GPU: MultiDiscrete / MultiBinary action heads and MultiDiscrete observations on the PPO2 learner.

Head kernels against float64 autograd (tests/_action_oracle.py restates MultiCategoricalPd / BernoulliPd of
common/distributions.py), the Discrete path as the one-segment case, parity of Model / Runner with the CPU oracle in
the form of test_ppo2_gpu.py, checkpoints, and the reference's learning test test_multidiscrete_identity
(common/tests/test_identity.py:43-56)."""
import math
import os

import numpy as np
import pytest
import torch

import _action_oracle as ao
import _loss_refs as lr
from oracle import nets

pytestmark = pytest.mark.gpu


def _pad(n, m):
    return (n + m - 1) // m * m


def _dev(a, dt=None):
    t = torch.as_tensor(np.ascontiguousarray(a))
    return (t if dt is None else t.to(dt)).cuda()


# ================================================================================================ 1. head kernels
HEADS = [("mcat", (1, 2, 3)), ("mcat", (3, 3)), ("mcat", (20, 30, 17)), ("bern", 5), ("bern", 33)]


def _seg_entropies(l64, nvec):
    out = []
    for blk in torch.split(l64, list(nvec), dim=1):
        lp = torch.log_softmax(blk, 1)
        out.append(-(lp.exp() * lp).sum(1))
    return torch.stack(out, 1)


def _within_fp16(got, ref):
    return np.abs(got - ref) <= 2.0 ** -11 * np.abs(ref) + 1e-6


@pytest.mark.parametrize("fused", [True, False], ids=["fused", "copy"])
@pytest.mark.parametrize("gather", [False, True], ids=["direct", "src_idx"])
@pytest.mark.parametrize("pd,arg", HEADS, ids=[f"{p}{a}" for p, a in HEADS])
def test_head_kernels_vs_float64_autograd(pd, arg, gather, fused):
    from baselines_b200 import ops
    rng = np.random.RandomState(11)
    B = 300                                                   # not a multiple of the 256-thread block
    nvec = list(arg) if pd == "mcat" else None
    nout = sum(nvec) if pd == "mcat" else arg
    k = len(nvec) if pd == "mcat" else arg
    seg = ops.segment_table(nvec, "cuda") if pd == "mcat" else None
    hb = lr.head_bufs(nout, B, "fused" if fused else "copy")
    lo, ld, vo, ldv, g, ld_g, dv, ld_dv = hb.ho, hb.ld, hb.vo, hb.ldv, hb.g, hb.ld_g, hb.dv, hb.ld_dv
    l32 = (rng.randn(B, nout) * 1.5).astype(np.float32)
    v32 = rng.randn(B).astype(np.float32)
    lo[:, :nout] = _dev(l32)
    vo[:, 0] = _dev(v32)
    # ---- act: injected noise, then the Philox stream
    adt = torch.int64 if pd == "mcat" else torch.float32
    a = torch.zeros(B, k, dtype=adt, device="cuda")
    val, nlp = torch.zeros(B, device="cuda"), torch.zeros(B, device="cuda")
    u = (rng.rand(B, nout) * 0.998 + 0.001).astype(np.float32)
    step = (lambda **kw: ops.cat_step(lo, ld, nout, vo, ldv, a, val, nlp, B, seg_off=seg, **kw)) if pd == "mcat" else \
        (lambda **kw: ops.bern_step(lo, ld, nout, vo, ldv, a, val, nlp, B, **kw))
    step(uniforms=_dev(u))
    torch.cuda.synchronize()
    got_a = a.cpu().numpy()
    l64 = torch.tensor(l32, dtype=torch.float64)
    if pd == "mcat":
        want_a = ao.mcat_sample(l64, torch.tensor(u, dtype=torch.float64), nvec).numpy()
        sc = l32.astype(np.float64) - np.log(-np.log(u.astype(np.float64)))
        clear = np.ones(B, bool)
        for blk in np.split(sc, np.cumsum(nvec)[:-1], axis=1):
            if blk.shape[1] > 1:
                top2 = np.sort(blk, 1)[:, -2:]
                clear &= (top2[:, 1] - top2[:, 0]) > 1e-4
    else:
        want_a = ao.bern_sample(l64, torch.tensor(u, dtype=torch.float64)).numpy()
        clear = np.all(np.abs(u - 1 / (1 + np.exp(-l32.astype(np.float64)))) > 1e-4, axis=1)
    assert clear.mean() > 0.9 and np.array_equal(got_a[clear], want_a[clear])
    assert np.array_equal(val.cpu().numpy(), v32)
    for _ in range(2):
        nlp_ref = ao.neglogp(pd, l64, None, torch.as_tensor(got_a).double() if pd == "bern" else torch.as_tensor(got_a),
                             nvec).numpy()
        assert np.allclose(nlp.cpu().numpy(), nlp_ref, rtol=1e-5, atol=1e-5)
        step(seed=77, offset=3)                               # Philox: same checks on what it drew
        torch.cuda.synchronize()
        got_a = a.cpu().numpy()
        if pd == "mcat":
            assert np.all((got_a >= 0) & (got_a < np.array(nvec)))
        else:
            assert set(np.unique(got_a)) <= {0.0, 1.0}
    # ---- loss + gradient
    Bbuf = B + 37 if gather else B
    src = rng.permutation(Bbuf)[:B] if gather else np.arange(B)
    acts_buf = np.stack([rng.randint(0, n, Bbuf) for n in nvec], 1) if pd == "mcat" else \
        (rng.rand(Bbuf, k) < 0.5).astype(np.float32)
    acts = acts_buf[src]
    nlp_cur = lr.ppo_ref(pd, l32, v32, acts, np.zeros(B), np.zeros(B), np.zeros(B), np.zeros(B), 0.2, 0.0, 0.0,
                         nvec=nvec).nlp
    oldnlp_buf = rng.randn(Bbuf).astype(np.float32)
    oldnlp_buf[src] = (nlp_cur + rng.randn(B) * 0.1).astype(np.float32)
    oldv_buf = (rng.randn(Bbuf)).astype(np.float32)
    oldv_buf[src] = (v32 + rng.randn(B) * 0.3).astype(np.float32)
    R_buf = (oldv_buf + rng.randn(Bbuf)).astype(np.float32)
    clip, ent_coef, vf_coef = 0.2, 0.3, 0.5
    idx = _dev(src.astype(np.int64)) if gather else None
    adv_st = torch.zeros(2, dtype=torch.float64, device="cuda")
    stats = torch.zeros(5, dtype=torch.float64, device="cuda")
    ops.adv_stats(_dev(R_buf), _dev(oldv_buf), idx, B, adv_st)
    loss = ops.cat_loss if pd == "mcat" else ops.bern_loss
    kw = dict(seg_off=seg) if pd == "mcat" else {}
    loss(lo, ld, nout, vo, ldv, _dev(acts_buf if gather else acts, adt), idx, _dev(R_buf if gather else R_buf[src]),
         _dev(oldv_buf if gather else oldv_buf[src]), _dev(oldnlp_buf if gather else oldnlp_buf[src]), adv_st, clip,
         ent_coef, vf_coef, g, ld_g, dv, ld_dv, stats, B, **kw)
    torch.cuda.synchronize()
    mean, std = adv_st.cpu().numpy()
    R, oldv, oldnlp = R_buf[src], oldv_buf[src], oldnlp_buf[src]
    adv = (((R - oldv).astype(np.float64) - mean) / (std + 1e-8)).astype(np.float32)
    ref = lr.ppo_ref(pd, l32, v32, acts, R, oldv, oldnlp, adv, clip, ent_coef, vf_coef, nvec=nvec)
    gl, gv, st = ref.dhead, ref.dv, ref.stats
    got_g = g[:, :nout].float().cpu().numpy()
    ok = _within_fp16(got_g, gl)
    assert ok.all(), (np.argwhere(~ok)[:5], float(np.abs(got_g - gl).max()))
    assert _within_fp16(dv[:, 0].float().cpu().numpy(), gv).all()
    if fused:                                                 # padding columns of the last store group are zero
        pad_cols = g[:, nout + 1:_pad(nout, 8)].float()
        assert pad_cols.numel() == 0 or float(pad_cols.abs().max()) == 0.0
    got_st = stats.cpu().numpy()
    for i in range(4):
        assert abs(got_st[i] - st[i]) <= 1e-5 * max(1.0, abs(st[i])) * B ** 0.5, (i, got_st[i], st[i])
    assert abs(got_st[4] - st[4]) <= 1.0
    # the comparison is sharp enough to see the two plausible mistakes of a multi-categorical entropy gradient
    if pd == "mcat" and len(nvec) > 1:
        p = torch.cat([torch.softmax(b, 1) for b in torch.split(l64, nvec, 1)], 1).numpy()
        Hs = _seg_entropies(l64, nvec).numpy()
        H_col = np.repeat(Hs, nvec, axis=1)
        wrong_total = gl + ent_coef * p * (Hs.sum(1, keepdims=True) - H_col)    # total H in place of H_s
        assert not _within_fp16(got_g, wrong_total).all()
        wrong_drop = lr.ppo_ref(pd, l32, v32, acts, R, oldv, oldnlp, adv, clip, ent_coef, vf_coef, nvec=nvec,
                                mutant="drop_last_entropy").dhead
        assert not _within_fp16(got_g, wrong_drop).all()


def test_multidiscrete_observation_encoding_kernel():
    from baselines_b200 import ops
    rng = np.random.RandomState(1)
    nvec = [3, 1, 7, 2, 9]
    seg = ops.segment_table(nvec, "cuda")
    x = np.stack([rng.randint(0, n, 200) for n in nvec], 1).astype(np.float32)
    idx = rng.randint(0, 200, 77)
    out = torch.full((77, 2 * 24), 7.0, dtype=torch.float16, device="cuda")
    ops.obs_encode(_dev(x), out, 77, len(nvec), sum(nvec), 24, src_idx=_dev(idx.astype(np.int64)), onehot_n=sum(nvec),
                   seg_off=seg)
    torch.cuda.synchronize()
    want = ao.encode_multidiscrete(x[idx].astype(np.int64), nvec).numpy()
    assert np.array_equal(out[:, :22].float().cpu().numpy(), want)
    assert float(out[:, 22:].float().abs().max()) == 0.0                 # padding and the lo half are zero


# ================================================================================================ models
class _Env:
    pass


def _spaces(ob, ac):
    from baselines_b200.common import spaces
    mk = {"box": lambda a: spaces.Box(-5, 5, a, np.float32), "u8": lambda a: spaces.Box(0, 255, a, np.uint8),
          "md": spaces.MultiDiscrete, "mb": spaces.MultiBinary, "disc": spaces.Discrete}
    return mk[ob[0]](ob[1]), mk[ac[0]](ac[1])


def _mk(network, ob, ac, value_network=None, nenv=64, nsteps=4, seed=0, **kw):
    from baselines_b200.common.policies import build_policy
    from baselines_b200.ppo2.model import Model
    env = _Env()
    env.observation_space, env.action_space = _spaces(ob, ac)
    env.num_envs = nenv
    np.random.seed(seed)
    policy = build_policy(env, network, value_network=value_network, **kw)
    model = Model(policy=policy, ob_space=env.observation_space, ac_space=env.action_space, nbatch_act=nenv,
                  nbatch_train=nenv * nsteps, nsteps=nsteps, ent_coef=0.01, vf_coef=0.5, max_grad_norm=0.5,
                  comm=False)
    return env, model


def _oracle_params(network, ob, ac, value_network=None, seed=0, **kw):
    np.random.seed(seed)
    ob_shape = (int(np.sum(ob[1])),) if ob[0] == "md" else tuple(ob[1])
    if ac[0] == "md":
        return ao.init_policy_params(network, ob_shape, "mcat", ac[1], value_network=value_network, **kw)
    return ao.init_policy_params(network, ob_shape, "bern", ac[1], value_network=value_network, **kw)


def _obs(rng, ob, B):
    if ob[0] == "md":
        return np.stack([rng.randint(0, n, B) for n in ob[1]], 1).astype(np.int64)
    if ob[0] == "u8":
        return rng.randint(0, 256, size=(B,) + tuple(ob[1])).astype(np.uint8)
    return np.clip(rng.randn(B, *ob[1]) * 3.0, -10.0, 10.0).astype(np.float32)


def _oracle_obs(ob, obs):
    return ao.encode_multidiscrete(obs, ob[1]).numpy() if ob[0] == "md" else obs


def _pd(ac):
    return ("mcat", list(ac[1])) if ac[0] == "md" else ("bern", None)


def _nout(ac):
    return int(np.sum(ac[1])) if ac[0] == "md" else int(ac[1])


CASES = {
    "mlp_md_obs_md_act": dict(network="mlp", ob=("md", (3, 3)), ac=("md", (3, 3))),
    "mlp_box_md_copy": dict(network="mlp", ob=("box", (7,)), ac=("md", (4, 2, 5)), value_network="copy"),
    "cnn_u8_md": dict(network="cnn", ob=("u8", (84, 84, 4)), ac=("md", (3, 4, 2))),
    "mlp_box_mb": dict(network="mlp", ob=("box", (6,)), ac=("mb", 5)),
    "mlp_md_matching_fc": dict(network="mlp", ob=("box", (5,)), ac=("md", (8, 8)), num_hidden=16),
}


def _case_kw(case):
    return {k: v for k, v in case.items() if k not in ("network", "ob", "ac", "value_network")}


def _check_same_init(model, oparams):
    mp = model.get_params()
    assert set(mp.keys()) == set(oparams.keys())
    for k, v in oparams.items():
        assert mp[k].shape == v.shape and np.array_equal(mp[k], v), k


@pytest.mark.parametrize("name", list(CASES))
def test_step_matches_oracle(name):
    case = CASES[name]
    B = 256
    env, model = _mk(case["network"], case["ob"], case["ac"], case.get("value_network"), nenv=B, **_case_kw(case))
    op = _oracle_params(case["network"], case["ob"], case["ac"], case.get("value_network"), **_case_kw(case))
    _check_same_init(model, op)
    assert ("ppo2_model/pi/w:0" in op) == (name != "mlp_md_matching_fc")
    rng = np.random.RandomState(1)
    obs = _obs(rng, case["ob"], B)
    nout = _nout(case["ac"])
    noise = (rng.rand(B, nout) * 0.998 + 0.001).astype(np.float32)
    a, v, s, nlp = model.step(obs, noise=noise)
    pd, nvec = _pd(case["ac"])
    a_o, v_o, nlp_o, pi_o = ao.policy_step(op, case["network"], _oracle_obs(case["ob"], obs), noise,
                                           case.get("value_network"), pd, nvec)
    pi = model.net.pi_out[:B, :nout].cpu().numpy()
    assert np.allclose(pi, pi_o, atol=3e-3, rtol=1e-2), float(np.abs(pi - pi_o).max())
    assert np.allclose(v, v_o, atol=3e-3 * max(1.0, float(np.abs(v_o).max())))
    if pd == "mcat":
        assert a.dtype == np.int32 and a.shape == (B, len(nvec))
        sc = pi_o - np.log(-np.log(noise))
        clear = np.ones(B, bool)
        for blk in np.split(sc, np.cumsum(nvec)[:-1], axis=1):
            top2 = np.sort(blk, 1)[:, -2:]
            clear &= (top2[:, 1] - top2[:, 0]) > 1e-2
    else:
        assert a.dtype == np.float32 and a.shape == (B, nout)
        clear = np.all(np.abs(noise - 1 / (1 + np.exp(-pi_o))) > 1e-2, axis=1)
    assert clear.mean() > 0.6 and np.array_equal(a[clear], a_o[clear])
    assert np.allclose(nlp[clear], nlp_o[clear], atol=3e-3)


@pytest.mark.parametrize("name", list(CASES))
def test_train_step_matches_oracle(name):
    case = CASES[name]
    M = 512 if case["network"] == "cnn" else 2048
    env, model = _mk(case["network"], case["ob"], case["ac"], case.get("value_network"), nenv=M // 4,
                     **_case_kw(case))
    op = _oracle_params(case["network"], case["ob"], case["ac"], case.get("value_network"), **_case_kw(case))
    pd, nvec = _pd(case["ac"])
    oracle = ao.PPO2Oracle(op, case["network"], 0.01, 0.5, 0.5, value_network=case.get("value_network"), pd=pd,
                           nvec=nvec)
    rng = np.random.RandomState(2)
    nout = _nout(case["ac"])
    worst = 0.0
    for it in range(3):
        obs = _obs(rng, case["ob"], M)
        oobs = _oracle_obs(case["ob"], obs)
        if pd == "mcat":
            actions = np.stack([rng.randint(0, n, M) for n in nvec], 1).astype(np.int32)
        else:
            actions = (rng.rand(M, nout) < 0.5).astype(np.float32)
        values = rng.randn(M).astype(np.float32)
        returns = (values + rng.randn(M) * 0.7).astype(np.float32)
        t = nets.to_torch(oracle.params_np())
        with torch.no_grad():
            pi, _, _ = nets.policy_forward(t, case["network"], torch.as_tensor(oobs), case.get("value_network"))
            nlp_cur = ao.neglogp(pd, pi, None, torch.as_tensor(actions), nvec).numpy()
        neglogpacs = (nlp_cur + rng.randn(M) * 0.05).astype(np.float32)
        lr, clip = 2.5e-4, 0.1
        st = model.train(lr, clip, obs, returns, None, actions, values, neglogpacs)
        st_o = oracle.train(lr, clip, oobs, returns, None, actions, values, neglogpacs)
        assert np.allclose(st[:4], st_o[:4], atol=3e-3, rtol=2e-2), (it, st, st_o)
        assert abs(st[4] - st_o[4]) <= 0.02, (st[4], st_o[4])
        g = model.net.store.export_tf("grads")
        num = sum(float(((g[k] - oracle.last_grads[k]) ** 2).sum()) for k in g)
        den = sum(float((oracle.last_grads[k] ** 2).sum()) for k in g)
        assert (num / den) ** 0.5 < 2e-2, (it, (num / den) ** 0.5)
        p, po = model.get_params(), oracle.params_np()
        err = max(float(np.abs(p[k] - po[k]).max()) for k in p)
        worst = max(worst, err)
        # the reference's tolerance.  Adam moves each element by at most ~lr per step whatever the gradient, so this
        # bounds the step and cannot detect a gradient error (see test_update_composition_gpu.py)
        assert err < 3e-3, (it, err)
    print(f"[{name}] max |param - oracle| after 3 steps = {worst:.3e}")


def test_one_segment_multidiscrete_is_bit_identical_to_discrete():
    """MultiDiscrete([6]) runs the segment-table instantiation of the categorical kernels; with the same parameters and
    noise it must reproduce Discrete(6) bit for bit (actions differ only in shape)."""
    B = 300
    outs = []
    for ac in (("disc", 6), ("md", [6])):
        env, model = _mk("mlp", ("box", (9,)), ac, nenv=B, nsteps=1)
        rng = np.random.RandomState(4)
        obs = _obs(rng, ("box", (9,)), B)
        noise = (rng.rand(B, 6) * 0.998 + 0.001).astype(np.float32)
        a, v, _, nlp = model.step(obs, noise=noise)
        model.net.rng_ctr.zero_()
        a2, _, _, nlp2 = model.step(obs)                              # Philox stream
        actions = rng.randint(0, 6, B)
        values = rng.randn(B).astype(np.float32)
        returns = (values + rng.randn(B)).astype(np.float32)
        oldnlp = (nlp + rng.randn(B) * 0.05).astype(np.float32)
        st = model.train(3e-4, 0.2, obs, returns, None, actions if ac[0] == "disc" else actions[:, None], values,
                         oldnlp)
        grads = model.net.store.export_tf("grads")
        outs.append((a.reshape(B), v, nlp, a2.reshape(B), nlp2, st, grads, model.get_params()))
    (a, v, nlp, a2, nlp2, st, g, p), (b, w, mlp, b2, mlp2, st2, g2, p2) = outs
    assert np.array_equal(a, b) and np.array_equal(a2, b2)
    for x, y in ((v, w), (nlp, mlp), (nlp2, mlp2), (np.array(st), np.array(st2))):
        assert np.array_equal(x, y)
    for k in g:
        assert np.array_equal(g[k], g2[k]) and np.array_equal(p[k], p2[k]), k


def test_train_chunking_and_indexed_gather_equivalence():
    """Chunked accumulation == one launch, and permuted buffer + src_idx == the materialised minibatch, for [*, k]
    MultiDiscrete action rows."""
    case = CASES["mlp_box_md_copy"]
    M = 384
    rng = np.random.RandomState(3)
    obs = _obs(rng, case["ob"], M)
    actions = np.stack([rng.randint(0, n, M) for n in case["ac"][1]], 1)
    values = rng.randn(M).astype(np.float32)
    returns = (values + rng.randn(M)).astype(np.float32)
    nlp = (np.log(40) + rng.randn(M) * 0.05).astype(np.float32)
    outs = []
    for chunk in (M, 100):
        os.environ["B200RL_TRAIN_CHUNK"] = str(chunk)
        try:
            env, model = _mk(case["network"], case["ob"], case["ac"], "copy", nenv=M // 4)
        finally:
            del os.environ["B200RL_TRAIN_CHUNK"]
        assert model.chunk == chunk
        st = model.train(2.5e-4, 0.1, obs, returns, None, actions, values, nlp)
        outs.append((st, model.get_params()))
    for k in outs[0][1]:
        assert np.allclose(outs[0][1][k], outs[1][1][k], atol=2e-5), k
    assert np.allclose(outs[0][0], outs[1][0], atol=1e-5)
    env, model = _mk(case["network"], case["ob"], case["ac"], "copy", nenv=M // 4)
    perm = rng.permutation(M)
    inv = np.argsort(perm)
    f = lambda z, dt: _dev(z[inv], dt)
    st = model.train_rollout(2.5e-4, 0.1, f(obs, torch.float32), f(actions, torch.int64), f(returns, torch.float32),
                             f(values, torch.float32), f(nlp, torch.float32), _dev(perm))
    assert np.allclose(st.cpu().numpy(), outs[0][0], atol=1e-5)
    p = model.get_params()
    for k in p:
        assert np.allclose(p[k], outs[0][1][k], atol=2e-5), k


def test_device_distributions_satisfy_reference_identities():
    """distributions.py:321-348 on the CUDA heads with the Philox stream (the reference's parameter vectors): E[neglogp]
    = entropy within 3 sigma; per-segment / per-bit frequencies within 4 sigma of softmax / sigmoid."""
    from baselines_b200 import ops
    N = 100000
    v = torch.zeros(N, 16, device="cuda")
    val, nlp = torch.zeros(N, device="cuda"), torch.zeros(N, device="cuda")
    nvec = [1, 2, 3]
    pm = np.array([-.2, .3, .5, .1, 1, -.1], np.float32)
    logits = torch.nn.functional.pad(_dev(np.repeat(pm[None], N, 0)), (0, 10)).contiguous()
    a = torch.zeros(N, 3, dtype=torch.int64, device="cuda")
    ops.cat_step(logits, 16, 6, v, 16, a, val, nlp, N, seed=4321, offset=2, seg_off=ops.segment_table(nvec, "cuda"))
    torch.cuda.synchronize()
    ent = float(ao.mcat_entropy(torch.tensor(pm[None].astype(np.float64)), nvec)[0])
    ll = nlp.double().cpu().numpy()
    assert abs(ll.mean() - ent) < 3 * ll.std() / math.sqrt(N)
    an = a.cpu().numpy()
    for i, blk in enumerate(np.split(pm.astype(np.float64), np.cumsum(nvec)[:-1])):
        sm = np.exp(blk) / np.exp(blk).sum()
        freq = np.bincount(an[:, i], minlength=nvec[i]) / N
        assert len(freq) == nvec[i] and np.all(np.abs(freq - sm) < 4 * np.sqrt(sm * (1 - sm) / N) + 1e-12)
    pb = np.array([-.2, .3, .5], np.float32)
    logits = torch.nn.functional.pad(_dev(np.repeat(pb[None], N, 0)), (0, 13)).contiguous()
    x = torch.zeros(N, 3, device="cuda")
    ops.bern_step(logits, 16, 3, v, 16, x, val, nlp, N, seed=99, offset=5)
    torch.cuda.synchronize()
    ent = float(ao.bern_entropy(torch.tensor(pb[None].astype(np.float64)))[0])
    ll = nlp.double().cpu().numpy()
    assert abs(ll.mean() - ent) < 3 * ll.std() / math.sqrt(N)
    p = 1 / (1 + np.exp(-pb.astype(np.float64)))
    assert np.all(np.abs(x.cpu().numpy().mean(0) - p) < 4 * np.sqrt(p * (1 - p) / N))


# ================================================================================================ runner / checkpoints
class _ReplayEnv:
    def __init__(self, obs_seq, rew, done, ob_space, ac_space):
        self.obs_seq, self.rew, self.done = obs_seq, rew, done
        self.num_envs = rew.shape[1]
        self.observation_space, self.action_space = ob_space, ac_space
        self.t = 0
        self.seen = []

    def reset(self):
        self.t = 0
        return self.obs_seq[0]

    def step(self, actions):
        self.seen.append(np.array(actions))
        r, d = self.rew[self.t], self.done[self.t]
        self.t += 1
        return self.obs_seq[self.t], r, d, [{} for _ in range(self.num_envs)]


@pytest.mark.parametrize("ac", [("md", (3, 3)), ("mb", 4)], ids=["multidiscrete", "multibinary"])
def test_runner_rollout_arrays(ac):
    from baselines_b200.ppo2.runner import Runner
    T, N = 8, 16
    ob = ("md", (3, 3)) if ac[0] == "md" else ("box", (5,))
    env0, model = _mk("mlp", ob, ac, nenv=N, nsteps=T)
    rng = np.random.RandomState(5)
    obs_seq = np.stack([_obs(rng, ob, N) for _ in range(T + 1)])
    env = _ReplayEnv(obs_seq, rng.randn(T, N).astype(np.float32), rng.rand(T, N) < 0.1, env0.observation_space,
                     env0.action_space)
    runner = Runner(env=env, model=model, nsteps=T, gamma=0.99, lam=0.95)
    obs, returns, masks, actions, values, nlp, states, _ = runner.run()
    from oracle.gae import sf01
    assert obs.dtype == obs_seq.dtype and np.array_equal(obs, sf01(obs_seq[:T]))       # returned bit-exact
    if ac[0] == "md":
        assert actions.shape == (N * T, 2) and actions.dtype == np.int32
        assert np.all((actions >= 0) & (actions < 3))
        assert env.seen[0].dtype == np.int32 and env.seen[0].shape == (N, 2)
    else:
        assert actions.shape == (N * T, 4) and actions.dtype == np.float32
        assert set(np.unique(actions)) <= {0.0, 1.0}
    assert np.array_equal(actions, sf01(np.stack(env.seen)))        # what the env was given
    # a graph-replayed (persistent) acting pass draws exactly what the eager one draws
    x = model.net.encode_obs(_obs(rng, ob, N))
    bufs = {p: (torch.zeros(model.net.action_shape(N), dtype=model.net.action_dtype, device="cuda"),
                torch.zeros(N, device="cuda"), torch.zeros(N, device="cuda")) for p in (False, True)}
    res = []
    for persistent in (False, True, True, True):             # eager; then first call, capture + replay, replay
        a, vv, nn_ = bufs[persistent]
        model.net.rng_ctr.zero_()
        model.step_device(x, a, vv, nn_, persistent=persistent)
        torch.cuda.synchronize()
        res.append((a.cpu().numpy(), vv.cpu().numpy(), nn_.cpu().numpy()))
    assert any(k[0] == "act" for k in model.graphs.graphs)
    for r in res[1:]:
        for p, q in zip(res[0], r):
            assert np.array_equal(p, q)


@pytest.mark.parametrize("case", ["cnn_u8_md", "mlp_md_matching_fc", "mlp_box_mb"])
def test_save_load_roundtrip(tmp_path, case):
    import joblib
    c = CASES[case]
    env, model = _mk(c["network"], c["ob"], c["ac"], c.get("value_network"), nenv=8, **_case_kw(c))
    rng = np.random.RandomState(6)
    M = 32
    pd, nvec = _pd(c["ac"])
    nout = _nout(c["ac"])
    acts = np.stack([rng.randint(0, n, M) for n in nvec], 1) if pd == "mcat" else (rng.rand(M, nout) < .5).astype(np.float32)
    model.train(1e-3, 0.2, _obs(rng, c["ob"], M), rng.randn(M).astype(np.float32), None, acts,
                rng.randn(M).astype(np.float32), np.full(M, 2.0, np.float32))
    path = str(tmp_path / "ckpt")
    model.save(path)
    d = joblib.load(path)
    assert not any("logstd" in k for k in d)
    lat = 512 if c["network"] == "cnn" else c.get("num_hidden", 64)
    if lat == nout:
        assert not any(k.startswith("ppo2_model/pi/w") or k.startswith("ppo2_model/pi/b") for k in d)
    else:
        assert d["ppo2_model/pi/w:0"].shape == (lat, nout) and d["ppo2_model/pi/b:0"].shape == (nout,)
        assert "ppo2_model/pi/w/Adam:0" in d
    assert d["ppo2_model/vf/w:0"].shape == (lat, 1)
    env2, model2 = _mk(c["network"], c["ob"], c["ac"], c.get("value_network"), nenv=8, seed=123, **_case_kw(c))
    model2.load(path)
    p1, p2 = model.get_params(), model2.get_params()
    for k in p1:
        assert np.array_equal(p1[k], p2[k]), k
    obs = _obs(rng, c["ob"], 8)
    noise = rng.rand(8, nout).astype(np.float32) * 0.98 + 0.01
    r1, r2 = model.step(obs, noise=noise), model2.step(obs, noise=noise)
    assert np.array_equal(r1[0], r2[0]) and np.array_equal(r1[1], r2[1]) and np.array_equal(r1[3], r2[3])
    assert model2.opt.t == model.opt.t


# ================================================================================================ learning
def test_multidiscrete_identity_learns():
    """common/tests/test_identity.py:43-56 with util.py:14-39 simple_test: MultiDiscreteIdentityEnv((3, 3),
    episode_len=100), one DummyVecEnv env seeded 0, ppo2 lr=1e-3, nsteps=64, ent_coef=0, gamma=0.9, seed=0,
    30000 steps; then 10000 trials must collect more than 0.9 of the reward."""
    from baselines_b200.common.vec_env import DummyVecEnv
    from baselines_b200.envs import MultiDiscreteIdentityEnv
    from baselines_b200.ppo2 import ppo2

    def seeded_env_fn():
        env = MultiDiscreteIdentityEnv((3, 3), episode_len=100)
        env.seed(0)
        return env

    np.random.seed(0)
    env = DummyVecEnv([seeded_env_fn])
    model = ppo2.learn(network="mlp", env=env, total_timesteps=30000, seed=0, lr=1e-3, nsteps=64, ent_coef=0.0,
                       gamma=0.9, log_interval=1000, comm=False)
    n_trials, sum_rew, done = 10000, 0.0, True
    for _ in range(n_trials):
        if done:
            obs = env.reset()
        a, v, _, _ = model.step(obs)
        obs, rew, done, _ = env.step(a)
        sum_rew += float(rew[0])
        done = bool(done[0])
    print(f"MultiDiscreteIdentityEnv((3, 3)): reward fraction {sum_rew / n_trials:.4f} over {n_trials} trials")
    assert sum_rew > 0.9 * n_trials, sum_rew / n_trials


def test_learn_is_bit_reproducible_with_a_seed():
    from baselines_b200.common.vec_env import DummyVecEnv
    from baselines_b200.envs import MultiDiscreteIdentityEnv
    from baselines_b200.ppo2 import ppo2
    params = []
    for _ in range(2):
        env = DummyVecEnv([lambda i=i: MultiDiscreteIdentityEnv((3, 4), episode_len=50) for i in range(4)])
        for i, e in enumerate(env.envs):
            e.seed(i)
        model = ppo2.learn(network="mlp", env=env, total_timesteps=2048, seed=3, lr=1e-3, nsteps=128, ent_coef=0.01,
                           log_interval=1000, comm=False)
        params.append(model.get_params())
    for k in params[0]:
        assert np.array_equal(params[0][k], params[1][k]), k


def test_command_line_trains_and_saves(tmp_path):
    import joblib
    from baselines_b200 import logger, run
    save = str(tmp_path / "model")
    try:
        model = run.main(["--alg=ppo2", "--env=MultiDiscreteIdentity-v0", "--num_timesteps=1024", "--num_env=2",
                          "--seed=0", "--nsteps=128", "--nminibatches=4", "--noptepochs=2", "--log_interval=1",
                          f"--log_path={tmp_path / 'log'}", f"--save_path={save}"])
    finally:
        logger.configure(None)
    ck = joblib.load(save)
    assert ck["ppo2_model/pi/mlp_fc0/w:0"].shape == (6, 64)          # one-hot of MultiDiscrete((3, 3)) observations
    assert ck["ppo2_model/pi/w:0"].shape == (64, 6) and "ppo2_model/pi/logstd:0" not in ck
    a, v, s, nlp = model.step(np.zeros((2, 2), np.int64))
    assert a.shape == (2, 2) and a.dtype == np.int32 and s is None
