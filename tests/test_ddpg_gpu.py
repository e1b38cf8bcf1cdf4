"""GPU: the DDPG kernels (csrc/ddpg.cu) against exact numpy restatements, whole train steps against the float64 mirror
of tests/_ddpg_refs.py, graph replay against eager, seeded determinism, learning and the command line."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import _ddpg_refs as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", autouse=True)
def _lib():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from baselines_b200 import build_ext
    build_ext.build()


def _c(a, dt=None):
    t = torch.as_tensor(np.ascontiguousarray(a)).cuda()
    return t if dt is None else t.to(dt)


def _decode(x0, in_pad):
    """fp16 [hi | lo] operand rows -> the float32 values they encode (hi + lo is exact in float32)."""
    x = x0.float().cpu().numpy()
    return (x[:, :in_pad] + x[:, in_pad:2 * in_pad]).astype(np.float32)


# ---------------------------------------------------------------------------------------------------------- kernels
def test_encode_normalises_clips_wraps_and_appends_actions():
    from baselines_b200 import ops
    rng = np.random.RandomState(0)
    limit, D, nA, B = 1000, 5, 3, 64
    obs = rng.randn(limit, D).astype(np.float32) * 4
    acts = rng.uniform(-1, 1, (limit, nA)).astype(np.float32)
    mean = rng.randn(D).astype(np.float32)
    std = rng.uniform(0.05, 3, D).astype(np.float32)
    start = limit - 7                                   # rows (start + idx) % limit wrap past the end
    idx = np.concatenate([np.arange(10), rng.randint(0, limit - 2, B - 10)]).astype(np.int64)
    sel = np.concatenate([[start], idx]).astype(np.int64)
    in_pad = 8
    out = torch.zeros(B, 2 * in_pad, dtype=torch.float16, device="cuda")
    ops.ddpg_encode(_c(obs), out, B, D, in_pad, sel=_c(sel), limit=limit, mean=_c(mean), std=_c(std), clip=5.0,
                    act=_c(acts), act_sel=True, nA=nA)
    rows = (start + idx) % limit
    want = np.clip((obs[rows] - mean) / (std + np.float32(1e-8)), np.float32(-5), np.float32(5))
    got = _decode(out, in_pad)
    # hi + lo holds a float32 to 2^-22 relative, exactly where the value is an fp16 + fp16 pair
    np.testing.assert_allclose(got[:, :D], want, rtol=2.5e-7, atol=3e-8)
    assert np.any(np.abs(want) == 5.0)
    np.testing.assert_allclose(got[:, D:D + nA], acts[rows], rtol=2.5e-7, atol=3e-8)
    assert np.all(got[:, D + nA:] == 0)
    # both fp16 halves bit for bit: hi = fp16(v), lo = fp16(v - float32(hi)) of the reference's float32 expression
    bits = lambda a: np.ascontiguousarray(a).view(np.uint16)
    dev = out.cpu().numpy()
    got_hi, got_lo = bits(dev[:, :D]), bits(dev[:, in_pad:in_pad + D])

    def halves(v):
        hi = v.astype(np.float16)
        return bits(hi), bits((v - hi.astype(np.float32)).astype(np.float16))
    want_hi, want_lo = halves(want)
    assert np.array_equal(got_hi, want_hi) and np.array_equal(got_lo, want_lo)
    # the reference divides by (std + 1e-8); an encoder that multiplied by the float32 reciprocal would round some values
    # one ulp apart, which the lo halves show
    inv = np.clip((obs[rows] - mean) * (np.float32(1) / (std + np.float32(1e-8))), np.float32(-5), np.float32(5))
    inv_hi, inv_lo = halves(inv)
    assert not (np.array_equal(got_hi, inv_hi) and np.array_equal(got_lo, inv_lo))


def test_soft_update_is_the_float32_expression_bit_for_bit():
    """ops.soft_update in DDPG's (1 - tau, tau) and HER's (polyak, 1 - polyak) forms, over two networks in one launch."""
    from baselines_b200 import ops
    rng = np.random.RandomState(1)
    t0, s0 = rng.randn(1001).astype(np.float32), rng.randn(1001).astype(np.float32)
    t1, s1 = rng.randn(77).astype(np.float32), rng.randn(77).astype(np.float32)
    a, b = _c(t0), _c(t1)
    ops.soft_update(a, _c(s0), 1.0 - 0.01, 0.01, b, _c(s1))
    assert np.array_equal(a.cpu().numpy(), R.polyak(t0, s0, 0.01))
    assert np.array_equal(b.cpu().numpy(), R.polyak(t1, s1, 0.01))
    a, b = _c(t0), _c(t1)
    ops.soft_update(a, _c(s0), 0.95, 1.0 - 0.95, b, _c(s1))
    her = lambda t, s: (np.float32(0.95) * t + np.float32(1.0 - 0.95) * s).astype(np.float32)
    assert np.array_equal(a.cpu().numpy().view(np.uint32), her(t0, s0).view(np.uint32))
    assert np.array_equal(b.cpu().numpy().view(np.uint32), her(t1, s1).view(np.uint32))


def test_obs_rms_is_bit_for_bit_over_thousands_of_rows():
    from baselines_b200 import ops
    rng = np.random.RandomState(2)
    D, limit, n = 7, 3000, 2500
    x = (rng.randn(limit, D) * 3 + 1).astype(np.float32)
    st0 = np.concatenate([np.zeros(D), np.full(D, 1e-2), [1e-2]])
    st, mean, std = _c(st0), torch.zeros(D, device="cuda"), torch.zeros(D, device="cuda")
    pos0 = 1200                                           # rows 1200 .. 2999, then 0 .. 699: the ring wraps
    ops.ddpg_obs_rms(_c(x), pos0, limit, 1800, D, st, mean, std)
    ops.ddpg_obs_rms(_c(x), (pos0 + 1800) % limit, limit, n - 1800, D, st, mean, std)
    rows = x[(pos0 + np.arange(n)) % limit]
    want = R.obs_rms_rows(st0, rows)
    assert np.array_equal(st.cpu().numpy(), want)
    m, s = R.rms_mean_std(want, D)
    assert np.array_equal(mean.cpu().numpy(), m) and np.array_equal(std.cpu().numpy(), s)


@pytest.mark.parametrize("B", [1, 7, 64, 129, 1000])
def test_ret_rms_pairwise_and_popart(B):
    from baselines_b200 import ops
    rng = np.random.RandomState(B)
    y = (rng.randn(B) * 5 + 2).astype(np.float32)
    st0 = np.array([3.0, 40.0, 5.01])
    m0, s0 = R.rms_mean_std(st0, 1)
    K = 64
    w0, w1 = rng.randn(K).astype(np.float32), rng.randn(K).astype(np.float32)
    b0, b1 = rng.randn(1).astype(np.float32), rng.randn(1).astype(np.float32)
    st, mean, std = _c(st0), _c(m0), _c(s0)
    W0, W1, B0, B1 = _c(w0), _c(w1), _c(b0), _c(b1)
    ops.ddpg_ret_rms(_c(y), B, st, mean, std, popart=(W0, B0, W1, B1))
    want = R.ret_rms_batch(st0, y)
    assert np.array_equal(st.cpu().numpy(), want)
    nm, ns = R.rms_mean_std(want, 1)
    assert np.array_equal(mean.cpu().numpy(), nm) and np.array_equal(std.cpu().numpy(), ns)
    f = np.float32
    for W, w in ((W0, w0), (W1, w1)):
        assert np.array_equal(W.cpu().numpy(), (w * s0[0] / ns[0]).astype(f))
    for Bb, b in ((B0, b0), (B1, b1)):
        assert np.array_equal(Bb.cpu().numpy(), ((b * s0[0] + m0[0] - nm[0]) / ns[0]).astype(f))


@pytest.mark.parametrize("norm", [False, True])
def test_target_and_loss_heads(norm):
    from baselines_b200 import ops
    rng = np.random.RandomState(3)
    B, limit = 300, 500
    q1 = rng.randn(B, 8).astype(np.float32)
    rew = rng.randn(limit).astype(np.float32)
    term = (rng.rand(limit) < 0.3).astype(np.float32)
    sel = np.concatenate([[450], rng.randint(0, limit - 2, B)]).astype(np.int64)
    rows = (450 + sel[1:]) % limit
    mean, std = (np.float32(0.7), np.float32(2.5)) if norm else (None, None)
    md = (_c(np.array([mean])), _c(np.array([std]))) if norm else (None, None)
    y = torch.zeros(B, device="cuda")
    ops.ddpg_target(_c(q1), 8, _c(sel), limit, _c(rew), _c(term), md[0], md[1], 0.99, y, B)
    f = np.float32
    qd = q1[:, 0] * std + mean if norm else q1[:, 0]
    want = rew[rows] + (f(1) - term[rows]) * f(0.99) * qd
    assert np.array_equal(y.cpu().numpy(), want.astype(f))
    assert np.any(term[rows] == 1) and np.any(term[rows] == 0)
    q = rng.randn(2 * B, 8).astype(np.float32)
    dq = torch.zeros(2 * B, 8, dtype=torch.float16, device="cuda")
    losses = torch.zeros(2, device="cuda")
    ops.ddpg_loss(_c(q), 8, y, md[0], md[1], B, dq, 8, losses)
    yv = want.astype(np.float64)
    yn = (yv - mean) / (float(std) + 1e-8) if norm else yv
    cl = np.mean((q[:B, 0] - yn) ** 2)
    qa = q[B:, 0] * (std if norm else 1.0) + (mean if norm else 0.0)
    l = losses.cpu().numpy()
    assert abs(l[0] - cl) <= 1e-5 * abs(cl) and abs(l[1] + np.mean(qa)) <= 1e-5 * (abs(np.mean(qa)) + 1)
    d = dq.float().cpu().numpy()[:, 0]
    np.testing.assert_allclose(d[:B], 2 * (q[:B, 0] - yn), rtol=1e-3, atol=1e-6)
    assert np.all(d[B:] == np.float16(-(float(std) if norm else 1.0)))


def test_l2_touches_only_its_segments():
    from baselines_b200 import ops
    rng = np.random.RandomState(4)
    w = rng.randn(100).astype(np.float32)
    g = rng.randn(100).astype(np.float32)
    segs = np.array([[0, 10], [40, 25]], np.int64)
    G, loss = _c(g), _c(np.array([1.5], np.float32))
    ops.ddpg_l2(_c(w), G, _c(segs), 0.01, loss)
    want = g.copy()
    for o, n in segs:
        want[o:o + n] = g[o:o + n] + np.float32(0.01) * w[o:o + n]
    assert np.array_equal(G.cpu().numpy(), want)
    reg = sum(0.01 * (w[o:o + n].astype(np.float64) ** 2).sum() / 2 for o, n in segs)
    assert abs(loss.item() - (1.5 + reg)) < 1e-5


def test_param_noise_distance_and_adaptation():
    from baselines_b200 import ops
    rng = np.random.RandomState(5)
    mu, ma = rng.randn(64, 3).astype(np.float32), rng.randn(64, 3).astype(np.float32) * 0.1
    sd, sd32, dist = _c(np.array([0.2])), torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
    ops.ddpg_pn_adapt(_c(mu), _c(mu + ma), mu.size, 0.2, sd, sd32, dist)
    want = np.sqrt(np.mean((ma.astype(np.float64)) ** 2))
    assert abs(dist.item() - want) < 1e-5
    spec = __import__("baselines_b200.ddpg.noise", fromlist=["x"]).AdaptiveParamNoiseSpec(0.2, 0.2)
    spec.adapt(float(dist.item()))
    assert sd.item() == spec.current_stddev and sd32.item() == np.float32(spec.current_stddev)


# ---------------------------------------------------------------------------------------------- whole train steps
def _make(cfg, B, seed=0, limit=5000, n_rows=1500, ob=6, nA=2):
    from baselines_b200.ddpg.ddpg_learner import DDPG
    from baselines_b200.ddpg.memory import Memory
    from baselines_b200.ddpg.models import Actor, Critic
    from baselines_b200.ddpg.noise import AdaptiveParamNoiseSpec
    np.random.seed(seed)
    kw = dict(num_layers=cfg["num_layers"], num_hidden=cfg.get("num_hidden", 64), layer_norm=cfg["layer_norm"])
    mem = Memory(limit, (nA,), (ob,))
    agent = DDPG(Actor(nA, **kw), Critic(**kw), mem, (ob,), (nA,), gamma=cfg["gamma"], tau=0.01,
                 normalize_returns=cfg["normalize_returns"], enable_popart=cfg["popart"],
                 normalize_observations=cfg["normalize_observations"], batch_size=B,
                 critic_l2_reg=cfg["critic_l2_reg"], clip_norm=cfg["clip_norm"], seed=seed,
                 param_noise=AdaptiveParamNoiseSpec(0.2, 0.2) if cfg.get("param_noise") else None)
    agent.initialize()
    rng = np.random.RandomState(seed + 1)
    for _ in range(n_rows // 10):
        o0 = (rng.randn(10, ob) * 2 + 0.5).astype(np.float32)
        agent.store_transition(o0, rng.uniform(-1, 1, (10, nA)).astype(np.float32), rng.randn(10),
                               (o0 + 0.1 * rng.randn(10, ob)).astype(np.float32), (rng.rand(10) < 0.2).astype(np.float32))
    return agent


BASE = dict(num_layers=2, layer_norm=False, gamma=0.99, normalize_returns=False, popart=False,
            normalize_observations=True, critic_l2_reg=1e-2, clip_norm=None)
CASES = {
    "plain": dict(),
    "layer_norm": dict(layer_norm=True),
    "no_obs_norm": dict(normalize_observations=False, critic_l2_reg=0.0),
    "popart": dict(normalize_returns=True, popart=True, layer_norm=True),
    "clip_some": dict(clip_norm=0.05),
    "clip_all": dict(clip_norm=1e-6, layer_norm=True),
    "clip_none": dict(clip_norm=1e6),
}


def _bound(dev, ref, scale):
    """max |dev - ref| over one variable, against a scale."""
    return float(np.max(np.abs(np.asarray(dev, np.float64) - ref))) / (scale + 1e-12)


def _layer_scales(rg):
    """Per variable, the largest reference entry of its layer (kernel and bias, or beta and gamma): a bias gradient is a
    sum over the batch that can cancel far below its layer's scale, which leaves the fp16 operand rounding exposed."""
    layer = lambda k: k.rsplit("/", 1)[0]
    top = {}
    for k, r in rg.items():
        top[layer(k)] = max(top.get(layer(k), 0.0), float(np.max(np.abs(r))))
    return {k: top[layer(k)] for k in rg}


def _state(agent):
    P = {}
    for net in (agent.actor, agent.critic, agent.target_actor, agent.target_critic):
        P.update(net.tf_variables())
    om = os_ = None
    if agent.obs_rms is not None:
        om, os_ = agent.obs_rms.mean.cpu().numpy(), agent.obs_rms.std.cpu().numpy()
    rs = agent.ret_rms.state.cpu().numpy() if agent.ret_rms is not None else None
    return P, om, os_, rs


def _batch(agent, idxs):
    m = agent.memory
    rows = (m.start + np.asarray(idxs)) % m.limit
    g = lambda t: t.cpu().numpy()[rows]
    return dict(obs0=g(m.obs0), obs1=g(m.obs1), actions=g(m.actions), rewards=g(m.rewards), terminals1=g(m.terminals1))


TOL = {1: 2e-2, 64: 1e-2, 1000: 1e-2}


@pytest.mark.parametrize("B", [1, 64, 1000])
@pytest.mark.parametrize("case", sorted(CASES))
def test_train_step_against_float64(case, B):
    cfg = dict(BASE, **CASES[case])
    agent = _make(cfg, B)
    # initialize() copies the online networks into the targets, bit for bit
    for t, s in ((agent.target_actor, agent.actor), (agent.target_critic, agent.critic)):
        assert torch.equal(t.store.params.view(torch.int32), s.store.params.view(torch.int32))
    for _ in range(2):
        agent.train_device()
        agent.update_target_net()
    # a target critic that answers about 3: the freshly initialised one answers about 0, and the (1 - d) of the
    # target would only move y by that much
    agent.target_critic.head.b.fill_(3.0)
    agent.target_critic.refresh()
    P, om, os_, rs = _state(agent)
    m_prev = {n: (net.store.export_tf("m"), net.store.export_tf("v")) for n, net in
              (("actor", agent.actor), ("critic", agent.critic))}
    idxs = agent.memory.sample_indices(B)
    batch = _batch(agent, idxs)
    ref = R.train_step(P, batch, cfg, om, os_, rs)
    losses = agent.train_device(idxs).cpu().numpy()
    tol = TOL[B]
    grads = {}
    for net, rg in ((agent.critic, ref["critic_grads"]), (agent.actor, ref["actor_grads"])):
        dg = net.store.export_tf("grads")
        sc = _layer_scales(rg)
        for k, r in rg.items():
            grads[k] = dg[k]
            assert _bound(dg[k], r, sc[k]) < tol, (case, B, k, _bound(dg[k], r, sc[k]))
    assert abs(losses[0] - ref["critic_loss"]) <= tol * (abs(ref["critic_loss"]) + 1e-3)
    assert abs(losses[1] - ref["actor_loss"]) <= tol * (abs(ref["actor_loss"]) + 1e-3)
    # Adam on each network from the device's own gradients (clipped per variable): m and v
    for name, net, t in (("actor", agent.actor, agent.actor_opt.t), ("critic", agent.critic, agent.critic_opt.t)):
        mm, vv = net.store.export_tf("m"), net.store.export_tf("v")
        for k in mm:
            g = R.clip_by_norm(grads[k].astype(np.float64), cfg["clip_norm"])
            m0, v0 = m_prev[name][0][k], m_prev[name][1][k]
            np.testing.assert_allclose(mm[k], 0.9 * m0 + 0.1 * g, rtol=1e-5, atol=1e-9 + 1e-6 * np.abs(g).max())
            np.testing.assert_allclose(vv[k], 0.999 * v0 + 0.001 * g * g, rtol=1e-4, atol=1e-12 + 1e-6 * (g * g).max())
    # Pop-Art reached both critics' output layers
    if cfg["popart"]:
        dv = agent.target_critic.tf_variables()
        for k in ("target_critic/output/kernel:0", "target_critic/output/bias:0"):
            np.testing.assert_allclose(dv[k], ref["P"][k], rtol=1e-5, atol=1e-7)
        bad = R.train_step(P, batch, cfg, om, os_, rs, skip_target_popart=True)
        assert not np.allclose(dv["target_critic/output/bias:0"], bad["P"]["target_critic/output/bias:0"],
                               rtol=1e-5, atol=1e-7)
    # the soft target update, bit for bit
    before = {**agent.target_actor.tf_variables(), **agent.target_critic.tf_variables()}
    agent.update_target_net()
    after = {**agent.target_actor.tf_variables(), **agent.target_critic.tf_variables()}
    online = {**agent.actor.tf_variables(), **agent.critic.tf_variables()}
    for k in before:
        src = online[k.replace("target_", "", 1)]
        assert np.array_equal(after[k], R.polyak(before[k], src, 0.01)), k
    # L2 reaches exactly the critic's hidden kernels: no bias, no LayerNorm variable, no output layer (the biases and the
    # output kernel are too small after three steps for a gradient bound to see reg * w on them)
    c = agent.critic
    want = sorted((c.store.offsets[c.tf_internal(k)], int(np.prod(c.store.tf_map[k][2]))) for k in c.tf_names
                  if k.endswith("/w:0") and "output" not in k)
    assert sorted(map(tuple, agent.l2_segs.cpu().numpy().tolist())) == want
    assert {k.split("/")[1] for k in c.tf_names if k.endswith("/w:0") and "output" not in k} == \
        {f"mlp_fc{i}" for i in range(cfg["num_layers"])}
    # every bound rejects the mistakes that this configuration can show
    if B >= 64 and case == "plain":
        mistakes = dict(actor_leak=("critic", True), actor_at_target=("actor", True), no_done_mask=("critic", True))
        for flag, (which, _) in mistakes.items():
            bad = R.train_step(P, batch, cfg, om, os_, rs, **{flag: True})
            rg = bad["critic_grads"] if which == "critic" else bad["actor_grads"]
            sc = _layer_scales(rg)
            worst = max(_bound(grads[k], rg[k], sc[k]) for k in rg)
            assert worst >= tol, (flag, worst)


# ------------------------------------------------------------------------------------------ replay and determinism
def test_graph_replay_equals_eager():
    cfg = dict(BASE, layer_norm=True, normalize_returns=True, popart=True, clip_norm=0.5, param_noise=True)
    outs = []
    for no_graphs in ("1", "0"):
        os.environ["B200RL_NO_GRAPHS"] = no_graphs
        try:
            agent = _make(cfg, 64)
            agent.reset()
            for _ in range(4):
                agent.adapt_param_noise_device()
                agent.train_device()
                agent.update_target_net()
            a, q, _, _ = agent.step(np.random.RandomState(9).randn(16, 6).astype(np.float32))
            outs.append((agent.get_variables(), a, q, float(agent.pn_stddev.item())))
        finally:
            os.environ.pop("B200RL_NO_GRAPHS", None)
    (v0, a0, q0, s0), (v1, a1, q1, s1) = outs
    assert v0.keys() == v1.keys()
    for k in v0:
        assert np.array_equal(v0[k], v1[k]), k
    assert np.array_equal(a0, a1) and np.array_equal(q0, q1) and s0 == s1


def test_acting_pass_perturbed_compute_q_and_clip():
    cfg = dict(BASE, layer_norm=True, param_noise=True)
    agent = _make(cfg, 64)
    agent.reset()
    obs = np.random.RandomState(3).randn(16, 6).astype(np.float32)
    a_clean, q_clean, _, _ = agent.step(obs, apply_noise=False, compute_Q=True)
    a_pert, q_pert, _, _ = agent.step(obs, apply_noise=True, compute_Q=True)
    a_noq, q_none, _, _ = agent.step(obs, apply_noise=False, compute_Q=False)
    assert q_none is None and np.array_equal(a_noq, a_clean)
    assert a_clean.shape == (16, 2) and q_clean.shape == (16, 1)
    assert np.array_equal(q_clean, q_pert)                     # Q is the unperturbed actor's (ddpg_learner.py:266)
    assert not np.array_equal(a_clean, a_pert)
    P, om, os_, _ = _state(agent)
    x = np.clip((obs - om) / (os_ + np.float32(1e-8)), -5, 5)
    mu = R.actor(R._t(x), {k: R._t(v) for k, v in P.items()}, "actor", 2, True).numpy()
    np.testing.assert_allclose(a_clean, mu, atol=2e-3)
    qr = R.critic(R._t(x), R._t(a_clean), {k: R._t(v) for k, v in P.items()}, "critic", 2, True).numpy()
    np.testing.assert_allclose(q_clean, qr, atol=2e-3 * (np.abs(qr).max() + 1e-3))
    from baselines_b200.ddpg.noise import NormalActionNoise
    agent.action_noise = NormalActionNoise(np.zeros(2), 50 * np.ones(2))
    a_big, _, _, _ = agent.step(obs, apply_noise=True)
    assert np.all(np.abs(a_big) <= 1.0) and np.any(np.abs(a_big) == 1.0)


def _learn(seed, **kw):
    from baselines_b200.common.vec_env import DummyVecEnv
    from baselines_b200.ddpg import ddpg
    from baselines_b200.envs import BoxIdentityEnv
    env = DummyVecEnv([lambda: BoxIdentityEnv((1,), 100)])
    env.seed(seed) if hasattr(env, "seed") else None
    return ddpg.learn("mlp", env, seed=seed, memory_limit=100000, **kw), env


def test_two_seeded_learn_runs_are_bit_identical():
    vs = []
    for _ in range(2):
        agent, _ = _learn(0, total_timesteps=2000, nb_epoch_cycles=5, nb_rollout_steps=100, nb_train_steps=10,
                          layer_norm=True)
        vs.append(agent.get_variables())
    for k in vs[0]:
        assert np.array_equal(vs[0][k], vs[1][k]), k


def test_continuous_identity_learns():
    """common/tests/test_identity.py test_continuous_identity['ddpg'] as its simple_test runs it: 30 000 steps, gamma 0.9,
    layer norm, seed 0, then 10 000 trials of the agent's default step (parameter noise applied), mean reward > -0.1."""
    from baselines_b200.common.vec_env import DummyVecEnv
    from baselines_b200.ddpg import ddpg
    from baselines_b200.envs import BoxIdentityEnv

    def env_fn():
        e = BoxIdentityEnv((1,), episode_len=100)
        e.seed(0)
        return e
    np.random.seed(0)
    env = DummyVecEnv([env_fn])
    agent = ddpg.learn(env=env, network="mlp", total_timesteps=30000, gamma=0.9, seed=0, layer_norm=True)
    total, done = 0.0, True
    for _ in range(10000):
        if done:
            obs = env.reset()
        a, _, _, _ = agent.step(obs)
        obs, rew, done, _ = env.step(a)
        total += float(rew[0])
    assert total > -0.1 * 10000, total


@pytest.mark.parametrize("flags", [
    ["--alg=ddpg", "--env=BoxIdentity-v0", "--num_timesteps=2000"],
    ["--alg=ddpg", "--env=BoxIdentity-v0", "--num_timesteps=2000", "--noise_type=normal_0.1"],
    ["--alg=ddpg", "--env=BoxIdentity-v0", "--num_timesteps=2000", "--noise_type=ou_0.1"],
    ["--alg=ddpg", "--env=BoxIdentity-v0", "--num_timesteps=2000", "--noise_type=adaptive-param_0.2,normal_0.1",
     "--normalize_returns=True", "--popart=True"],
])
def test_cli_smoke_flag_sets(flags, tmp_path):
    """ddpg/test_smoke.py's four flag sets, one epoch each through the command line."""
    env = dict(os.environ, PYTHONPATH=ROOT)
    p = subprocess.run([sys.executable, "-m", "baselines_b200.run"] + flags + ["--memory_limit=10000",
                        f"--log_path={tmp_path}"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    out = p.stdout
    for key in ("rollout/return", "train/loss_actor", "train/loss_critic", "train/param_noise_distance",
                "total/steps", "reference_Q_mean", "obs_rms_mean"):
        assert key in out, key


# ------------------------------------------------------------------------------- variables, creation order, noise sets
def _expected_variables(ob, nA, L, H, ln, pn, nobs, nret):
    """(TF name, shape) of every variable in the reference's creation order (ddpg_learner.py:102-169, models.py,
    common/models.py mlp, mpi_running_mean_std.py)."""
    out = []
    for scope, on, shape in (("obs_rms", nobs, (ob,)), ("ret_rms", nret, ())):
        if on:
            out += [(f"{scope}/runningsum:0", shape), (f"{scope}/runningsumsq:0", shape), (f"{scope}/count:0", ())]
    scopes = ["actor", "critic", "target_actor", "target_critic"] + (
        ["param_noise_actor", "adaptive_param_noise_actor"] if pn else [])
    for sc in scopes:
        critic = sc.endswith("critic")
        nin = ob + (nA if critic else 0)
        for i in range(L):
            out += [(f"{sc}/mlp_fc{i}/w:0", (nin, H)), (f"{sc}/mlp_fc{i}/b:0", (H,))]
            if ln:
                lsc = "LayerNorm" if i == 0 else f"LayerNorm_{i}"
                out += [(f"{sc}/{lsc}/beta:0", (H,)), (f"{sc}/{lsc}/gamma:0", (H,))]
            nin = H
        head = "output" if critic else "dense"
        nout = 1 if critic else nA
        out += [(f"{sc}/{head}/kernel:0", (H, nout)), (f"{sc}/{head}/bias:0", (nout,))]
    return scopes, out


@pytest.mark.parametrize("ln,pn,nobs,nret", [(True, True, True, True), (False, False, False, False),
                                             (True, False, True, False)])
def test_variable_names_shapes_order_and_numpy_draws(ln, pn, nobs, nret):
    """Every variable under the reference's TF name and shape, in its creation order; each copy takes its orthogonal
    initialisers from numpy's global stream in that order, so the stream after building the agent is the reference's
    (noise and memory sampling draw from it next)."""
    from baselines_b200 import nn
    from baselines_b200.ddpg.ddpg_learner import DDPG
    from baselines_b200.ddpg.memory import Memory
    from baselines_b200.ddpg.models import Actor, Critic
    from baselines_b200.ddpg.noise import AdaptiveParamNoiseSpec
    ob, nA, L, H = 5, 3, 3, 16
    np.random.seed(7)
    kw = dict(num_layers=L, num_hidden=H, layer_norm=ln)
    agent = DDPG(Actor(nA, **kw), Critic(**kw), Memory(100, (nA,), (ob,)), (ob,), (nA,), batch_size=8,
                 normalize_observations=nobs, normalize_returns=nret, seed=3,
                 param_noise=AdaptiveParamNoiseSpec(0.2, 0.2) if pn else None)
    got = agent.get_variables()
    scopes, want = _expected_variables(ob, nA, L, H, ln, pn, nobs, nret)
    assert [(k, tuple(np.shape(v))) for k, v in got.items()] == want
    rs = np.random.RandomState(7)
    for sc in scopes:
        nin = ob + (nA if sc.endswith("critic") else 0)
        for i in range(L):
            w = nn.ortho_init((nin, H), np.sqrt(2), rs)
            assert np.array_equal(got[f"{sc}/mlp_fc{i}/w:0"], w), (sc, i)
            nin = H
        assert np.all(np.abs(got[f"{sc}/{'output' if sc.endswith('critic') else 'dense'}/kernel:0"]) <= 3e-3)
    s_got, s_want = np.random.get_state(), rs.get_state()
    assert np.array_equal(s_got[1], s_want[1]) and s_got[2:] == s_want[2:]
    # the L2 term's variables: the critic's hidden kernels
    c = agent.critic
    reg = sorted(map(tuple, agent.l2_segs.cpu().numpy().tolist()))
    assert reg == sorted((c.store.offsets[c.tf_internal(f"critic/mlp_fc{i}/w:0")], (ob + nA if i == 0 else H) * H)
                         for i in range(L))


def test_perturbed_copies_keep_layer_norm_variables():
    """After reset (param_noise_actor) and adapt_param_noise (adaptive_param_noise_actor), each copy's LayerNorm
    variables are the actor's exactly and every other variable differs in every element (models.py:18-20)."""
    cfg = dict(BASE, layer_norm=True, param_noise=True)
    agent = _make(cfg, 64)
    agent.reset()
    agent.adapt_param_noise_device()
    actor = agent.actor.tf_variables()
    for net in (agent.param_noise_actor, agent.adaptive_param_noise_actor):
        for k, v in net.tf_variables().items():
            a = actor[k.replace(net.scope, "actor", 1)]
            if "LayerNorm" in k:
                assert np.array_equal(v, a), k
            else:
                assert np.all(v != a), k
