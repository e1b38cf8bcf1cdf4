"""CPU: DDPG's host side -- noise parsing and streams, the replay ring's bookkeeping and sampling stream against fixtures
the reference's own numpy modules produced, the float64 mirror against loops and central differences, the refusals,
and the command-line dispatch."""
import os
import types

import numpy as np
import pytest
import torch

import _ddpg_refs as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_noise_type_parsing():
    from baselines_b200.ddpg.noise import (AdaptiveParamNoiseSpec, NormalActionNoise, OrnsteinUhlenbeckActionNoise,
                                           parse_noise_type)
    a, p = parse_noise_type('adaptive-param_0.2', 3)
    assert a is None and isinstance(p, AdaptiveParamNoiseSpec)
    assert p.initial_stddev == 0.2 and p.desired_action_stddev == 0.2 and p.current_stddev == 0.2
    a, p = parse_noise_type(' ou_0.3 , adaptive-param_0.1', 2)
    assert isinstance(a, OrnsteinUhlenbeckActionNoise) and np.array_equal(a.sigma, [0.3, 0.3])
    assert p.desired_action_stddev == 0.1
    a, p = parse_noise_type('normal_0.5,none', 4)
    assert isinstance(a, NormalActionNoise) and p is None and a.mu.shape == (4,)
    assert parse_noise_type('none', 1) == (None, None) and parse_noise_type(None, 1) == (None, None)
    with pytest.raises(RuntimeError, match='unknown noise type'):
        parse_noise_type('adaptive-param_0.2,gaussian_0.1', 1)


def test_host_noise_streams_match_the_reference():
    from baselines_b200.ddpg.noise import AdaptiveParamNoiseSpec, NormalActionNoise, OrnsteinUhlenbeckActionNoise
    g = np.load(os.path.join(GOLDEN, "ddpg_noise.npz"))
    np.random.seed(1)
    ou = OrnsteinUhlenbeckActionNoise(mu=np.zeros(3), sigma=0.2 * np.ones(3))
    seq = [ou() for _ in range(20)]
    ou.reset()
    seq += [ou() for _ in range(30)]
    assert np.array_equal(np.array(seq), g["ou"])
    np.random.seed(2)
    nn_ = NormalActionNoise(mu=np.zeros(3), sigma=0.1 * np.ones(3))
    assert np.array_equal(np.array([nn_() for _ in range(50)]), g["normal"])
    spec = AdaptiveParamNoiseSpec(0.2, 0.2)
    trace = []
    for d in g["dists"]:
        spec.adapt(d)
        trace.append(spec.current_stddev)
    assert np.array_equal(np.array(trace), g["adapt"])


def _ring(limit):
    """A Memory's host bookkeeping without its device arrays."""
    from baselines_b200.ddpg.memory import Memory
    m = types.SimpleNamespace(limit=limit, start=0, length=0)
    m.advance = types.MethodType(Memory._advance, m)
    return m, Memory


def test_ring_bookkeeping_and_sampling_stream_match_the_reference():
    g = np.load(os.path.join(GOLDEN, "ddpg_memory.npz"))
    m, Memory = _ring(10)
    data = {k: np.zeros((10,) + g[k].shape[1:], np.float32) for k in ("obs0", "obs1", "actions", "rewards", "terminals1")}
    k = 0
    for n in (12, 27):
        while k < n:
            row = m.advance()
            for key in data:
                data[key][row] = g[key][k]
            k += 1
        assert m.start == int(g[f"n{n}_start"]) and m.length == int(g[f"n{n}_length"])
        np.random.seed(n)
        stub = types.SimpleNamespace(nb_entries=m.length)
        idx = Memory.sample_indices(stub, 16)
        sel = Memory.selection(m, idx)
        rows = (sel[0] + sel[1:]) % m.limit
        for key in data:
            assert np.array_equal(data[key][rows].reshape(g[f"n{n}_{key}"].shape), g[f"n{n}_{key}"]), (n, key)


def test_sampling_never_draws_the_last_two_entries():
    from baselines_b200.ddpg.memory import Memory
    np.random.seed(0)
    idx = Memory.sample_indices(types.SimpleNamespace(nb_entries=5), 10000)
    assert idx.max() == 2 and idx.min() == 0
    np.random.seed(0)
    assert not np.array_equal(idx, np.random.randint(5, size=10000))   # the tempting randint(nb_entries)


def test_networks_other_than_mlp_and_bad_arguments_are_refused():
    from baselines_b200.ddpg.models import Actor, Critic
    for net in ("cnn", "lstm", "conv_only", "cnn_lstm"):
        with pytest.raises(NotImplementedError):
            Actor(2, network=net)
        with pytest.raises(NotImplementedError):
            Critic(network=net)
    with pytest.raises(TypeError):
        Critic(network="mlp", nlstm=128)
    spec = Actor(3, num_layers=3, num_hidden=32, layer_norm=True)
    assert (spec.num_layers, spec.num_hidden, spec.layer_norm, spec.nb_actions) == (3, 32, True, 3)


def test_asymmetric_action_space_is_refused():
    from baselines_b200.common import spaces
    from baselines_b200.ddpg import ddpg

    class Env:
        observation_space = spaces.Box(-1.0, 1.0, (2,), np.float32)
        action_space = spaces.Box(np.array([-1.0, 0.0], np.float32), np.array([1.0, 1.0], np.float32),
                                  dtype=np.float32)
    with pytest.raises(AssertionError):
        ddpg.learn("mlp", Env(), total_timesteps=100)


def test_learn_function_dispatch():
    from baselines_b200.ddpg import ddpg
    from baselines_b200.run import get_learn_function, get_learn_function_defaults
    assert get_learn_function('ddpg') is ddpg.learn
    assert get_learn_function_defaults('ddpg', 'mujoco') == {}


# ------------------------------------------------------------------------------------------------ the float64 mirror
def _params(ob, nA, L=2, H=8, ln=False, seed=0):
    rng = np.random.RandomState(seed)
    P = {}
    for sc in ("actor", "critic", "target_actor", "target_critic"):
        nin = ob + (nA if "critic" in sc else 0)
        for i in range(L):
            P[f"{sc}/mlp_fc{i}/w:0"] = rng.randn(nin, H) * 0.5
            P[f"{sc}/mlp_fc{i}/b:0"] = rng.randn(H) * 0.1
            if ln:
                P[f"{sc}/{R.ln_scope(i)}/beta:0"] = rng.randn(H) * 0.1
                P[f"{sc}/{R.ln_scope(i)}/gamma:0"] = 1 + rng.randn(H) * 0.1
            nin = H
        head = "dense" if "actor" in sc else "output"
        P[f"{sc}/{head}/kernel:0"] = rng.randn(H, nA if "actor" in sc else 1) * 0.5
        P[f"{sc}/{head}/bias:0"] = rng.randn(nA if "actor" in sc else 1) * 0.1
    return P


def _batch(ob, nA, B, seed=1):
    rng = np.random.RandomState(seed)
    return dict(obs0=rng.randn(B, ob), obs1=rng.randn(B, ob), actions=rng.uniform(-1, 1, (B, nA)),
                rewards=rng.randn(B), terminals1=(rng.rand(B) < 0.3).astype(np.float64))


def test_mirror_forward_against_loops():
    P = _params(3, 2, ln=True)
    x = np.random.RandomState(2).randn(4, 3)
    T = {k: R._t(v) for k, v in P.items()}
    got = R.actor(R._t(x), T, "actor", 2, True).numpy()
    for b in range(4):
        h = list(x[b])
        for i in range(2):
            W, bb = P[f"actor/mlp_fc{i}/w:0"], P[f"actor/mlp_fc{i}/b:0"]
            z = [sum(h[k] * W[k, j] for k in range(len(h))) + bb[j] for j in range(W.shape[1])]
            m = sum(z) / len(z)
            v = sum((zz - m) ** 2 for zz in z) / len(z)
            ga, be = P[f"actor/{R.ln_scope(i)}/gamma:0"], P[f"actor/{R.ln_scope(i)}/beta:0"]
            h = [np.tanh((zz - m) / np.sqrt(v + R.LN_EPS) * ga[j] + be[j]) for j, zz in enumerate(z)]
        K, bk = P["actor/dense/kernel:0"], P["actor/dense/bias:0"]
        mu = [np.tanh(sum(h[k] * K[k, j] for k in range(len(h))) + bk[j]) for j in range(2)]
        np.testing.assert_allclose(got[b], mu, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("cfg", [
    dict(num_layers=2, layer_norm=False, gamma=0.99, normalize_returns=False, popart=False, critic_l2_reg=1e-2),
    dict(num_layers=2, layer_norm=True, gamma=0.9, normalize_returns=True, popart=True, critic_l2_reg=0.0),
])
def test_mirror_gradients_against_central_differences(cfg):
    ob, nA, B = 3, 2, 5
    P = _params(ob, nA, ln=cfg["layer_norm"])
    batch = _batch(ob, nA, B)
    om, os_ = np.array([0.1, -0.2, 0.3], np.float32), np.array([1.5, 0.7, 1.1], np.float32)
    rs = np.array([3.0, 40.0, 5.01]) if cfg["normalize_returns"] else None
    ref = R.train_step(P, batch, cfg, om, os_, rs)
    Pp = ref["P"]                                       # after Pop-Art: the parameters the losses are taken at

    def losses(Q):
        out = R.train_step(Q, batch, dict(cfg, popart=False), om, os_,
                           ref["ret_state"] if cfg["normalize_returns"] else None)
        return out["critic_loss"], out["actor_loss"]
    # the target is fixed by the step's y: perturbing critic / actor variables leaves the targets alone
    h = 1e-6
    for name, which in (("critic/mlp_fc0/w:0", 0), ("critic/output/bias:0", 0), ("actor/dense/kernel:0", 1),
                        ("actor/mlp_fc1/b:0", 1)):
        idx = (0,) * Pp[name].ndim
        Qp = {k: v.copy() for k, v in Pp.items()}
        Qm = {k: v.copy() for k, v in Pp.items()}
        Qp[name][idx] += h
        Qm[name][idx] -= h
        num = (losses(Qp)[which] - losses(Qm)[which]) / (2 * h)
        g = (ref["critic_grads"] if which == 0 else ref["actor_grads"])[name][idx]
        assert abs(num - g) <= 1e-6 * max(1.0, abs(g)), (name, num, g)


def test_mirror_running_stats_against_the_definition():
    rows = np.random.RandomState(3).randn(50, 4).astype(np.float32)
    st = R.obs_rms_rows(np.concatenate([np.zeros(4), np.full(4, 1e-2), [1e-2]]), rows)
    np.testing.assert_allclose(st[:4], rows.astype(np.float64).sum(0), rtol=1e-12)
    np.testing.assert_allclose(st[4:8], 1e-2 + (rows.astype(np.float64) ** 2).sum(0), rtol=1e-12)
    assert st[8] == 1e-2 + 50
    m, s = R.rms_mean_std(st, 4)
    np.testing.assert_allclose(m, rows.mean(0), rtol=1e-3, atol=1e-4)
    np.testing.assert_allclose(s, rows.std(0), rtol=1e-2)


def test_mirror_polyak_and_adam():
    t, s = np.float32([1.0, -2.0]), np.float32([3.0, 0.5])
    assert np.array_equal(R.polyak(t, s, 0.01), np.float32(0.99) * t + np.float32(0.01) * s)
    p, m, v = R.adam(np.array([1.0]), np.array([0.5]), np.zeros(1), np.zeros(1), 1, 1e-3)
    np.testing.assert_allclose(p, 1.0 - 1e-3 * np.sqrt(0.001) / 0.1 * 0.05 / (np.sqrt(0.001 * 0.25) + 1e-8))
    assert np.allclose(R.clip_by_norm(np.array([3.0, 4.0]), 1.0), [0.6, 0.8])
    assert np.array_equal(R.clip_by_norm(np.array([3.0, 4.0]), None), [3.0, 4.0])
