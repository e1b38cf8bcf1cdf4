"""Recurrent policies (lstm, cnn_lstm) without a GPU: the fixed-sequence env, the variables and their creation order,
and every configuration outside what the LSTM kernels cover."""
import numpy as np
import pytest

from baselines_b200 import nn
from baselines_b200.common import spaces
from baselines_b200.common.policies import build_policy
from baselines_b200.envs import FixedSequenceEnv


class _Env:
    def __init__(self, ob, ac):
        self.observation_space, self.action_space, self.num_envs = ob, ac, 1


def test_fixed_sequence_env():
    e = FixedSequenceEnv(n_actions=10, episode_len=5)
    assert e.observation_space.n == 1 and e.action_space.n == 10
    seq = list(e.sequence)
    r = np.random.RandomState(0)
    assert seq == [int(r.randint(0, 10)) for _ in range(5)]
    assert e.reset() == 0
    rews, dones = [], []
    for t in range(5):
        ob, r, d, info = e.step(seq[t])
        assert ob == 0 and info == {}
        rews.append(r), dones.append(d)
    assert rews == [1] * 5 and dones == [False] * 4 + [True]
    e.reset()
    assert e.step((seq[0] + 1) % 10)[1] == 0
    e.seed(3)
    assert e.sequence == seq                       # reseeding keeps the sequence


def _rng_draws(shapes):
    rng = np.random.RandomState(11)
    return [nn.ortho_init(s, sc, rng) for s, sc in shapes]


def test_lstm_variables_in_creation_order():
    rng = np.random.RandomState(11)
    store = nn.ParamStore(None)
    t = nn.Tower(store, "lstm", (7,), "pi", "ppo2_model/pi", rng, 4, nlstm=64)
    assert t.latent_dim == 64
    assert {k: v[2] for k, v in store.tf_map.items()} == {
        "ppo2_model/pi/lstm/wx:0": (7, 256), "ppo2_model/pi/lstm/b:0": (256,), "ppo2_model/pi/lstm/wh:0": (64, 256)}
    wx, wh = _rng_draws([((7, 256), 1.0), ((64, 256), 1.0)])
    specs = {n: init for n, _, init in store._specs}
    assert np.array_equal(specs["pi/lstm/wx/w"], wx) and np.array_equal(specs["pi/lstm/wh"], wh)
    assert not specs["pi/lstm/wx/b"].any()


def test_cnn_lstm_variables_in_creation_order():
    rng = np.random.RandomState(11)
    store = nn.ParamStore(None)
    nn.Tower(store, "cnn_lstm", (84, 84, 4), "pi", "ppo2_model/pi", rng, 4, nlstm=128)
    names = list(store.tf_map)
    assert names[:8] == [f"ppo2_model/pi/{l}/{v}:0" for l in ("c1", "c2", "c3", "fc1") for v in ("w", "b")]
    assert names[8:] == ["ppo2_model/pi/lstm/wx:0", "ppo2_model/pi/lstm/b:0", "ppo2_model/pi/lstm/wh:0"]
    draws = _rng_draws([((8, 8, 4, 32), np.sqrt(2)), ((4, 4, 32, 64), np.sqrt(2)), ((3, 3, 64, 64), np.sqrt(2)),
                        ((3136, 512), np.sqrt(2)), ((512, 512), 1.0), ((128, 512), 1.0)])
    specs = {n: init for n, _, init in store._specs}
    assert np.array_equal(specs["pi/lstm/wx/w"], draws[4]) and np.array_equal(specs["pi/lstm/wh"], draws[5])


@pytest.mark.parametrize("network,kw", [("lnlstm", {}), ("cnn_lnlstm", {}), ("lstm", {"layer_norm": True}),
                                        ("cnn_lstm", {"layer_norm": True}), ("impala_cnn", {}),
                                        ("impala_cnn_lstm", {})])
def test_out_of_scope_networks_raise(network, kw):
    with pytest.raises(NotImplementedError):
        build_policy(_Env(spaces.Box(-1, 1, (4,)), spaces.Discrete(2)), network, **kw)


@pytest.mark.parametrize("network", ["lstm", "cnn_lstm"])
def test_copy_value_network_with_recurrence_raises(network):
    with pytest.raises(NotImplementedError, match="recurrent"):
        build_policy(_Env(spaces.Box(-1, 1, (4,)), spaces.Discrete(2)), network, value_network="copy")


@pytest.mark.parametrize("nlstm", [32, 100, 256])
def test_unsupported_lstm_sizes_raise(nlstm):
    with pytest.raises(NotImplementedError, match="nlstm"):
        nn.Tower(nn.ParamStore(None), "lstm", (4,), "pi", "ppo2_model/pi", np.random.RandomState(0), 4, nlstm=nlstm)


def test_recurrent_deepq_raises():
    from baselines_b200.deepq.build_graph import QNet
    with pytest.raises(NotImplementedError, match="recurrent"):
        QNet((4,), 2, "lstm", 4, None, np.random.RandomState(0), "deepq/q_func")


def test_microbatched_model_refuses_states():
    from baselines_b200.ppo2.microbatched_model import MicrobatchedModel
    m = MicrobatchedModel.__new__(MicrobatchedModel)
    with pytest.raises(AssertionError, match="microbatches with recurrent models are not supported yet"):
        m.train(3e-4, 0.2, None, None, None, None, None, None, states=np.zeros((1, 256)))
