"""Layer normalisation without a GPU: the float64 references against the definition and central differences, and the
variables `layer_norm=True` creates (names, shapes, order, and an untouched ortho_init / xavier draw sequence)."""
import numpy as np
import pytest
import torch

import _layer_norm_refs as L
from baselines_b200 import nn
from oracle import nets


def _case(rows, N, seed=0):
    rng = np.random.RandomState(seed)
    z = rng.randn(rows, N) * rng.uniform(0.1, 3.0, (rows, 1)) + rng.uniform(-2, 2, (rows, 1))
    return z, rng.uniform(0.5, 1.5, N), rng.randn(N) * 0.3, rng.randn(rows, N)


def test_forward_is_the_definition():
    z, gamma, beta, _ = _case(5, 24)
    _, u, xhat, _ = L.ln_forward(z, gamma, beta, eps=1e-12)
    assert np.allclose(u, L.ln_forward_loops(z, gamma, beta, 1e-12), rtol=1e-12, atol=1e-12)
    assert np.allclose(xhat.mean(1), 0, atol=1e-12) and np.allclose((xhat ** 2).mean(1), 1, atol=1e-9)   # biased variance
    for act, f in ((1, lambda v: np.maximum(v, 0)), (2, np.tanh)):
        assert np.array_equal(L.ln_forward(z, gamma, beta, act)[0], f(u))
    assert np.allclose(L.ln_torch(torch.tensor(z), torch.tensor(gamma), torch.tensor(beta)).numpy(), u, rtol=1e-12)


def test_backward_matches_central_differences():
    z, gamma, beta, du = _case(4, 16, seed=1)
    loss = lambda z_, g_, b_: float((L.ln_forward(z_, g_, b_)[1] * du).sum())
    dz, dgamma, dbeta = L.ln_backward(du, z, gamma)
    h = 1e-6
    for arr, grad in ((z, dz), (gamma, dgamma), (beta, dbeta)):
        num = np.zeros_like(arr)
        for i in np.ndindex(arr.shape):
            a, b = arr.copy(), arr.copy()
            a[i] += h
            b[i] -= h
            args = [a if x is arr else x for x in (z, gamma, beta)], [b if x is arr else x for x in (z, gamma, beta)]
            num[i] = (loss(*args[0]) - loss(*args[1])) / (2 * h)
        assert np.allclose(grad, num, rtol=1e-5, atol=1e-7)


def test_one_pass_variance_is_the_mistake_the_bound_must_catch():
    """Rows with mean 1e3 and spread 1e-2: float32 E[x^2] - E[x]^2 has lost the variance, the two-pass form has not."""
    rng = np.random.RandomState(2)
    z = (1e3 + 1e-2 * rng.randn(8, 64)).astype(np.float32)
    ref = L.ln_forward(z, np.ones(64), np.zeros(64))[0]
    bad = L.ln_forward_one_pass(z, np.ones(64), np.zeros(64))
    assert np.abs(ref).max() < 5 and np.abs(bad - ref).max() > 0.5


def test_dbeta_order_emulation_sums_every_row_once():
    du = np.random.RandomState(3).randint(-4, 5, (300, 16)).astype(np.float16)      # integers: every order is exact
    for lanes in (8, 32):
        assert np.array_equal(L.dbeta_in_kernel_order(du, 0.5, lanes), 0.5 * du.astype(np.float32).sum(0))


def test_mlp_layer_norm_variables_in_creation_order():
    rng = np.random.RandomState(11)
    store = nn.ParamStore(None)
    t = nn.Tower(store, "mlp", (7,), "pi", "ppo2_model/pi", rng, 4, layer_norm=True)
    assert t.latent_dim == 64
    assert [(k, v[2]) for k, v in store.tf_map.items()] == [
        ("ppo2_model/pi/mlp_fc0/w:0", (7, 64)), ("ppo2_model/pi/mlp_fc0/b:0", (64,)),
        ("ppo2_model/pi/LayerNorm/beta:0", (64,)), ("ppo2_model/pi/LayerNorm/gamma:0", (64,)),
        ("ppo2_model/pi/mlp_fc1/w:0", (64, 64)), ("ppo2_model/pi/mlp_fc1/b:0", (64,)),
        ("ppo2_model/pi/LayerNorm_1/beta:0", (64,)), ("ppo2_model/pi/LayerNorm_1/gamma:0", (64,))]
    specs = {n: init for n, _, init in store._specs}
    assert not specs["pi/mlp_ln0/beta"].any() and np.all(specs["pi/mlp_ln1/gamma"] == 1)
    # the norms draw nothing: the weights are those of the un-normed tower from the same seed
    plain = nn.ParamStore(None)
    nn.Tower(plain, "mlp", (7,), "pi", "ppo2_model/pi", np.random.RandomState(11), 4)
    for n, _, init in plain._specs:
        assert np.array_equal(specs[n], init), n


def test_policy_reference_names_match_the_tower():
    op = L.with_policy_norms(nets.init_policy_params("mlp", (7,), "box", 3, value_network="copy", seed=0))
    names = [k for k in op if "/vf/" in k and "mlp" not in k and k.count("/") == 3]
    assert names == ["ppo2_model/vf/LayerNorm/beta:0", "ppo2_model/vf/LayerNorm/gamma:0",
                     "ppo2_model/vf/LayerNorm_1/beta:0", "ppo2_model/vf/LayerNorm_1/gamma:0"]
    store = nn.ParamStore(None)
    rng = np.random.RandomState(0)
    nn.Tower(store, "mlp", (7,), "pi", "ppo2_model/pi", rng, 4, layer_norm=True)
    nn.Tower(store, "mlp", (7,), "vf", "ppo2_model/vf", rng, 4, layer_norm=True)
    tower_names = list(store.tf_map)
    assert tower_names == [k for k in op if "mlp_fc" in k or "LayerNorm" in k]


@pytest.mark.parametrize("kind", ["cnn", "conv_only", "lstm", "cnn_lstm"])
def test_layer_norm_is_an_mlp_argument(kind):
    ob = (84, 84, 4) if "cnn" in kind or kind == "conv_only" else (4,)
    with pytest.raises(NotImplementedError, match="layer_norm"):
        nn.Tower(nn.ParamStore(None), kind, ob, "pi", "ppo2_model/pi", np.random.RandomState(0), 4, layer_norm=True)


def test_q_reference_norms_only_in_the_streams():
    qp = L.with_q_norms(nets.init_q_params("mlp", (8,), 4, hiddens=(32, 16), seed=0), n_hidden=2)
    ln = [k for k in qp if "LayerNorm" in k]
    assert ln == [f"deepq/q_func/{s}/{sc}/{v}:0" for s in ("action_value", "state_value")
                  for sc in ("LayerNorm", "LayerNorm_1") for v in ("beta", "gamma")]
    assert qp["deepq/q_func/action_value/LayerNorm_1/gamma:0"].shape == (16,)
    with L.layer_norm_nets():
        obs = torch.randn(5, 8, dtype=torch.float64)
        tp = nets.to_torch(qp, torch.float64)
        q = nets.q_forward(tp, "mlp", obs, "deepq/q_func", 2, True)
        tp["deepq/q_func/action_value/LayerNorm_1/gamma:0"][0] = 3.0
        assert not torch.allclose(q, nets.q_forward(tp, "mlp", obs, "deepq/q_func", 2, True))
    assert nets.q_forward is L._Q_FORWARD and nets.mlp is L._MLP
