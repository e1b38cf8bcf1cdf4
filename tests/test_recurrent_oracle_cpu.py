"""Anchors of the recurrent oracle (tests/_lstm_oracle.py) that do not go through its own torch code: definition-level
numpy loops of the reference cell, float64 central finite differences of its autograd gradients, the exact state
reset of the masks, and the variable creation order of the product's networks."""
import numpy as np
import torch

import _lstm_oracle as lo
from baselines_b200 import nn


def _small(seed=0, nenv=3, T=4, nin=5, H=4):
    rng = np.random.RandomState(seed)
    xs = rng.randn(nenv, T, nin)
    ms = (rng.rand(nenv, T) < 0.3).astype(np.float64)
    s = rng.randn(nenv, 2 * H) * 0.5
    wx, wh, b = rng.randn(nin, 4 * H) * 0.5, rng.randn(H, 4 * H) * 0.5, rng.randn(4 * H) * 0.1
    return xs, ms, s, wx, wh, b


def test_oracle_cell_matches_numpy_loops():
    xs, ms, s, wx, wh, b = _small()
    t = lambda a: torch.as_tensor(a, dtype=torch.float64)
    h, snew = lo.lstm_cell_seq(t(xs), t(ms), t(s), t(wx), t(wh), t(b))
    hr, sr = lo.lstm_numpy_loop(xs, ms, s, wx, wh, b)
    assert np.abs(h.numpy() - hr).max() < 1e-12
    assert np.abs(snew.numpy() - sr).max() < 1e-12


def test_oracle_gradients_match_central_differences():
    xs, ms, s, wx, wh, b = _small(1)
    t = lambda a, g=False: torch.tensor(a, dtype=torch.float64, requires_grad=g)
    rng = np.random.RandomState(2)
    cw = rng.randn(3, 4, 4)                                   # a fixed linear read-out of every h_t

    def loss(wx_, wh_, b_, s_):
        h, sn = lo.lstm_cell_seq(t(xs), t(ms), s_, wx_, wh_, b_)
        return (h * torch.as_tensor(cw)).sum() + (sn ** 2).sum()
    args = [t(wx, True), t(wh, True), t(b, True), t(s, True)]
    grads = torch.autograd.grad(loss(*args), args)
    eps = 1e-6
    for j, (a, g) in enumerate(zip(args, grads)):
        n = a.numel()
        for i in range(0, n, max(1, n // 12)):
            vals = []
            for d in (eps, -eps):
                pert = [x.detach().clone() for x in args]
                pert[j].view(-1)[i] += d
                vals.append(float(loss(*pert)))
            fd = (vals[0] - vals[1]) / (2 * eps)
            assert abs(fd - float(g.reshape(-1)[i])) <= 1e-6 * max(1.0, abs(fd)), (i, fd, float(g.reshape(-1)[i]))


def test_masks_reset_the_state_exactly():
    xs, ms, s, wx, wh, b = _small(3)
    ms[:] = 0
    ms[:, 2] = 1                                              # every environment's episode restarts at step 2
    t = lambda a: torch.as_tensor(a, dtype=torch.float64)
    h, _ = lo.lstm_cell_seq(t(xs), t(ms), t(s), t(wx), t(wh), t(b))
    h2, _ = lo.lstm_cell_seq(t(xs[:, 2:]), t(np.zeros_like(ms[:, 2:])), t(np.zeros_like(s)), t(wx), t(wh), t(b))
    assert torch.equal(h[:, 2:], h2)


def _tower_params(kind, ob_shape, nlstm, seed):
    rng = np.random.RandomState(seed)
    store = nn.ParamStore(None)
    t = nn.Tower(store, kind, ob_shape, "pi", "ppo2_model/pi", rng, 4, nlstm=nlstm)
    specs = {n: init for n, _, init in store._specs}
    out = {}
    for tf_name, (internal, sl, shape) in store.tf_map.items():
        a = specs[internal]
        if tf_name in store.row_perms:
            b = np.empty_like(a)
            b[store.row_perms[tf_name]] = a
            a = b
        out[tf_name] = a.reshape(shape)
    return out, t


def test_oracle_creation_order_matches_the_towers():
    for kind, ob_shape, nlstm in (("lstm", (7,), 64), ("cnn_lstm", (84, 84, 4), 128)):
        tp, _ = _tower_params(kind, ob_shape, nlstm, 5)
        op = lo.init_recurrent_params(kind, ob_shape, "discrete", 3, nlstm=nlstm, seed=5)
        for k, v in tp.items():
            assert np.array_equal(v, op[k]), (kind, k)
