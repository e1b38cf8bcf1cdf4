"""A graph-replayed PPO2 Model whose minibatch index buffer grows between calls.  train_rollout at nbatch_train (the
second call captures the step), at 2 * nbatch_train (the index buffer is reallocated), then at nbatch_train again
with new indices must compute what the same calls compute eagerly: the last call may not replay the graph captured
over the buffer the growth replaced, which would read the indices from freed memory."""
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from test_ppo2_gpu import CASES, _mk      # noqa: E402  (shared builders)


def _calls():
    """Parameters, Adam moments, statistics and graph replays of each call after four train_rollout calls."""
    from baselines_b200 import _lib
    _, model, _ = _mk(nenv=64, nsteps=8, nminibatches=2, **CASES["cnn_cat"])
    M, N, dev = model.nbatch_train, 512, model.device
    g = torch.Generator(device=dev).manual_seed(0)
    obs = torch.randint(0, 256, (N, 84, 84, 4), dtype=torch.uint8, device=dev, generator=g)
    actions = torch.randint(0, 6, (N,), dtype=torch.int64, device=dev, generator=g)
    values = torch.randn(N, device=dev, generator=g)
    returns = values + torch.randn(N, device=dev, generator=g)
    nlp = math.log(6) + 0.05 * torch.randn(N, device=dev, generator=g)
    rng = np.random.RandomState(1)
    stats, replays, stale = [], [], None
    for i, m in enumerate((M, M, 2 * M, M)):
        idx = torch.as_tensor(rng.permutation(N)[:m]).to(dev)
        r0 = _lib.REPLAYS
        st = model.train_rollout(2.5e-4 * (1.0 - 0.1 * i), 0.2 - 0.02 * i, obs, actions, returns, values, nlp, idx)
        stats.append(st.cpu().numpy())
        replays.append(_lib.REPLAYS - r0)
        if i == 2:
            stale = [k for k in model.graphs.graphs if k[:2] == ("train", M)]
    torch.cuda.synchronize()
    s = model.net.store
    return {k: t.cpu().numpy().copy() for k, t in (("params", s.params), ("m", s.m), ("v", s.v))}, stats, replays, stale


def test_growing_index_buffer_never_replays_a_stale_graph():
    out = {}
    for mode in ("eager", "eager2", "graphs"):
        if mode.startswith("eager"):
            os.environ["B200RL_NO_GRAPHS"] = "1"
        try:
            out[mode] = _calls()
        finally:
            os.environ.pop("B200RL_NO_GRAPHS", None)
    assert out["eager"][2] == [0, 0, 0, 0]
    # call 2 captures and replays; the growth in call 3 drops that graph, so call 4 runs eagerly
    assert out["graphs"][2] == [0, 1, 0, 0], out["graphs"][2]
    assert out["graphs"][3] == [], out["graphs"][3]
    # test_round2_gpu.py's graph-versus-eager criterion, on the parameters and on both Adam moments (whose floor is
    # scaled to their size: a stale index set changes every gradient, so it moves them by a large fraction)
    e, e2, gr = out["eager"][0], out["eager2"][0], out["graphs"][0]
    for k in ("params", "m", "v"):
        mspread, mdiff = float(np.abs(e[k] - e2[k]).mean()), float(np.abs(e[k] - gr[k]).mean())
        floor = 2e-6 if k == "params" else 1e-3 * float(np.abs(e[k]).mean())
        print(f"{k}: eager-vs-eager mean {mspread:.2e}, graphs-vs-eager mean {mdiff:.2e}")
        assert mdiff <= 10 * mspread + floor, (k, mdiff, mspread)
    assert float(np.abs(e["params"] - gr["params"]).max()) <= 1e-3
    for i, (a, b) in enumerate(zip(out["eager"][1], out["graphs"][1])):
        assert np.allclose(a, b, rtol=5e-3, atol=5e-3), (i, a, b)
