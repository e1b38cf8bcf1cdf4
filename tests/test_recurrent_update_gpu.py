"""Whole recurrent PPO2 updates against the torch-CPU restatement of the reference (tests/_lstm_oracle.py), the Runner
against the reference's acting loop, and resuming a recurrent model through learn(load_path=...)."""
import numpy as np
import pytest
import torch

import _lstm_oracle as lo
from test_recurrent_gpu import DEV, _model, _spaces, _vec_env

pytestmark = pytest.mark.gpu

CASES = {
    "box_lstm": dict(kind="box", network="lstm", nlstm=128, chunk=None),
    "discrete_lstm": dict(kind="discrete", network="lstm", nlstm=64, chunk=None),
    "atari_cnn_lstm": dict(kind="atari", network="cnn_lstm", nlstm=128, chunk=None),
    # 4 environments per minibatch, 2 per chunk: two chunks accumulate into every minibatch
    "box_lstm_chunked": dict(kind="box", network="lstm", nlstm=64, chunk=16),
    "atari_cnn_lstm_chunked": dict(kind="atari", network="cnn_lstm", nlstm=64, chunk=16),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_recurrent_update_matches_oracle(name):
    """One recurrent update (ppo2.py:167-180), 2 minibatches x 2 epochs over a Runner rollout, against the oracle: the
    initial variables (creation order), every minibatch's statistics, every parameter afterwards within the reference's
    own equivalence tolerance (3e-3, ppo2/test_microbatches.py:31-32), and the gradient of the last minibatch."""
    from baselines_b200.ppo2.ppo2 import run_epochs
    from baselines_b200.ppo2.runner import Runner
    case = CASES[name]
    N, T, nmb, nep = 8, 8, 2, 2
    ob, ac = _spaces(case["kind"])
    model = _model(case["network"], ob, ac, N, T, nminibatches=nmb, nlstm=case["nlstm"], train_chunk=case["chunk"])
    onehot = ob.n if case["kind"] == "discrete" else 0
    p0 = lo.init_recurrent_params(case["network"], getattr(ob, "shape", ()), "discrete", ac.n, nlstm=case["nlstm"],
                                  seed=0, onehot_n=onehot)
    mp = model.get_params()
    assert set(mp) == set(p0)
    for k in p0:
        assert np.array_equal(mp[k], p0[k]), k
    runner = Runner(env=_vec_env(case["kind"], N, 4), model=model, nsteps=T, gamma=0.99, lam=0.95)
    runner.run()                                   # a first rollout, so the second starts from non-zero states
    obs, returns, masks, actions, values, neglogpacs, states, _ = runner.run()
    assert np.abs(states).max() > 0 and masks.any()
    oracle = lo.RecurrentPPO2Oracle(model.get_params(), case["network"], 0.01, 0.5, 0.5, T, onehot_n=onehot)
    rng = np.random.RandomState(7)
    perms = [rng.permutation(N) for _ in range(nep)]
    lr, clip = 3e-4, 0.2
    got = [s.cpu().numpy() for s in run_epochs(model, runner.rollout, lr, clip, N * T, N * T // nmb, nep, DEV,
                                                 perms=perms)]
    flatinds = np.arange(N * T).reshape(N, T)
    envsper = N // nmb
    want = []
    for ep in range(nep):
        for start in range(0, N, envsper):
            mbenv = perms[ep][start:start + envsper]
            mbflat = flatinds[mbenv].ravel()
            want.append(oracle.train(lr, clip, obs[mbflat], returns[mbflat], masks[mbflat], actions[mbflat],
                                     values[mbflat], neglogpacs[mbflat], states[mbenv]))
    M = envsper * T
    for i, (g, w) in enumerate(zip(got, want)):
        assert np.allclose(g[:4], w[:4], atol=3e-3, rtol=2e-2), (i, g, w)
        assert abs(g[4] - w[4]) <= max(0.02, 2.5 / M), (i, g[4], w[4])      # a sample or two may flip side
    assert got[0][3] == 0.0 and got[0][4] == 0.0                            # the acting pass, bit for bit
    gm = model.net.store.export_tf("grads")
    num = sum(float(((gm[k] - oracle.last_grads[k]) ** 2).sum()) for k in gm)
    den = sum(float((oracle.last_grads[k] ** 2).sum()) for k in gm)
    assert (num / den) ** 0.5 < 2e-2, (num / den) ** 0.5
    p, po = model.get_params(), oracle.params_np()
    err = max(float(np.abs(p[k] - po[k]).max()) for k in p)
    assert err < 3e-3, err


def test_runner_matches_reference_acting_loop():
    """runner.py:20-50 with S=self.states, M=self.dones: same actions, values, neglogp, masks and states as the
    reference's loop over model.step, with the state carried across steps and reset where an episode ended."""
    from baselines_b200.ppo2.runner import Runner
    N, T, nA = 6, 12, 4
    ob, ac = _spaces("box")
    model = _model("lstm", ob, ac, N, T)
    noise = np.random.RandomState(3).uniform(0.01, 0.99, (2, T, N, nA)).astype(np.float32)
    runner = Runner(env=_vec_env("box", N, 9), model=model, nsteps=T, gamma=0.99, lam=0.95)
    outs = [runner.run(noise=noise[r]) for r in range(2)]
    env = _vec_env("box", N, 9)
    o = env.reset()
    S, dones = model.initial_state, np.zeros(N, bool)
    for r in range(2):
        mb = {k: [] for k in ("a", "v", "nlp", "d")}
        s_start = np.asarray(S, np.float32).copy()
        for t in range(T):
            a, v, S, nlp = model.step(o, S=S, M=dones, noise=noise[r, t])
            mb["a"].append(a), mb["v"].append(v), mb["nlp"].append(nlp), mb["d"].append(dones)
            o, _, dones, _ = env.step(a)
        sf = lambda x: np.asarray(x).swapaxes(0, 1).reshape(N * T)
        obs_r, _, masks_r, actions_r, values_r, nlp_r, states_r, _ = outs[r]
        assert np.array_equal(states_r, s_start)
        assert np.array_equal(masks_r, sf(mb["d"]))
        assert np.array_equal(actions_r, sf(mb["a"]))
        assert np.array_equal(values_r, sf(mb["v"]))
        assert np.array_equal(nlp_r, sf(mb["nlp"]))
        assert masks_r.any()
    assert np.array_equal(runner.states, S)


@pytest.mark.parametrize("H", [64, 128])
def test_sequence_rows_identical_across_batch_sizes(H):
    """A row's h, state and saved tensors do not depend on how many rows run with it (B = 1, 7, 8, 9, 200)."""
    from baselines_b200 import ops
    rng = np.random.default_rng(5)
    T, Bmax = 9, 200
    xg = torch.from_numpy(rng.standard_normal((T, Bmax, 4 * H)).astype(np.float32)).to(DEV)
    wh = torch.from_numpy((rng.standard_normal((H, 4 * H)) / np.sqrt(H)).astype(np.float16)).to(DEV)
    m = torch.from_numpy((rng.random((T, Bmax)) < 0.2).astype(np.uint8)).to(DEV)
    s0 = torch.from_numpy(rng.standard_normal((Bmax, 2 * H)).astype(np.float32)).to(DEV)
    res = {}
    for B in (1, 7, 8, 9, 200):
        h = torch.zeros(T * B, H, dtype=torch.float16, device=DEV)
        g = torch.zeros(T * B, 4 * H, device=DEV)
        so = torch.zeros(B, 2 * H, device=DEV)
        ops.lstm_seq_fwd(xg[:, :B].contiguous().view(T * B, 4 * H), 4 * H, wh, m[:, :B].contiguous().view(-1), s0[:B],
                         h, H, T, B, H, state_out=so, gates_out=g)
        res[B] = (h.view(T, B, H)[:, :1].clone(), g.view(T, B, 4 * H)[:, :1].clone(), so[:1].clone())
    for B in res:
        for a, b in zip(res[B], res[1]):
            assert torch.equal(a, b), B


def test_learn_resumes_from_a_checkpoint(tmp_path):
    """learn(total_timesteps=0, load_path=...) restores a recurrent model's variables."""
    from baselines_b200.ppo2 import ppo2
    ob, ac = _spaces("box")
    m1 = _model("lstm", ob, ac, 4, 8, nlstm=64, seed=3)
    path = str(tmp_path / "ck")
    m1.save(path)
    m2 = ppo2.learn(network="lstm", env=_vec_env("box", 4, 1), total_timesteps=0, seed=0, nsteps=8, nlstm=64,
                    load_path=path)
    p1, p2 = m1.get_params(), m2.get_params()
    assert set(p1) == set(p2)
    for k in p1:
        assert np.array_equal(p1[k], p2[k]), k
