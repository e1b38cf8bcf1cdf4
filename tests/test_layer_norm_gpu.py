"""Layer normalisation on the GPU: the ln_fwd / ln_bwd kernels against float64, and the networks that use them
(PPO2 `mlp(layer_norm=True)`, deepq `layer_norm=True`) against the float64 / float32 restatements of _layer_norm_refs."""
import numpy as np
import pytest
import torch

import _layer_norm_refs as L

pytestmark = pytest.mark.gpu

R16 = 2.0 ** -11           # one rounding of an fp16 output


def _ops():
    from baselines_b200 import ops
    return ops


def _fwd(z, gamma, beta, act, eps=L.EPS, ld_z=None, ld_y=None):
    ops = _ops()
    rows, N = z.shape
    ld_z, ld_y = ld_z or N, ld_y or N
    zd = torch.full((rows, ld_z), 7.0, dtype=torch.float32, device="cuda")      # the padding must not be read
    zd[:, :N] = torch.as_tensor(z, dtype=torch.float32)
    y = torch.full((rows, ld_y), -3.0, dtype=torch.float16, device="cuda")       # nor the output's written
    c = lambda a: torch.as_tensor(np.asarray(a, np.float32)).cuda()
    ops.ln_fwd(zd, ld_z, c(gamma), c(beta), y, ld_y, rows, N, act, eps)
    torch.cuda.synchronize()
    if ld_y > N:
        assert torch.all(y[:, N:] == -3.0)
    return y[:, :N].cpu().numpy()


def _bwd(du, z, gamma, alpha=1.0, eps=L.EPS, ld=None, in_place=False, acc0=0.0):
    ops = _ops()
    rows, N = z.shape
    ld = ld or N
    c = lambda a: torch.as_tensor(np.asarray(a, np.float32)).cuda()
    zd = torch.zeros(rows, ld, dtype=torch.float32, device="cuda")
    zd[:, :N] = torch.as_tensor(z, dtype=torch.float32)
    dud = torch.zeros(rows, ld, dtype=torch.float16, device="cuda")
    dud[:, :N] = torch.as_tensor(np.asarray(du, np.float16))
    dz = dud if in_place else torch.full((rows, ld), 5.0, dtype=torch.float16, device="cuda")
    dg = torch.full((N,), acc0, dtype=torch.float32, device="cuda")
    db = torch.full((N,), acc0, dtype=torch.float32, device="cuda")
    ops.ln_bwd(dud, ld, zd, ld, c(gamma), dz, ld, dg, db, rows, N, alpha, eps)
    torch.cuda.synchronize()
    if ld > N and not in_place:
        assert torch.all(dz[:, N:] == 5.0)
    return dz[:, :N].cpu().numpy(), dg.cpu().numpy(), db.cpu().numpy()


def _data(rows, N, seed):
    rng = np.random.RandomState(seed)
    z = (rng.randn(rows, N) * rng.uniform(0.2, 3.0, (rows, 1)) + rng.uniform(-2, 2, (rows, 1))).astype(np.float32)
    gamma = rng.uniform(0.5, 1.5, N).astype(np.float32)
    beta = (rng.randn(N) * 0.3).astype(np.float32)
    du = (rng.randn(rows, N) * 0.1).astype(np.float16)
    return z, gamma, beta, du


def _fwd_bound(ref, u):
    """fp16 rounding of the result plus float32 arithmetic on the way: xhat carries a few float32 roundings, scaled by
    |gamma * xhat| <= |u| + |beta|, and the activation has slope <= 1."""
    return R16 * np.abs(ref) + 1e-5 * (1.0 + np.abs(u)) + 1e-7


# every (lanes per row, chunks per lane) instance of csrc/layer_norm.cu LN_DISPATCH, each with full and partial last chunks:
# <8,1> N <= 64, <32,1> N <= 256, <32,2> N <= 512, <32,4> beyond
LN_WIDTHS = [8, 64, 72, 256, 264, 384, 512, 520, 1000, 1024]


@pytest.mark.parametrize("N", LN_WIDTHS)
@pytest.mark.parametrize("rows", [1, 31, 32, 33, 1000])
def test_ln_fwd_matches_float64(N, rows):
    z, gamma, beta, _ = _data(rows, N, seed=N + rows)
    for act in (0, 1, 2):
        ref, u, _, _ = L.ln_forward(z, gamma, beta, act)
        got = _fwd(z, gamma, beta, act, ld_z=N + 8 * (act == 1), ld_y=N + 16 * (act == 2))
        assert np.all(np.abs(got - ref) <= _fwd_bound(ref, u)), (act, float(np.abs(got - ref).max()))


@pytest.mark.parametrize("N", [64, 256])
def test_ln_many_rows_and_rows_do_not_depend_on_their_neighbours(N):
    """131072 rows against float64, and every row bit-identical to the same row normalised in a 1-, 33- or 1000-row
    launch: a row's result is a function of the row alone."""
    rows = 131072
    z, gamma, beta, _ = _data(rows, N, seed=5)
    ref, u, _, _ = L.ln_forward(z, gamma, beta, 2)
    got = _fwd(z, gamma, beta, 2)
    assert np.all(np.abs(got - ref) <= _fwd_bound(ref, u))
    for n in (1, 33, 1000):
        assert np.array_equal(_fwd(z[:n], gamma, beta, 2), got[:n])
        assert np.array_equal(_fwd(z[-n:], gamma, beta, 2), got[-n:])


@pytest.mark.parametrize("N", [8, 64, 256, 1024])
def test_constant_rows_give_exactly_the_activation_of_beta(N):
    """Variance 0: xhat = 0 * (1 / sqrt(eps)) = 0 exactly.  (Constants with short mantissas and N a power of two, so that
    the float32 mean is the constant itself.)"""
    consts = np.array([0.0, 0.5, -3.0, 1024.0, -0.015625], np.float32)
    z = np.repeat(consts[:, None], N, axis=1)
    _, gamma, beta, _ = _data(1, N, seed=9)
    for act in (0, 1, 2):
        want = L.ACTS[act](beta.astype(np.float64)).astype(np.float16)
        assert np.array_equal(_fwd(z, gamma, beta, act), np.repeat(want[None], len(consts), 0))


def test_large_mean_small_spread_keeps_its_variance():
    """Rows with mean 1e3 and spread 1e-2.  The bound that accepts the kernel rejects the one-pass variance
    E[x^2] - E[x]^2 in float32."""
    rng = np.random.RandomState(4)
    N = 256
    z = (1e3 + 1e-2 * rng.randn(64, N)).astype(np.float32)
    gamma, beta = np.ones(N, np.float32), np.zeros(N, np.float32)
    ref, u, _, _ = L.ln_forward(z, gamma, beta, 0)
    # the float32 mean of 256 values near 1e3 can be off by ~1e-4, i.e. 1e-2 spreads: a shift every column of a row
    # shares, far below what losing the variance does
    bound = _fwd_bound(ref, u) + 3e-2
    got = _fwd(z, gamma, beta, 0)
    assert np.all(np.abs(got - ref) <= bound), float(np.abs(got - ref).max())
    bad = L.ln_forward_one_pass(z, gamma, beta, 0)
    assert np.mean(np.abs(bad - ref) > bound) > 0.5


@pytest.mark.parametrize("N", LN_WIDTHS)
@pytest.mark.parametrize("rows", [1, 33, 127, 128, 129, 1000])
def test_ln_bwd_matches_float64(N, rows):
    z, gamma, _, du = _data(rows, N, seed=3 * N + rows)
    alpha = 1.0 / rows
    dz_r, dg_r, db_r = L.ln_backward(du, z, gamma)
    dz, dg, db = _bwd(du, z, gamma, alpha=alpha, ld=N + 8, acc0=0.25)
    scale = np.abs(dz_r).max(axis=1, keepdims=True) + 1e-6
    assert np.all(np.abs(dz - dz_r) <= R16 * np.abs(dz_r) + 1e-5 * scale + 1e-7), float(np.abs(dz - dz_r).max())
    # the accumulators keep what they held: dgamma += alpha * sum, dbeta += alpha * sum
    xhat = L.ln_forward(z, gamma, np.zeros(N), 0)[2]
    tol_g = 1e-5 * alpha * (np.abs(du.astype(np.float64)) * (np.abs(xhat) + 1.0)).sum(0) + 1e-7
    tol_b = 1e-5 * alpha * np.abs(du.astype(np.float64)).sum(0) + 1e-7
    assert np.all(np.abs(dg - (0.25 + alpha * dg_r)) <= tol_g + 3e-8)
    assert np.all(np.abs(db - (0.25 + alpha * db_r)) <= tol_b + 3e-8)
    if rows > 1:                                                      # those bounds notice one dropped row
        assert np.any(alpha * np.abs(du[-1].astype(np.float64) * xhat[-1]) > tol_g + 3e-8)
        assert np.any(alpha * np.abs(du[-1].astype(np.float64)) > tol_b + 3e-8)
    # in place (du's buffer receives dz): same bits
    dz2, dg2, db2 = _bwd(du, z, gamma, alpha=alpha, ld=N + 8, in_place=True, acc0=0.25)
    assert np.array_equal(dz2, dz) and np.array_equal(dg2, dg) and np.array_equal(db2, db)


@pytest.mark.parametrize("N,lanes", [(64, 8), (256, 32), (384, 32), (1000, 32)])
def test_norm_gradients_repeat_and_follow_the_documented_order(N, lanes):
    """dgamma / dbeta are the same bits on every run, and dbeta is the float32 sum in the order csrc/layer_norm.cu
    documents (fixed 128-row slices, whatever the grid): an order that only depends on the data."""
    rows = 128 * 21 + 57
    z, gamma, _, du = _data(rows, N, seed=8)
    runs = [_bwd(du, z, gamma, alpha=0.125) for _ in range(3)]
    for r in runs[1:]:
        assert all(np.array_equal(a, b) for a, b in zip(r, runs[0]))
    assert np.array_equal(runs[0][2], L.dbeta_in_kernel_order(du, 0.125, lanes))
    # row r's dz is the same bits when the rows before it are gone (another slice position, another grid)
    assert np.array_equal(_bwd(du[300:], z[300:], gamma)[0], runs[0][0][300:])


# --------------------------------------------------------------------------------------------------- PPO2
PPO_CASES = {
    "gauss_copy": dict(network="mlp", ob_shape=(376,), ob_dtype=np.float32, discrete=False, nA=17, value_network="copy"),
    "cat_shared": dict(network="mlp", ob_shape=(4,), ob_dtype=np.float32, discrete=True, nA=2, value_network=None),
}


def _mk_ppo(case, M, seed=0):
    from baselines_b200.common import spaces
    from baselines_b200.common.policies import build_policy
    from baselines_b200.ppo2.model import Model
    from oracle import nets

    class E:
        observation_space = spaces.Box(-5, 5, case["ob_shape"], np.float32)
        action_space = spaces.Discrete(case["nA"]) if case["discrete"] else spaces.Box(-1, 1, (case["nA"],), np.float32)
        num_envs = M // 4
    np.random.seed(seed)
    model = Model(policy=build_policy(E, "mlp", value_network=case["value_network"], layer_norm=True),
                  ob_space=E.observation_space, ac_space=E.action_space, nbatch_act=M // 4, nbatch_train=M, nsteps=4,
                  ent_coef=0.01, vf_coef=0.5, max_grad_norm=0.5, comm=False)
    np.random.seed(seed)
    # init_policy_params knows nothing of layer_norm, and needs not: the norms draw nothing
    oparams = nets.init_policy_params("mlp", case["ob_shape"], "discrete" if case["discrete"] else "box", case["nA"],
                                      value_network=case["value_network"])
    return E, model, L.with_policy_norms(oparams)


def _randomise_norms(model, oparams, seed):
    """gamma = 1, beta = 0 would leave the forward blind to both: give them values, in the model and the reference."""
    L.randomise_norms(oparams, np.random.RandomState(seed))
    model.set_params(oparams)


def _ppo_batch(rng, case, M, oracle):
    from oracle import nets
    from test_ppo2_gpu import _obs
    nA = case["nA"]
    obs = _obs(rng, case, M)
    actions = rng.randint(0, nA, M).astype(np.int64) if case["discrete"] else rng.randn(M, nA).astype(np.float32)
    values = rng.randn(M).astype(np.float32)
    returns = (values + rng.randn(M) * 0.7).astype(np.float32)
    t = nets.to_torch(oracle.params_np())
    with torch.no_grad():
        pi, ls, _ = nets.policy_forward(t, case["network"], torch.as_tensor(obs), case["value_network"])
        nlp = (nets.cat_neglogp(pi, torch.as_tensor(actions)) if case["discrete"]
               else nets.gauss_neglogp(pi, ls, torch.as_tensor(actions))).numpy()
    return obs, returns, actions, values, (nlp + rng.randn(M) * 0.05).astype(np.float32)


@pytest.mark.parametrize("name", list(PPO_CASES))
def test_ppo2_layer_norm_train_matches_float64(name):
    """ppo2/model.py:133-158 with mlp(layer_norm=True) for 3 minibatches against the float64 restatement: statistics,
    every gradient (the norms' too), parameters; at the tolerances of test_ppo2_gpu.test_train_step_matches_oracle."""
    from oracle import nets
    case, M = PPO_CASES[name], 2048
    env, model, oparams = _mk_ppo(case, M)
    mp = model.get_params()
    assert set(mp) == set(oparams)
    for k, v in oparams.items():
        assert np.array_equal(mp[k], v), k                            # same draws: the norms consume none
    assert not model.net.fuse0
    _randomise_norms(model, oparams, 1)
    rng = np.random.RandomState(2)
    with L.layer_norm_nets():
        oracle = nets.PPO2Oracle(oparams, "mlp", 0.01, 0.5, 0.5, value_network=case["value_network"], dtype=torch.float64)
        for it in range(3):
            obs, returns, actions, values, nlp = _ppo_batch(rng, case, M, oracle)
            st = model.train(2.5e-4, 0.1, obs, returns, None, actions, values, nlp)
            st_o = oracle.train(2.5e-4, 0.1, obs, returns, None, actions, values, nlp)
            assert np.allclose(st[:4], st_o[:4], atol=3e-3, rtol=2e-2), (it, st, st_o)
            assert abs(st[4] - st_o[4]) <= 0.02
            g = model.net.store.export_tf("grads")
            assert set(g) == set(oracle.last_grads)
            rel = lambda keys: (sum(float(((g[k] - oracle.last_grads[k]) ** 2).sum()) for k in keys) /
                                sum(float((oracle.last_grads[k] ** 2).sum()) for k in keys)) ** 0.5
            assert rel(list(g)) < 2e-2, (it, rel(list(g)))
            norms = [k for k in g if "LayerNorm" in k]
            assert len(norms) == (8 if case["value_network"] else 4) and rel(norms) < 2e-2, (it, rel(norms))
            p, po = model.get_params(), oracle.params_np()
            assert max(float(np.abs(p[k] - po[k]).max()) for k in p) < 3e-3


def test_ppo2_layer_norm_acting_rows_are_the_training_rows():
    """The acting pass and the training forward run the same kernels on the same operands: per row, bit for bit."""
    case = PPO_CASES["gauss_copy"]
    env, model, oparams = _mk_ppo(case, 256)
    _randomise_norms(model, oparams, 3)
    from test_ppo2_gpu import _obs
    obs = _obs(np.random.RandomState(0), case, 64)
    net = model.net
    x = net.encode_obs(obs)
    net.forward(x, 64)
    pi64, v64 = net.pi_out[:64].clone(), net.v_out[:64].clone()
    net.forward(x[:1], 1, masks=False)
    assert torch.equal(net.pi_out[:1], pi64[:1]) and torch.equal(net.v_out[:1], v64[:1])
    assert np.array_equal(model.value(obs[:7]), v64[:7, 0].cpu().numpy())


def test_ppo2_layer_norm_graph_replay_equals_eager(monkeypatch, tmp_path):
    """Three updates replayed from captured launch sequences and three run eagerly leave the same bits; the checkpoint
    carries the norms under the reference's names and restores them."""
    case, M = PPO_CASES["cat_shared"], 512
    finals = []
    for no_graphs in ("0", "1"):
        monkeypatch.setenv("B200RL_NO_GRAPHS", no_graphs)
        env, model, oparams = _mk_ppo(case, M)
        _randomise_norms(model, oparams, 4)
        rng = np.random.RandomState(6)
        from test_ppo2_gpu import _obs
        for it in range(4):
            obs = _obs(rng, case, M)
            actions = rng.randint(0, 2, M).astype(np.int64)
            values = rng.randn(M).astype(np.float32)
            returns = (values + rng.randn(M) * 0.7).astype(np.float32)
            model.train(2.5e-4, 0.1, obs, returns, None, actions, values, np.full(M, np.log(2), np.float32))
        finals.append((model, model.get_params(), model.step(obs[:M // 4], noise=np.full((M // 4, 2), 0.5, np.float32))))
    (m0, p0, s0), (_, p1, s1) = finals
    for k in p0:
        assert np.array_equal(p0[k], p1[k]), k
    assert np.array_equal(s0[0], s1[0]) and np.array_equal(s0[1], s1[1]) and np.array_equal(s0[3], s1[3])
    path = str(tmp_path / "ckpt")
    m0.save(path)
    import joblib
    d = joblib.load(path)
    for k in ("ppo2_model/pi/LayerNorm/beta:0", "ppo2_model/pi/LayerNorm_1/gamma:0",
              "ppo2_model/pi/LayerNorm_1/gamma/Adam:0", "ppo2_model/pi/LayerNorm/beta/Adam_1:0"):
        assert k in d and d[k].shape == (64,), k
    assert not np.array_equal(d["ppo2_model/pi/LayerNorm_1/gamma:0"], oparams["ppo2_model/pi/LayerNorm_1/gamma:0"])
    env, fresh, _ = _mk_ppo(case, M, seed=5)
    fresh.load(path)
    for k, v in fresh.get_params().items():
        assert np.array_equal(v, p0[k]), k
    s2 = fresh.step(obs[:M // 4], noise=np.full((M // 4, 2), 0.5, np.float32))
    assert np.array_equal(s2[0], s0[0]) and np.array_equal(s2[1], s0[1])


# --------------------------------------------------------------------------------------------------- deepq
@pytest.mark.parametrize("network,ob_shape,dtype,dueling,hiddens", [("mlp", (8,), np.float32, True, (256,)),
                                                                    ("mlp", (8,), np.float32, False, (64, 32)),
                                                                    ("conv_only", (84, 84, 4), np.uint8, True, (256,))])
def test_dqn_layer_norm_train_step_matches_float64(network, ob_shape, dtype, dueling, hiddens):
    """deepq/build_graph.py:380-444 with layer_norm=True (norms in the streams only, deepq/models.py:24-25,34-35):
    one step from identical state, three times, as test_deepq_gpu.test_dqn_train_step_matches_oracle does."""
    from baselines_b200.deepq.build_graph import DQNModel
    from oracle import nets
    from test_deepq_gpu import _space
    nA, seed = 6, 3
    B = 256 if dtype == np.uint8 else 64
    model = DQNModel(_space(ob_shape, dtype), nA, network, lr=1e-4, gamma=0.99, grad_norm_clipping=10, batch_cap=B,
                     seed=seed, hiddens=hiddens, dueling=dueling, layer_norm=True)
    nh = len(hiddens)
    qp = L.with_q_norms(nets.init_q_params(network, ob_shape, nA, hiddens=hiddens, dueling=dueling, seed=seed), nh)
    mp = model.q.store.export_tf("params")
    assert set(mp) == set(qp)
    assert not any("LayerNorm" in k and "_value/" not in k for k in mp)
    for k in qp:
        assert np.array_equal(mp[k], qp[k]), k
    rng = np.random.RandomState(0)
    L.randomise_norms(qp, rng)
    obs = (lambda: rng.randint(0, 256, (B,) + ob_shape).astype(np.uint8)) if dtype == np.uint8 else \
          (lambda: (rng.randn(B, *ob_shape) * 2.0).astype(np.float32))
    dev = model.device
    f = lambda a: torch.as_tensor(a).to(dev)
    with L.layer_norm_nets():
        oracle = nets.DQNOracle(qp, network, 0.99, n_hidden=nh, dueling=dueling, grad_norm_clipping=10.0,
                                dtype=torch.float64)
        for it in range(3):
            model.q.store.import_tf({k: v.numpy() for k, v in oracle.tp.items()}, "params")
            model.q.store.import_tf({k: v.numpy() for k, v in oracle.m.items()}, "m")
            model.q.store.import_tf({k: v.numpy() for k, v in oracle.v.items()}, "v")
            model.qt.store.import_tf({k: v.numpy() for k, v in oracle.tt.items()}, "params")
            model.opt.t = oracle.t
            model.q.refresh()
            model.qt.refresh()
            o_t, o_1 = obs(), obs()
            act = rng.randint(0, nA, B).astype(np.int64)
            rew = rng.randn(B).astype(np.float32)
            done = (rng.rand(B) < 0.1).astype(np.float32)
            w = (rng.rand(B) * 0.9 + 0.1).astype(np.float32)
            qn = np.sort(oracle.q_values(o_1), axis=1)
            done[(qn[:, -1] - qn[:, -2]) < 3e-2] = 1.0                # double-Q argmax ties inside the fp16 error
            td = model.train_device(f(o_t), f(o_1), f(act), f(rew), f(done), f(w), None, B).cpu().numpy()
            td_o = oracle.train(1e-4, o_t, act, rew, o_1, done, w)
            assert np.allclose(td, td_o, atol=5e-3 * max(1.0, np.abs(td_o).max())), (it, np.abs(td - td_o).max())
            g = model.q.store.export_tf("grads")
            rel = lambda keys: (sum(float(((g[k] - oracle.last_grads[k]) ** 2).sum()) for k in keys) /
                                sum(float((oracle.last_grads[k] ** 2).sum()) for k in keys)) ** 0.5
            norms = [k for k in g if "LayerNorm" in k]
            assert len(norms) == 2 * nh * (2 if dueling else 1)
            assert rel(list(g)) < 5e-2 and rel(norms) < 5e-2, (it, rel(list(g)), rel(norms))
            p, po = model.q.store.export_tf("params"), {k: v.numpy() for k, v in oracle.tp.items()}
            assert max(float(np.abs(p[k] - po[k]).max()) for k in p) < 3e-3
            if it == 1:
                model.update_target()
                oracle.update_target()
        assert np.allclose(model.q_values(o_t[:8]), oracle.q_values(o_t[:8]), atol=2e-2)


def test_deepq_learn_with_layer_norm_solves_identity_env(tmp_path):
    """deepq.learn(layer_norm=True) on the contextual-bandit identity env of test_deepq_gpu, at its step budget and
    threshold; the saved act function reloads with the norms and picks the same actions."""
    from baselines_b200 import deepq
    from baselines_b200.common import spaces

    class Env:
        def __init__(self, n=5, ep_len=50):
            self.n, self.ep_len = n, ep_len
            self.observation_space = spaces.Box(0, 1, (n,), np.float32)
            self.action_space = spaces.Discrete(n)
            self.rng = np.random.RandomState(0)

        def _ob(self):
            o = np.zeros(self.n, np.float32)
            o[self.s] = 1
            return o

        def reset(self):
            self.s, self.t = self.rng.randint(self.n), 0
            return self._ob()

        def step(self, a):
            r = 1.0 if int(a) == self.s else 0.0
            self.s, self.t = self.rng.randint(self.n), self.t + 1
            return self._ob(), r, self.t >= self.ep_len, {}

    env = Env()
    act = deepq.learn(env, "mlp", seed=0, lr=1e-3, total_timesteps=4000, buffer_size=2000, exploration_fraction=0.3,
                      exploration_final_eps=0.02, train_freq=1, batch_size=32, print_freq=None, checkpoint_freq=None,
                      learning_starts=200, gamma=0.0, target_network_update_freq=200, prioritized_replay=True,
                      hiddens=(64,), dueling=True, layer_norm=True)
    eye = np.eye(5, dtype=np.float32)
    picks = act(eye, stochastic=False)
    ob, tot = env.reset(), 0.0
    for _ in range(200):
        ob, r, d, _ = env.step(act(ob[None], stochastic=False)[0])
        tot += r
        if d:
            ob = env.reset()
    assert tot / 200 > 0.9, tot / 200
    path = str(tmp_path / "act.pkl")
    act.save_act(path)
    again = deepq.load_act(path)
    assert np.array_equal(again(eye, stochastic=False), picks)
