"""GPU parity of the PPO2 learner (Model / Runner / learn) against the CPU oracle restatement of the
reference's TF1 graph (oracle/nets.py; PARITY UNPINNED at the TF boundary, see oracle/__init__.py).

Tolerances: the CUDA path uses fp16 operands with fp32 accumulation; the reference's own tolerance for "same
update computed another way" is atol=3e-3 on parameters (ppo2/test_microbatches.py:31-32).  We assert that and
report much tighter observed errors."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _mk(network, ob_shape, ob_dtype, discrete, nA, value_network, nenv, nsteps, nminibatches, seed=0, **kw):
    from baselines_b200.common import spaces
    from baselines_b200.common.policies import build_policy
    from baselines_b200.ppo2.model import Model
    from oracle import nets

    class E:
        pass
    env = E()
    env.observation_space = spaces.Box(0, 255, ob_shape, ob_dtype) if ob_dtype == np.uint8 else spaces.Box(-5, 5, ob_shape, ob_dtype)
    env.action_space = spaces.Discrete(nA) if discrete else spaces.Box(-1, 1, (nA,), np.float32)
    env.num_envs = nenv
    np.random.seed(seed)
    policy = build_policy(env, network, value_network=value_network, **kw)
    nbatch_train = nenv * nsteps // nminibatches
    model = Model(policy=policy, ob_space=env.observation_space, ac_space=env.action_space, nbatch_act=nenv,
                  nbatch_train=nbatch_train, nsteps=nsteps, ent_coef=0.01, vf_coef=0.5, max_grad_norm=0.5, comm=False)
    np.random.seed(seed)
    okw = {k: v for k, v in kw.items() if k != "normalize_observations"}
    oparams = nets.init_policy_params(network, ob_shape, "discrete" if discrete else "box", nA,
                                      value_network=value_network, **okw)
    return env, model, oparams


def _check_same_init(model, oparams):
    mp = model.get_params()
    assert set(mp.keys()) == set(oparams.keys())
    for k, v in oparams.items():
        assert mp[k].shape == v.shape, k
        assert np.array_equal(mp[k], v), k            # same ortho_init draws in the same order


CASES = {
    "cnn_cat": dict(network="cnn", ob_shape=(84, 84, 4), ob_dtype=np.uint8, discrete=True, nA=6, value_network=None),
    "mlp_cat": dict(network="mlp", ob_shape=(4,), ob_dtype=np.float32, discrete=True, nA=2, value_network=None),
    "mlp_gauss_copy": dict(network="mlp", ob_shape=(376,), ob_dtype=np.float32, discrete=False, nA=17,
                           value_network="copy"),
    "mlp_gauss_shared": dict(network="mlp", ob_shape=(11,), ob_dtype=np.float32, discrete=False, nA=3,
                             value_network=None),
    # 2 * 256 hidden units: the two first layers run as separate GEMMs (the fused one takes 2 * hidden <= 256)
    "mlp_gauss_copy_unfused": dict(network="mlp", ob_shape=(11,), ob_dtype=np.float32, discrete=False, nA=3,
                                   value_network="copy", num_hidden=256),
}


def _obs(rng, case, B):
    if case["ob_dtype"] == np.uint8:
        return rng.randint(0, 256, size=(B,) + case["ob_shape"]).astype(np.uint8)
    # un-rounded float32, at the scale VecNormalize hands out (clipped to +-10, vec_normalize.py:39): the product
    # may not narrow observations (common/input.py:56-57 to_float) -- they reach the first GEMM as fp16 hi/lo pairs
    return np.clip(rng.randn(B, *case["ob_shape"]) * 3.0, -10.0, 10.0).astype(np.float32)


@pytest.mark.parametrize("name", list(CASES))
def test_step_matches_oracle(name):
    from oracle import nets
    case = CASES[name]
    B = 256
    env, model, oparams = _mk(nenv=B, nsteps=4, nminibatches=1, **case)
    _check_same_init(model, oparams)
    rng = np.random.RandomState(1)
    obs = _obs(rng, case, B)
    nA = case["nA"]
    noise = (rng.rand(B, nA) * 0.998 + 0.001).astype(np.float32) if case["discrete"] else rng.randn(B, nA).astype(np.float32)
    a, v, s, nlp = model.step(obs, noise=noise)
    assert s is None
    a_o, v_o, nlp_o, pi_o = nets.policy_step(oparams, case["network"], obs, noise, case["value_network"])
    pi = model.net.pi_out[:B, :nA].cpu().numpy()
    assert np.allclose(pi, pi_o, atol=3e-3, rtol=1e-2), float(np.abs(pi - pi_o).max())
    assert np.allclose(v, v_o, atol=3e-3 * max(1.0, float(np.abs(v_o).max()))), float(np.abs(v - v_o).max())
    assert np.allclose(model.value(obs), v_o, atol=3e-3 * max(1.0, float(np.abs(v_o).max())))
    if case["discrete"]:
        # Gumbel-max with injected noise: identical unless the top-2 scores are closer than the fp16 logit error
        sc = pi_o - np.log(-np.log(noise))
        top2 = np.sort(sc, axis=1)[:, -2:]
        clear = (top2[:, 1] - top2[:, 0]) > 1e-2
        assert np.array_equal(a[clear], a_o[clear]) and clear.mean() > 0.9
        assert np.allclose(nlp[clear], nlp_o[clear], atol=3e-3)
    else:
        assert np.allclose(a, a_o, atol=3e-3)
        # neglogp of the sampled action depends only on the injected noise
        assert np.allclose(nlp, nlp_o, atol=1e-3)


@pytest.mark.parametrize("name", list(CASES))
def test_train_step_matches_oracle(name):
    """ppo2/model.py:133-158 for 3 consecutive minibatches: loss statistics, gradients, post-step parameters."""
    from oracle import nets
    case = CASES[name]
    M = 512 if case["network"] == "cnn" else 2048
    env, model, oparams = _mk(nenv=M // 4, nsteps=4, nminibatches=1, **case)
    oracle = nets.PPO2Oracle(oparams, case["network"], 0.01, 0.5, 0.5, value_network=case["value_network"])
    rng = np.random.RandomState(2)
    nA = case["nA"]
    worst = 0.0
    for it in range(3):
        obs = _obs(rng, case, M)
        if case["discrete"]:
            actions = rng.randint(0, nA, M).astype(np.int64)
        else:
            actions = rng.randn(M, nA).astype(np.float32)
        values = rng.randn(M).astype(np.float32)
        returns = (values + rng.randn(M) * 0.7).astype(np.float32)
        _, _, nlp_cur, _ = nets.policy_step(oracle.params_np(), case["network"], obs,
                                            np.full((M, nA), 0.5, np.float32), case["value_network"])
        if case["discrete"]:
            t = nets.to_torch(oracle.params_np())
            with torch.no_grad():
                pi, _, _ = nets.policy_forward(t, case["network"], torch.as_tensor(obs), case["value_network"])
                nlp_cur = nets.cat_neglogp(pi, torch.as_tensor(actions)).numpy()
        else:
            t = nets.to_torch(oracle.params_np())
            with torch.no_grad():
                pi, ls, _ = nets.policy_forward(t, case["network"], torch.as_tensor(obs), case["value_network"])
                nlp_cur = nets.gauss_neglogp(pi, ls, torch.as_tensor(actions)).numpy()
        neglogpacs = (nlp_cur + rng.randn(M) * 0.05).astype(np.float32)
        lr, clip = 2.5e-4, 0.1
        st = model.train(lr, clip, obs, returns, None, actions, values, neglogpacs)
        st_o = oracle.train(lr, clip, obs, returns, None, actions, values, neglogpacs)
        assert np.allclose(st[:4], st_o[:4], atol=3e-3, rtol=2e-2), (it, st, st_o)
        assert abs(st[4] - st_o[4]) <= 0.02, (st[4], st_o[4])            # clipfrac: a few samples may flip side
        # gradients (mean loss, before clipping): cosine + relative L2 per tensor family
        g = model.net.store.export_tf("grads")
        num = sum(float(((g[k] - oracle.last_grads[k]) ** 2).sum()) for k in g)
        den = sum(float((oracle.last_grads[k] ** 2).sum()) for k in g)
        rel = (num / den) ** 0.5
        assert rel < 2e-2, (it, rel)
        p, po = model.get_params(), oracle.params_np()
        err = max(float(np.abs(p[k] - po[k]).max()) for k in p)
        worst = max(worst, err)
        # test_microbatches.py:31-32 tolerance.  Adam moves each element by at most ~lr per step whatever the
        # gradient, so this bounds the step and cannot detect a gradient error; every tensor's gradient and the Adam
        # step are checked in test_update_composition_gpu.py
        assert err < 3e-3, (it, err)
    print(f"[{name}] max |param - oracle| after 3 steps = {worst:.3e}")


def test_train_chunking_and_indexed_gather_equivalence():
    """MicrobatchedModel contract (ppo2/microbatched_model.py:35-75, test_microbatches.py): chunked
    accumulation == one big launch; and the index-gather path == the materialised-minibatch path."""
    case = CASES["cnn_cat"]
    M = 384
    rng = np.random.RandomState(3)
    obs = _obs(rng, case, M)
    actions = rng.randint(0, 6, M).astype(np.int64)
    values = rng.randn(M).astype(np.float32)
    returns = (values + rng.randn(M)).astype(np.float32)
    nlp = (np.log(6) + rng.randn(M) * 0.05).astype(np.float32)
    outs = []
    for chunk in (M, 100):
        os.environ["B200RL_TRAIN_CHUNK"] = str(chunk)
        try:
            env, model, _ = _mk(nenv=M // 4, nsteps=4, nminibatches=1, **case)
        finally:
            del os.environ["B200RL_TRAIN_CHUNK"]
        st = model.train(2.5e-4, 0.1, obs, returns, None, actions, values, nlp)
        outs.append((st, model.get_params()))
    for k in outs[0][1]:
        assert np.allclose(outs[0][1][k], outs[1][1][k], atol=3e-3), k      # reference tolerance; observed ~1e-6
        assert np.allclose(outs[0][1][k], outs[1][1][k], atol=2e-5), k
    assert np.allclose(outs[0][0], outs[1][0], atol=1e-5)
    # indexed path: permuted buffer + src_idx must give the same step
    env, model, _ = _mk(nenv=M // 4, nsteps=4, nminibatches=1, **case)
    perm = rng.permutation(M)
    inv = np.argsort(perm)
    dev = model.device
    f = lambda z, dt: torch.as_tensor(np.ascontiguousarray(z[inv]), dtype=dt).to(dev)
    st = model.train_rollout(2.5e-4, 0.1, f(obs, torch.uint8), f(actions, torch.int64), f(returns, torch.float32),
                             f(values, torch.float32), f(nlp, torch.float32), torch.as_tensor(perm).to(dev))
    assert np.allclose(st.cpu().numpy(), outs[0][0], atol=1e-5)
    p = model.get_params()
    for k in p:
        assert np.allclose(p[k], outs[0][1][k], atol=2e-5), k


class _ReplayEnv:
    """Deterministic VecEnv replaying pre-drawn rewards / dones (same idea as oracle/gen_golden.py FakeEnv)."""

    def __init__(self, obs_seq, rew, done, ob_space, ac_space):
        self.obs_seq, self.rew, self.done = obs_seq, rew, done
        self.num_envs = rew.shape[1]
        self.observation_space, self.action_space = ob_space, ac_space
        self.t = 0

    def reset(self):
        self.t = 0
        return self.obs_seq[0]

    def step(self, actions):
        r, d = self.rew[self.t], self.done[self.t]
        self.t += 1
        return self.obs_seq[self.t], r, d, [{} for _ in range(self.num_envs)]


def test_runner_matches_reference_semantics():
    """Runner.run(): mb_dones shift (runner.py:34), bootstrap from the last obs (:50), GAE (:53-65), sf01 (:69-74).
    GAE is checked bit-exactly against the oracle on the values the device itself produced."""
    from baselines_b200.ppo2.runner import Runner
    from oracle.gae import gae_reference_order, sf01
    case = CASES["mlp_cat"]
    T, N = 16, 32
    env0, model, oparams = _mk(nenv=N, nsteps=T, nminibatches=1, **case)
    rng = np.random.RandomState(5)
    obs_seq = (rng.randn(2 * T + 1, N, 4) * 3.0).astype(np.float32)          # not representable in fp16
    rew = rng.randn(2 * T, N).astype(np.float32)
    done = rng.rand(2 * T, N) < 0.15
    env = _ReplayEnv(obs_seq, rew, done, env0.observation_space, env0.action_space)
    runner = Runner(env=env, model=model, nsteps=T, gamma=0.99, lam=0.95)
    for k in range(2):
        obs, returns, masks, actions, values, neglogpacs, states, epinfos = runner.run()
        assert states is None and epinfos == []
        assert obs.shape == (N * T, 4) and returns.shape == (N * T,) and masks.dtype == np.bool_
        assert obs.dtype == np.float32 and np.array_equal(obs, sf01(obs_seq[k * T:(k + 1) * T]))   # returned bit-exact
        dones_before = np.concatenate([(done[k * T - 1] if k else np.zeros(N, bool))[None], done[k * T:(k + 1) * T - 1]], 0)
        assert np.array_equal(masks, sf01(dones_before))
        val_tn = values.reshape(N, T).T.copy()
        last_val = model.value(obs_seq[(k + 1) * T])
        adv_o, ret_o = gae_reference_order(rew[k * T:(k + 1) * T], val_tn, dones_before, last_val, done[(k + 1) * T - 1],
                                           0.99, 0.95)
        assert np.array_equal(returns, sf01(ret_o))                       # bit exact given the same values
        assert actions.shape == (N * T,) and actions.dtype == np.int64
        assert np.all((actions >= 0) & (actions < 2))


def test_learn_runs_and_improves_on_identity_env():
    """Reference learning test shape (common/tests/test_identity.py:28-41, envs/identity_env.py): the agent must
    repeat the observed one-hot state; ppo2 kwargs lr=1e-3, nsteps=64, ent_coef=0 (:19)."""
    from baselines_b200.common import spaces
    from baselines_b200.common.vec_env import DummyVecEnv
    from baselines_b200.ppo2 import ppo2

    class IdentityEnv:
        """Discrete identity env with one-hot float observations (the reference feeds Discrete obs through a
        one-hot encoder, common/input.py:52-53)."""

        def __init__(self, dim, ep_len=100, seed=0):
            self.dim, self.ep_len = dim, ep_len
            self.observation_space = spaces.Box(0, 1, (dim,), np.float32)
            self.action_space = spaces.Discrete(dim)
            self.rng = np.random.RandomState(seed)

        def _ob(self):
            o = np.zeros(self.dim, np.float32)
            o[self.state] = 1
            return o

        def reset(self):
            self.state, self.t = self.rng.randint(self.dim), 0
            return self._ob()

        def step(self, a):
            rew = 1.0 if int(a) == self.state else 0.0
            self.state, self.t = self.rng.randint(self.dim), self.t + 1
            return self._ob(), rew, self.t >= self.ep_len, {}

    env = DummyVecEnv([lambda i=i: IdentityEnv(10, seed=i) for i in range(8)])
    model = ppo2.learn(network="mlp", env=env, total_timesteps=30000, seed=0, lr=1e-3, nsteps=64, ent_coef=0.0,
                       gamma=0.9, log_interval=1000, comm=False)
    # evaluate like tests/util.py:14-39: fraction of reward over N trials
    obs = env.reset()
    tot = 0.0
    for _ in range(100):
        a, v, _, _ = model.step(obs)
        obs, rew, done, _ = env.step(a)
        tot += float(rew.sum())
    assert tot / (100 * 8) > 0.9, tot / 800


def test_save_load_roundtrip(tmp_path):
    """common/tests/test_serialization.py:77-82 contract: save -> load -> variables equal (atol 0.01 there; exact
    here), file is a joblib dict keyed by the reference's TF variable names."""
    import joblib
    case = CASES["cnn_cat"]
    env, model, oparams = _mk(nenv=8, nsteps=4, nminibatches=1, **case)
    rng = np.random.RandomState(6)
    M = 32
    model.train(1e-3, 0.2, _obs(rng, case, M), rng.randn(M).astype(np.float32), None, rng.randint(0, 6, M),
                rng.randn(M).astype(np.float32), np.full(M, 1.79, np.float32))
    path = str(tmp_path / "ckpt")
    model.save(path)
    d = joblib.load(path)
    for k in ("ppo2_model/pi/c1/w:0", "ppo2_model/pi/c1/b:0", "ppo2_model/pi/fc1/w:0", "ppo2_model/pi/w:0",
              "ppo2_model/vf/w:0", "ppo2_model/vf/b:0", "ppo2_model/pi/fc1/w/Adam:0", "ppo2_model/pi/fc1/w/Adam_1:0"):
        assert k in d, k
    assert d["ppo2_model/pi/c1/w:0"].shape == (8, 8, 4, 32) and d["ppo2_model/pi/c1/b:0"].shape == (1, 32, 1, 1)
    assert d["ppo2_model/pi/w:0"].shape == (512, 6) and d["ppo2_model/vf/w:0"].shape == (512, 1)
    env2, model2, _ = _mk(nenv=8, nsteps=4, nminibatches=1, seed=123, **case)
    model2.load(path)
    p1, p2 = model.get_params(), model2.get_params()
    for k in p1:
        assert np.array_equal(p1[k], p2[k]), k
    obs = _obs(rng, case, 8)
    assert np.array_equal(model.value(obs), model2.value(obs))
    assert model2.opt.t == model.opt.t


def test_runner_device_frame_stack_equals_host_stacked_upload():
    """VecFrameStack handled on the device (new frames uploaded, stack kept in the rollout buffer) must give the
    same rollout, bit for bit, as uploading the reference-style host-stacked observations."""
    from baselines_b200.common import spaces
    from baselines_b200.common.vec_env import VecEnv, VecFrameStack
    from baselines_b200.ppo2.runner import Runner
    case = CASES["cnn_cat"]
    T, N = 6, 8
    env0, model, _ = _mk(nenv=N, nsteps=T, nminibatches=1, **case)
    rng = np.random.RandomState(3)
    frames = rng.randint(0, 256, (2 * T + 1, N, 84, 84, 1)).astype(np.uint8)
    rew = rng.randn(2 * T, N).astype(np.float32)
    done = rng.rand(2 * T, N) < 0.3

    class Scripted(VecEnv):
        def __init__(self):
            super().__init__(N, spaces.Box(0, 255, (84, 84, 1), np.uint8), env0.action_space)
            self.t = 0

        def reset(self):
            self.t = 0
            return frames[0]

        def step_async(self, actions):
            pass

        def step_wait(self):
            r, d = rew[self.t], done[self.t]
            self.t += 1
            return frames[self.t], r, d, [{} for _ in range(N)]

    noise = rng.rand(2, T, N, 6).astype(np.float32) * 0.98 + 0.01
    outs = []
    for device_stack in (True, False):
        env = VecFrameStack(Scripted(), 4)
        if not device_stack:
            env.frame_stack_device = False                 # force the host np.roll path + full upload
        runner = Runner(env=env, model=model, nsteps=T, gamma=0.99, lam=0.95)
        assert runner.fs == device_stack
        res = []
        for k in range(2):
            o, ret, masks, act, val, nlp, _, _ = runner.run(noise=noise[k])
            res.append((o.copy(), ret.copy(), masks.copy(), act.copy(), val.copy(), nlp.copy()))
        outs.append(res)
    for a, b in zip(*outs):
        for x, y in zip(a, b):
            assert np.array_equal(x, y)


def test_command_line_trains_and_saves(tmp_path):
    """`python -m baselines_b200.run` control flow (run.py:52-84,202-222): worker-process envs with Monitor files,
    progress.csv, checkpoint in the reference's variable-name format."""
    import joblib
    from baselines_b200 import logger, run
    log_dir, save = str(tmp_path / "log"), str(tmp_path / "model")
    try:
        model = run.main(["--alg=ppo2", "--env=CartPole-v0", "--num_timesteps=2048", "--num_env=2", "--seed=0",
                          "--network=mlp", "--nsteps=256", "--nminibatches=4", "--noptepochs=2", "--log_interval=1",
                          "--lr=1e-3", f"--log_path={log_dir}", f"--save_path={save}"])
    finally:
        logger.configure(None)
    assert os.path.exists(os.path.join(log_dir, "progress.csv"))
    rows = open(os.path.join(log_dir, "progress.csv")).read().splitlines()
    assert len(rows) == 1 + 4 and "eprewmean" in rows[0] and "loss/policy_loss" in rows[0]
    for k in (0, 1):
        mon = open(os.path.join(log_dir, f"0.{k}.monitor.csv")).read().splitlines()
        assert mon[0].startswith("#") and mon[1] == "r,l,t" and len(mon) > 3        # CartPole episodes are short
    ck = joblib.load(save)
    assert "ppo2_model/pi/mlp_fc0/w:0" in ck and ck["ppo2_model/pi/mlp_fc0/w:0"].shape == (4, 64)
    a, v, s, nlp = model.step(np.zeros((2, 4), np.float32))
    assert a.shape == (2,) and s is None


def test_command_line_play_loop(tmp_path, monkeypatch, capsys):
    """--play (run.py:222-247): after training the trained model is stepped on the env forever, rendering each step
    and printing `episode_rew=<return>` when an env finishes.  The loop has no exit in the reference either; the test
    bounds it by making the (otherwise unused) render hook raise after a fixed number of steps."""
    from baselines_b200 import logger, run
    from baselines_b200.common import vec_env

    class _Stop(Exception):
        pass

    calls = {"n": 0}

    def render(self, *a, **k):
        calls["n"] += 1
        if calls["n"] >= 400:
            raise _Stop

    for cls in (vec_env.VecEnv, vec_env.DummyVecEnv, vec_env.SubprocVecEnv, vec_env.VecEnvWrapper):
        monkeypatch.setattr(cls, "render", render, raising=False)
    try:
        with pytest.raises(_Stop):
            run.main(["--alg=ppo2", "--env=CartPole-v0", "--num_timesteps=512", "--num_env=1", "--seed=0",
                      "--network=mlp", "--nsteps=128", "--nminibatches=4", "--noptepochs=1", "--log_interval=100",
                      f"--log_path={tmp_path / 'log'}", "--play"])
    finally:
        logger.configure(None)
    out = capsys.readouterr().out
    rets = [float(l.split("=")[1]) for l in out.splitlines() if l.startswith("episode_rew=")]
    # CartPole-v0 pays +1 per step and ends within 200 steps: 400 play steps finish at least one episode and every
    # printed return is that episode's step count
    assert calls["n"] == 400 and len(rets) >= 1
    assert all(r == int(r) and 1 <= r <= 200 for r in rets) and sum(rets) <= 400
