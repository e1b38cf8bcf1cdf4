"""GPU: VecNormalize on the device (csrc/vec_normalize.cu) equals the numpy wrapper bit for bit -- the kernels against
the order-explicit restatement (tests/_vec_normalize_refs.py, itself pinned to numpy by test_vec_normalize_cpu.py),
and the PPO2 Runner / ppo2.learn on the device path against the host path."""
import numpy as np
import pytest
import torch

from _vec_normalize_refs import RefVecNormalize, batch_moments

pytestmark = pytest.mark.gpu

SHAPES = [(1,), (2,), (5,), (3, 5), (376,)]
NS = [1, 2, 7, 8, 9, 127, 128, 129, 8191, 8192, 8193, 16384, 65536]


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True) and \
        np.array_equal(np.signbit(a) | np.isnan(a), np.signbit(b) | np.isnan(b))


def _grid():
    for shape in SHAPES:
        for N in NS:
            if N * int(np.prod(shape)) <= (1 << 22):
                yield shape, N


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("shape,N", list(_grid()))
def test_moments_kernel_equals_numpy(shape, N, dtype):
    from baselines_b200 import ops
    rng = np.random.RandomState(N % 997)
    D = int(np.prod(shape))
    ws = torch.zeros(2 * D, dtype=torch.float64, device="cuda")
    for x in ((1e4 + rng.randn(N, *shape)).astype(dtype), (rng.randn(N, *shape) * 3).astype(dtype)):
        ops.vecnorm_moments(torch.from_numpy(x).cuda(), ws)
        m, v = batch_moments(x)
        got = ws.cpu().numpy()
        assert _same(got[:D], m.ravel().astype(np.float64)) and _same(got[D:], v.ravel().astype(np.float64))


def _run_both(shape, N, T, dtype, rdtype=None, ob=True, ret=True, special=False, news_mode="mixed", seed=0):
    """Drive the device filter (VecNormalize.dev_reset / dev_step on CUDA tensors) and the restatement with the same
    raw steps; compare every output and the final statistics."""
    from baselines_b200.common import spaces
    from baselines_b200.common.vec_env import VecEnv, VecNormalize
    rdtype = rdtype or dtype
    rng = np.random.RandomState(seed)
    obs = (1e4 + rng.randn(T + 1, N, *shape)).astype(dtype) if not special else \
        (rng.randn(T + 1, N, *shape) * 2).astype(dtype)
    rews = (rng.randn(T, N) * 4).astype(rdtype)
    if special:
        flat = obs.reshape(T + 1, N, -1)
        flat[1:, 0, 0] = 0.0
        flat[1:, -1, -1] = -0.0
        flat[2, N // 2, 0] = 1e6                         # far above the clip bound
        flat[3, N // 2, -1] = -1e6
        rews[1, 0] = 1e5
        rews[2, -1] = -1e5
        rews[3, N // 2] = -0.0
    news = {"none": np.zeros((T, N), bool), "all": np.ones((T, N), bool),
            "mixed": rng.rand(T, N) < 0.3}[news_mode]

    class Null(VecEnv):
        def reset(self):
            pass

        def step_async(self, a):
            pass

        def step_wait(self):
            pass

    env = VecNormalize(Null(N, spaces.Box(-np.inf, np.inf, shape, dtype), spaces.Discrete(2)), ob=ob, ret=ret)
    ref = RefVecNormalize(shape, N, ob=ob, ret=ret)
    D = int(np.prod(shape))
    out = torch.zeros(N, D, device="cuda")
    rout = torch.zeros(N, device="cuda")
    env.dev_reset(torch.from_numpy(obs[0]).cuda(), out)
    assert _same(out.cpu().numpy(), ref.reset(obs[0]).reshape(N, D))
    for t in range(T):
        env.dev_step(torch.from_numpy(obs[t + 1]).cuda(), torch.from_numpy(rews[t]).cuda(),
                     torch.from_numpy(news[t].astype(np.uint8)).cuda(), out, rout)
        o, r = ref.step(obs[t + 1], rews[t], news[t])
        assert _same(out.cpu().numpy(), o.reshape(N, D)), t
        assert _same(rout.cpu().numpy(), r), t
    if ob:
        assert _same(env.ob_rms.mean, ref.ob[0]) and _same(env.ob_rms.var, ref.ob[1]) and env.ob_rms.count == ref.ob[2]
    if ret:
        assert _same(env.ret_rms.mean, ref.rt[0]) and _same(env.ret_rms.var, ref.rt[1])
        assert env.ret_rms.count == ref.rt[2]
    assert _same(env.ret, ref.ret)
    return env


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("shape,N", [((1,), 9), ((1,), 8193), ((2,), 127), ((5,), 129), ((3, 5), 7), ((376,), 8192),
                                     ((376,), 1), ((2,), 65536)])
def test_filter_steps_equal_restatement(shape, N, dtype):
    _run_both(shape, N, 4, dtype)


@pytest.mark.parametrize("news_mode", ["none", "all", "mixed"])
@pytest.mark.parametrize("rdtype", [np.float32, np.float64])
@pytest.mark.parametrize("shape", [(1,), (5,)])
def test_clip_signed_zero_and_episode_ends(shape, rdtype, news_mode):
    _run_both(shape, 64, 5, np.float32, rdtype=rdtype, special=True, news_mode=news_mode)


@pytest.mark.parametrize("ob,ret", [(False, True), (True, False), (False, False)])
def test_halves_switched_off(ob, ret):
    _run_both((5,), 33, 4, np.float64, ob=ob, ret=ret)


def test_nan_and_inf_behave_like_np_clip():
    """Normalising NaN / +-inf with given statistics: np.clip keeps NaN and clips the infinities."""
    from baselines_b200 import ops
    D, N = 3, 4
    x = np.array([[np.nan, np.inf, -np.inf], [0.0, -0.0, 1.0], [25.0, -25.0, 2.0], [np.nan, 0.5, -1e300]])
    mean, var = np.array([0.5, -0.25, 0.0]), np.array([1.0, 4.0, 0.25])
    rms = torch.from_numpy(np.concatenate([mean, var, np.sqrt(var + 1e-8), [3.0]])).cuda()
    out = torch.zeros(N, D, device="cuda")
    ops.vecnorm_normalize(torch.from_numpy(x).cuda(), rms, 10.0, out)
    want = np.clip((x - mean) / np.sqrt(var + 1e-8), -10.0, 10.0).astype(np.float32)
    assert _same(out.cpu().numpy(), want)


def test_cfg3_shape_four_steps():
    """The MuJoCo Humanoid shape of cfg-3: 16384 envs x 376 float32, 4 steps."""
    _run_both((376,), 16384, 4, np.float32, seed=3)


def test_host_refuses_bad_operands():
    from baselines_b200 import ops
    ws = torch.zeros(4, dtype=torch.float64, device="cuda")
    with pytest.raises(RuntimeError):
        ops.vecnorm_moments(torch.zeros(4, 2, dtype=torch.float16, device="cuda"), ws)
    with pytest.raises(RuntimeError):
        ops.vecnorm_moments(torch.zeros(200000, 1, device="cuda"), ws)        # beyond the pairwise CTA's leaves
    with pytest.raises(RuntimeError):
        ops.vecnorm_moments(torch.zeros(4, 2), ws)                              # host tensor


# ------------------------------------------------------------------------------------------- Runner and learn
class _Scripted:
    """Deterministic vector env (actions ignored) with episode ends; obs of `dtype`, rewards float32."""

    def __init__(self, N, shape, dtype, act_dim=2, seed=0, period=7):
        from baselines_b200.common import spaces
        rng = np.random.RandomState(seed)
        self.num_envs = N
        self.observation_space = spaces.Box(-np.inf, np.inf, shape, dtype)
        self.action_space = spaces.Box(-1.0, 1.0, (act_dim,), np.float32)
        self.obs = (5.0 + 3.0 * rng.randn(period, N, *shape)).astype(dtype)
        self.rews = (rng.randn(period, N) * 2).astype(np.float32)
        self.news = rng.rand(period, N) < 0.2
        self.t = 0

    def reset(self):
        self.t = 0
        return self.obs[0]

    def step_async(self, actions):
        pass

    def step_wait(self):
        self.t += 1
        k = self.t % len(self.obs)
        infos = [{"episode": {"r": 1.0, "l": self.t, "t": 0.0}} if d else {} for d in self.news[k]]
        return self.obs[k].copy(), self.rews[k], self.news[k], infos

    def close(self):
        pass


def _forwarding(venv):
    """The same VecNormalize hidden under a plain wrapper: no longer outermost, so the Runner takes the host path."""
    from baselines_b200.common.vec_env import VecEnvWrapper

    class Fwd(VecEnvWrapper):
        def reset(self):
            return self.venv.reset()

        def step_wait(self):
            return self.venv.step_wait()
    return Fwd(venv)


def _model(network, env, nsteps, **kw):
    from baselines_b200.common.policies import build_policy
    from baselines_b200.ppo2.model import Model
    np.random.seed(0)
    policy = build_policy(env, network, **kw)
    return Model(policy=policy, ob_space=env.observation_space, ac_space=env.action_space, nbatch_act=env.num_envs,
                 nbatch_train=env.num_envs * nsteps, nsteps=nsteps, ent_coef=0.01, vf_coef=0.5, max_grad_norm=0.5,
                 comm=False)


RUNNER_CASES = {
    "f32": dict(shape=(6,), dtype=np.float32, network="mlp"),
    "f64": dict(shape=(6,), dtype=np.float64, network="mlp"),
    "ob_off": dict(shape=(6,), dtype=np.float32, network="mlp", ob=False),
    "ret_off": dict(shape=(6,), dtype=np.float64, network="mlp", ret=False),
    "d1": dict(shape=(1,), dtype=np.float32, network="mlp"),
    "copy": dict(shape=(6,), dtype=np.float32, network="mlp", value_network="copy"),
    "lstm": dict(shape=(6,), dtype=np.float32, network="lstm", nlstm=64),
}


@pytest.mark.parametrize("name", list(RUNNER_CASES))
def test_runner_device_path_equals_host_path(name):
    from baselines_b200.common.vec_env import VecNormalize
    from baselines_b200.ppo2.runner import Runner
    c = dict(RUNNER_CASES[name])
    shape, dtype, network = c.pop("shape"), c.pop("dtype"), c.pop("network")
    vkw = {k: c.pop(k) for k in ("ob", "ret") if k in c}
    N, T = 16, 5
    rng = np.random.RandomState(1)
    noise = rng.randn(2, T, N, 2).astype(np.float32)
    results, envs = [], []
    for device in (True, False):
        vn = VecNormalize(_Scripted(N, shape, dtype), **vkw)
        env = vn if device else _forwarding(vn)
        model = _model(network, env, T, **c)
        runner = Runner(env=env, model=model, nsteps=T, gamma=0.99, lam=0.95)
        assert runner.vn == device
        res = []
        for k in range(2):
            out = runner.run(noise=noise[k])
            ro = runner.rollout
            res.append([np.copy(a) for a in out[:6]] + [ro.rewards.cpu().numpy(), ro.advs.cpu().numpy(),
                                                        ro.obs.cpu().numpy()])
        results.append(res)
        envs.append(vn)
    for a, b in zip(*results):
        for x, y in zip(a, b):
            assert _same(x, y)
    d, h = envs
    for attr in ("ob_rms", "ret_rms"):
        rd, rh = getattr(d, attr), getattr(h, attr)
        assert (rd is None) == (rh is None)
        if rd is not None:
            assert _same(rd.mean, rh.mean) and _same(rd.var, rh.var) and rd.count == rh.count
    assert _same(d.ret, h.ret)


def test_host_steps_continue_from_the_device_state():
    """After a device rollout, host env.step() calls continue exactly as a run that stayed on the host."""
    from baselines_b200.common.vec_env import VecNormalize
    from baselines_b200.ppo2.runner import Runner
    N, T = 12, 6
    dev = VecNormalize(_Scripted(N, (4,), np.float32))
    host = VecNormalize(_Scripted(N, (4,), np.float32))
    runner = Runner(env=dev, model=_model("mlp", dev, T), nsteps=T, gamma=0.99, lam=0.95)
    assert runner.vn
    runner.run()
    host.reset()
    for _ in range(T):
        host.step(None)
    for _ in range(3):
        od, rd, nd, _ = dev.step(None)
        oh, rh, nh, _ = host.step(None)
        assert _same(od, oh) and _same(rd, rh) and _same(nd, nh)
    # and a rollout after host steps starts from the host-updated state
    dev.ob_rms.mean = dev.ob_rms.mean + 1.0
    host.ob_rms.mean = host.ob_rms.mean + 1.0
    runner.run()
    for _ in range(T):
        host.step(None)
    assert _same(dev.ob_rms.mean, host.ob_rms.mean) and _same(dev.ret_rms.var, host.ret_rms.var)
    assert _same(dev.ret, host.ret)


def test_device_env_under_vec_normalize():
    """VecNormalize(DeviceSyntheticVecEnv) normalises in HBM (no host step) and equals the same batches on the host."""
    from baselines_b200.common.vec_env import DeviceSyntheticVecEnv, VecNormalize
    from baselines_b200.ppo2.runner import Runner
    N, T = 64, 4
    results = []
    for device in (True, False):
        vn = VecNormalize(DeviceSyntheticVecEnv(N, ob_shape=(10,), ob_dtype=np.float32, act_dim=3, pool=3))
        env = vn if device else _forwarding(vn)
        runner = Runner(env=env, model=_model("mlp", env, T), nsteps=T, gamma=0.99, lam=0.95)
        assert runner.vn_dev_env == device
        noise = np.random.RandomState(0).randn(T, N, 3).astype(np.float32)
        out = runner.run(noise=noise)
        results.append([np.copy(a) for a in out[:6]] + [runner.rollout.rewards.cpu().numpy()])
    for x, y in zip(*results):
        assert _same(x, y)


def test_learn_two_updates_same_parameters():
    from baselines_b200.common.vec_env import VecNormalize
    from baselines_b200.ppo2 import ppo2
    params = []
    for device in (True, False):
        vn = VecNormalize(_Scripted(8, (5,), np.float32))
        env = vn if device else _forwarding(vn)
        model = ppo2.learn(network="mlp", env=env, total_timesteps=2 * 8 * 16, seed=0, nsteps=16, nminibatches=2,
                           noptepochs=2, log_interval=100)
        params.append(model.get_params())
    assert params[0].keys() == params[1].keys()
    for k in params[0]:
        assert _same(params[0][k], params[1][k]), k


def test_command_line_mujoco_type_takes_device_path(monkeypatch):
    from baselines_b200 import logger, run
    from baselines_b200.ppo2 import ppo2, runner as runner_mod
    seen = []

    class Recording(runner_mod.Runner):
        def __init__(self, **kw):
            super().__init__(**kw)
            seen.append(self.vn)
    monkeypatch.setattr(ppo2, "Runner", Recording)
    try:
        run.main(["--alg=ppo2", "--env=CartPole-v0", "--env_type=mujoco", "--num_env=8", "--num_timesteps=2e4"])
    finally:
        logger.configure(None)
    assert seen and seen[0] is True
