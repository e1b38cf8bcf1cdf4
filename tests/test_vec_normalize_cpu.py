"""CPU: the order-explicit restatement of VecNormalize (tests/_vec_normalize_refs.py), which the device kernels are
checked against, equals np.mean / np.var and the host VecNormalize bit for bit.  If numpy ever changes its summation
order, this file fails before the GPU tests do."""
import numpy as np
import pytest

from _vec_normalize_refs import RefVecNormalize, batch_moments, pairwise_sum

SHAPES = [(1,), (2,), (5,), (3, 5), (376,)]
NS = [1, 2, 7, 8, 9, 127, 128, 129, 8191, 8192, 8193, 16384, 65536]


def _grid():
    for shape in SHAPES:
        for N in NS:
            if N * int(np.prod(shape)) <= (1 << 24):
                yield shape, N


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("shape,N", list(_grid()))
def test_batch_moments_equal_numpy(shape, N, dtype):
    rng = np.random.RandomState(N % 1000 + len(shape))
    for x in ((1e4 + rng.randn(N, *shape)).astype(dtype), rng.randn(N, *shape).astype(dtype)):
        m, v = batch_moments(x)
        em, ev = np.mean(x, axis=0), np.var(x, axis=0)
        assert m.dtype == em.dtype and v.dtype == ev.dtype
        assert np.array_equal(m, em) and np.array_equal(v, ev)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_pairwise_sum_equals_add_reduce(dtype):
    rng = np.random.RandomState(0)
    for n in list(range(1, 300)) + [8191, 8192, 8193, 16384, 65535, 65536]:
        a = (1e5 + 1e3 * rng.randn(n)).astype(dtype)
        assert pairwise_sum(a) == np.add.reduce(a), n
    z = np.full(20, -0.0, dtype)
    assert not np.signbit(pairwise_sum(z)) and not np.signbit(np.add.reduce(z))


class _Scripted:
    def __init__(self, obs, rews, news):
        from baselines_b200.common import spaces
        self.obs, self.rews, self.news = obs, rews, news
        self.num_envs = obs.shape[1]
        self.observation_space = spaces.Box(-np.inf, np.inf, obs.shape[2:], obs.dtype)
        self.action_space = spaces.Discrete(2)
        self.t = 0

    def reset(self):
        self.t = 0
        return self.obs[0]

    def step_async(self, actions):
        pass

    def step_wait(self):
        self.t += 1
        return self.obs[self.t], self.rews[self.t - 1], self.news[self.t - 1], [{}] * self.num_envs

    def close(self):
        pass


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("shape,N,ob,ret", [((5,), 9, True, True), ((1,), 300, True, True), ((3, 5), 3, True, True),
                                            ((376,), 64, True, True), ((2,), 16, False, True),
                                            ((2,), 16, True, False)])
def test_restatement_equals_host_vec_normalize(shape, N, ob, ret, dtype):
    from baselines_b200.common.vec_env import VecNormalize
    rng = np.random.RandomState(1)
    T = 6
    obs = (3.0 + 2.0 * rng.randn(T + 1, N, *shape)).astype(dtype)
    obs[2, 0] = 40.0                                              # hits the clip bound
    rews = (rng.randn(T, N) * 5).astype(dtype)
    news = rng.rand(T, N) < 0.3
    env = VecNormalize(_Scripted(obs, rews, news), ob=ob, ret=ret)
    ref = RefVecNormalize(shape, N, ob=ob, ret=ret)
    assert np.array_equal(env.reset().astype(np.float32), ref.reset(obs[0]))
    for t in range(T):
        o, r, _, _ = env.step(None)
        ro, rr = ref.step(obs[t + 1], rews[t], news[t])
        assert np.array_equal(np.asarray(o).astype(np.float32), ro), t
        assert np.array_equal(np.asarray(r, dtype=np.float32), rr), t
    if ob:
        assert np.array_equal(env.ob_rms.mean, ref.ob[0]) and np.array_equal(env.ob_rms.var, ref.ob[1])
        assert env.ob_rms.count == ref.ob[2]
    if ret:
        assert env.ret_rms.mean == ref.rt[0] and env.ret_rms.var == ref.rt[1] and env.ret_rms.count == ref.rt[2]
    assert np.array_equal(env.ret, ref.ret)


def test_statistics_stay_assignable_on_the_host():
    """ob_rms / ret_rms / ret are properties now; without a device runner they are plain host objects."""
    from baselines_b200.common.vec_env import VecNormalize
    rng = np.random.RandomState(2)
    obs = rng.randn(3, 4, 2).astype(np.float32)
    env = VecNormalize(_Scripted(obs, np.ones((2, 4), np.float32), np.zeros((2, 4), bool)))
    env.reset()
    env.ob_rms.mean = np.array([1.0, 2.0])
    env.ret = np.full(4, 0.5)
    assert np.array_equal(env.ob_rms.mean, [1.0, 2.0]) and np.array_equal(env.ret, np.full(4, 0.5))
    env.step(None)
    assert np.array_equal(env.ret, 0.5 * 0.99 + 1.0 + np.zeros(4))
