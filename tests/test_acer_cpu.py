"""ACER host logic and the float64 mirror, without a GPU: the mirror against definition-level loops and central
differences, the re-stacking rule against VecFrameStack's own stacks, the schedules, the policy's variables and numpy
draws, dispatch and the refusals."""
import numpy as np
import pytest

import _acer_refs as AR
from baselines_b200.acer import acer as A
from baselines_b200.common import spaces
from baselines_b200.common.vec_env import VecEnv, VecFrameStack


def _head_inputs(rng, nenv, nsteps, nA, p_done=0.2):
    R = nenv * (nsteps + 1)
    pi, q, pol = rng.randn(R, nA), rng.randn(R, nA), rng.randn(R, nA)
    actions = rng.randint(0, nA, nenv * nsteps)
    rewards = rng.randn(nenv * nsteps)
    dones = rng.rand(nenv * nsteps) < p_done
    mus = AR.softmax(rng.randn(nenv * nsteps, nA))
    return pi, q, pol, actions, rewards, dones, mus


def test_retrace_against_a_definition_level_loop():
    rng = np.random.RandomState(0)
    nenv, T = 3, 6
    R, D, qi, rho = rng.randn(nenv, T), rng.rand(nenv, T) < 0.3, rng.randn(nenv, T), rng.rand(nenv, T) * 2
    v = rng.randn(nenv, T + 1)
    out = AR.retrace(R, D, qi, v, rho, nenv, T, 0.9)
    for e in range(nenv):
        for t in range(T):
            # Q_ret(t) = r_t + gamma (1 - d_t) [rho_bar_{t+1} (Q_ret(t+1) - q_{t+1}) + v_{t+1}], with Q_ret(T) = v_T
            nxt = v[e, T] if t == T - 1 else min(1.0, rho[e, t + 1]) * (out[e, t + 1] - qi[e, t + 1]) + v[e, t + 1]
            assert out[e, t] == pytest.approx(R[e, t] + 0.9 * (1 - D[e, t]) * nxt, abs=1e-12)


@pytest.mark.parametrize("nA", [2, 6])
def test_head_gradient_against_central_differences(nA):
    """Without the trust region dpi / dq are N * d loss / d (logits, q) with the reference's stop-gradients."""
    rng = np.random.RandomState(nA)
    nenv, T = 2, 4
    pi, q, pol, a, r, d, mus = _head_inputs(rng, nenv, T, nA)
    base = AR.head(pi, q, pol, a, r, d, mus, nenv, T, trust_region=False)
    N = nenv * T
    F0 = AR.softmax(pi).reshape(nenv, T + 1, nA)[:, :T]
    V0 = base.v.reshape(nenv, T + 1)[:, :T]
    qret = base.qret.reshape(nenv, T)
    rho0 = F0 / (mus.reshape(nenv, T, nA) + AR.EPS)
    A_ = a.reshape(nenv, T)
    rho_i0 = np.take_along_axis(rho0, A_[..., None], -1)[..., 0]
    Af = (qret - V0) * np.minimum(10.0, rho_i0)
    Bm = (q.reshape(nenv, T + 1, nA)[:, :T] - V0[..., None]) * np.maximum(0, 1 - 10.0 / (rho0 + AR.EPS)) * F0

    def loss(pi_, q_):                       # the stopped terms are constants at the base point
        f = AR.softmax(pi_).reshape(nenv, T + 1, nA)[:, :T]
        qi = np.take_along_axis(q_.reshape(nenv, T + 1, nA)[:, :T], A_[..., None], -1)[..., 0]
        fi = np.take_along_axis(f, A_[..., None], -1)[..., 0]
        lf = -np.mean(np.log(fi + AR.EPS) * Af)
        lbc = -np.mean((np.log(f + AR.EPS) * Bm).sum(-1))
        ent = np.mean(-(f * np.log(f + 1e-6)).sum(-1))
        return lf + lbc + 0.5 * np.mean(0.5 * (qret - qi) ** 2) - 0.01 * ent
    h = 1e-6
    for X, dX in ((pi, base.dpi), (q, base.dq)):
        num = np.zeros_like(X)
        for idx in np.ndindex(*X.shape):
            Xp, Xm = X.copy(), X.copy()
            Xp[idx] += h
            Xm[idx] -= h
            args_p = (Xp, q) if X is pi else (pi, Xp)
            args_m = (Xm, q) if X is pi else (pi, Xm)
            num[idx] = (loss(*args_p) - loss(*args_m)) / (2 * h)
        np.testing.assert_allclose(dX / N, num, atol=1e-7, rtol=1e-5)
    assert np.isclose(base.stats[0], loss(pi, q))


def test_trust_region_projection_is_the_kl_constrained_step():
    """adj makes k . g' <= delta where the constraint is active, and leaves g alone where it is not."""
    rng = np.random.RandomState(1)
    nenv, T, nA = 4, 5, 6
    pi, q, pol, a, r, d, mus = _head_inputs(rng, nenv, T, nA)
    q *= 50
    h = AR.head(pi, q, pol, a, r, d, mus, nenv, T, delta=0.1)
    assert (h.adj > 0).any() and (h.adj == 0).any()
    ht = AR.head(pi, q, pol, a, r, d, mus, nenv, T, trust_region=False)
    assert np.abs(h.dpi - ht.dpi).max() > 0
    np.testing.assert_allclose(h.dq, ht.dq)


def test_rmsprop_ema_definition():
    rng = np.random.RandomState(2)
    p, g, ms, sh = rng.randn(10), rng.randn(10), np.ones(10), rng.randn(10)
    p1, ms1, sh1 = AR.rmsprop_ema(p, g, ms, sh, 0.1, 0.0)
    m = 1 + (g * g - 1) * 0.01
    np.testing.assert_allclose(ms1, m)
    np.testing.assert_allclose(p1, p - 0.1 * g / np.sqrt(m + 1e-5))
    np.testing.assert_allclose(sh1, sh - (sh - p1) * 0.01)


class _Frames(VecEnv):
    """Scripted frames and dones for VecFrameStack."""

    def __init__(self, nenv, frame, nc, dtype, dones, seed):
        super().__init__(nenv, spaces.Box(0, 255, frame + (nc,), dtype), spaces.Discrete(3))
        self.rng = np.random.RandomState(seed)
        self.dones, self.t, self.frame, self.nc, self.dtype = dones, 0, frame, nc, dtype

    def _obs(self):
        x = self.rng.randint(1, 256, (self.num_envs,) + self.frame + (self.nc,))
        return x.astype(self.dtype) if self.dtype == np.uint8 else (x - 128.5).astype(self.dtype)

    def reset(self):
        return self._obs()

    def step_async(self, actions):
        pass

    def step_wait(self):
        d = self.dones[self.t]
        self.t += 1
        return self._obs(), np.zeros(self.num_envs, np.float32), d, [{} for _ in range(self.num_envs)]


@pytest.mark.parametrize("nstack,nc,dtype", [(4, 1, np.uint8), (1, 3, np.uint8), (4, 1, np.float32), (2, 1, np.float32),
                                              (1, 4, np.float32), (4, 2, np.uint8), (2, 3, np.float32)])
def test_restacked_segment_against_the_frame_stacks_the_runner_saw(nstack, nc, dtype):
    """The on-policy batch is mb_obs (runner.py:32,43).  With one channel per frame, or no stacking, re-stacking the
    segment's single frames with the shifted dones gives the same values, with dones at the first and last steps and a
    done in the segment before.  With several channels per frame VecFrameStack rolls the stack by one CHANNEL per step
    (vec_frame_stack.py:19), so its stacks are not _stack_obs's: the runner then trains from the stacks themselves."""
    nenv, T, frame = 3, 7, (2, 3)
    rng = np.random.RandomState(nstack)
    dones = rng.rand(2 * T, nenv) < 0.3
    dones[T, 0] = dones[2 * T - 1, 1] = True
    venv = VecFrameStack(_Frames(nenv, frame, nc, dtype, dones, 5), nstack)
    obs = venv.reset()
    for _ in range(T):                          # one segment first, so the start stack already holds cleared frames
        obs, _, _, _ = venv.step(np.zeros(nenv, np.int64))
    enc = list(np.split(venv.stackedobs, nstack, axis=-1))
    mb_obs, mb_dones = [obs.copy()], []
    for _ in range(T):
        obs, _, d, _ = venv.step(np.zeros(nenv, np.int64))
        mb_obs.append(obs.copy())
        mb_dones.append(d)
        enc.append(obs[..., -nc:])
    enc = np.asarray(enc, dtype).swapaxes(1, 0)
    mb_obs = np.asarray(mb_obs, dtype).swapaxes(1, 0)
    mb_dones = np.asarray(mb_dones, bool).swapaxes(1, 0)
    got = AR.stack_obs(enc, mb_dones, T)
    assert got.dtype == mb_obs.dtype and got.shape == mb_obs.shape
    if nc == 1 or nstack == 1:
        np.testing.assert_array_equal(got, mb_obs)
    else:
        assert not np.array_equal(got, mb_obs)


def test_scheduler_schedules():
    s = A.Scheduler(v=7e-4, nvalues=1000, schedule='linear')
    assert s.value_steps(0) == 7e-4 and s.value_steps(250) == 7e-4 * 0.75
    assert A.Scheduler(7e-4, 1000, 'constant').value_steps(999) == 7e-4
    assert A.Scheduler(1.0, 100, 'middle_drop').value_steps(30) == 0.75 * 0.1
    assert A.Scheduler(1.0, 100, 'double_linear_con').value_steps(46) == 0.125
    assert A.Scheduler(1.0, 100, 'double_middle_drop').value_steps(80) == 0.125
    s = A.Scheduler(1.0, 4, 'linear')
    assert [s.value() for _ in range(3)] == [1.0, 0.75, 0.5]


def test_episode_stats():
    es = A.EpisodeStats(3, 2)
    es.feed(np.array([[1, 2, 3], [4, 5, 6]], np.float32), np.array([[0, 1, 0], [0, 0, 0]], bool))
    es.feed(np.array([[1, 1, 1], [1, 1, 1]], np.float32), np.array([[0, 0, 1], [1, 0, 0]], bool))
    assert list(es.lenbuffer) == [2, 4, 4] and list(es.rewbuffer) == [3.0, 6.0, 16.0]
    assert es.mean_length() == pytest.approx(10 / 3)


def test_dispatch_and_defaults():
    from baselines_b200 import run
    assert run.get_learn_function('acer') is A.learn
    assert run.get_learn_function_defaults('acer', 'atari') == dict(lrschedule='constant')
    assert run.get_learn_function_defaults('acer', 'classic_control') == {}
    import inspect
    sig = inspect.signature(A.learn)
    want = dict(nsteps=20, q_coef=0.5, ent_coef=0.01, max_grad_norm=10, lr=7e-4, lrschedule='linear',
                rprop_epsilon=1e-5, rprop_alpha=0.99, gamma=0.99, log_interval=100, buffer_size=50000,
                replay_ratio=4, replay_start=10000, c=10.0, trust_region=True, alpha=0.99, delta=1, load_path=None)
    for k, v in want.items():
        assert sig.parameters[k].default == v, k


class _E:
    def __init__(self, ob, ac, n=2):
        self.observation_space, self.action_space, self.num_envs = ob, ac, n


def test_refusals():
    from baselines_b200.common.policies import build_policy
    box = spaces.Box(-1, 1, (4,), np.float32)
    with pytest.raises(NotImplementedError):
        build_policy(_E(box, spaces.Box(-1, 1, (2,), np.float32)), 'mlp', estimate_q=True)
    for net in ('lstm', 'cnn_lstm'):
        with pytest.raises(NotImplementedError):
            A.check_supported(build_policy(_E(spaces.Box(0, 255, (84, 84, 4), np.uint8), spaces.Discrete(3)), net,
                                           estimate_q=True))
    with pytest.raises(NotImplementedError):
        A.check_supported(build_policy(_E(spaces.Discrete(5), spaces.Discrete(3)), 'mlp', estimate_q=True))


def test_learn_refuses_mpi(monkeypatch):
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(NotImplementedError):
        A.learn('mlp', None)
