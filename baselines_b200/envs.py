"""Gym-free environments and a tiny id registry for the command line (`python -m baselines_b200.run --env=...`).

`gym` is a third-party dependency of the reference (run.py:5, cmd_util.py:11) and is not installed here; when it IS
importable, cmd_util.make_env uses `gym.make` for ids that are not registered below.  The built-in ids cover the
reference's plumbing tests and the benchmark workload:

  DiscreteIdentity-v0 / BoxIdentity-v0   common/tests/envs/identity_env.py:7-90 (test_identity.py)
  MultiDiscreteIdentity-v0               identity_env.py:62-74 with dims (3, 3) (test_identity.py:43-56)
  CartPole-v0 / CartPole-v1              classic cart-pole of common/tests/test_cartpole.py:14 (gym's dynamics: Barto,
                                         Sutton & Anderson 1983, Euler step, tau = 0.02)
  SyntheticAtari-v0                      84x84x1 uint8 frames, 6 actions: the bench.py workload as a steppable env
"""
import math
from collections import deque

import numpy as np

from .common import spaces


class EnvSpec:
    def __init__(self, id, entry_point, env_type, max_episode_steps=None, kwargs=None):
        self.id, self.entry_point, self.env_type = id, entry_point, env_type
        self.max_episode_steps, self.kwargs = max_episode_steps, dict(kwargs or {})


registry = {}


def register(id, entry_point, env_type, max_episode_steps=None, **kwargs):
    registry[id] = EnvSpec(id, entry_point, env_type, max_episode_steps, kwargs)


def make(id, **kwargs):
    spec = registry[id]
    kw = dict(spec.kwargs)
    kw.update(kwargs)
    env = spec.entry_point(**kw)
    env.spec = spec
    if spec.max_episode_steps is not None:
        env = TimeLimit(env, spec.max_episode_steps)
    return env


class Env:
    """The subset of gym.Env the host pipeline relies on."""
    spec = None
    observation_space = action_space = None

    def reset(self):
        raise NotImplementedError

    def step(self, action):
        raise NotImplementedError

    def seed(self, seed=None):
        self.np_random = np.random.RandomState(seed)
        return [seed]

    def render(self, mode="human"):
        return None

    def close(self):
        pass


class TimeLimit(Env):
    """Episode cap (gym.wrappers.TimeLimit): done after max_episode_steps, flagged in info['TimeLimit.truncated']."""

    def __init__(self, env, max_episode_steps):
        self.env, self.max_episode_steps = env, max_episode_steps
        self.observation_space, self.action_space, self.spec = env.observation_space, env.action_space, env.spec
        self._t = 0

    def reset(self):
        self._t = 0
        return self.env.reset()

    def step(self, action):
        ob, rew, done, info = self.env.step(action)
        self._t += 1
        if self._t >= self.max_episode_steps and not done:
            info = dict(info)
            info["TimeLimit.truncated"] = True
            done = True
        return ob, rew, done, info

    def seed(self, seed=None):
        return self.env.seed(seed)

    def render(self, mode="human"):
        return self.env.render(mode)

    def close(self):
        self.env.close()


# ------------------------------------------------------------------------------------------------ identity envs
class IdentityEnv(Env):
    """identity_env.py:7-46: the observation is a sample of the action space; reward for repeating it back
    (after `delay` steps)."""

    def __init__(self, episode_len=None, delay=0, zero_first_rewards=True):
        self.observation_space = self.action_space
        self.episode_len, self.delay, self.zero_first_rewards = episode_len, delay, zero_first_rewards
        self.time = 0
        self.q = deque(maxlen=delay + 1)

    def reset(self):
        self.q.clear()
        for _ in range(self.delay + 1):
            self.q.append(self.action_space.sample())
        self.time = 0
        return self.q[-1]

    def step(self, actions):
        rew = self._get_reward(self.q.popleft(), actions)
        if self.zero_first_rewards and self.time < self.delay:
            rew = 0
        self.q.append(self.action_space.sample())
        self.time += 1
        done = self.episode_len is not None and self.time >= self.episode_len
        return self.q[-1], rew, done, {}

    def seed(self, seed=None):
        self.action_space.seed(seed)
        return [seed]


class FixedSequenceEnv(Env):
    """A memory task (common/tests/envs/fixed_sequence_env.py): the observation is always 0 (Discrete(1)); at step t
    of an episode the action that earns reward 1 is the t-th entry of one sequence of `episode_len` actions, drawn once
    when the env is built from a RandomState seeded 0.  Only a policy that counts steps (a recurrent one) can follow it.
    The episode ends after `episode_len` steps; seed() reseeds the env's generator but keeps the sequence."""

    def __init__(self, n_actions=10, episode_len=100):
        self.action_space = spaces.Discrete(n_actions)
        self.observation_space = spaces.Discrete(1)
        self.np_random = np.random.RandomState(0)
        self.episode_len = episode_len
        self.sequence = [int(self.np_random.randint(0, n_actions)) for _ in range(episode_len)]
        self.time = 0

    def reset(self):
        self.time = 0
        return 0

    def step(self, actions):
        rew = 1 if actions == self.sequence[self.time] else 0
        self.time += 1
        done = bool(self.episode_len) and self.time >= self.episode_len
        return 0, rew, done, {}

    def seed(self, seed=None):
        self.np_random.seed(seed)
        return [seed]


class DiscreteIdentityEnv(IdentityEnv):
    def __init__(self, dim, episode_len=None, delay=0, zero_first_rewards=True):
        self.action_space = spaces.Discrete(dim)
        super().__init__(episode_len=episode_len, delay=delay, zero_first_rewards=zero_first_rewards)

    def _get_reward(self, state, actions):
        return 1 if state == actions else 0


class MultiDiscreteIdentityEnv(IdentityEnv):
    """identity_env.py:62-74: observation and action are MultiDiscrete(dims); reward 1 iff every component matches."""

    def __init__(self, dims, episode_len=None, delay=0):
        self.action_space = spaces.MultiDiscrete(dims)
        super().__init__(episode_len=episode_len, delay=delay)

    def _get_reward(self, state, actions):
        return 1 if np.all(np.asarray(state) == np.asarray(actions)) else 0


class BoxIdentityEnv(IdentityEnv):
    def __init__(self, shape, episode_len=None):
        self.action_space = spaces.Box(low=-1.0, high=1.0, shape=shape, dtype=np.float32)
        super().__init__(episode_len=episode_len)

    def _get_reward(self, state, actions):
        diff = np.asarray(actions, dtype=np.float64).reshape(-1) - np.asarray(state, dtype=np.float64).reshape(-1)
        return -0.5 * float(np.dot(diff, diff))


# ------------------------------------------------------------------------------------------------ cart-pole
class CartPoleEnv(Env):
    """Pole balancing (Barto, Sutton & Anderson 1983) with gym's constants: force +-10 N, tau 0.02 s explicit Euler,
    failure at |x| > 2.4 or |theta| > 12 deg, reward 1 per step, start state U(-0.05, 0.05)^4."""
    gravity, masscart, masspole, length, force_mag, tau = 9.8, 1.0, 0.1, 0.5, 10.0, 0.02
    theta_threshold = 12 * 2 * math.pi / 360
    x_threshold = 2.4

    def __init__(self):
        high = np.array([self.x_threshold * 2, np.finfo(np.float32).max, self.theta_threshold * 2,
                         np.finfo(np.float32).max], dtype=np.float32)
        self.observation_space = spaces.Box(-high, high, dtype=np.float32)
        self.action_space = spaces.Discrete(2)
        self.seed()
        self.state = None

    def reset(self):
        self.state = self.np_random.uniform(-0.05, 0.05, size=(4,))
        return np.array(self.state, dtype=np.float32)

    def step(self, action):
        x, x_dot, th, th_dot = self.state
        force = self.force_mag if int(action) == 1 else -self.force_mag
        total_mass = self.masspole + self.masscart
        pml = self.masspole * self.length
        cos, sin = math.cos(th), math.sin(th)
        temp = (force + pml * th_dot ** 2 * sin) / total_mass
        th_acc = (self.gravity * sin - cos * temp) / (self.length * (4.0 / 3.0 - self.masspole * cos ** 2 / total_mass))
        x_acc = temp - pml * th_acc * cos / total_mass
        x, x_dot = x + self.tau * x_dot, x_dot + self.tau * x_acc
        th, th_dot = th + self.tau * th_dot, th_dot + self.tau * th_acc
        self.state = (x, x_dot, th, th_dot)
        done = bool(x < -self.x_threshold or x > self.x_threshold or th < -self.theta_threshold or
                    th > self.theta_threshold)
        return np.array(self.state, dtype=np.float32), 1.0, done, {}


# ------------------------------------------------------------------------------------------------ synthetic frames
class SyntheticAtariEnv(Env):
    """One 84x84x1 uint8 frame per step from a small pre-drawn pool (the cost of a real emulator is NOT modelled),
    N(0,1) rewards, Bernoulli(p_done) episode ends: the bench.py workload as a single steppable env."""

    def __init__(self, n_actions=6, pool=16, p_done=0.01):
        self.observation_space = spaces.Box(0, 255, (84, 84, 1), np.uint8)
        self.action_space = spaces.Discrete(n_actions)
        self.pool_size, self.p_done = pool, p_done
        self.seed(0)

    def seed(self, seed=None):
        out = super().seed(seed)
        self.frames = self.np_random.randint(0, 256, size=(self.pool_size, 84, 84, 1)).astype(np.uint8)
        self.t = 0
        return out

    def reset(self):
        self.t += 1
        return self.frames[self.t % self.pool_size]

    def step(self, action):
        self.t += 1
        return (self.frames[self.t % self.pool_size], float(self.np_random.randn()),
                bool(self.np_random.rand() < self.p_done), {})


register("DiscreteIdentity-v0", DiscreteIdentityEnv, "identity", dim=10, episode_len=100)
register("MultiDiscreteIdentity-v0", MultiDiscreteIdentityEnv, "identity", dims=(3, 3), episode_len=100)
register("BoxIdentity-v0", BoxIdentityEnv, "identity", shape=(1,), episode_len=100)
register("CartPole-v0", CartPoleEnv, "classic_control", max_episode_steps=200)
register("CartPole-v1", CartPoleEnv, "classic_control", max_episode_steps=500)
register("SyntheticAtari-v0", SyntheticAtariEnv, "atari")
