"""Environment construction and argument parsing for the command line -- the call surface of the reference's
baselines/common/cmd_util.py:22-210 (`make_vec_env`, `make_env`, `common_arg_parser`, `parse_unknown_args`).

Ids registered in baselines_b200.envs are built without gym; any other id goes to `gym.make` when gym is importable
(atari ids additionally need the reference's atari wrappers, which are out of scope here: see DESIGN.md 7)."""
import argparse
import os

import numpy as np

from .. import logger
from ..bench import Monitor
from .misc_util import set_global_seeds
from . import spaces
from .vec_env import DummyVecEnv, SubprocVecEnv


def _rank():
    try:
        import torch.distributed as dist
        return dist.get_rank() if dist.is_available() and dist.is_initialized() else int(os.environ.get("RANK", 0))
    except Exception:
        return 0


class ClipActionsWrapper:
    """common/wrappers.py:22-29: clip continuous actions to the action-space bounds before stepping."""

    def __init__(self, env):
        self.env = env
        self.observation_space, self.action_space = env.observation_space, env.action_space

    def __getattr__(self, name):
        if name.startswith('_'):
            raise AttributeError(name)
        return getattr(self.env, name)

    def step(self, action):
        import numpy as np
        action = np.nan_to_num(action)
        return self.env.step(np.clip(action, self.action_space.low, self.action_space.high))

    def reset(self, **kwargs):
        return self.env.reset(**kwargs)


class FlattenObservation:
    """gym.wrappers.FlattenObservation: a Dict observation as the concatenation of its parts in key order."""

    def __init__(self, env):
        self.env = env
        parts = env.observation_space.spaces
        n = sum(int(np.prod(s.shape)) for s in parts.values())
        self.observation_space = spaces.Box(-np.inf, np.inf, (n,), np.float32)
        self.action_space = env.action_space

    def __getattr__(self, name):
        if name.startswith('_'):
            raise AttributeError(name)
        return getattr(self.env, name)

    def _flat(self, ob):
        return np.concatenate([np.asarray(ob[k], np.float32).ravel() for k in self.env.observation_space.spaces])

    def step(self, action):
        ob, rew, done, info = self.env.step(action)
        return self._flat(ob), rew, done, info

    def reset(self, **kwargs):
        return self._flat(self.env.reset(**kwargs))


class RewardScaler:
    """retro_wrappers.py:147-157: multiply rewards by a constant (PPO is sensitive to reward scale)."""

    def __init__(self, env, scale=0.01):
        self.env, self.scale = env, scale
        self.observation_space, self.action_space = env.observation_space, env.action_space

    def __getattr__(self, name):
        if name.startswith('_'):
            raise AttributeError(name)
        return getattr(self.env, name)

    def step(self, action):
        ob, rew, done, info = self.env.step(action)
        return ob, rew * self.scale, done, info

    def reset(self, **kwargs):
        return self.env.reset(**kwargs)


def make_env(env_id, env_type, mpi_rank=0, subrank=0, seed=None, reward_scale=1.0, gamestate=None,
             flatten_dict_observations=True, wrapper_kwargs=None, env_kwargs=None, logger_dir=None, initializer=None):
    """cmd_util.py:64-111: one seeded, monitored env."""
    from .. import envs as builtin
    if initializer is not None:
        initializer(mpi_rank=mpi_rank, subrank=subrank)
    env_kwargs = env_kwargs or {}
    if ':' in env_id:                                        # "module:EnvId" imports the module first
        import importlib
        module_name, env_id = env_id.split(':', 1)
        importlib.import_module(module_name)
    if env_id in builtin.registry:
        env = builtin.make(env_id, **env_kwargs)
    else:
        try:
            import gym
        except ImportError as e:
            raise RuntimeError(f"env id {env_id!r} is not built in ({sorted(builtin.registry)}) and gym is not "
                               f"installed") from e
        if env_type in ('atari', 'retro'):
            raise NotImplementedError("gym atari / retro ids need the reference's emulator wrappers (out of scope)")
        env = gym.make(env_id, **env_kwargs)
    env.seed(seed + subrank if seed is not None else None)
    if flatten_dict_observations and spaces.is_dict(env.observation_space):
        env = FlattenObservation(env)
    env = Monitor(env, logger_dir and os.path.join(logger_dir, str(mpi_rank) + '.' + str(subrank)),
                  allow_early_resets=True)
    if hasattr(env.action_space, "low") and hasattr(env.action_space, "high"):
        env = ClipActionsWrapper(env)
    if reward_scale != 1:
        env = RewardScaler(env, reward_scale)
    return env


def make_vec_env(env_id, env_type, num_env, seed, wrapper_kwargs=None, env_kwargs=None, start_index=0,
                 reward_scale=1.0, flatten_dict_observations=True, gamestate=None, initializer=None,
                 force_dummy=False):
    """cmd_util.py:22-61: `num_env` monitored copies; worker processes when num_env > 1.  Seeds are
    seed + 10000 * rank + subrank (cmd_util.py:37, SURVEY 8e)."""
    rank = _rank()
    seed = seed + 10000 * rank if seed is not None else None
    logger_dir = logger.get_dir()

    def make_thunk(subrank, initializer=None):
        return lambda: make_env(env_id=env_id, env_type=env_type, mpi_rank=rank, subrank=subrank, seed=seed,
                                reward_scale=reward_scale, gamestate=gamestate,
                                flatten_dict_observations=flatten_dict_observations, wrapper_kwargs=wrapper_kwargs,
                                env_kwargs=env_kwargs, logger_dir=logger_dir, initializer=initializer)

    set_global_seeds(seed)
    if not force_dummy and num_env > 1:
        return SubprocVecEnv([make_thunk(i + start_index, initializer=initializer) for i in range(num_env)])
    return DummyVecEnv([make_thunk(i + start_index) for i in range(num_env)])


def arg_parser():
    return argparse.ArgumentParser(formatter_class=argparse.ArgumentDefaultsHelpFormatter)


def common_arg_parser():
    """cmd_util.py:156-178: the flags of `python -m baselines.run`."""
    parser = arg_parser()
    parser.add_argument('--env', help='environment ID', type=str, default='CartPole-v0')
    parser.add_argument('--env_type', help='type of environment, used when the environment type cannot be '
                                           'automatically determined', type=str)
    parser.add_argument('--seed', help='RNG seed', type=int, default=None)
    parser.add_argument('--alg', help='Algorithm', type=str, default='ppo2')
    parser.add_argument('--num_timesteps', type=float, default=1e6)
    parser.add_argument('--network', help='network type (mlp, cnn, conv_only)', default=None)
    parser.add_argument('--gamestate', help='game state to load (retro only; unused)', default=None)
    parser.add_argument('--num_env', help='Number of environment copies being run in parallel. When not specified, '
                                          'set to number of cpus for Atari, and to 1 otherwise', default=None, type=int)
    parser.add_argument('--reward_scale', help='Reward scale factor. Default: 1.0', default=1.0, type=float)
    parser.add_argument('--save_path', help='Path to save trained model to', default=None, type=str)
    parser.add_argument('--save_video_interval', help='(unsupported; must be 0)', default=0, type=int)
    parser.add_argument('--save_video_length', help='(unsupported)', default=200, type=int)
    parser.add_argument('--log_path', help='Directory to save learning curve data.', default=None, type=str)
    parser.add_argument('--play', default=False, action='store_true')
    return parser


def parse_unknown_args(args):
    """cmd_util.py:191-210: `--key=value` / `--key value` leftovers -> dict of strings."""
    retval, key, pending = {}, None, False
    for arg in args:
        if arg.startswith('--'):
            if '=' in arg:
                k, v = arg[2:].split('=', 1)
                retval[k] = v
                pending = False
            else:
                key, pending = arg[2:], True
        elif pending:
            retval[key] = arg
            pending = False
    return retval
