"""`python -m baselines_b200.run --alg=ppo2 --env=CartPole-v0 --num_timesteps=1e5 [--num_env=8] [--network=mlp]
[--save_path=...] [--log_path=...] [--play] [--<learn kwarg>=<python literal> ...]`

Command-line front end with the flags, defaults lookup and control flow of the reference's baselines/run.py:52-247
(train / build_env / get_env_type / get_learn_function(_defaults) / parse_cmdline_kwargs / main).  Algorithms: the
ones this package accelerates (ppo2, deepq, ddpg, her, acer).  Under `torchrun` every rank runs the same command (the reference's
`mpirun -np K python -m baselines.run ...`); only rank 0 logs and saves.
"""
import multiprocessing
import os
import os.path as osp
import sys
from importlib import import_module

import numpy as np

from . import envs as builtin_envs
from . import logger
from .common.cmd_util import common_arg_parser, make_env, make_vec_env, parse_unknown_args
from .common.vec_env import VecEnv, VecFrameStack, VecNormalize


def _init_distributed():
    """torchrun sets RANK / WORLD_SIZE: join the process group so Model's DataParallel finds it (NCCL on GPU)."""
    if int(os.environ.get("WORLD_SIZE", "1")) <= 1:
        return 0
    import torch
    import torch.distributed as dist
    if not dist.is_initialized():
        if torch.cuda.is_available():
            torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
        dist.init_process_group("nccl" if torch.cuda.is_available() else "gloo")
    return dist.get_rank()


def get_env_type(args):
    """run.py:120-147: explicit --env_type wins; an env TYPE given as --env picks one of its ids; otherwise the
    registry (ours, then gym's when importable) is searched; `module:Id` takes the module name."""
    env_id = args.env
    if args.env_type is not None:
        return args.env_type, env_id
    by_type = {}
    for spec in builtin_envs.registry.values():
        by_type.setdefault(spec.env_type, set()).add(spec.id)
    try:
        import gym
        for spec in gym.envs.registry.all():
            by_type.setdefault(spec.entry_point.split(':')[0].split('.')[-1], set()).add(spec.id)
    except Exception:
        pass
    if env_id in by_type:
        return env_id, sorted(by_type[env_id])[0]
    env_type = next((t for t, ids in by_type.items() if env_id in ids), None)
    if ':' in env_id:
        env_type = env_id.split(':', 1)[0]
    assert env_type is not None, 'env_id {} is not recognized in env types {}'.format(env_id, sorted(by_type))
    return env_type, env_id


def get_default_network(env_type):
    return 'cnn' if env_type in {'atari', 'retro'} else 'mlp'


def get_alg_module(alg, submodule=None):
    return import_module('.'.join([__package__, alg, submodule or alg]))


def get_learn_function(alg):
    return get_alg_module(alg).learn


def get_learn_function_defaults(alg, env_type):
    try:
        return getattr(get_alg_module(alg, 'defaults'), env_type)()
    except (ImportError, AttributeError):
        return {}


def parse_cmdline_kwargs(args):
    """run.py:178-191: leftover `--k=v` pairs, values evaluated as python when possible (`--lr=3e-4`,
    `--lr='lambda f: 3e-4*f'`)."""
    def parse(v):
        assert isinstance(v, str)
        try:
            return eval(v)
        except (NameError, SyntaxError):
            return v
    return {k: parse(v) for k, v in parse_unknown_args(args).items()}


def build_env(args):
    """run.py:87-117: atari-type envs -> num_env (default: #cpus) copies + VecFrameStack(4) (deepq: one env with
    the stack built in); everything else -> num_env (default 1) copies, mujoco additionally VecNormalize."""
    ncpu = multiprocessing.cpu_count()
    nenv = args.num_env or ncpu
    env_type, env_id = get_env_type(args)
    if env_type in {'atari', 'retro'}:
        if args.alg == 'deepq':
            venv = make_vec_env(env_id, env_type, 1, args.seed, reward_scale=args.reward_scale, force_dummy=True)
            return _SingleEnv(VecFrameStack(venv, 4))
        venv = make_vec_env(env_id, env_type, nenv, args.seed, gamestate=args.gamestate, reward_scale=args.reward_scale)
        return VecFrameStack(venv, 4)
    if args.alg == 'deepq':
        return make_env(env_id, env_type, seed=args.seed, reward_scale=args.reward_scale, logger_dir=logger.get_dir())
    flatten_dict_observations = args.alg not in {'her'}
    venv = make_vec_env(env_id, env_type, args.num_env or 1, args.seed, reward_scale=args.reward_scale,
                        flatten_dict_observations=flatten_dict_observations)
    if env_type == 'mujoco':
        venv = VecNormalize(venv)
    return venv


class _SingleEnv:
    """A one-env VecEnv seen as a plain env (deepq.learn steps a single env, deepq.py:243-262)."""

    def __init__(self, venv):
        assert venv.num_envs == 1
        self.venv = venv
        self.observation_space, self.action_space = venv.observation_space, venv.action_space

    def reset(self):
        return self.venv.reset()[0]

    def step(self, action):
        ob, rew, done, infos = self.venv.step(np.asarray([action]))
        return ob[0], float(rew[0]), bool(done[0]), infos[0]

    def close(self):
        self.venv.close()


def train(args, extra_args):
    env_type, env_id = get_env_type(args)
    print('env_type: {}'.format(env_type))
    assert args.save_video_interval == 0, "video recording is not supported"
    learn = get_learn_function(args.alg)
    alg_kwargs = get_learn_function_defaults(args.alg, env_type)
    alg_kwargs.update(extra_args)
    env = build_env(args)
    if args.network:
        alg_kwargs['network'] = args.network
    elif alg_kwargs.get('network') is None:
        alg_kwargs['network'] = get_default_network(env_type)
    print('Training {} on {}:{} with arguments \n{}'.format(args.alg, env_type, env_id, alg_kwargs))
    model = learn(env=env, seed=args.seed, total_timesteps=int(args.num_timesteps), **alg_kwargs)
    return model, env


def configure_logger(log_path, **kwargs):
    if log_path is not None:
        logger.configure(log_path, **kwargs)
    else:
        logger.configure(**kwargs)


def main(args):
    args, unknown_args = common_arg_parser().parse_known_args(args)
    extra_args = parse_cmdline_kwargs(unknown_args)
    rank = _init_distributed()
    if rank == 0:
        configure_logger(args.log_path)
    else:
        configure_logger(args.log_path, format_strs=[], quiet=True)
    model, env = train(args, extra_args)
    if args.save_path is not None and rank == 0:
        model.save(osp.expanduser(args.save_path))
    if args.play:
        logger.log("Running trained model")
        obs = env.reset()
        is_vec = isinstance(env, VecEnv)
        episode_rew = np.zeros(env.num_envs) if is_vec else np.zeros(1)
        while True:
            actions = model.step(obs)[0] if hasattr(model, "step") else model(obs)[0]
            obs, rew, done, _ = env.step(actions)
            episode_rew += rew
            if hasattr(env, "render"):
                env.render()
            for i in np.nonzero(np.atleast_1d(done))[0]:
                print('episode_rew={}'.format(episode_rew[i]))
                episode_rew[i] = 0
            if not is_vec and done:
                obs = env.reset()
    env.close()
    return model


if __name__ == '__main__':
    main(sys.argv)
