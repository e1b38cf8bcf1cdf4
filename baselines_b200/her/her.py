"""her.learn (baselines/her/her.py): the same epochs / cycles / batches, params.json, logger keys and policy pickles,
with the agent of her/ddpg.py on the device.

Out of scope: MPI (one process: the reference's averages over one rank are identities) and demonstrations
(demo_file, the bc_loss / q_filter path)."""
import os
import json

import numpy as np

from .. import logger
from ..common.misc_util import set_global_seeds
from .experiment import config
from .rollout import RolloutWorker


def mpi_average(value):
    if not isinstance(value, list):
        value = [value]
    if not any(value):
        value = [0.]
    return np.mean(np.array(value, dtype=np.float64), axis=0)


def train(*, policy, rollout_worker, evaluator, n_epochs, n_test_rollouts, n_cycles, n_batches, policy_save_interval,
          save_path, demo_file, **kwargs):
    if save_path:
        latest_policy_path = os.path.join(save_path, 'policy_latest.pkl')
        best_policy_path = os.path.join(save_path, 'policy_best.pkl')
        periodic_policy_path = os.path.join(save_path, 'policy_{}.pkl')
        os.makedirs(save_path, exist_ok=True)

    logger.info("Training...")
    best_success_rate = -1
    for epoch in range(n_epochs):
        rollout_worker.clear_history()
        for _ in range(n_cycles):
            episode = rollout_worker.generate_rollouts()
            policy.store_episode(episode)
            for _ in range(n_batches):
                policy.train_device()
            policy.update_target_net()

        evaluator.clear_history()
        for _ in range(n_test_rollouts):
            evaluator.generate_rollouts()

        logger.record_tabular('epoch', epoch)
        for key, val in evaluator.logs('test'):
            logger.record_tabular(key, mpi_average(val))
        for key, val in rollout_worker.logs('train'):
            logger.record_tabular(key, mpi_average(val))
        for key, val in policy.logs():
            logger.record_tabular(key, mpi_average(val))
        logger.dump_tabular()

        success_rate = mpi_average(evaluator.current_success_rate())
        if success_rate >= best_success_rate and save_path:
            best_success_rate = success_rate
            logger.info('New best success rate: {}. Saving policy to {} ...'.format(best_success_rate,
                                                                                  best_policy_path))
            evaluator.save_policy(best_policy_path)
            evaluator.save_policy(latest_policy_path)
        if policy_save_interval > 0 and epoch % policy_save_interval == 0 and save_path:
            policy_path = periodic_policy_path.format(epoch)
            logger.info('Saving periodic policy to {} ...'.format(policy_path))
            evaluator.save_policy(policy_path)

        # the reference draws one uniform per epoch to check that ranks differ (her.py:83-88)
        np.random.uniform(size=(1,))
    return policy


def learn(*, network, env, total_timesteps, seed=None, eval_env=None, replay_strategy='future',
          policy_save_interval=5, clip_return=True, demo_file=None, override_params=None, load_path=None,
          save_path=None, **kwargs):
    if demo_file is not None:
        raise NotImplementedError("her demonstrations (demo_file: the bc_loss / q_filter path) are not supported")
    if replay_strategy not in ('future', 'none'):
        raise NotImplementedError(f"replay_strategy {replay_strategy!r}: only 'future' and 'none' exist")
    override_params = override_params or {}
    set_global_seeds(seed)

    params = dict(config.DEFAULT_PARAMS)
    env_name = env.spec.id
    params['env_name'] = env_name
    params['replay_strategy'] = replay_strategy
    if env_name in config.DEFAULT_ENV_PARAMS:
        params.update(config.DEFAULT_ENV_PARAMS[env_name])
    params.update(**override_params)
    if logger.get_dir():
        with open(os.path.join(logger.get_dir(), 'params.json'), 'w') as f:
            json.dump(params, f)
    params = config.prepare_params(params)
    params['rollout_batch_size'] = env.num_envs
    params.update(kwargs)
    params['seed'] = seed
    config.log_params(params, logger=logger)

    dims = config.configure_dims(params)
    policy = config.configure_ddpg(dims=dims, params=params, clip_return=clip_return)
    if load_path is not None:
        policy.load(load_path)

    rollout_params = {'exploit': False, 'use_target_net': False, 'use_demo_states': True, 'compute_Q': False,
                      'T': params['T']}
    eval_params = {'exploit': True, 'use_target_net': params['test_with_polyak'], 'use_demo_states': False,
                   'compute_Q': True, 'T': params['T']}
    for name in ['T', 'rollout_batch_size', 'gamma', 'noise_eps', 'random_eps']:
        rollout_params[name] = params[name]
        eval_params[name] = params[name]

    eval_env = eval_env or env
    rollout_worker = RolloutWorker(env, policy, dims, logger, monitor=True, **rollout_params)
    evaluator = RolloutWorker(eval_env, policy, dims, logger, **eval_params)

    n_cycles = params['n_cycles']
    n_epochs = total_timesteps // n_cycles // rollout_worker.T // rollout_worker.rollout_batch_size
    return train(save_path=save_path, policy=policy, rollout_worker=rollout_worker, evaluator=evaluator,
                 n_epochs=n_epochs, n_test_rollouts=params['n_test_rollouts'], n_cycles=params['n_cycles'],
                 n_batches=params['n_batches'], policy_save_interval=policy_save_interval, demo_file=demo_file)
