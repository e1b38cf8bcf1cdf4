"""ddpg.learn (baselines/ddpg/ddpg.py:21-275): the same epochs / cycles / rollout / train loop and logger keys, with the
agent of ddpg_learner on the device.

Out of scope: MPI (one process; the reference's allreduces over one rank are identities), rendering, and the
env_state.pkl dumps (the reference agent has no save / load either).
"""
import time
from collections import deque

import numpy as np

from .. import logger
from .ddpg_learner import DDPG
from .memory import Memory
from .models import Actor, Critic
from .noise import parse_noise_type


def _set_global_seeds(seed):
    if seed is None:
        return
    import random
    import torch
    np.random.seed(seed)
    random.seed(seed)
    torch.manual_seed(seed)


def learn(network, env,
          seed=None,
          total_timesteps=None,
          nb_epochs=None,
          nb_epoch_cycles=20,
          nb_rollout_steps=100,
          reward_scale=1.0,
          render=False,
          render_eval=False,
          noise_type='adaptive-param_0.2',
          normalize_returns=False,
          normalize_observations=True,
          critic_l2_reg=1e-2,
          actor_lr=1e-4,
          critic_lr=1e-3,
          popart=False,
          gamma=0.99,
          clip_norm=None,
          nb_train_steps=50,
          nb_eval_steps=100,
          batch_size=64,
          tau=0.01,
          eval_env=None,
          param_noise_adaption_interval=50,
          memory_limit=int(1e6),
          **network_kwargs):
    """Returns the agent.  memory_limit: the replay ring's rows (the reference's fixed 1e6)."""
    if render or render_eval:
        raise NotImplementedError("ddpg rendering is not supported")
    _set_global_seeds(seed)
    if total_timesteps is not None:
        assert nb_epochs is None
        nb_epochs = int(total_timesteps) // (nb_epoch_cycles * nb_rollout_steps)
    else:
        nb_epochs = 500

    nb_actions = env.action_space.shape[-1]
    assert (np.abs(env.action_space.low) == env.action_space.high).all()  # symmetric actions

    memory = Memory(limit=int(memory_limit), action_shape=env.action_space.shape,
                    observation_shape=env.observation_space.shape)
    critic = Critic(network=network, **network_kwargs)
    actor = Actor(nb_actions, network=network, **network_kwargs)
    action_noise, param_noise = parse_noise_type(noise_type, nb_actions)

    max_action = env.action_space.high
    logger.info('scaling actions by {} before executing in env'.format(max_action))

    obs = env.reset()
    nenvs = obs.shape[0]
    agent = DDPG(actor, critic, memory, env.observation_space.shape, env.action_space.shape,
                 gamma=gamma, tau=tau, normalize_returns=normalize_returns,
                 normalize_observations=normalize_observations, batch_size=batch_size, action_noise=action_noise,
                 param_noise=param_noise, critic_l2_reg=critic_l2_reg, actor_lr=actor_lr, critic_lr=critic_lr,
                 enable_popart=popart, clip_norm=clip_norm, reward_scale=reward_scale,
                 act_cap=max(nenvs, 256 if eval_env is None else max(256, eval_env.num_envs)),
                 seed=seed)
    logger.info('Using agent with the following configuration:')
    logger.info(str(agent.__dict__.items()))

    eval_episode_rewards_history = deque(maxlen=100)
    episode_rewards_history = deque(maxlen=100)
    agent.initialize()
    agent.reset()

    if eval_env is not None:
        eval_obs = eval_env.reset()

    episode_reward = np.zeros(nenvs, dtype=np.float32)
    episode_step = np.zeros(nenvs, dtype=int)
    episodes = 0
    t = 0
    start_time = time.time()

    epoch_episode_rewards = []
    epoch_episode_steps = []
    epoch_actions = []
    epoch_qs = []
    epoch_episodes = 0
    for epoch in range(nb_epochs):
        for cycle in range(nb_epoch_cycles):
            if nenvs > 1:
                # several envs step together: the agent resets per cycle, not per episode
                agent.reset()
            for t_rollout in range(nb_rollout_steps):
                action, q, _, _ = agent.step(obs, apply_noise=True, compute_Q=True)
                new_obs, r, done, info = env.step(max_action * action)
                t += 1
                episode_reward += r
                episode_step += 1
                epoch_actions.append(action)
                epoch_qs.append(q)
                agent.store_transition(obs, action, r, new_obs, done)
                obs = new_obs
                for d in range(len(done)):
                    if done[d]:
                        epoch_episode_rewards.append(episode_reward[d])
                        episode_rewards_history.append(episode_reward[d])
                        epoch_episode_steps.append(episode_step[d])
                        episode_reward[d] = 0.
                        episode_step[d] = 0
                        epoch_episodes += 1
                        episodes += 1
                        if nenvs == 1:
                            agent.reset()

            # the losses and distances stay on the device until the epoch's statistics
            epoch_losses = []
            epoch_adaptive_distances = []
            for t_train in range(nb_train_steps):
                if memory.nb_entries >= batch_size and t_train % param_noise_adaption_interval == 0:
                    distance = agent.adapt_param_noise_device()
                    if distance is not None:
                        epoch_adaptive_distances.append(distance.clone())
                    else:
                        epoch_adaptive_distances.append(0.)
                epoch_losses.append(agent.train_device().clone())
                agent.update_target_net()

            eval_episode_rewards = []
            eval_qs = []
            if eval_env is not None:
                nenvs_eval = eval_obs.shape[0]
                eval_episode_reward = np.zeros(nenvs_eval, dtype=np.float32)
                for t_rollout in range(nb_eval_steps):
                    eval_action, eval_q, _, _ = agent.step(eval_obs, apply_noise=False, compute_Q=True)
                    eval_obs, eval_r, eval_done, eval_info = eval_env.step(max_action * eval_action)
                    eval_episode_reward += eval_r
                    eval_qs.append(eval_q)
                    for d in range(len(eval_done)):
                        if eval_done[d]:
                            eval_episode_rewards.append(eval_episode_reward[d])
                            eval_episode_rewards_history.append(eval_episode_reward[d])
                            eval_episode_reward[d] = 0.0

        losses = np.stack([x.cpu().numpy() for x in epoch_losses]) if epoch_losses else np.zeros((0, 2), np.float32)
        dists = [float(x.item()) if hasattr(x, 'item') else x for x in epoch_adaptive_distances]
        duration = time.time() - start_time
        stats = agent.get_stats()
        combined_stats = stats.copy()
        combined_stats['rollout/return'] = np.mean(epoch_episode_rewards)
        combined_stats['rollout/return_std'] = np.std(epoch_episode_rewards)
        combined_stats['rollout/return_history'] = np.mean(episode_rewards_history)
        combined_stats['rollout/return_history_std'] = np.std(episode_rewards_history)
        combined_stats['rollout/episode_steps'] = np.mean(epoch_episode_steps)
        combined_stats['rollout/actions_mean'] = np.mean(epoch_actions)
        combined_stats['rollout/Q_mean'] = np.mean(epoch_qs)
        combined_stats['train/loss_actor'] = np.mean(losses[:, 1])
        combined_stats['train/loss_critic'] = np.mean(losses[:, 0])
        combined_stats['train/param_noise_distance'] = np.mean(dists)
        combined_stats['total/duration'] = duration
        combined_stats['total/steps_per_second'] = float(t) / float(duration)
        combined_stats['total/episodes'] = episodes
        combined_stats['rollout/episodes'] = epoch_episodes
        combined_stats['rollout/actions_std'] = np.std(epoch_actions)
        if eval_env is not None:
            combined_stats['eval/return'] = eval_episode_rewards
            combined_stats['eval/return_history'] = np.mean(eval_episode_rewards_history)
            combined_stats['eval/Q'] = eval_qs
            combined_stats['eval/episodes'] = len(eval_episode_rewards)
        # one process: the reference's allreduce over ranks keeps each value's first element
        combined_stats = {k: np.array(v).flatten()[0] for k, v in combined_stats.items()}
        combined_stats['total/epochs'] = epoch + 1
        combined_stats['total/steps'] = t
        for key in sorted(combined_stats.keys()):
            logger.logkv(key, combined_stats[key])
        logger.dumpkvs()
        logger.info('')
    return agent
