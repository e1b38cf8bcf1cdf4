"""rollout.py: RolloutWorker on the host, with the reference's episode dict, success-rate and mean_Q histories and
logs.  The policy's get_actions runs on the device; its noise draws stay on numpy's global stream."""
import pickle
from collections import deque

import numpy as np


def convert_episode_to_batch_major(episode):
    """util.py:112-121: make inputs batch-major instead of time-major."""
    episode_batch = {}
    for key in episode.keys():
        val = np.array(episode[key]).copy()
        episode_batch[key] = val.swapaxes(0, 1)
    return episode_batch


def transitions_in_episode_batch(episode_batch):
    shape = episode_batch['u'].shape
    return shape[0] * shape[1]


class RolloutWorker:
    def __init__(self, venv, policy, dims, logger, T, rollout_batch_size=1, exploit=False, use_target_net=False,
                 compute_Q=False, noise_eps=0, random_eps=0, history_len=100, render=False, monitor=False, **kwargs):
        assert T > 0
        if render:
            raise NotImplementedError("her rendering is not supported")
        self.venv, self.policy, self.dims, self.logger, self.T = venv, policy, dims, logger, T
        self.rollout_batch_size, self.exploit, self.use_target_net = rollout_batch_size, exploit, use_target_net
        self.compute_Q, self.noise_eps, self.random_eps = compute_Q, noise_eps, random_eps
        self.history_len, self.render, self.monitor = history_len, render, monitor
        self.info_keys = [key.replace('info_', '') for key in dims.keys() if key.startswith('info_')]
        self.success_history = deque(maxlen=history_len)
        self.Q_history = deque(maxlen=history_len)
        self.n_episodes = 0
        self.reset_all_rollouts()
        self.clear_history()

    def reset_all_rollouts(self):
        self.obs_dict = self.venv.reset()
        self.initial_o = self.obs_dict['observation']
        self.initial_ag = self.obs_dict['achieved_goal']
        self.g = self.obs_dict['desired_goal']

    def generate_rollouts(self):
        """rollout_batch_size rollouts in parallel for up to T steps (rollout.py:50-134)."""
        self.reset_all_rollouts()
        o = np.empty((self.rollout_batch_size, self.dims['o']), np.float32)
        ag = np.empty((self.rollout_batch_size, self.dims['g']), np.float32)
        o[:] = self.initial_o
        ag[:] = self.initial_ag
        obs, achieved_goals, acts, goals, successes = [], [], [], [], []
        dones = []
        info_values = [np.empty((self.T - 1, self.rollout_batch_size, self.dims['info_' + key]), np.float32)
                       for key in self.info_keys]
        Qs = []
        for t in range(self.T):
            policy_output = self.policy.get_actions(
                o, ag, self.g, compute_Q=self.compute_Q,
                noise_eps=self.noise_eps if not self.exploit else 0.,
                random_eps=self.random_eps if not self.exploit else 0.,
                use_target_net=self.use_target_net)
            if self.compute_Q:
                u, Q = policy_output
                Qs.append(Q)
            else:
                u = policy_output
            if u.ndim == 1:
                u = u.reshape(1, -1)
            obs_dict_new, _, done, info = self.venv.step(u)
            o_new = obs_dict_new['observation']
            ag_new = obs_dict_new['achieved_goal']
            success = np.array([i.get('is_success', 0.0) for i in info])
            if any(done):
                # the vec env has already reset the finished envs: their observations start the next episode
                break
            for i, info_dict in enumerate(info):
                for idx, key in enumerate(self.info_keys):
                    info_values[idx][t, i] = info[i][key]
            if np.isnan(o_new).any():
                self.logger.warn('NaN caught during rollout generation. Trying again...')
                self.reset_all_rollouts()
                return self.generate_rollouts()
            dones.append(done)
            obs.append(o.copy())
            achieved_goals.append(ag.copy())
            successes.append(success.copy())
            acts.append(u.copy())
            goals.append(self.g.copy())
            o[...] = o_new
            ag[...] = ag_new
        obs.append(o.copy())
        achieved_goals.append(ag.copy())
        episode = dict(o=obs, u=acts, g=goals, ag=achieved_goals)
        for key, value in zip(self.info_keys, info_values):
            episode['info_{}'.format(key)] = value
        successful = np.array(successes)[-1, :]
        assert successful.shape == (self.rollout_batch_size,)
        success_rate = np.mean(successful)
        self.success_history.append(success_rate)
        if self.compute_Q:
            self.Q_history.append(np.mean(Qs))
        self.n_episodes += self.rollout_batch_size
        return convert_episode_to_batch_major(episode)

    def clear_history(self):
        self.success_history.clear()
        self.Q_history.clear()

    def current_success_rate(self):
        return np.mean(self.success_history)

    def current_mean_Q(self):
        return np.mean(self.Q_history)

    def save_policy(self, path):
        with open(path, 'wb') as f:
            pickle.dump(self.policy, f)

    def logs(self, prefix='worker'):
        logs = []
        logs += [('success_rate', np.mean(self.success_history))]
        if self.compute_Q:
            logs += [('mean_Q', np.mean(self.Q_history))]
        logs += [('episode', self.n_episodes)]
        if prefix != '' and not prefix.endswith('/'):
            return [(prefix + '/' + key, val) for key, val in logs]
        return logs
