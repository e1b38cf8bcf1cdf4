"""her_sampler.py: the `future` goal relabelling.  The host draws the sample from numpy's global stream in the
reference's order and float64 arithmetic (her_sampler.py:27-37); `draw` returns only the integers the device needs."""
import numpy as np


def make_sample_her_transitions(replay_strategy, replay_k, reward_fun):
    """-> sample(episode_batch, batch_size): the reference's host function over a dict of episode arrays, with
    sample.draw(n_episodes, T, batch_size) -> (episode_idxs, t_samples, future_t with -1 where the goal is kept)."""
    if replay_strategy == 'future':
        future_p = 1 - (1. / (1 + replay_k))
    elif replay_strategy == 'none':
        future_p = 0
    else:
        raise NotImplementedError(f"replay_strategy {replay_strategy!r}: only 'future' and 'none' exist")

    def draw(n_episodes, T, batch_size):
        episode_idxs = np.random.randint(0, n_episodes, batch_size)
        t_samples = np.random.randint(T, size=batch_size)
        her = np.random.uniform(size=batch_size) < future_p
        future_offset = np.random.uniform(size=batch_size) * (T - t_samples)
        future_offset = future_offset.astype(int)
        future_t = np.where(her, t_samples + 1 + future_offset, -1)
        return episode_idxs, t_samples, future_t

    def _sample_her_transitions(episode_batch, batch_size_in_transitions):
        """episode_batch is {key: array(buffer_size x T x dim_key)}"""
        T = episode_batch['u'].shape[1]
        batch_size = batch_size_in_transitions
        episode_idxs, t_samples, future_t = draw(episode_batch['u'].shape[0], T, batch_size)
        transitions = {key: episode_batch[key][episode_idxs, t_samples].copy() for key in episode_batch.keys()}
        her = future_t >= 0
        transitions['g'][her] = episode_batch['ag'][episode_idxs[her], future_t[her]]
        info = {key.replace('info_', ''): value for key, value in transitions.items() if key.startswith('info_')}
        transitions['r'] = reward_fun(ag_2=transitions['ag_2'], g=transitions['g'], info=info)
        return {k: transitions[k].reshape(batch_size, *transitions[k].shape[1:]) for k in transitions.keys()}

    _sample_her_transitions.draw = draw
    _sample_her_transitions.future_p = future_p
    _sample_her_transitions.reward_fun = reward_fun
    _sample_her_transitions.device_reward = None      # (reward_type, distance_threshold) once the rule is verified
    return _sample_her_transitions
