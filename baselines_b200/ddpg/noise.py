"""Exploration noise of DDPG (baselines/ddpg/noise.py), on the host: one noise vector per call, drawn from numpy's global
stream as the reference draws it, and broadcast over the environments by the agent."""
import numpy as np


class AdaptiveParamNoiseSpec:
    """Parameter-space noise whose scale follows the action-space distance it causes (Plappert et al. 2017).  The agent
    keeps its own float64 copy of current_stddev on the device and writes it back here when it reports statistics."""

    def __init__(self, initial_stddev=0.1, desired_action_stddev=0.1, adoption_coefficient=1.01):
        self.initial_stddev = initial_stddev
        self.desired_action_stddev = desired_action_stddev
        self.adoption_coefficient = adoption_coefficient
        self.current_stddev = initial_stddev

    def adapt(self, distance):
        if distance > self.desired_action_stddev:
            self.current_stddev /= self.adoption_coefficient
        else:
            self.current_stddev *= self.adoption_coefficient

    def get_stats(self):
        return {'param_noise_stddev': self.current_stddev}

    def __repr__(self):
        return (f'AdaptiveParamNoiseSpec(initial_stddev={self.initial_stddev}, '
                f'desired_action_stddev={self.desired_action_stddev}, '
                f'adoption_coefficient={self.adoption_coefficient})')


class ActionNoise:
    def reset(self):
        pass


class NormalActionNoise(ActionNoise):
    def __init__(self, mu, sigma):
        self.mu, self.sigma = mu, sigma

    def __call__(self):
        return np.random.normal(self.mu, self.sigma)

    def __repr__(self):
        return f'NormalActionNoise(mu={self.mu}, sigma={self.sigma})'


class OrnsteinUhlenbeckActionNoise(ActionNoise):
    """Euler-Maruyama steps of dx = theta (mu - x) dt + sigma dW."""

    def __init__(self, mu, sigma, theta=.15, dt=1e-2, x0=None):
        self.theta, self.mu, self.sigma, self.dt, self.x0 = theta, mu, sigma, dt, x0
        self.reset()

    def __call__(self):
        x = (self.x_prev + self.theta * (self.mu - self.x_prev) * self.dt +
             self.sigma * np.sqrt(self.dt) * np.random.normal(size=self.mu.shape))
        self.x_prev = x
        return x

    def reset(self):
        self.x_prev = self.x0 if self.x0 is not None else np.zeros_like(self.mu)

    def __repr__(self):
        return f'OrnsteinUhlenbeckActionNoise(mu={self.mu}, sigma={self.sigma})'


def parse_noise_type(noise_type, nb_actions):
    """-> (action_noise, param_noise) for a comma list such as 'adaptive-param_0.2,ou_0.2' (ddpg.py:67-84); a later
    entry of the same kind replaces an earlier one.  RuntimeError on an unknown type."""
    action_noise = param_noise = None
    if noise_type is None:
        return action_noise, param_noise
    for current in noise_type.split(','):
        current = current.strip()
        if current == 'none':
            pass
        elif 'adaptive-param' in current:
            _, stddev = current.split('_')
            param_noise = AdaptiveParamNoiseSpec(initial_stddev=float(stddev), desired_action_stddev=float(stddev))
        elif 'normal' in current:
            _, stddev = current.split('_')
            action_noise = NormalActionNoise(mu=np.zeros(nb_actions), sigma=float(stddev) * np.ones(nb_actions))
        elif 'ou' in current:
            _, stddev = current.split('_')
            action_noise = OrnsteinUhlenbeckActionNoise(mu=np.zeros(nb_actions),
                                                        sigma=float(stddev) * np.ones(nb_actions))
        else:
            raise RuntimeError(f'unknown noise type "{current}"')
    return action_noise, param_noise
