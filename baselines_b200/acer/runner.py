"""acer/runner.py's Runner with the segment kept on the device.

Each run() writes one segment per env into a one-slot `Segment`: the single frames enc_obs (the split stacked
observation of the first step, then the newest `nc` channels of every step), the actions and mus the device sampled,
and the rewards, dones and masks of the environment.  The training batch of the on-policy call is re-stacked from
those frames by the same kernel that serves replay (`ops.acer_stack_obs`).  That equals the reference's mb_obs when a frame has one
channel (Atari) or nothing is stacked (classic control behind VecFrameStack(env, 1)), because VecFrameStack then clears
a stack exactly where _stack_obs masks it.  With several channels per frame and nstack > 1 VecFrameStack rolls its
stack by one channel per step (vec_frame_stack.py:19), which _stack_obs does not restate; the runner then also keeps
the stacked observations themselves (`mb_obs`) and the on-policy call trains from those, as the reference does.
"""
import numpy as np
import torch

from ..common import spaces
from ..common.vec_env import VecFrameStack
from .buffer import Segment, frame_layout


class Runner(object):

    def __init__(self, env, model, nsteps):
        assert spaces.is_discrete(env.action_space), 'This ACER implementation works only with discrete action spaces!'
        assert isinstance(env, VecFrameStack)
        self.env, self.model, self.nsteps = env, model, nsteps
        self.nenv = nenv = env.num_envs
        self.nact = env.action_space.n
        self.nbatch = nenv * nsteps
        self.batch_ob_shape = (nenv * (nsteps + 1),) + env.observation_space.shape
        self.obs = env.reset()
        self.obs_dtype = env.observation_space.dtype
        self.nstack = self.env.nstack
        self.nc = self.batch_ob_shape[-1] // self.nstack
        self.states = model.initial_state
        self.dones = np.array([False for _ in range(nenv)])
        frame, nc, nstack = frame_layout(env)
        self.seg = Segment(1, nenv, nsteps, nstack, frame, nc, self.obs_dtype, self.nact, model.device)
        self._a = torch.zeros(nenv, dtype=torch.int64, device=model.device)
        self._mu = torch.zeros(nenv, self.nact, dtype=torch.float32, device=model.device)
        self.mb_obs = None
        if nc > 1 and nstack > 1:
            self.mb_obs = torch.zeros((nenv, nsteps + 1) + tuple(env.observation_space.shape),
                                      dtype=self.seg.enc_obs.dtype, device=model.device)

    def _frames(self, x):
        """[nenv, *frame, k * nc] host -> [nenv, k, *frame, nc] device (the split of runner.py:28)."""
        nenv, nc = self.nenv, self.nc
        k = x.shape[-1] // nc
        t = torch.from_numpy(np.ascontiguousarray(x).reshape(x.shape[:-1] + (k, nc)))
        return t.movedim(-2, 1).to(self.model.device, non_blocking=True)

    def run(self):
        """One segment (runner.py:26-60) into self.seg slot 0.  Returns the host rewards [nenv, nsteps] and dones
        [nenv, nsteps] (for EpisodeStats); everything the learner trains from stays in self.seg."""
        seg, T, S = self.seg, self.nsteps, self.nstack
        seg.enc_obs[0, :, :S].copy_(self._frames(self.env.stackedobs))
        mb_rewards, mb_dones = [], []
        for t in range(T):
            if self.mb_obs is not None:
                self.mb_obs[:, t].copy_(torch.from_numpy(np.ascontiguousarray(self.obs)))
            self.model.step_device(self.obs, self._a, self._mu)
            seg.actions[0, :, t].copy_(self._a)
            seg.mus[0, :, t].copy_(self._mu)
            actions = self._a.cpu().numpy()
            mb_dones.append(self.dones)
            obs, rewards, dones, _ = self.env.step(actions)
            self.dones = np.asarray(dones, dtype=bool)
            self.obs = obs
            mb_rewards.append(np.asarray(rewards, dtype=np.float32))
            seg.enc_obs[0, :, S + t].copy_(self._frames(obs[..., -self.nc:])[:, 0])
        mb_dones.append(self.dones)
        if self.mb_obs is not None:
            self.mb_obs[:, T].copy_(torch.from_numpy(np.ascontiguousarray(self.obs)))
        mb_rewards = np.asarray(mb_rewards, dtype=np.float32).swapaxes(1, 0)
        mb_dones = np.asarray(mb_dones, dtype=bool).swapaxes(1, 0)
        mb_masks = mb_dones  # Used for statefull models like LSTM's to mask state when done
        mb_dones = mb_dones[:, 1:]  # Used for calculating returns. The dones array is now aligned with rewards
        seg.rewards[0].copy_(torch.from_numpy(np.ascontiguousarray(mb_rewards)))
        seg.dones[0].copy_(torch.from_numpy(mb_dones.astype(np.uint8)))
        seg.masks[0].copy_(torch.from_numpy(mb_masks.astype(np.uint8)))
        return mb_rewards, mb_dones
