"""Replay helpers for tests/golden/acer_*.npz (written by tools/gen_acer_golden.py from the reference's own code)."""
import os

import numpy as np
import torch

from baselines_b200.common import spaces
from baselines_b200.common.vec_env import VecEnv

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# (name, nenv, nsteps, frame, nc, nstack, dtype), as the generator's CASES
CASES = [("u8_s4", 3, 5, (4, 3), 1, 4, np.uint8), ("f32_s1", 2, 6, (), 4, 1, np.float32),
         ("f32_s4c2", 2, 4, (3,), 2, 4, np.float32), ("u8_s1", 2, 3, (2, 2), 3, 1, np.uint8)]
NA = 5


def load(which):
    return np.load(os.path.join(GOLDEN, f"acer_{which}.npz"))


def segment(g, name, i):
    return tuple(g[f"{name}/seg{i}/{k}"] for k in ("enc", "act", "rew", "mus", "dones", "masks"))


class ScriptedEnv(VecEnv):
    """The generator's scripted environment: reset() returns frames[0], step k returns frames[k + 1]."""

    def __init__(self, frames, rewards, dones, nA):
        lo, hi = (0, 255) if frames.dtype == np.uint8 else (-10.0, 10.0)
        super().__init__(frames.shape[1], spaces.Box(lo, hi, frames.shape[2:], frames.dtype), spaces.Discrete(nA))
        self.frames, self.rewards, self.dones, self.k = frames, rewards, dones, 0

    def reset(self):
        return self.frames[0].copy()

    def step_async(self, actions):
        self.actions = actions

    def step_wait(self):
        k = self.k
        self.k += 1
        return (self.frames[k + 1].copy(), self.rewards[k].copy(), self.dones[k].copy(),
                [{} for _ in range(self.num_envs)])


class ScriptedModel:
    """Stands in for acer.Model in Runner: step_device writes actions[k] and mus[k] on call k."""

    def __init__(self, actions, mus, device):
        self.actions, self.mus, self.k, self.device, self.initial_state = actions, mus, 0, torch.device(device), None

    def step_device(self, observation, actions, mu):
        actions.copy_(torch.from_numpy(self.actions[self.k]))
        mu.copy_(torch.from_numpy(self.mus[self.k]))
        self.k += 1


class BufferEnv:
    def __init__(self, frame, nc, nstack, dtype, nenv):
        self.observation_space = spaces.Box(0, 255, frame + (nc * nstack,), dtype)
        self.action_space = spaces.Discrete(NA)
        self.num_envs, self.nstack = nenv, nstack
