"""Replay buffers with device-resident storage and fp64 sum / min segment trees in HBM.

Same classes, constructor arguments and method names as baselines/deepq/replay_buffer.py (ReplayBuffer :7-68,
PrioritizedReplayBuffer :71-191); `sample` / `update_priorities` keep the numpy return types of the reference.
`sample_device` / `update_priorities_device` are the resident fast path used by this repo's deepq.learn: the
sampled transitions never leave HBM (the train step gathers observations by index), only the scalar
max-priority is read back.

Randomness: like the reference, sampling positions come from python's `random` module (replay_buffer.py:67,112),
so a seeded run draws the same strata; the uniforms (8 bytes each) are uploaded.
"""
import random

import numpy as np
import torch

from .. import ops


class ReplayBuffer(object):
    STAGE = 64          # transitions staged in pinned host memory between uploads

    def __init__(self, size, device=None):
        self._maxsize = int(size)
        self._next_idx = 0
        self._n = 0
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self._obs_t = self._obs_tp1 = None          # allocated on first add (shape / dtype known then)
        dev = self.device
        self._actions = torch.zeros(self._maxsize, dtype=torch.int64, device=dev)
        self._rewards = torch.zeros(self._maxsize, dtype=torch.float32, device=dev)
        self._dones = torch.zeros(self._maxsize, dtype=torch.float32, device=dev)
        # `add` (one transition per env step, deepq.py:283) only writes a pinned host record; the records are uploaded
        # with a few asynchronous slice copies the next time the device arrays are read (every train_freq steps)
        self._pend = 0
        self._pend_first = 0
        self._stage_done = torch.cuda.Event()
        P = min(self.STAGE, self._maxsize)
        self._stage_cap = P
        self._p_act = torch.zeros(P, dtype=torch.int64).pin_memory()
        self._p_rew = torch.zeros(P, dtype=torch.float32).pin_memory()
        self._p_done = torch.zeros(P, dtype=torch.float32).pin_memory()
        self._p_obs_t = self._p_obs_tp1 = None

    def __len__(self):
        return self._n

    def _alloc(self, obs):
        obs = np.asarray(obs)
        dt = torch.uint8 if obs.dtype == np.uint8 else torch.float32
        self._obs_t = torch.zeros((self._maxsize,) + obs.shape, dtype=dt, device=self.device)
        self._obs_tp1 = torch.zeros_like(self._obs_t)
        self._p_obs_t = torch.zeros((self._stage_cap,) + obs.shape, dtype=dt).pin_memory()
        self._p_obs_tp1 = torch.zeros_like(self._p_obs_t).pin_memory()

    def add(self, obs_t, action, reward, obs_tp1, done):
        """replay_buffer.py:24-31: ring write at _next_idx (staged; see _flush)."""
        if self._obs_t is None:
            self._alloc(obs_t)
        if self._pend == self._stage_cap:
            self._flush()
        if self._pend == 0:
            self._stage_done.synchronize()           # the previous upload has finished reading the staging records
            self._pend_first = self._next_idx
        k = self._pend
        self._p_obs_t[k].numpy()[...] = obs_t
        self._p_obs_tp1[k].numpy()[...] = obs_tp1
        self._p_act[k] = int(action)
        self._p_rew[k] = float(reward)
        self._p_done[k] = float(done)
        self._pend = k + 1
        i = self._next_idx
        self._next_idx = (self._next_idx + 1) % self._maxsize
        self._n = min(self._n + 1, self._maxsize)
        return i

    def _flush(self):
        """Upload the staged transitions into their ring slots (at most two contiguous ranges when the ring wraps)."""
        k = self._pend
        if k == 0:
            return
        first = self._pend_first
        with torch.cuda.device(self.device):
            done = 0
            while done < k:
                lo = (first + done) % self._maxsize
                n = min(k - done, self._maxsize - lo)
                src, dst = slice(done, done + n), slice(lo, lo + n)
                self._obs_t[dst].copy_(self._p_obs_t[src], non_blocking=True)
                self._obs_tp1[dst].copy_(self._p_obs_tp1[src], non_blocking=True)
                self._actions[dst].copy_(self._p_act[src], non_blocking=True)
                self._rewards[dst].copy_(self._p_rew[src], non_blocking=True)
                self._dones[dst].copy_(self._p_done[src], non_blocking=True)
                self._on_flush_range(lo, n)
                done += n
            self._stage_done.record()
        self._pend = 0

    def _on_flush_range(self, lo, n):
        pass

    def add_batch(self, obs_t, actions, rewards, obs_tp1, dones):
        """Vectorised add of k transitions (device or host arrays); same ring semantics."""
        k = len(actions)
        if self._obs_t is None:
            self._alloc(np.asarray(obs_t[0].cpu() if torch.is_tensor(obs_t) else obs_t[0]))
        self._flush()
        idx = (self._next_idx + np.arange(k)) % self._maxsize
        it = torch.from_numpy(idx).to(self.device)
        as_t = lambda x, dt: (x if torch.is_tensor(x) else torch.from_numpy(np.ascontiguousarray(x))).to(self.device, dt)
        self._obs_t[it] = as_t(obs_t, self._obs_t.dtype)
        self._obs_tp1[it] = as_t(obs_tp1, self._obs_t.dtype)
        self._actions[it] = as_t(actions, torch.int64)
        self._rewards[it] = as_t(rewards, torch.float32)
        self._dones[it] = as_t(dones, torch.float32)
        self._next_idx = int((self._next_idx + k) % self._maxsize)
        self._n = min(self._n + k, self._maxsize)
        return idx

    def _encode_sample(self, idxes):
        """replay_buffer.py:33-43 (rewards / dones come back float64 there: python floats)."""
        self._flush()
        it = torch.as_tensor(np.asarray(idxes, dtype=np.int64)).to(self.device)
        return (self._obs_t[it].cpu().numpy(), self._actions[it].cpu().numpy(),
                self._rewards[it].cpu().numpy().astype(np.float64), self._obs_tp1[it].cpu().numpy(),
                self._dones[it].cpu().numpy().astype(np.float64))

    def sample(self, batch_size):
        idxes = [random.randint(0, self._n - 1) for _ in range(batch_size)]      # replay_buffer.py:67
        return self._encode_sample(idxes)

    def sample_device(self, batch_size):
        self._flush()
        idxes = [random.randint(0, self._n - 1) for _ in range(batch_size)]
        idx = torch.as_tensor(np.asarray(idxes, dtype=np.int64)).to(self.device)
        return idx, torch.ones(batch_size, dtype=torch.float32, device=self.device)


class PrioritizedReplayBuffer(ReplayBuffer):
    def __init__(self, size, alpha, device=None):
        super().__init__(size, device)
        assert alpha >= 0
        self._alpha = alpha
        it_capacity = 1
        while it_capacity < size:                                                # replay_buffer.py:92-94
            it_capacity *= 2
        self._cap = it_capacity
        dev = self.device
        self._it_sum = torch.zeros(2 * it_capacity, dtype=torch.float64, device=dev)
        self._it_min = torch.full((2 * it_capacity,), float("inf"), dtype=torch.float64, device=dev)
        # running max of the priorities (replay_buffer.py:98,191) lives on the device so that the resident train loop
        # never reads it back; the host attribute `_max_priority` is a view that synchronises only when somebody asks
        self._maxp_dev = torch.ones(1, dtype=torch.float64, device=dev)
        self._arange = torch.arange(self._stage_cap, dtype=torch.int64, device=dev)
        self._new_val = torch.zeros(self._stage_cap, dtype=torch.float64, device=dev)
        # the reference asserts `priority > 0` (replay_buffer.py:186).  The kernels set a sticky device flag instead;
        # it is copied to pinned memory without waiting and raised on by the first sample / update call that finds the
        # copy complete, which is the first one after the host has synchronised with the stream (deepq.learn: after the
        # next act), so the train loop never waits for it
        self._bad_dev = torch.zeros(1, dtype=torch.int32, device=dev)
        self._bad_host = torch.zeros(1, dtype=torch.int32).pin_memory()
        self._bad_copied = torch.cuda.Event()
        self._bad_pending = False
        self._bad_seen = False

    @property
    def _max_priority(self):
        return float(self._maxp_dev.item())

    @_max_priority.setter
    def _max_priority(self, v):
        self._maxp_dev.fill_(float(v))

    def _set_priorities(self, idx_t, vals_t):
        ops.tree_set(self._it_sum, self._it_min, self._cap, idx_t, vals_t)

    def _copy_bad_flag(self):
        with torch.cuda.device(self.device):
            self._bad_host.copy_(self._bad_dev, non_blocking=True)
            self._bad_copied.record()
        self._bad_pending = True

    def _check_priorities(self):
        if self._bad_pending and self._bad_copied.query():
            self._bad_pending = False
            self._bad_seen = bool(int(self._bad_host[0]))                        # the device flag is sticky
        if self._bad_seen:
            raise AssertionError("assert priority > 0 failed: an update wrote a priority that is not > 0 "
                                 "(NaN or zero |td| + eps); the sum / min trees are invalid")

    def add(self, *args, **kwargs):
        """replay_buffer.py:100-105: new transitions enter with max_priority ** alpha.  max_priority only changes in
        update_priorities, which flushes the staged transitions first, so every staged transition shares one value and
        the tree writes happen with the upload (one launch per range)."""
        return super().add(*args, **kwargs)

    def _on_flush_range(self, lo, n):
        ops.per_pow(self._maxp_dev, self._alpha, self._new_val[:1])             # scalar bookkeeping, stays on the device
        self._set_priorities(self._arange[:n] + lo, self._new_val[:1].expand(n).contiguous())

    def add_batch(self, *args, **kwargs):
        idx = super().add_batch(*args, **kwargs)
        it = torch.from_numpy(np.asarray(idx, dtype=np.int64)).to(self.device)
        ops.per_pow(self._maxp_dev, self._alpha, self._new_val[:1])
        self._set_priorities(it, self._new_val[:1].expand(len(idx)).contiguous())
        return idx

    def sample_device(self, batch_size, beta, uniforms=None):
        """Stratified proportional sampling + importance weights on device (replay_buffer.py:107-115,157-165).
        Returns (idx int64[B], weights float32[B], weights float64[B]) device tensors."""
        assert beta > 0
        self._check_priorities()
        self._flush()
        if uniforms is None:
            uniforms = [random.random() for _ in range(batch_size)]              # replay_buffer.py:112
        u = torch.as_tensor(np.asarray(uniforms, dtype=np.float64)).to(self.device)
        idx = torch.empty(batch_size, dtype=torch.int64, device=self.device)
        w64 = torch.empty(batch_size, dtype=torch.float64, device=self.device)
        w32 = torch.empty(batch_size, dtype=torch.float32, device=self.device)
        ops.per_sample(self._it_sum, self._it_min, self._cap, self._n, u, beta, idx, w64, w32, self._bad_dev)
        return idx, w32, w64

    def sample(self, batch_size, beta):
        """Reference return tuple: (obs_t, act, rew, obs_tp1, done, weights float64, idxes)."""
        idx, _, w64 = self.sample_device(batch_size, beta)
        self._copy_bad_flag()
        idxes = idx.cpu().numpy()
        self._check_priorities()
        return tuple(list(self._encode_sample(idxes)) + [w64.cpu().numpy(), list(idxes)])

    def update_priorities(self, idxes, priorities):
        """replay_buffer.py:169-191.  priority ** alpha is evaluated with python floats like the reference."""
        assert len(idxes) == len(priorities)
        self._check_priorities()
        self._flush()
        pr = [float(p) for p in priorities]
        assert all(p > 0 for p in pr)
        assert all(0 <= int(i) < self._n for i in idxes)
        it = torch.as_tensor(np.asarray(idxes, dtype=np.int64)).to(self.device)
        vals = torch.as_tensor(np.array([p ** self._alpha for p in pr], dtype=np.float64)).to(self.device)
        self._set_priorities(it, vals)
        self._max_priority = max(self._max_priority, max(pr))

    def update_priorities_device(self, idx, td_errors, eps):
        """new_priorities = |td| + eps in float32 (deepq.py:302); p ** alpha and the running max are computed on device.
        A priority that is not > 0 raises AssertionError here or in a later sample / update call (see __init__)."""
        self._check_priorities()
        self._flush()
        powered = torch.empty(idx.numel(), dtype=torch.float64, device=self.device)
        ops.per_priorities(td_errors, eps, self._alpha, powered, self._maxp_dev, self._bad_dev)
        self._set_priorities(idx, powered)
        self._copy_bad_flag()
