"""DDPG's replay memory (baselines/ddpg/memory.py) as one device ring: float32 obs0, obs1, actions, rewards and
terminals1 rows, with RingBuffer's bookkeeping (`start`, `length`; item i at row (start + i) % limit).  Sample indices
come from numpy's global stream exactly as the reference draws them, including its quirk: randint(nb_entries - 2), so the
last two entries are never drawn."""
import numpy as np
import torch


class Memory:
    def __init__(self, limit, action_shape, observation_shape, device=None):
        if not torch.cuda.is_available():
            raise RuntimeError("baselines_b200.ddpg needs a CUDA device: no CPU fallback on the hot path")
        self.limit = int(limit)
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.action_shape, self.observation_shape = tuple(action_shape), tuple(observation_shape)
        self.ob_dim = int(np.prod(self.observation_shape))
        self.nA = int(np.prod(self.action_shape))
        self.start = self.length = 0
        f32 = dict(dtype=torch.float32, device=self.device)
        self.obs0 = torch.zeros(self.limit, self.ob_dim, **f32)
        self.obs1 = torch.zeros(self.limit, self.ob_dim, **f32)
        self.actions = torch.zeros(self.limit, self.nA, **f32)
        self.rewards = torch.zeros(self.limit, **f32)
        self.terminals1 = torch.zeros(self.limit, **f32)

    @property
    def nb_entries(self):
        return self.length

    def _advance(self):
        """RingBuffer.append's bookkeeping for one row; -> the ring row it writes."""
        if self.length < self.limit:
            self.length += 1
        else:
            self.start = (self.start + 1) % self.limit
        return (self.start + self.length - 1) % self.limit

    def append_batch(self, obs0, action, reward, obs1, terminal1):
        """Append n rows in order (one RingBuffer.append each); -> (ring row of the first, n).  The rows follow each
        other modulo limit."""
        obs0 = np.asarray(obs0, np.float32).reshape(-1, self.ob_dim)
        n = obs0.shape[0]
        host = np.empty((n, 2 * self.ob_dim + self.nA + 2), np.float32)
        host[:, :self.ob_dim] = obs0
        host[:, self.ob_dim:2 * self.ob_dim] = np.asarray(obs1, np.float32).reshape(n, self.ob_dim)
        host[:, 2 * self.ob_dim:2 * self.ob_dim + self.nA] = np.asarray(action, np.float32).reshape(n, self.nA)
        host[:, -2] = np.asarray(reward, np.float32).reshape(n)
        host[:, -1] = np.asarray(terminal1, np.float32).reshape(n)
        rows = [self._advance() for _ in range(n)]
        dev = torch.from_numpy(host).to(self.device)
        i = 0
        while i < n:                                      # at most two contiguous pieces: the ring wraps once
            p, k = rows[i], min(n - i, self.limit - rows[i])
            src = dev[i:i + k]
            self.obs0[p:p + k].copy_(src[:, :self.ob_dim])
            self.obs1[p:p + k].copy_(src[:, self.ob_dim:2 * self.ob_dim])
            self.actions[p:p + k].copy_(src[:, 2 * self.ob_dim:2 * self.ob_dim + self.nA])
            self.rewards[p:p + k].copy_(src[:, -2])
            self.terminals1[p:p + k].copy_(src[:, -1])
            i += k
        return rows[0], n

    def append(self, obs0, action, reward, obs1, terminal1, training=True):
        if not training:
            return
        self.append_batch(np.asarray(obs0)[None], np.asarray(action)[None], [reward], np.asarray(obs1)[None],
                          [terminal1])

    def sample_indices(self, batch_size):
        """memory.py:54: the batch's item indices, from numpy's global stream."""
        return np.random.randint(self.nb_entries - 2, size=batch_size)

    def selection(self, idxs):
        """The int64 host vector [start, idx...] the kernels read a sample through."""
        return np.concatenate([[self.start], np.asarray(idxs, np.int64)]).astype(np.int64)

    def sample(self, batch_size):
        """memory.py:52-69 with host arrays: the batch dict of the reference."""
        idxs = self.sample_indices(batch_size)
        rows = torch.from_numpy((self.start + idxs) % self.limit).to(self.device)
        take = lambda t: t.index_select(0, rows).cpu().numpy()
        return {'obs0': take(self.obs0), 'obs1': take(self.obs1), 'rewards': take(self.rewards).reshape(-1, 1),
                'actions': take(self.actions), 'terminals1': take(self.terminals1).reshape(-1, 1)}
