"""replay_buffer.py: the episode ring on the device.  Like the reference's np.empty buffers the values are float64:
o and ag hold T+1 steps per episode, g, u and the info_* keys T (T: transitions per episode).  The info_* keys are
column views of one [size, T, n_info] tensor so that one kernel argument reaches all of them."""
import numpy as np
import torch


class ReplayBuffer:
    def __init__(self, buffer_shapes, size_in_transitions, T, sample_transitions, device=None):
        """buffer_shapes: {key: (steps, dim)}; T: the time horizon the size is counted in (the reference's T)."""
        if not torch.cuda.is_available():
            raise RuntimeError("baselines_b200.her needs a CUDA device: no CPU fallback on the hot path")
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.buffer_shapes = buffer_shapes
        self.size = size_in_transitions // T
        self.T = T
        self.sample_transitions = sample_transitions
        f64 = dict(dtype=torch.float64, device=self.device)
        self.info_keys = sorted(k for k in buffer_shapes if k.startswith('info_'))
        self.info_off, n = {}, 0
        for k in self.info_keys:
            self.info_off[k] = (n, buffer_shapes[k][1])
            n += buffer_shapes[k][1]
        self.info = torch.zeros(self.size, buffer_shapes['u'][0], n, **f64)
        self.buffers = {}
        for key, shape in buffer_shapes.items():
            if key in self.info_off:
                o, d = self.info_off[key]
                self.buffers[key] = self.info[:, :, o:o + d]
            else:
                self.buffers[key] = torch.zeros(self.size, *shape, **f64)
        self.current_size = 0
        self.n_transitions_stored = 0

    @property
    def full(self):
        return self.current_size == self.size

    @property
    def ring(self):
        """(o, ag, g, u, info) for the kernels."""
        b = self.buffers
        return b['o'], b['ag'], b['g'], b['u'], self.info

    def draw(self, batch_size):
        """The sample's (episode, t, future_t) rows as an int64 [B, 3] host array, drawn as sample() draws them."""
        assert self.current_size > 0
        ep, t, ft = self.sample_transitions.draw(self.current_size, self.buffer_shapes['u'][0], batch_size)
        return np.stack([ep, t, ft], axis=1).astype(np.int64)

    def sample(self, batch_size):
        """The reference's sample() on host copies (for inspection; training samples on the device)."""
        assert self.current_size > 0
        buffers = {key: v[:self.current_size].cpu().numpy() for key, v in self.buffers.items()}
        buffers['o_2'] = buffers['o'][:, 1:, :]
        buffers['ag_2'] = buffers['ag'][:, 1:, :]
        return self.sample_transitions(buffers, batch_size)

    def store_episode(self, episode_batch, staged=None):
        """episode_batch: {key: array(batch x (T+1 or T) x dim)}.  staged: the same batch already on the device
        ({key: float64 tensor}); -> the ring slots written."""
        batch_sizes = [len(episode_batch[key]) for key in episode_batch.keys()]
        assert np.all(np.array(batch_sizes) == batch_sizes[0])
        batch_size = batch_sizes[0]
        idxs = np.atleast_1d(self._get_storage_idx(batch_size))
        # numpy's buffers[key][idxs] = batch: with a repeated slot the last episode stays
        last = {int(s): i for i, s in enumerate(idxs)}
        slots = torch.tensor(list(last.keys()), dtype=torch.int64, device=self.device)
        rows = torch.tensor(list(last.values()), dtype=torch.int64, device=self.device)
        for key in self.buffers.keys():
            src = staged[key] if staged is not None else \
                torch.from_numpy(np.asarray(episode_batch[key], np.float64)).to(self.device)
            self.buffers[key][slots] = src.index_select(0, rows)
        self.n_transitions_stored += batch_size * self.T
        return idxs

    def get_current_episode_size(self):
        return self.current_size

    def get_current_size(self):
        return self.current_size * self.T

    def get_transitions_stored(self):
        return self.n_transitions_stored

    def clear_buffer(self):
        self.current_size = 0

    def _get_storage_idx(self, inc=None):
        idx, self.current_size = storage_idx(self.current_size, self.size, inc)
        return idx


def storage_idx(current_size, size, inc=None):
    """replay_buffer.py:89-108: the slots of the next `inc` episodes, consecutive until the ring is full, then drawn
    with numpy's randint; -> (slots, the new current size)."""
    inc = inc or 1
    assert inc <= size, "Batch committed to replay is too large!"
    if current_size + inc <= size:
        idx = np.arange(current_size, current_size + inc)
    elif current_size < size:
        overflow = inc - (size - current_size)
        idx_a = np.arange(current_size, size)
        idx_b = np.random.randint(0, current_size, overflow)
        idx = np.concatenate([idx_a, idx_b])
    else:
        idx = np.random.randint(0, size, inc)
    current_size = min(size, current_size + inc)
    if inc == 1:
        idx = idx[0]
    return idx, current_size
