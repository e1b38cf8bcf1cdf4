"""acer/buffer.py's Buffer with its ring in device memory.

The ring keeps the reference's layout: per slot and env the `nsteps + nstack` single frames of a segment (enc_obs) and
the segment's per-step arrays.  `get()` draws one slot per env with `np.random.randint(0, num_in_buffer, nenv)` from
numpy's global stream, as the reference does, and hands the slots to the device through a pinned buffer; the frames
are re-stacked there by `ops.acer_stack_obs` (_stack_obs, buffer.py:124-140).
"""
import numpy as np
import torch

from .. import ops


class Segment:
    """One segment per env on the device, stored as a ring of `slots` slots:
    enc_obs [slots, nenv, nsteps + nstack, *frame, nc] (uint8 or float32), actions int64 / rewards float32 /
    dones uint8 [slots, nenv, nsteps], mus float32 [slots, nenv, nsteps, nA], masks uint8 [slots, nenv, nsteps + 1]."""

    def __init__(self, slots, nenv, nsteps, nstack, frame, nc, obs_dtype, nact, device):
        self.slots, self.nenv, self.nsteps, self.nstack, self.nact = slots, nenv, nsteps, nstack, nact
        self.frame, self.nc = tuple(frame), nc
        dt = torch.uint8 if np.dtype(obs_dtype) == np.uint8 else torch.float32
        self.enc_obs = torch.zeros((slots, nenv, nsteps + nstack) + self.frame + (nc,), dtype=dt, device=device)
        self.actions = torch.zeros(slots, nenv, nsteps, dtype=torch.int64, device=device)
        self.rewards = torch.zeros(slots, nenv, nsteps, dtype=torch.float32, device=device)
        self.mus = torch.zeros(slots, nenv, nsteps, nact, dtype=torch.float32, device=device)
        self.dones = torch.zeros(slots, nenv, nsteps, dtype=torch.uint8, device=device)
        self.masks = torch.zeros(slots, nenv, nsteps + 1, dtype=torch.uint8, device=device)

    @staticmethod
    def nbytes(slots, nenv, nsteps, nstack, frame, nc, obs_dtype, nact):
        per = (nsteps + nstack) * int(np.prod(frame, dtype=np.int64)) * nc * np.dtype(obs_dtype).itemsize
        per += nsteps * (8 + 4 + 4 * nact + 1) + nsteps + 1
        return int(slots) * nenv * per

    def arrays(self):
        return (self.enc_obs, self.actions, self.rewards, self.mus, self.dones, self.masks)


def frame_layout(env):
    """(frame shape, channels per frame, nstack) of a VecFrameStack env (buffer.py:9-14)."""
    shape = tuple(env.observation_space.shape)
    nstack = env.nstack
    return shape[:-1], shape[-1] // nstack, nstack


class Buffer(object):
    # gets obs, actions, rewards, mu's, (states, masks), dones
    def __init__(self, env, nsteps, size=50000, device=None):
        self.nenv = env.num_envs
        self.nsteps = nsteps
        self.obs_shape = env.observation_space.shape
        self.obs_dtype = env.observation_space.dtype
        self.frame, self.nc, self.nstack = frame_layout(env)
        self.nact = env.action_space.n
        self.nbatch = self.nenv * self.nsteps
        self.size = size // (self.nsteps)  # Each loc contains nenv * nsteps frames, thus total buffer is nenv * size frames
        if self.size < 1:
            raise ValueError(f"buffer_size={size} holds no segment of nsteps={nsteps} steps")
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        need = Segment.nbytes(self.size, self.nenv, nsteps, self.nstack, self.frame, self.nc, self.obs_dtype, self.nact)
        free, total = torch.cuda.mem_get_info(self.device)
        if need > free:
            raise MemoryError(f"the ACER replay ring needs {need / 2**30:.2f} GiB of device memory ({self.size} slots x "
                              f"{self.nenv} envs x {nsteps + self.nstack} frames) but {free / 2**30:.2f} GiB of "
                              f"{total / 2**30:.2f} GiB are free: lower buffer_size or the number of envs")
        self.ring = Segment(self.size, self.nenv, nsteps, self.nstack, self.frame, self.nc, self.obs_dtype, self.nact,
                            self.device)
        # the slots drawn by get(), staged in pinned memory; the copy must finish before the next draw overwrites them
        self._idx_host = torch.zeros(self.nenv, dtype=torch.int64).pin_memory()
        self.idx = torch.zeros(self.nenv, dtype=torch.int64, device=self.device)
        self._idx_copied = torch.cuda.Event()
        self._out = None

        # Size indexes
        self.next_idx = 0
        self.num_in_buffer = 0

    def has_atleast(self, frames):
        # Frames per env, so total (nenv * frames) Frames needed
        # Each buffer loc has nenv * nsteps frames
        return self.num_in_buffer >= (frames // self.nsteps)

    def can_sample(self):
        return self.num_in_buffer > 0

    def put(self, enc_obs, actions, rewards, mus, dones, masks):
        """enc_obs [nenv, nsteps + nstack, *frame, nc]; actions, rewards, dones [nenv, nsteps]; mus [nenv, nsteps, nact];
        masks [nenv, nsteps + 1].  Device tensors (a Runner segment's slot) or host arrays."""
        for dst, src in zip(self.ring.arrays(), (enc_obs, actions, rewards, mus, dones, masks)):
            t = src if torch.is_tensor(src) else torch.from_numpy(np.ascontiguousarray(src))
            dst[self.next_idx].copy_(t.reshape(dst.shape[1:]).to(dst.dtype), non_blocking=True)
        self.next_idx = (self.next_idx + 1) % self.size
        self.num_in_buffer = min(self.size, self.num_in_buffer + 1)

    def sample_slots(self):
        """Draw one slot per env like Buffer.get (buffer.py:86) and stage them on the device -> int64 [nenv]."""
        assert self.can_sample()
        idx = np.random.randint(0, self.num_in_buffer, self.nenv)
        self._idx_copied.synchronize()
        self._idx_host.numpy()[:] = idx
        self.idx.copy_(self._idx_host, non_blocking=True)
        self._idx_copied.record()
        return self.idx

    def get(self):
        """buffer.py:77-97 on the device: (obs [nenv * (nsteps + 1), *obs_shape], actions, rewards, mus, dones, masks),
        device tensors shaped as the reference's arrays."""
        idx = self.sample_slots()
        if self._out is None:
            dev, nenv, ns = self.device, self.nenv, self.nsteps
            self._out = (torch.empty((nenv * (ns + 1),) + tuple(self.obs_shape), dtype=self.ring.enc_obs.dtype,
                                     device=dev),
                         torch.empty(nenv, ns, dtype=torch.int64, device=dev),
                         torch.empty(nenv, ns, dtype=torch.float32, device=dev),
                         torch.empty(nenv, ns, self.nact, dtype=torch.float32, device=dev),
                         torch.empty(nenv, ns, dtype=torch.uint8, device=dev),
                         torch.empty(nenv, ns + 1, dtype=torch.uint8, device=dev))
        obs, actions, rewards, mus, dones, masks = self._out
        ops.acer_stack_obs(self.ring.enc_obs, idx, self.nenv, self.nsteps, self.nstack, self.ring.dones, obs)
        ops.acer_take(idx, self.nenv, self.nsteps, self.nact, self.ring.arrays()[1:], (actions, rewards, mus, dones,
                                                                                      masks))
        return obs.reshape((self.nenv, self.nsteps + 1) + tuple(self.obs_shape)), actions, rewards, mus, dones, masks

