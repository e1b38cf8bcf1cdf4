"""VecEnv boundary (host side).  Env stepping stays on host CPU (north star); this module only restates the
interface the learner consumes -- reference: baselines/common/vec_env/vec_env.py:29-138 (VecEnv ABC),
dummy_vec_env.py:5-81 (auto-reset on done, obs buffers), plus synthetic envs for benchmarks (SURVEY 8d).

Any object with the same attributes works with Runner (the reference's own SubprocVecEnv / DummyVecEnv do).
"""
from abc import ABC, abstractmethod

import numpy as np
import torch

from . import spaces


def obs_space_info(obs_space):
    """vec_env/util.py:obs_space_info: (keys, shapes, dtypes) of the observation's parts; a non-Dict space is the
    single part None."""
    if spaces.is_dict(obs_space):
        subspaces = obs_space.spaces
    else:
        subspaces = {None: obs_space}
    keys = list(subspaces.keys())
    return keys, {k: tuple(subspaces[k].shape) for k in keys}, {k: np.dtype(subspaces[k].dtype) for k in keys}


def dict_to_obs(obs_dict):
    """vec_env/util.py:dict_to_obs: {None: array} -> array, any other dict as it is."""
    if set(obs_dict.keys()) == {None}:
        return obs_dict[None]
    return obs_dict


def _copy_obs_dict(obs):
    return {k: np.copy(v) for k, v in obs.items()}


class VecEnv(ABC):
    """vec_env.py:29-138: batched env; reset() -> obs[N,...]; step(a[N]) -> (obs, rews f32[N], dones bool[N], infos)."""
    closed = False

    def __init__(self, num_envs, observation_space, action_space):
        self.num_envs = num_envs
        self.observation_space = observation_space
        self.action_space = action_space

    @abstractmethod
    def reset(self):
        pass

    @abstractmethod
    def step_async(self, actions):
        pass

    @abstractmethod
    def step_wait(self):
        pass

    def step(self, actions):
        self.step_async(actions)
        return self.step_wait()

    def close(self):
        self.closed = True


class DummyVecEnv(VecEnv):
    """Sequential in-process VecEnv (dummy_vec_env.py:5-81): envs are created from thunks, stepped in a loop,
    and reset automatically when done (the returned obs is then the first obs of the next episode)."""

    def __init__(self, env_fns):
        self.envs = [fn() for fn in env_fns]
        env = self.envs[0]
        super().__init__(len(self.envs), env.observation_space, env.action_space)
        self.spec = getattr(env, "spec", None)
        self.keys, shapes, dtypes = obs_space_info(env.observation_space)
        self.buf_obs = {k: np.zeros((self.num_envs,) + shapes[k], dtype=dtypes[k]) for k in self.keys}
        self.buf_dones = np.zeros((self.num_envs,), dtype=np.bool_)
        self.buf_rews = np.zeros((self.num_envs,), dtype=np.float32)
        self.buf_infos = [{} for _ in range(self.num_envs)]
        self.actions = None

    def step_async(self, actions):
        self.actions = actions

    def step_wait(self):
        for e in range(self.num_envs):
            a = self.actions[e]
            obs, self.buf_rews[e], self.buf_dones[e], self.buf_infos[e] = self.envs[e].step(a)
            if self.buf_dones[e]:
                obs = self.envs[e].reset()
            self._save_obs(e, obs)
        return self._obs_from_buf(), self.buf_rews.copy(), self.buf_dones.copy(), list(self.buf_infos)

    def reset(self):
        for e in range(self.num_envs):
            self._save_obs(e, self.envs[e].reset())
        return self._obs_from_buf()

    def _save_obs(self, e, obs):
        for k in self.keys:
            self.buf_obs[k][e] = obs if k is None else obs[k]

    def _obs_from_buf(self):
        return dict_to_obs(_copy_obs_dict(self.buf_obs))


def _subproc_worker(remote, parent_remote, fns_pickled, obs_buf, first):
    """Worker of SubprocVecEnv: owns `len(fns)` envs (run in series), writes their observations straight into
    rows [first, first+len) of the shared observation buffer and answers (rews, dones, infos) over the pipe."""
    import pickle
    parent_remote.close()
    fns = pickle.loads(fns_pickled) if isinstance(fns_pickled, bytes) else fns_pickled
    envs = [fn() for fn in fns]
    views = {k: b.numpy() for k, b in obs_buf.items()}

    def put(i, ob):
        for k, v in views.items():
            v[i] = ob if k is None else ob[k]
    try:
        while True:
            cmd, data = remote.recv()
            if cmd == 'step':
                out = []
                for k, (env, a) in enumerate(zip(envs, data)):
                    ob, rew, done, info = env.step(a)
                    if done:
                        ob = env.reset()                          # subproc_vec_env.py:8-12: auto-reset
                    put(first + k, ob)
                    out.append((rew, done, info))
                remote.send(out)
            elif cmd == 'reset':
                for k, env in enumerate(envs):
                    put(first + k, env.reset())
                remote.send(None)
            elif cmd == 'get_spaces_spec':
                remote.send((envs[0].observation_space, envs[0].action_space, getattr(envs[0], "spec", None)))
            elif cmd == 'close':
                remote.close()
                break
            else:
                raise NotImplementedError(cmd)
    except KeyboardInterrupt:
        pass
    finally:
        for env in envs:
            if hasattr(env, "close"):
                env.close()


class SubprocVecEnv(VecEnv):
    """Envs stepped in worker processes (subproc_vec_env.py:39-140, with the shared observation buffer of
    shmem_vec_env.py:23-140): `in_series` envs per process, pipes carry only actions / rewards / dones / infos.
    The observation batch lives in ONE shared-memory tensor that the workers fill in place; when CUDA is present the
    parent page-locks that memory (cudaHostRegister), so Runner uploads it with a single async copy and no
    host-side stacking -- `step_wait` hands out the same array every time (copy it if you keep it)."""

    def __init__(self, env_fns, spaces=None, context='fork', in_series=1):
        import multiprocessing as mp
        self.waiting = self.closed = False
        nenvs = len(env_fns)
        assert nenvs % in_series == 0, "Number of envs must be divisible by number of envs to run in series"
        self.nremotes, self.in_series = nenvs // in_series, in_series
        groups = [list(env_fns[i * in_series:(i + 1) * in_series]) for i in range(self.nremotes)]
        ctx = mp.get_context(context)
        if spaces is None:                                   # ask a throw-away env, like shmem_vec_env.py:35-41
            probe = env_fns[0]()
            spaces = (probe.observation_space, probe.action_space)
            self.spec = getattr(probe, "spec", None)
            if hasattr(probe, "close"):
                probe.close()
        ob_space, ac_space = spaces
        super().__init__(nenvs, ob_space, ac_space)
        self.keys, shapes, dtypes = obs_space_info(ob_space)
        self._bufs = {k: torch.zeros((nenvs,) + shapes[k], dtype=torch.from_numpy(np.zeros(1, dtypes[k])).dtype)
                      .share_memory_() for k in self.keys}
        self._obs = self._bufs[None] if self.keys == [None] else None
        self._pinned = False
        if torch.cuda.is_available() and self._obs is not None:
            try:
                rc = torch.cuda.cudart().cudaHostRegister(self._obs.data_ptr(), self._obs.numel() * self._obs.element_size(), 0)
                self._pinned = int(rc) == 0
            except Exception:
                self._pinned = False
        self.remotes, self.work_remotes = zip(*[ctx.Pipe() for _ in range(self.nremotes)])
        self.ps = []
        for k, (work_remote, remote, fns) in enumerate(zip(self.work_remotes, self.remotes, groups)):
            payload = fns
            if context != 'fork':
                import cloudpickle
                payload = cloudpickle.dumps(fns)
            proc = ctx.Process(target=_subproc_worker, args=(work_remote, remote, payload, self._bufs, k * in_series),
                               daemon=True)                  # a crashed parent must not leave workers behind
            proc.start()
            self.ps.append(proc)
        for r in self.work_remotes:
            r.close()

    def step_async(self, actions):
        assert not self.closed
        actions = np.asarray(actions)
        for k, remote in enumerate(self.remotes):
            remote.send(('step', actions[k * self.in_series:(k + 1) * self.in_series]))
        self.waiting = True

    def step_wait(self):
        assert not self.closed
        results = [r for remote in self.remotes for r in remote.recv()]
        self.waiting = False
        rews, dones, infos = zip(*results)
        return self._obs_out(), np.asarray(rews, dtype=np.float32), np.asarray(dones, dtype=np.bool_), list(infos)

    def reset(self):
        assert not self.closed
        for remote in self.remotes:
            remote.send(('reset', None))
        for remote in self.remotes:
            remote.recv()
        return self._obs_out()

    def _obs_out(self):
        """The shared observation array itself, or a dict of copies of the parts of a Dict observation."""
        if self._obs is not None:
            return self._obs.numpy()
        return {k: b.numpy().copy() for k, b in self._bufs.items()}

    def close(self):
        if self.closed:
            return
        if self.waiting:
            for remote in self.remotes:
                remote.recv()
        for remote in self.remotes:
            remote.send(('close', None))
        for proc in self.ps:
            proc.join()
        if self._pinned:
            try:
                torch.cuda.cudart().cudaHostUnregister(self._obs.data_ptr())
            except Exception:
                pass
        self.closed = True

    def __del__(self):
        if not getattr(self, "closed", True):
            self.close()


class VecEnvWrapper(VecEnv):
    """vec_env.py:140-175: a wrapper over a whole batch of envs; unknown public attributes fall through to venv."""

    def __init__(self, venv, observation_space=None, action_space=None):
        self.venv = venv
        super().__init__(venv.num_envs, observation_space or venv.observation_space,
                         action_space or venv.action_space)

    def step_async(self, actions):
        self.venv.step_async(actions)

    def close(self):
        return self.venv.close()

    def __getattr__(self, name):
        if name.startswith('_'):
            raise AttributeError("attempted to get missing private attribute '{}'".format(name))
        return getattr(self.venv, name)


class VecFrameStack(VecEnvWrapper):
    """vec_frame_stack.py:6-31: stack the last `nstack` observations along the channel axis; the stack of an env is
    cleared when its episode ends.

    reset()/step_wait() are the reference's host implementation (np.roll on a [N, H, W, nstack*c] array).  The
    device Runner does not call them: it sees `frame_stack_device`, pulls the UNSTACKED frames with step_frames()
    (1/nstack of the bytes over PCIe) and applies the same update to the HBM-resident rollout buffer with
    b200rl_frame_stack -- the previous stacked observation is already there as rollout.obs[t-1]."""
    frame_stack_device = True

    def __init__(self, venv, nstack):
        self.nstack = nstack
        wos = venv.observation_space
        low = np.repeat(wos.low, nstack, axis=-1)
        high = np.repeat(wos.high, nstack, axis=-1)
        self.frame_channels = int(wos.shape[-1])
        self.stackedobs = np.zeros((venv.num_envs,) + low.shape, low.dtype)
        ob_space = spaces.Box(low=low, high=high, dtype=wos.dtype)
        super().__init__(venv, observation_space=ob_space)

    def step_wait(self):
        obs, rews, news, infos = self.venv.step_wait()
        self.stackedobs = np.roll(self.stackedobs, shift=-1, axis=-1)
        self.stackedobs[np.asarray(news, dtype=np.bool_)] = 0
        self.stackedobs[..., -obs.shape[-1]:] = obs
        return self.stackedobs, rews, news, infos

    def reset(self):
        obs = self.venv.reset()
        self.stackedobs[...] = 0
        self.stackedobs[..., -obs.shape[-1]:] = obs
        return self.stackedobs

    # ---- unstacked access for the device-side stack
    def reset_frames(self):
        return self.venv.reset()

    def step_frames(self, actions):
        """(new frames [N, ..., c], rews, news, infos): the wrapped env's step; stacking is left to the caller."""
        self.venv.step_async(actions)
        return self.venv.step_wait()


class VecNormalize(VecEnvWrapper):
    """vec_normalize.py:4-49: running normalisation of observations and of rewards (by the std of the discounted
    return), both clipped.  Host numpy, float64 statistics (the reference's use_tf=True variant only changes where
    the three statistics are stored).

    reset()/step_wait() are the reference's host implementation.  The device Runner does not call them: it sees
    `normalize_device`, pulls the RAW batches with reset_raw()/step_raw() (or, over a device env, the HBM tensors of
    reset_raw_device()/step_raw_device()) and applies the same update, bit for bit, with the b200rl_vecnorm kernels
    (dev_reset / dev_step).  From then on the statistics and `ret` live on the device; `ob_rms`, `ret_rms` and `ret`
    read them back when accessed (and what is assigned through them is uploaded before the next device step), and a
    host reset()/step_wait() continues from the device state."""
    normalize_device = True

    def __init__(self, venv, ob=True, ret=True, clipob=10., cliprew=10., gamma=0.99, epsilon=1e-8, use_tf=False):
        super().__init__(venv)
        from .running_mean_std import RunningMeanStd
        self._ob_rms = RunningMeanStd(shape=self.observation_space.shape) if ob else None
        self._ret_rms = RunningMeanStd(shape=()) if ret else None
        self.clipob, self.cliprew, self.gamma, self.epsilon = clipob, cliprew, gamma, epsilon
        self._ret = np.zeros(self.num_envs)
        self._dev = None                 # _VecNormDevice once a device Runner has stepped through this wrapper
        self._on_device = False          # the device copy is the current state (the host copy is stale)

    # ---- the statistics, wherever they currently live
    @property
    def ob_rms(self):
        self._pull()
        return self._ob_rms

    @ob_rms.setter
    def ob_rms(self, v):
        self._pull()
        self._ob_rms = v

    @property
    def ret_rms(self):
        self._pull()
        return self._ret_rms

    @ret_rms.setter
    def ret_rms(self, v):
        self._pull()
        self._ret_rms = v

    @property
    def ret(self):
        self._pull()
        return self._ret

    @ret.setter
    def ret(self, v):
        self._pull()
        self._ret = np.asarray(v, dtype=np.float64)

    def _pull(self):
        """Make the host copy current (device -> host) and the host its owner."""
        if self._on_device:
            self._dev.download(self)
            self._on_device = False

    def _push(self, device):
        """Make the device copy current (host -> device) and the device its owner."""
        if self._dev is None or not self._dev.fits(self, device):
            self._pull()
            self._dev = _VecNormDevice(self, device)
        if not self._on_device:
            self._dev.upload(self)
            self._on_device = True
        return self._dev

    # ---- host implementation
    def _obfilt(self, obs):
        if self._ob_rms is None:
            return obs
        self._ob_rms.update(obs)
        return np.clip((obs - self._ob_rms.mean) / np.sqrt(self._ob_rms.var + self.epsilon), -self.clipob, self.clipob)

    def step_wait(self):
        obs, rews, news, infos = self.venv.step_wait()
        self._pull()
        self._ret = self._ret * self.gamma + rews
        obs = self._obfilt(obs)
        if self._ret_rms is not None:
            self._ret_rms.update(self._ret)
            rews = np.clip(rews / np.sqrt(self._ret_rms.var + self.epsilon), -self.cliprew, self.cliprew)
        self._ret[np.asarray(news, dtype=np.bool_)] = 0.
        return obs, rews, news, infos

    def reset(self):
        self._pull()
        self._ret = np.zeros(self.num_envs)
        return self._obfilt(self.venv.reset())

    # ---- raw access and the device implementation (ppo2 Runner)
    def reset_raw(self):
        return self.venv.reset()

    def step_raw(self, actions):
        """(raw obs, raw rews, news, infos): the wrapped env's step; normalisation is left to the caller."""
        self.venv.step_async(actions)
        return self.venv.step_wait()

    def reset_raw_device(self):
        return self.venv.reset_device()

    def step_raw_device(self, actions):
        return self.venv.step_device(actions)

    def dev_reset(self, obs, out):
        """reset() on the device: ret = 0, out float32 [N, D] = the filtered observations obs [N, ...] (float32 or
        float64 CUDA tensor), ob_rms updated."""
        dev = self._push(obs.device)
        dev.ret.zero_()
        self._dev_obfilt(dev, obs, out)

    def dev_step(self, obs, rews, news, obs_out, rew_out):
        """step_wait() on the device from the raw step: obs [N, ...] and rews [N] (float32 or float64), news uint8 [N];
        writes the float32 observations [N, D] and rewards [N] the Runner stores."""
        from .. import ops
        dev = self._push(obs.device)
        ops.vecnorm_rewards(rews, news, dev.ret, dev.rt, self.gamma, self.epsilon, self.cliprew, rew_out)
        self._dev_obfilt(dev, obs, obs_out)

    def _dev_obfilt(self, dev, obs, out):
        from .. import ops
        if dev.ob is not None:
            ops.vecnorm_moments(obs, dev.ws)
            ops.vecnorm_combine(dev.ob, dev.ws, obs.shape[0], self.epsilon, obs.dtype == torch.float32)
        ops.vecnorm_normalize(obs, dev.ob, self.clipob, out)


class _VecNormDevice:
    """Device copy of VecNormalize's state: float64 [mean(D) | var(D) | std(D) | count] per RunningMeanStd (the
    layout of the b200rl_vecnorm kernels), ret [N], and the batch-moment workspace."""

    def __init__(self, vn, device):
        self.device = device
        f64 = dict(dtype=torch.float64, device=device)
        D = int(np.prod(vn.observation_space.shape))
        self.ob = torch.zeros(3 * D + 1, **f64) if vn._ob_rms is not None else None
        self.rt = torch.zeros(4, **f64) if vn._ret_rms is not None else None
        self.ret = torch.zeros(vn.num_envs, **f64)
        self.ws = torch.zeros(2 * D, **f64)

    def fits(self, vn, device):
        return self.device == device and (self.ob is None) == (vn._ob_rms is None) and \
            (self.rt is None) == (vn._ret_rms is None) and self.ret.numel() == np.size(vn._ret)

    @staticmethod
    def _pack(rms, eps):
        mean = np.asarray(rms.mean, np.float64).ravel()
        var = np.asarray(rms.var, np.float64).ravel()
        return np.concatenate([mean, var, np.sqrt(var + eps), [np.float64(rms.count)]])

    def upload(self, vn):
        if self.ob is not None:
            self.ob.copy_(torch.from_numpy(self._pack(vn._ob_rms, vn.epsilon)))
        if self.rt is not None:
            self.rt.copy_(torch.from_numpy(self._pack(vn._ret_rms, vn.epsilon)))
        self.ret.copy_(torch.from_numpy(np.ascontiguousarray(vn._ret, dtype=np.float64)))

    def download(self, vn):
        for t, rms in ((self.ob, vn._ob_rms), (self.rt, vn._ret_rms)):
            if t is None:
                continue
            a = t.cpu().numpy()
            shape = np.shape(rms.mean)
            n = int(np.prod(shape))
            rms.mean = a[:n].reshape(shape).copy()
            rms.var = a[n:2 * n].reshape(shape).copy()
            rms.count = np.float64(a[3 * n])
        vn._ret = self.ret.cpu().numpy().copy()


class VecMonitor(VecEnvWrapper):
    """vec_monitor.py:7-55: per-env episode return / length bookkeeping for a whole VecEnv; finished episodes are
    reported as info['episode'] = {'r','l','t'} (what ppo2.learn's epinfobuf consumes) and optionally appended to a
    monitor.csv."""

    def __init__(self, venv, filename=None, keep_buf=0, info_keywords=()):
        import time
        from collections import deque
        super().__init__(venv)
        self.eprets = self.eplens = None
        self.epcount = 0
        self.tstart = time.time()
        self.info_keywords = info_keywords
        self.results_writer = None
        if filename:
            from ..bench.monitor import ResultsWriter
            self.results_writer = ResultsWriter(filename, header={'t_start': self.tstart}, extra_keys=info_keywords)
        self.keep_buf = keep_buf
        if keep_buf:
            self.epret_buf, self.eplen_buf = deque([], maxlen=keep_buf), deque([], maxlen=keep_buf)

    def reset(self):
        obs = self.venv.reset()
        self.eprets = np.zeros(self.num_envs, 'f')
        self.eplens = np.zeros(self.num_envs, 'i')
        return obs

    def step_wait(self):
        import time
        obs, rews, dones, infos = self.venv.step_wait()
        self.eprets += rews
        self.eplens += 1
        infos = list(infos)
        for i in np.nonzero(np.asarray(dones))[0]:
            info = dict(infos[i])
            ep = {'r': self.eprets[i], 'l': self.eplens[i], 't': round(time.time() - self.tstart, 6)}
            ep.update({k: info[k] for k in self.info_keywords})
            info['episode'] = ep
            if self.keep_buf:
                self.epret_buf.append(ep['r'])
                self.eplen_buf.append(ep['l'])
            self.epcount += 1
            self.eprets[i], self.eplens[i] = 0, 0
            if self.results_writer:
                self.results_writer.write_row(ep)
            infos[i] = info
        return obs, rews, dones, infos


class EpisodeStats:
    """What bench.Monitor contributes to the learner (bench/monitor.py:58-75): info['episode'] = {r, l, t}."""

    def __init__(self, env):
        import time
        self.env, self._t0, self._time = env, time.time(), time
        self.observation_space, self.action_space = env.observation_space, env.action_space
        self.r, self.l = 0.0, 0

    def reset(self):
        self.r, self.l = 0.0, 0
        return self.env.reset()

    def step(self, a):
        ob, rew, done, info = self.env.step(a)
        self.r += float(rew)
        self.l += 1
        if done:
            info = dict(info)
            info['episode'] = {"r": round(self.r, 6), "l": self.l, "t": round(self._time.time() - self._t0, 6)}
        return ob, rew, done, info


class SyntheticVecEnv(VecEnv):
    """Zero-cost host VecEnv for throughput measurement (SURVEY 8d): observations cycle through a pool of
    pre-generated batches held in PINNED host memory, rewards ~ N(0,1), dones ~ Bernoulli(p_done)."""

    def __init__(self, num_envs, ob_shape=(84, 84, 4), ob_dtype=np.uint8, n_actions=6, act_dim=None, pool=8,
                 p_done=0.01, seed=0):
        ob_space = spaces.Box(0, 255, ob_shape, ob_dtype) if np.dtype(ob_dtype) == np.uint8 else \
            spaces.Box(-10.0, 10.0, ob_shape, ob_dtype)
        ac_space = spaces.Discrete(n_actions) if act_dim is None else spaces.Box(-1.0, 1.0, (act_dim,), np.float32)
        super().__init__(num_envs, ob_space, ac_space)
        rng = np.random.RandomState(seed)
        self.pool = []
        for _ in range(pool):
            if np.dtype(ob_dtype) == np.uint8:
                a = rng.randint(0, 256, size=(num_envs,) + tuple(ob_shape), dtype=np.uint8)
            else:
                a = np.clip(rng.randn(num_envs, *ob_shape), -10, 10).astype(ob_dtype)    # vec_normalize.py:10,39 clip
            t = torch.from_numpy(a)
            if torch.cuda.is_available():
                t = t.pin_memory()
            self.pool.append(t)
        self.rews = rng.randn(64, num_envs).astype(np.float32)
        self.dones = rng.rand(64, num_envs) < p_done
        self.t = 0

    def reset(self):
        self.t = 0
        return self.pool[0].numpy()

    def step_async(self, actions):
        self.actions = actions

    def step_wait(self):
        self.t += 1
        return (self.pool[self.t % len(self.pool)].numpy(), self.rews[self.t % 64], self.dones[self.t % 64],
                _EMPTY_INFOS[:self.num_envs] if self.num_envs <= len(_EMPTY_INFOS) else [{}] * self.num_envs)


_EMPTY_INFOS = [{} for _ in range(65536)]


class DeviceSyntheticVecEnv(VecEnv):
    """Same synthetic process with every array resident in HBM (inputs already on device when the timed
    region starts: bench.py's `value`).  Exposes reset_device / step_device, which Runner detects."""

    def __init__(self, num_envs, ob_shape=(84, 84, 4), ob_dtype=np.uint8, n_actions=6, act_dim=None, pool=8,
                 p_done=0.01, seed=0, device=None):
        host = SyntheticVecEnv(num_envs, ob_shape, ob_dtype, n_actions, act_dim, pool, p_done, seed)
        super().__init__(num_envs, host.observation_space, host.action_space)
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.pool = [p.to(self.device) for p in host.pool]
        self.rews = torch.from_numpy(host.rews).to(self.device)
        self.dones = torch.from_numpy(host.dones.astype(np.uint8)).to(self.device)
        self.t = 0

    def reset_device(self):
        self.t = 0
        return self.pool[0]

    def step_device(self, actions):
        self.t += 1
        return self.pool[self.t % len(self.pool)], self.rews[self.t % 64], self.dones[self.t % 64]

    def reset(self):
        return self.reset_device().cpu().numpy()

    def step_async(self, actions):
        self.actions = actions

    def step_wait(self):
        o, r, d = self.step_device(None)
        return o.cpu().numpy(), r.cpu().numpy(), d.cpu().numpy().astype(np.bool_), [{}] * self.num_envs
