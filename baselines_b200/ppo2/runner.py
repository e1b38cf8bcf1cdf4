"""PPO2 rollout collection with an HBM-resident rollout buffer and the GAE scan on device.

Drop-in for baselines/ppo2/runner.py Runner (+ common/runners.py AbstractEnvRunner):
  * `Runner(env=, model=, nsteps=, gamma=, lam=)`, `.run()` returns the reference tuple
    (obs, returns, masks, actions, values, neglogpacs, states, epinfos) as flat env-major numpy arrays
    (sf01 layout, runner.py:66-74) -- used for parity tests and by foreign callers;
  * `.run_device()` returns a `Rollout` handle whose arrays never leave HBM; the learner indexes it with
    the shuffled minibatch indices (ppo2.py:157-165) through `Rollout.src_index`.
Per env step only the observation (host->device) and the actions (device->host) cross PCIe.
"""
import numpy as np
import torch

from .. import ops


class Rollout:
    """Time-major [T, N] rollout arrays in HBM.  Flat env-major index i = e*T + t (runner.py:69-74) maps to
    buffer offset t*N + e."""

    def __init__(self, T, N, obs_store_shape, obs_dtype, discrete, act_dim, device, act_dtype=None, state_dim=0):
        """discrete: int64 [T, N] actions (Discrete); otherwise [T, N, act_dim] rows of act_dtype (float32 for Box and
        MultiBinary, int64 for MultiDiscrete).  state_dim > 0 (recurrent policies): states0 float32 [N, state_dim] holds
        the policy state at the start of the rollout (runner.py:31 mb_states)."""
        self.T, self.N, self.device = T, N, device
        f32 = dict(dtype=torch.float32, device=device)
        self.obs = torch.zeros((T, N) + tuple(obs_store_shape), dtype=obs_dtype, device=device)
        self.rewards = torch.zeros(T, N, **f32)
        self.values = torch.zeros(T, N, **f32)
        self.neglogpacs = torch.zeros(T, N, **f32)
        self.dones = torch.zeros(T, N, dtype=torch.uint8, device=device)        # done BEFORE step t (runner.py:34)
        self.actions = torch.zeros((T, N) if discrete else (T, N, act_dim),
                                   dtype=torch.int64 if discrete else (act_dtype or torch.float32), device=device)
        self.advs = torch.zeros(T, N, **f32)
        self.returns = torch.zeros(T, N, **f32)
        self.last_values = torch.zeros(N, **f32)
        self.last_dones = torch.zeros(N, dtype=torch.uint8, device=device)
        self.states0 = torch.zeros(N, state_dim, **f32) if state_dim else None
        self._arange = None

    @property
    def nbatch(self):
        return self.T * self.N

    def flat(self, name):
        a = getattr(self, name)
        return a.view((self.T * self.N,) + tuple(a.shape[2:]))

    def shuffle_buffer(self):
        """Device home of the current epoch's shuffled sample offsets (ops.shuffle_indices)."""
        if self._arange is None:
            self._arange = torch.empty(self.T * self.N, dtype=torch.int64, device=self.device)
        return self._arange

    def src_index(self, inds):
        """env-major flat indices (device int64) -> buffer offsets."""
        return (inds % self.T) * self.N + torch.div(inds, self.T, rounding_mode="floor")

    def to_reference_numpy(self, name):
        """sf01(arr): swap axes 0,1 and flatten (runner.py:69-74) on the host copy."""
        a = getattr(self, name).cpu().numpy()
        s = a.shape
        return a.swapaxes(0, 1).reshape(s[0] * s[1], *s[2:])


class Runner:
    def __init__(self, *, env, model, nsteps, gamma, lam):
        self.env, self.model, self.nsteps = env, model, nsteps
        self.lam, self.gamma = lam, gamma
        self.nenv = nenv = env.num_envs if hasattr(env, 'num_envs') else 1
        ob_space = env.observation_space
        self.batch_ob_shape = (nenv * nsteps,) + tuple(ob_space.shape)
        self.device = model.device
        net = model.net
        from ..common.vec_env import VecEnvWrapper
        # wrappers forward unknown attributes to the env they wrap: a device env hidden under a wrapper must be
        # stepped through the wrapper, not around it
        self.device_env = hasattr(env, "step_device") and not isinstance(env, VecEnvWrapper)
        self.u8 = net.tower_pi.in_u8
        # vector observations are kept as the float32 the env produced (the reference never narrows them,
        # common/input.py:56-57); the encode kernel reads them through the minibatch indices
        store_shape = tuple(ob_space.shape) if self.u8 else (net.tower_pi.raw_dim,)
        self.rollout = Rollout(nsteps, nenv, store_shape, torch.uint8 if self.u8 else torch.float32, net.pd == "cat",
                               net.act_dim, self.device, act_dtype=net.action_dtype,
                               state_dim=2 * net.nlstm if net.recurrent else 0)
        # pinned staging for the per-step host<->device traffic
        pin = torch.cuda.is_available()
        np_dtype = np.dtype(ob_space.dtype.name) if hasattr(ob_space.dtype, "name") else np.dtype(ob_space.dtype)
        self._obs_pin = torch.zeros((nenv,) + tuple(ob_space.shape), dtype=torch.from_numpy(np.zeros(1, np_dtype)).dtype)
        if pin:
            self._obs_pin = self._obs_pin.pin_memory()
        self.obs = self._obs_pin.numpy()                                       # runners.py:10 self.obs
        self._act_pin = torch.zeros(net.action_shape(nenv), dtype=net.action_dtype)
        self._rew_host = torch.zeros(nsteps, nenv, dtype=torch.float32)
        self._done_host = torch.zeros(nsteps, nenv, dtype=torch.uint8)
        if pin:
            self._act_pin, self._rew_host, self._done_host = (t.pin_memory() for t in
                                                              (self._act_pin, self._rew_host, self._done_host))
        self._f32_pin = None
        if not self.u8:
            self._f32_pin = torch.zeros(nenv, net.tower_pi.raw_dim, dtype=torch.float32)
            if pin:
                self._f32_pin = self._f32_pin.pin_memory()
        # host copy of the encoder's out-of-range flag (vector observations), read after a synchronisation the runner
        # makes anyway: per step with a host env, at the start of the next rollout with a device env
        self._over_pin = torch.zeros(1, dtype=torch.int32)
        if pin:
            self._over_pin = self._over_pin.pin_memory()
        self._over_ev = torch.cuda.Event()
        self._f32_sync = torch.cuda.Event()
        self._ro_copied = torch.cuda.Event()          # end-of-rollout H2D copies of the pinned reward / done staging
        self._cur = torch.zeros((nenv,) + store_shape, dtype=self.rollout.obs.dtype, device=self.device)
        self._obs_src = None
        # VecFrameStack on the device: only the new frames cross PCIe, the stack lives in the rollout buffer
        # (only when VecFrameStack is the OUTERMOST wrapper: step_frames() would bypass anything wrapped around it)
        from ..common.vec_env import VecFrameStack, VecNormalize
        self.fs = isinstance(env, VecFrameStack) and bool(env.frame_stack_device) and self.u8 and \
            not self.device_env and pin
        # VecNormalize on the device (likewise only when OUTERMOST): the raw float observations and rewards are
        # normalised by the b200rl_vecnorm kernels straight into the rollout buffer, the statistics stay in HBM
        self.vn = isinstance(env, VecNormalize) and bool(env.normalize_device) and not self.u8 and \
            not getattr(net.tower_pi, "onehot_n", 0) and np_dtype in (np.float32, np.float64) and pin
        self.vn_dev_env = self.vn and hasattr(env.venv, "step_device") and not isinstance(env.venv, VecEnvWrapper)
        if self.device_env:
            self._dev_obs = env.reset_device()
        elif self.vn:
            self._vn_obs = torch.zeros(tuple(self._obs_pin.shape), dtype=self._obs_pin.dtype, device=self.device)
            self._vn_rew = {}                                # reward dtype -> (pinned staging, device buffer)
            self._news_pin = torch.zeros(nenv, dtype=torch.uint8).pin_memory()
            self._news_dev = torch.zeros(nenv, dtype=torch.uint8, device=self.device)
            with torch.cuda.device(self.device):
                if self.vn_dev_env:
                    env.dev_reset(env.reset_raw_device(), self._cur)
                else:
                    self._vn_stage(env.reset_raw())
                    env.dev_reset(self._vn_obs, self._cur)
        elif self.fs:
            c = env.frame_channels
            fshape = (nenv,) + tuple(ob_space.shape[:-1]) + (c,)
            self._frame_pin = torch.zeros(fshape, dtype=torch.uint8).pin_memory()
            self._frame_dev = torch.zeros(fshape, dtype=torch.uint8, device=self.device)
            self._news_pin = torch.ones(nenv, dtype=torch.uint8).pin_memory()
            self._news_dev = torch.zeros(nenv, dtype=torch.uint8, device=self.device)
            self._zero_obs = torch.zeros_like(self._cur)
            # the upload of the new frames (PCIe-bound: 29 MB per step at cfg-2) is pipelined against the acting
            # forward: the envs are cut into chunks, and while chunk k+1 is still in flight on the copy stream the
            # frame-stack update and the policy forward of chunk k already run
            import os
            k = int(os.environ.get("B200RL_ACT_CHUNKS", 4 if (nenv % 4 == 0 and nenv >= 2048) else 1))
            self.act_chunks = k if (k > 1 and nenv % k == 0) else 1
            self._copy_stream = torch.cuda.Stream(device=self.device)
            self._chunk_ev = [torch.cuda.Event() for _ in range(self.act_chunks)]
            # reset(): stack = 0, newest slot = first frame  (vec_frame_stack.py:27-31)
            self._stack_frames(env.reset_frames(), np.ones(nenv, dtype=np.bool_), self._zero_obs, self._cur)
        else:
            self._take_obs(env.reset())                                        # runners.py:11
        self.states = model.initial_state
        self.dones = np.zeros(nenv, dtype=np.bool_)                            # runners.py:14
        self._dev_dones = torch.zeros(nenv, dtype=torch.uint8, device=self.device)
        # recurrent policies (runner.py:31-36): the state lives on the device and is advanced in place by every acting
        # pass; the mask of step t (done before step t) reaches the device before that step's pass
        self.recurrent = net.recurrent
        if self.recurrent:
            st = np.zeros((nenv, 2 * net.nlstm), np.float32) if self.states is None else self.states
            self._state_dev = torch.from_numpy(np.ascontiguousarray(st, dtype=np.float32)).to(self.device)
            self._mask_dev = torch.zeros(nenv, dtype=torch.uint8, device=self.device)

    @property
    def _dev_steps(self):
        """The env is stepped on the device (no per-step host synchronisation): a device env, bare or under the
        device VecNormalize."""
        return self.device_env or self.vn_dev_env

    def _rnn(self):
        """step_device / value_device keywords of a recurrent policy: the state and this step's mask."""
        if not self.recurrent:
            return {}
        if self._dev_steps:
            self._mask_dev.copy_(self._dev_dones)
        else:
            self._mask_dev.copy_(torch.from_numpy(self.dones.astype(np.uint8)))
        return dict(state=self._state_dev, mask=self._mask_dev)

    def _take_obs(self, obs):
        """`self.obs[:] = obs` of the reference (runner.py:38), except that an env which already hands out
        PINNED host memory is uploaded from directly (no extra host memcpy)."""
        t = torch.from_numpy(obs) if isinstance(obs, np.ndarray) and obs.flags.c_contiguous else None
        if t is not None and t.dtype == self._obs_pin.dtype and t.shape == self._obs_pin.shape and \
                torch.cuda.is_available() and t.is_pinned():
            self._obs_src, self.obs = t, obs
        else:
            self._obs_src = None
            self.obs = self._obs_pin.numpy()
            self.obs[:] = obs

    def _vn_stage(self, obs, rews=None, news=None):
        """Raw host step -> device buffers through pinned staging (the obs directly when the env already hands out
        pinned memory of the right dtype); returns the device rewards (float32, or float64 for any other dtype)."""
        t = torch.from_numpy(obs) if isinstance(obs, np.ndarray) and obs.flags.c_contiguous else None
        if t is not None and t.dtype == self._obs_pin.dtype and t.shape == self._obs_pin.shape and t.is_pinned():
            src = t
        else:
            self._obs_pin.numpy()[...] = np.asarray(obs).reshape(self._obs_pin.shape)
            src = self._obs_pin
        self._vn_obs.copy_(src, non_blocking=True)
        if rews is None:
            return None
        rews = np.asarray(rews)
        rdt = np.float32 if rews.dtype == np.float32 else np.float64
        if rdt not in self._vn_rew:
            tdt = torch.float32 if rdt == np.float32 else torch.float64
            self._vn_rew[rdt] = (torch.zeros(self.nenv, dtype=tdt).pin_memory(),
                                 torch.zeros(self.nenv, dtype=tdt, device=self.device))
        pin, dev = self._vn_rew[rdt]
        pin.numpy()[...] = rews.reshape(self.nenv)
        dev.copy_(pin, non_blocking=True)
        self._news_pin.numpy()[...] = np.asarray(news, dtype=np.uint8).reshape(self.nenv)
        self._news_dev.copy_(self._news_pin, non_blocking=True)
        return dev

    def _stack_frames(self, frames, news, prev, out):
        """out = VecFrameStack.step_wait update (vec_frame_stack.py:17-25) of the stacked observation `prev` with
        the freshly stepped frames; frames and the done flags are the only host->device traffic."""
        t = torch.from_numpy(frames) if isinstance(frames, np.ndarray) and frames.flags.c_contiguous else None
        if t is not None and t.dtype == torch.uint8 and t.shape == self._frame_pin.shape and t.is_pinned():
            src = t
        else:
            self._frame_pin.numpy()[...] = frames
            src = self._frame_pin
        self._frame_dev.copy_(src, non_blocking=True)
        self._news_pin.numpy()[...] = np.asarray(news, dtype=np.uint8)
        self._news_dev.copy_(self._news_pin, non_blocking=True)
        ops.frame_stack(prev, self._frame_dev, self._news_dev, out, self.env.nstack, self.env.frame_channels)

    def _stack_and_act_chunked(self, frames, news, prev, t1):
        """Frames of step t1 arrive: per env chunk, upload (copy stream) -> frame-stack update into rollout.obs[t1] ->
        policy step into the rollout slots of t1, so the forward of chunk k overlaps the upload of chunk k+1."""
        ro, model, K = self.rollout, self.model, self.act_chunks
        tsrc = torch.from_numpy(frames) if isinstance(frames, np.ndarray) and frames.flags.c_contiguous else None
        if tsrc is not None and tsrc.dtype == torch.uint8 and tsrc.shape == self._frame_pin.shape and tsrc.is_pinned():
            src = tsrc
        else:
            self._frame_pin.numpy()[...] = frames
            src = self._frame_pin
        self._news_pin.numpy()[...] = np.asarray(news, dtype=np.uint8)
        step = self.nenv // K
        cur = torch.cuda.current_stream()
        out = ro.obs[t1]
        for k in range(K):
            sl = slice(k * step, (k + 1) * step)
            with torch.cuda.stream(self._copy_stream):
                self._frame_dev[sl].copy_(src[sl], non_blocking=True)
                self._news_dev[sl].copy_(self._news_pin[sl], non_blocking=True)
                self._chunk_ev[k].record(self._copy_stream)
            cur.wait_event(self._chunk_ev[k])
            ops.frame_stack(prev[sl], self._frame_dev[sl], self._news_dev[sl], out[sl], self.env.nstack,
                            self.env.frame_channels)
            model.step_device(out[sl], ro.actions[t1][sl], ro.values[t1][sl], ro.neglogpacs[t1][sl], persistent=True)

    # -- stage the current observation into `dst` (rollout.obs[t] or a temp) in the network's input format
    def _upload_obs(self, dst):
        if self.device_env:
            src = self._dev_obs
            dst.copy_(src if self.u8 else src.reshape(self.nenv, -1))
            return
        src = self._obs_src if self._obs_src is not None else self._obs_pin
        if self.u8:
            dst.copy_(src, non_blocking=True)
        elif src.dtype == torch.float32:
            dst.copy_(src.reshape(self.nenv, -1), non_blocking=True)
        else:
            # integer (Discrete) / float64 observations: to_float on the host, one H2D copy (input.py:54-57)
            self._f32_sync.synchronize()                     # the previous upload has left the staging buffer
            np.copyto(self._f32_pin.numpy(), src.numpy().reshape(self.nenv, -1), casting="unsafe")
            dst.copy_(self._f32_pin, non_blocking=True)
            self._f32_sync.record()

    def run_device(self, noise=None):
        """Collect nsteps transitions; returns (Rollout, epinfos).  noise: optional [T, N, nout] float32 host
        array of injected sampling noise (parity tests; nout = nA, sum(nvec), n or d)."""
        ro, model, T, N = self.rollout, self.model, self.nsteps, self.nenv
        epinfos = []
        with torch.cuda.device(self.device):
            nz = None if noise is None else torch.as_tensor(np.ascontiguousarray(noise), dtype=torch.float32).to(self.device)
            # the previous rollout's asynchronous upload of _rew_host / _done_host must have read the staging buffers
            # before this rollout overwrites row 0 (callers need not synchronise between run_device calls)
            self._ro_copied.synchronize()
            if not self.u8:                    # the previous rollout's flag (device envs)
                self._over_ev.synchronize()
                flag = int(self._over_pin[0])
                self._over_pin.zero_()
                model.net.check_obs_range(flag)
            if self.fs or self.vn:
                ro.obs[0].copy_(self._cur)
            if self.recurrent:
                ro.states0.copy_(self._state_dev)                              # runner.py:31 mb_states = self.states
            # chunked acting overlaps step t+1's pass with the upload; a recurrent pass waits for step t+1's mask instead
            chunked = self.fs and self.act_chunks > 1 and nz is None and not self.recurrent
            acted = False                      # step t's policy pass already issued (chunk-wise, with the upload)
            for t in range(T):
                if not (self.fs or self.vn):
                    self._upload_obs(ro.obs[t])
                if not acted:
                    model.step_device(ro.obs[t], ro.actions[t], ro.values[t], ro.neglogpacs[t],
                                      noise=None if nz is None else nz[t], persistent=True, **self._rnn())
                acted = False
                nxt = ro.obs[t + 1] if t + 1 < T else self._cur
                if self.vn_dev_env:
                    ro.dones[t].copy_(self._dev_dones)
                    obs, rew, self._dev_dones = self.env.step_raw_device(ro.actions[t])
                    self.env.dev_step(obs, rew, self._dev_dones, nxt, ro.rewards[t])
                    continue
                if self.device_env:
                    ro.dones[t].copy_(self._dev_dones)
                    self._dev_obs, rew, self._dev_dones = self.env.step_device(ro.actions[t])
                    ro.rewards[t].copy_(rew)
                    continue
                self._done_host[t] = torch.from_numpy(self.dones.astype(np.uint8))       # mb_dones.append(self.dones)
                self._act_pin.copy_(ro.actions[t], non_blocking=True)
                if not self.u8:
                    self._over_pin.copy_(model.net.tower_pi.obs_overflow, non_blocking=True)
                torch.cuda.current_stream().synchronize()
                if not self.u8:
                    model.net.check_obs_range(int(self._over_pin[0]))
                actions = self._act_pin.numpy()
                if self.model.net.pd == "mcat":
                    actions = actions.astype(np.int32)                      # distributions.py:222 tf.int32
                if self.fs:
                    frames, rewards, self.dones, infos = self.env.step_frames(actions)
                    self.dones = np.asarray(self.dones, dtype=np.bool_)
                    if chunked and t + 1 < T:
                        self._stack_and_act_chunked(frames, self.dones, ro.obs[t], t + 1)
                        acted = True
                    else:
                        self._stack_frames(frames, self.dones, ro.obs[t], ro.obs[t + 1] if t + 1 < T else self._cur)
                elif self.vn:
                    obs, rewards, self.dones, infos = self.env.step_raw(actions)
                    self.dones = np.asarray(self.dones, dtype=np.bool_)
                    rew_dev = self._vn_stage(obs, rewards, self.dones)
                    self.env.dev_step(self._vn_obs, rew_dev, self._news_dev, nxt, ro.rewards[t])
                else:
                    obs, rewards, self.dones, infos = self.env.step(actions)             # runner.py:38
                    self._take_obs(obs)
                    self.dones = np.asarray(self.dones, dtype=np.bool_)
                for info in infos:
                    maybeepinfo = info.get('episode') if info else None
                    if maybeepinfo:
                        epinfos.append(maybeepinfo)
                if not self.vn:                  # the device VecNormalize has written ro.rewards[t] already
                    self._rew_host[t] = torch.from_numpy(np.asarray(rewards, dtype=np.float32))
            # bootstrap value of the final observation (runner.py:50)
            if not (self.fs or self.vn):
                self._upload_obs(self._cur)
            model.value_device(self._cur, ro.last_values, persistent=True, **self._rnn())   # runner.py:50
            if self._dev_steps:
                ro.last_dones.copy_(self._dev_dones)
                if not self.u8:
                    self._over_pin.copy_(model.net.tower_pi.obs_overflow, non_blocking=True)
                    self._over_ev.record()
            else:
                if not self.vn:
                    ro.rewards.copy_(self._rew_host, non_blocking=True)
                ro.dones.copy_(self._done_host, non_blocking=True)
                self._ro_copied.record()
                ro.last_dones.copy_(torch.from_numpy(self.dones.astype(np.uint8)))
            # GAE(lambda) + returns (runner.py:53-65) in one kernel over the resident buffers
            ops.gae_scan(ro.rewards, ro.values, ro.dones, ro.last_values, ro.last_dones, ro.advs, ro.returns,
                         self.gamma, self.lam)
        return ro, epinfos

    def run(self, noise=None):
        """Reference-compatible return value (numpy, flat env-major)."""
        ro, epinfos = self.run_device(noise=noise)
        torch.cuda.synchronize(self.device)
        if self.u8:
            obs = ro.to_reference_numpy("obs")
        else:
            sp = self.env.observation_space
            o = ro.obs.cpu().numpy().reshape((self.nsteps, self.nenv) + tuple(sp.shape))
            obs = o.swapaxes(0, 1).reshape(self.batch_ob_shape).astype(np.dtype(sp.dtype), copy=False)
        masks = ro.to_reference_numpy("dones").astype(np.bool_)
        actions = ro.to_reference_numpy("actions")
        if self.model.net.pd == "mcat":
            actions = actions.astype(np.int32)                              # distributions.py:222 tf.int32
        states = None
        if self.recurrent:
            states = ro.states0.cpu().numpy()                               # the states at the start of the rollout
            self.states = self._state_dev.cpu().numpy()
        return (obs, ro.to_reference_numpy("returns"), masks, actions,
                ro.to_reference_numpy("values"), ro.to_reference_numpy("neglogpacs"), states, epinfos)
