"""acer.learn (baselines/acer/acer.py): ACER on the sm_90a kernels.

The train net and the Polyak-averaged net are two PolicyNets of `build_policy(..., estimate_q=True)` over the same
structure; the Polyak net's parameter buffer is the ExponentialMovingAverage shadow.  One train call is one
graph-replayed launch sequence: gather + re-stack of the segment, train forward, Polyak forward, the loss head
(ops.acer_loss), backward, global norm, clip + RMSProp + moving average (ops.clip_rmsprop_ema), and the fp16 operand
refresh of both nets.

Out of scope: recurrent networks (the reference's own serialization test skips them for ACER), non-Discrete action
spaces, Discrete observations, and MPI / several GPUs (the reference's ACER has no MPI either).
"""
import functools
import os
import time
from collections import deque

import numpy as np
import torch

from .. import graphs, logger, ops
from ..common import spaces
from ..common.misc_util import set_global_seeds
from ..common.policies import RECURRENT_NETWORKS, PolicyNet, build_policy
from ..common.vec_env import VecFrameStack
from .buffer import Buffer
from .runner import Runner


# a2c/utils.py:161-195
def constant(p):
    return 1


def linear(p):
    return 1 - p


def middle_drop(p):
    eps = 0.75
    if 1 - p < eps:
        return eps * 0.1
    return 1 - p


def double_linear_con(p):
    p *= 2
    eps = 0.125
    if 1 - p < eps:
        return eps
    return 1 - p


def double_middle_drop(p):
    eps1 = 0.75
    eps2 = 0.25
    if 1 - p < eps1:
        if 1 - p < eps2:
            return eps2 * 0.5
        return eps1 * 0.1
    return 1 - p


schedules = {
    'linear': linear,
    'constant': constant,
    'double_linear_con': double_linear_con,
    'middle_drop': middle_drop,
    'double_middle_drop': double_middle_drop
}


class Scheduler(object):
    """a2c/utils.py:197-212."""

    def __init__(self, v, nvalues, schedule):
        self.n = 0.
        self.v = v
        self.nvalues = nvalues
        self.schedule = schedules[schedule]

    def value(self):
        current_value = self.v * self.schedule(self.n / self.nvalues)
        self.n += 1.
        return current_value

    def value_steps(self, steps):
        return self.v * self.schedule(steps / self.nvalues)


class EpisodeStats:
    """a2c/utils.py:214-249."""

    def __init__(self, nsteps, nenvs):
        self.episode_rewards = []
        for i in range(nenvs):
            self.episode_rewards.append([])
        self.lenbuffer = deque(maxlen=40)  # rolling buffer for episode lengths
        self.rewbuffer = deque(maxlen=40)  # rolling buffer for episode rewards
        self.nsteps = nsteps
        self.nenvs = nenvs

    def feed(self, rewards, masks):
        rewards = np.reshape(rewards, [self.nenvs, self.nsteps])
        masks = np.reshape(masks, [self.nenvs, self.nsteps])
        for i in range(0, self.nenvs):
            for j in range(0, self.nsteps):
                self.episode_rewards[i].append(rewards[i][j])
                if masks[i][j]:
                    l = len(self.episode_rewards[i])
                    s = sum(self.episode_rewards[i])
                    self.lenbuffer.append(l)
                    self.rewbuffer.append(s)
                    self.episode_rewards[i] = []

    def mean_length(self):
        if self.lenbuffer:
            return np.mean(self.lenbuffer)
        else:
            return 0  # on the first params dump, no episodes are finished

    def mean_reward(self):
        if self.rewbuffer:
            return np.mean(self.rewbuffer)
        else:
            return 0


NAMES = ['loss', 'loss_q', 'entropy', 'loss_policy', 'loss_f', 'loss_bc', 'explained_variance', 'norm_grads']
NAMES_TR = ['norm_grads_q', 'norm_grads_policy', 'avg_norm_grads_f', 'avg_norm_k', 'avg_norm_g', 'avg_norm_k_dot_g',
            'avg_norm_adj']


def check_supported(policy):
    if policy.network in RECURRENT_NETWORKS or policy.network in ("lnlstm", "cnn_lnlstm"):
        raise NotImplementedError(f"acer: recurrent networks ({policy.network!r}) are not supported")
    if not spaces.is_discrete(policy.ac_space):
        raise NotImplementedError("acer works only with Discrete action spaces")
    if spaces.is_discrete(policy.ob_space) or spaces.is_multi_discrete(policy.ob_space):
        raise NotImplementedError("acer: Discrete / MultiDiscrete observations are not supported")


class Model(object):
    def __init__(self, policy, ob_space, ac_space, nenvs, nsteps, ent_coef, q_coef, gamma, max_grad_norm, lr,
                 rprop_alpha, rprop_epsilon, total_timesteps, lrschedule,
                 c, trust_region, alpha, delta, device=None):
        if not torch.cuda.is_available():
            raise RuntimeError("baselines_b200.acer.Model needs a CUDA device: the learner hot path is hand-written "
                               "sm_90a CUDA and has no CPU fallback")
        check_supported(policy)
        self.device = dev = torch.device(device) if device is not None else torch.device("cuda",
                                                                                          torch.cuda.current_device())
        self.nenvs, self.nsteps, self.nact = nenvs, nsteps, ac_space.n
        self.nbatch = nenvs * nsteps
        self.rows = R = nenvs * (nsteps + 1)
        self.ent_coef, self.q_coef, self.gamma = float(ent_coef), float(q_coef), float(gamma)
        self.max_grad_norm = max_grad_norm
        self.rprop_alpha, self.rprop_epsilon = float(rprop_alpha), float(rprop_epsilon)
        self.c, self.trust_region, self.alpha, self.delta = float(c), bool(trust_region), float(alpha), float(delta)
        self.ob_shape = tuple(ob_space.shape)
        with torch.cuda.device(dev):
            # acer_model/...: the numpy global stream feeds ortho_init, in the reference's creation order
            self.net = PolicyNet(policy, R, dev, rng=np.random, scope="acer_model")
            # the Polyak net: same structure, no draws from the global stream; its parameters are the moving average
            self.polyak = PolicyNet(policy, R, dev, rng=np.random.RandomState(0), scope="acer_model")
            self.shadow = self.polyak.store.params
            self.shadow.copy_(self.net.store.params)
            self.polyak.refresh()
            self.ms = self.net.store.m                         # RMSProp slot, initialised to ones (TF's default)
            self.ms.fill_(1.0)
            self.lr_dev = torch.zeros(1, dtype=torch.float32, device=dev)
            self.sumsq = torch.zeros(3, dtype=torch.float64, device=dev)
            self.head_stats = torch.zeros(12, dtype=torch.float64, device=dev)
            self.stats_out = torch.zeros(15, dtype=torch.float64, device=dev)
            in_u8 = self.net.tower_pi.in_u8
            self.obs_buf = torch.zeros((R,) + self.ob_shape, dtype=torch.uint8 if in_u8 else torch.float32, device=dev)
            self.a_buf = torch.zeros(nenvs, nsteps, dtype=torch.int64, device=dev)
            self.r_buf = torch.zeros(nenvs, nsteps, dtype=torch.float32, device=dev)
            self.mu_buf = torch.zeros(nenvs, nsteps, self.nact, dtype=torch.float32, device=dev)
            self.d_buf = torch.zeros(nenvs, nsteps, dtype=torch.uint8, device=dev)
            self.m_buf = torch.zeros(nenvs, nsteps + 1, dtype=torch.uint8, device=dev)
            self._gsave = torch.zeros_like(self.net.store.grads)
            net = self.net
            self._dsave = [torch.zeros_like(t) for t in ((net.dhead,) if net.head is not None else (net.dpi, net.dv))]
            self._act_x = torch.zeros((nenvs,) + self.ob_shape, dtype=self.obs_buf.dtype, device=dev)
            self._act_a = torch.zeros(nenvs, dtype=torch.int64, device=dev)
            self._act_mu = torch.zeros(nenvs, self.nact, dtype=torch.float32, device=dev)
            self._act_v = torch.zeros(nenvs, dtype=torch.float32, device=dev)
            self._act_nlp = torch.zeros(nenvs, dtype=torch.float32, device=dev)
        self.lr = Scheduler(v=lr, nvalues=total_timesteps, schedule=lrschedule)
        self.names_ops = NAMES + (NAMES_TR if self.trust_region else [])
        # the sampler's Philox key comes from torch's generator (seeded by set_global_seeds), so numpy's global
        # stream sees exactly the reference's draws
        self._rng_seed = int(torch.randint(0, 2 ** 31 - 1, (1,)).item())
        self.graphs = graphs.GraphCache()
        self.initial_state = None
        self.train_model = self.step_model = self

    # ------------------------------------------------------------------------------------ act path
    def _stage_obs(self, observation):
        x = torch.from_numpy(np.ascontiguousarray(observation)) if not torch.is_tensor(observation) else observation
        B = x.shape[0]
        if B > self.rows:
            raise ValueError(f"batch {B} exceeds the workspace capacity {self.rows}")
        dst = self._act_x if B == self.nenvs else torch.zeros((B,) + self.ob_shape, dtype=self.obs_buf.dtype,
                                                              device=self.device)
        dst.copy_(x.reshape(dst.shape).to(dst.dtype))
        return dst, B

    def step_device(self, observation, actions, mu):
        """acer.py:213-214 `_step` into device tensors actions int64 [B] and mu float32 [B, nA]."""
        with torch.cuda.device(self.device):
            x, B = self._stage_obs(observation)
            net = self.net

            def body():
                net.forward(x, B, masks=False)
                ops.acer_step(net.pi_out, net.ld_pi, self.nact, actions, mu, B, seed=self._rng_seed,
                              offset_dev=net.rng_ctr)
                ops.counter_add(net.rng_ctr, 1)
            if B == self.nenvs:
                self.graphs.run(("act", actions.data_ptr(), mu.data_ptr()), body)
            else:
                body()

    def _step(self, observation, **kwargs):
        """(actions, mus, states) as numpy, like step_model._evaluate([action, step_model_p, state])."""
        with torch.cuda.device(self.device):
            B = np.shape(observation)[0]
            a, mu = (self._act_a, self._act_mu) if B == self.nenvs else (
                torch.zeros(B, dtype=torch.int64, device=self.device),
                torch.zeros(B, self.nact, dtype=torch.float32, device=self.device))
            self.step_device(observation, a, mu)
            return a.cpu().numpy(), mu.cpu().numpy(), None

    def step(self, observation, **kwargs):
        """PolicyWithValue.step (policies.py:77-96): (actions, q rows [B, nA], state None, neglogp)."""
        with torch.cuda.device(self.device):
            x, B = self._stage_obs(observation)
            net = self.net
            v = torch.zeros(B, dtype=torch.float32, device=self.device)
            a = torch.zeros(B, dtype=torch.int64, device=self.device)
            nlp = torch.zeros(B, dtype=torch.float32, device=self.device)
            net.forward(x, B, masks=False)
            ops.cat_step(net.pi_out, net.ld_pi, self.nact, net.v_out, net.ld_v, a, v, nlp, B, seed=self._rng_seed,
                         offset_dev=net.rng_ctr)
            ops.counter_add(net.rng_ctr, 1)
            q = net.v_out[:B, :self.nact].cpu().numpy()
            return a.cpu().numpy(), q, None, nlp.cpu().numpy()

    # ------------------------------------------------------------------------------------ train path
    def _backward_norm(self, slot):
        """Backward of the current head gradients into store.grads, the frozen identity block zeroed, and its squared
        global norm into sumsq[slot]."""
        store = self.net.store
        store.grads.zero_()
        self.net.backward(self.rows, 1.0 / self.nbatch)
        self.net.freeze_identity()
        ops.sumsq(store.grads, self.sumsq[slot:slot + 1])

    def _partial_norms(self):
        """norm_grads_policy / norm_grads_q (acer.py:175-176): the trunk receives both parts, so each is a backward of
        its own from the head gradient with the other part zeroed.  The fused gradient is saved and put back, so the
        update does not depend on whether the statistics were asked for."""
        net, store = self.net, self.net.store
        self._gsave.copy_(store.grads)
        heads = (net.dhead,) if net.head is not None else (net.dpi, net.dv)
        for s, h in zip(self._dsave, heads):
            s.copy_(h)
        net.dv.zero_()
        self._backward_norm(2)                                  # policy part
        for s, h in zip(self._dsave, heads):
            h.copy_(s)
        net.dpi[:, :self.nact].zero_()
        self._backward_norm(1)                                  # Q part
        for s, h in zip(self._dsave, heads):
            h.copy_(s)
        store.grads.copy_(self._gsave)

    def _train_body(self, src, idx, with_stats, obs):
        net, pol = self.net, self.polyak
        R, nA = self.rows, self.nact
        if obs is not None:
            self.obs_buf.copy_(obs.reshape(self.obs_buf.shape))
        elif src is not None:
            ops.acer_stack_obs(src.enc_obs, idx, self.nenvs, self.nsteps, src.nstack, src.dones, self.obs_buf)
        if src is not None:
            ops.acer_take(idx, self.nenvs, self.nsteps, nA, src.arrays()[1:],
                          (self.a_buf, self.r_buf, self.mu_buf, self.d_buf, self.m_buf))
        x = self.obs_buf.reshape(R, -1) if not net.tower_pi.in_u8 else self.obs_buf
        net.forward(x, R)
        pol.forward(x, R, masks=False)
        ops.acer_loss(net.pi_out, net.ld_pi, net.v_out, net.ld_v, pol.pi_out, pol.ld_pi, self.a_buf, self.r_buf,
                      self.d_buf, self.mu_buf, self.nenvs, self.nsteps, nA, self.gamma, self.c, self.delta,
                      self.q_coef, self.ent_coef, self.trust_region, net.dpi, net.ld_dpi, net.dv, net.ld_dv,
                      self.head_stats)
        self._backward_norm(0)
        if with_stats:
            self._partial_norms()
        store = net.store
        ops.clip_rmsprop_ema(store.params, store.grads, self.ms, self.shadow, self.lr_dev, self.max_grad_norm or 0.0,
                             self.sumsq, self.rprop_alpha, self.rprop_epsilon, self.alpha)
        net.refresh()
        pol.refresh()

    def train_device(self, src, idx, steps, with_stats=True, obs=None):
        """One train call (acer.py:202-211) from a device segment ring `src` (buffer.Segment) at slots idx
        (int64 [nenv], None: slot 0), or, src None, from the model's staging buffers.  obs: stacked observations
        [nenv, nsteps + 1, *ob_shape] to train from instead of re-stacking src's frames.  Returns the device float64
        statistics: the 12 of ops.acer_loss, then sumsq of the full / Q / policy gradients."""
        with torch.cuda.device(self.device):
            ops.set_scalars(self.lr_dev, self.lr.value_steps(steps))
            key = ("train", with_stats) + tuple(None if t is None else t.data_ptr() for t in (
                None if src is None else src.enc_obs, idx, obs))
            self.graphs.run(key, lambda: self._train_body(src, idx, with_stats, obs))
            return self.head_stats, self.sumsq

    def values_of(self, head_stats, sumsq):
        """The reference's run_ops values (8, or 15 with the trust region) from the device statistics."""
        h = head_stats.cpu().numpy()
        s = np.sqrt(sumsq.cpu().numpy())
        vals = list(h[:7]) + [s[0]]
        if self.trust_region:
            vals += [s[1], s[2], h[11], h[7], h[8], h[9], h[10]]
        return vals

    def train(self, obs, actions, rewards, dones, mus, states, masks, steps):
        """acer.py:202-211 on host arrays: obs [nenv * (nsteps + 1), *ob_shape] env-major, actions / rewards / dones
        [nenv * nsteps], mus [nenv * nsteps, nA]; states and masks are for recurrent policies, which are not
        supported.  Returns (names_ops, values)."""
        if states is not None:
            raise NotImplementedError("acer: recurrent policies are not supported")
        with torch.cuda.device(self.device):
            up = lambda a, dst: dst.copy_(torch.from_numpy(np.ascontiguousarray(a)).reshape(dst.shape).to(dst.dtype))
            up(obs, self.obs_buf)
            up(actions, self.a_buf)
            up(rewards, self.r_buf)
            up(np.asarray(dones).astype(np.uint8), self.d_buf)
            up(mus, self.mu_buf)
            h, s = self.train_device(None, None, steps)
            return list(self.names_ops), self.values_of(h, s)

    # ------------------------------------------------------------------------------------ checkpoints
    def save(self, save_path):
        """tf_util.save_variables: {TF name: array} of the trainable variables only, like the reference (the Polyak
        shadow and the RMSProp slots are not saved)."""
        import joblib
        d = dict(self.net.store.export_tf("params"))
        dirname = os.path.dirname(save_path)
        if dirname:
            os.makedirs(dirname, exist_ok=True)
        joblib.dump(d, save_path)

    def load(self, load_path):
        """tf_util.load_variables: the trainable variables; the shadow and the RMSProp slots keep their values."""
        import joblib
        d = joblib.load(os.path.expanduser(load_path))
        self.net.store.import_tf({k: v for k, v in d.items() if k in self.net.store.tf_map}, "params")
        self.net.refresh()

    def get_params(self):
        return self.net.store.export_tf("params")

    def get_polyak_params(self):
        return self.polyak.store.export_tf("params")


class Acer():
    def __init__(self, runner, model, buffer, log_interval):
        self.runner = runner
        self.model = model
        self.buffer = buffer
        self.log_interval = log_interval
        self.tstart = None
        self.episode_stats = EpisodeStats(runner.nsteps, runner.nenv)
        self.steps = None

    def call(self, on_policy):
        runner, model, buffer, steps = self.runner, self.model, self.buffer, self.steps
        log = on_policy and (int(steps / runner.nbatch) % self.log_interval == 0)
        if on_policy:
            rewards, dones = runner.run()
            self.episode_stats.feed(rewards, dones)
            if buffer is not None:
                buffer.put(*[a[0] for a in runner.seg.arrays()])
            h, s = model.train_device(runner.seg, None, steps, with_stats=log, obs=runner.mb_obs)
        else:
            # get obs, actions, rewards, mus, dones from buffer.
            idx = buffer.sample_slots()
            h, s = model.train_device(buffer.ring, idx, steps, with_stats=log)

        if log:
            values_ops = model.values_of(h, s)
            logger.record_tabular("total_timesteps", steps)
            logger.record_tabular("fps", int(steps / (time.time() - self.tstart)))
            # IMP: In EpisodicLife env, during training, we get done=True at each loss of life, not just at the terminal state.
            # Thus, this is mean until end of life, not end of episode.
            # For true episode rewards, see the monitor files in the log folder.
            logger.record_tabular("mean_episode_length", self.episode_stats.mean_length())
            logger.record_tabular("mean_episode_reward", self.episode_stats.mean_reward())
            for name, val in zip(model.names_ops, values_ops):
                logger.record_tabular(name, float(val))
            logger.dump_tabular()


def learn(network, env, seed=None, nsteps=20, total_timesteps=int(80e6), q_coef=0.5, ent_coef=0.01,
          max_grad_norm=10, lr=7e-4, lrschedule='linear', rprop_epsilon=1e-5, rprop_alpha=0.99, gamma=0.99,
          log_interval=100, buffer_size=50000, replay_ratio=4, replay_start=10000, c=10.0,
          trust_region=True, alpha=0.99, delta=1, load_path=None, **network_kwargs):
    '''
    Main entrypoint for ACER (Actor-Critic with Experience Replay) algorithm (https://arxiv.org/pdf/1611.01224.pdf),
    with the reference's parameters and defaults (baselines/acer/acer.py:275-343).  Returns the Model.
    '''
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        raise NotImplementedError("acer runs on one GPU in one process (the reference's ACER has no MPI)")
    print("Running Acer Simple")
    print(locals())
    set_global_seeds(seed)
    if not isinstance(env, VecFrameStack):
        env = VecFrameStack(env, 1)

    policy = build_policy(env, network, estimate_q=True, **network_kwargs)
    check_supported(policy)
    nenvs = env.num_envs
    ob_space = env.observation_space
    ac_space = env.action_space

    model = Model(policy=policy, ob_space=ob_space, ac_space=ac_space, nenvs=nenvs, nsteps=nsteps,
                  ent_coef=ent_coef, q_coef=q_coef, gamma=gamma,
                  max_grad_norm=max_grad_norm, lr=lr, rprop_alpha=rprop_alpha, rprop_epsilon=rprop_epsilon,
                  total_timesteps=total_timesteps, lrschedule=lrschedule, c=c,
                  trust_region=trust_region, alpha=alpha, delta=delta)

    if load_path is not None:
        model.load(load_path)

    runner = Runner(env=env, model=model, nsteps=nsteps)
    if replay_ratio > 0:
        buffer = Buffer(env=env, nsteps=nsteps, size=buffer_size, device=model.device)
    else:
        buffer = None
    nbatch = nenvs * nsteps
    acer = Acer(runner, model, buffer, log_interval)
    acer.tstart = time.time()

    for acer.steps in range(0, total_timesteps, nbatch):  # nbatch samples, 1 on_policy call and multiple off-policy calls
        acer.call(on_policy=True)
        if replay_ratio > 0 and buffer.has_atleast(replay_start):
            n = np.random.poisson(replay_ratio)
            for _ in range(n):
                acer.call(on_policy=False)  # no simulation steps in this

    return model
