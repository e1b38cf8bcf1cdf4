"""The DDPG agent (baselines/ddpg/ddpg_learner.py) on the H100 kernels.

A train step is one fixed launch sequence, captured once per batch size and replayed (graphs.GraphCache): the sample's
ring selection is the only per-step input, uploaded into a fixed buffer, and Adam's step sizes go to the device.  The
sequence (csrc/ddpg.cu, nn.py):
  target actor on obs1 -> target critic on [obs1 | mu'(obs1)] -> y = r + (1 - d) gamma Q' -> (ret_rms + Pop-Art) ->
  actor on obs0 -> ONE critic pass over 2B rows [obs0 | a] and [obs0 | mu(obs0)] -> both losses and head gradients ->
  critic backward (weight gradients from the first B rows; the second B rows only carry d/d mu down to the action
  columns) -> L2 -> actor backward through tanh' -> per-variable clip + Adam on each network.
Both gradients are taken at the parameters the step started from, as in the reference's single sess.run (:322-329).
"""
from collections import OrderedDict

import numpy as np
import torch

from .. import graphs, ops
from .models import Net


class _RunningMeanStd:
    """common/mpi_running_mean_std.py on the device: float64 state [sum(D) | sumsq(D) | count], initialised to (0,
    epsilon, epsilon), and the float32 mean / std the graph reads."""

    def __init__(self, D, device, epsilon=1e-2):
        self.D = D
        self.state = torch.zeros(2 * D + 1, dtype=torch.float64, device=device)
        self.state[D:].fill_(epsilon)
        self.mean = torch.zeros(D, dtype=torch.float32, device=device)
        self.std = torch.ones(D, dtype=torch.float32, device=device)      # sqrt(max(eps / eps - 0^2, 1e-2))

    def tf_variables(self, scope):
        st = self.state.cpu().numpy()
        shape = (self.D,) if scope == 'obs_rms' else ()
        return OrderedDict([(f'{scope}/runningsum:0', st[:self.D].reshape(shape)),
                            (f'{scope}/runningsumsq:0', st[self.D:2 * self.D].reshape(shape)),
                            (f'{scope}/count:0', st[2 * self.D])])


class DDPG:
    def __init__(self, actor, critic, memory, observation_shape, action_shape, param_noise=None, action_noise=None,
                 gamma=0.99, tau=0.001, normalize_returns=False, enable_popart=False, normalize_observations=True,
                 batch_size=128, observation_range=(-5., 5.), action_range=(-1., 1.), return_range=(-np.inf, np.inf),
                 critic_l2_reg=0., actor_lr=1e-4, critic_lr=1e-3, clip_norm=None, reward_scale=1., act_cap=256,
                 seed=None):
        """actor / critic: models.Actor / models.Critic specs.  The six network copies are built in the reference's
        creation order (actor, critic, target_actor, target_critic, param_noise_actor, adaptive_param_noise_actor), each
        taking its orthogonal initialisers from numpy's global stream; the uniform head initialisers come from their own
        stream (seeded by `seed`).  act_cap: the most observations one step() takes."""
        if observation_range[0] != -observation_range[1]:
            raise NotImplementedError("observation_range must be symmetric")
        if tuple(return_range) != (-np.inf, np.inf):
            raise NotImplementedError("return_range other than (-inf, inf)")
        from .. import nn
        self.memory, self.device = memory, memory.device
        self.gamma, self.tau = float(gamma), float(tau)
        self.normalize_observations, self.normalize_returns = bool(normalize_observations), bool(normalize_returns)
        self.enable_popart = bool(enable_popart)
        self.action_noise, self.param_noise = action_noise, param_noise
        self.action_range, self.observation_range, self.return_range = action_range, observation_range, return_range
        self.actor_lr, self.critic_lr, self.clip_norm = actor_lr, critic_lr, clip_norm
        self.reward_scale, self.batch_size = reward_scale, int(batch_size)
        self.critic_l2_reg = float(critic_l2_reg)
        self.stats_sample = None
        self.initial_state = None
        self.ob_dim = int(np.prod(observation_shape))
        self.nA = int(np.prod(action_shape))
        dev = self.device
        cap = max(self.batch_size, int(act_cap))
        self.cap = cap
        urng = np.random.RandomState(seed)
        with torch.cuda.device(dev):
            self.obs_rms = _RunningMeanStd(self.ob_dim, dev) if self.normalize_observations else None
            self.ret_rms = _RunningMeanStd(1, dev) if self.normalize_returns else None
            mk = lambda spec, kind, scope, rows: Net(spec, kind, scope, self.ob_dim, self.nA, rows, dev, np.random, urng)
            self.actor = mk(actor, 'actor', 'actor', cap)
            self.critic = mk(critic, 'critic', 'critic', 2 * cap)
            self.target_actor = mk(actor, 'actor', 'target_actor', cap)
            self.target_critic = mk(critic, 'critic', 'target_critic', cap)
            self.param_noise_actor = self.adaptive_param_noise_actor = None
            if param_noise is not None:
                self.param_noise_actor = mk(actor, 'actor', 'param_noise_actor', cap)
                self.adaptive_param_noise_actor = mk(actor, 'actor', 'adaptive_param_noise_actor', cap)
            per_var = clip_norm is not None
            self.actor_opt = nn.Optimizer(self.actor.store, eps=1e-8, max_grad_norm=clip_norm, per_variable=per_var)
            self.critic_opt = nn.Optimizer(self.critic.store, eps=1e-8, max_grad_norm=clip_norm, per_variable=per_var)
            reg = self.critic.segments(lambda k: k.endswith('/w:0') and 'output' not in k)
            self.l2_segs = torch.tensor(reg, dtype=torch.int64, device=dev)
            self.y = torch.zeros(cap, dtype=torch.float32, device=dev)
            self.losses = torch.zeros(2, dtype=torch.float32, device=dev)       # critic_loss, actor_loss
            self.q_act = torch.zeros(cap, dtype=torch.float32, device=dev)
            if param_noise is not None:
                st = self.actor.store
                jobs = []
                for k in self.actor.tf_names:
                    internal = self.actor.tf_internal(k)
                    n = int(np.prod(st.tf_map[k][2]))
                    jobs.append((st.offsets[internal], st.offsets[internal], n, 0 if 'LayerNorm' in k else 1))
                self.pn_jobs = torch.tensor(jobs, dtype=torch.int64, device=dev)
                self.pn_njobs, self.pn_max_len = len(jobs), max(j[2] for j in jobs)
                self.pn_stddev = torch.full((1,), float(param_noise.current_stddev), dtype=torch.float64, device=dev)
                self.pn_stddev32 = torch.full((1,), float(np.float32(param_noise.current_stddev)), dtype=torch.float32,
                                              device=dev)
                self.pn_dist = torch.zeros(1, dtype=torch.float32, device=dev)
                self.pn_ctr = torch.zeros(1, dtype=torch.int64, device=dev)
                self.pn_seed = int(urng.randint(0, 2 ** 31 - 1))
        self.graphs = graphs.GraphCache()

    # ---- helpers ----------------------------------------------------------------------------------------------------
    def _obs_norm(self):
        return (self.obs_rms.mean, self.obs_rms.std) if self.obs_rms is not None else (None, None)

    def _ret_norm(self):
        return (self.ret_rms.mean, self.ret_rms.std) if self.ret_rms is not None else (None, None)

    def _encode(self, net, obs, B, sel=None, act=None, act_sel=False, out=None):
        m = self.memory
        mean, std = self._obs_norm()
        ops.ddpg_encode(obs, net.x0 if out is None else out, B, self.ob_dim, net.in_pad, sel=sel, limit=m.limit,
                        mean=mean, std=std, clip=self.observation_range[1], act=act, act_sel=act_sel,
                        nA=self.nA if act is not None else 0)

    def _critic_pass(self, obs, B, sel, act, act_sel):
        """The critic over 2B rows: [obs | act] (ring rows when act_sel) and [obs | mu(obs)] of the actor's last pass."""
        c = self.critic
        self._encode(c, obs, B, sel=sel, act=act, act_sel=act_sel, out=c.x0[:B])
        self._encode(c, obs, B, sel=sel, act=self.actor.mu, out=c.x0[B:2 * B])
        c.forward(2 * B)

    def _perturb(self, dst):
        """dst <- actor + N(0, float32(current_stddev)^2) on every variable outside LayerNorm (:50-63)."""
        ops.param_perturb(self.actor.store.params, dst.store.params, self.pn_jobs, self.pn_njobs, self.pn_max_len,
                          self.pn_stddev32, self.pn_seed, self.pn_ctr)
        ops.counter_add(self.pn_ctr, 1)
        dst.refresh()

    # ---- the reference's interface ----------------------------------------------------------------------------------
    def initialize(self, sess=None):
        """Target networks <- online ones (:333-338)."""
        with torch.cuda.device(self.device):
            self.target_actor.store.params.copy_(self.actor.store.params)
            self.target_critic.store.params.copy_(self.critic.store.params)
            self.target_actor.refresh()
            self.target_critic.refresh()

    def step(self, obs, apply_noise=True, compute_Q=True):
        obs = np.asarray(obs, dtype=np.float32).reshape(-1, self.ob_dim)
        n = obs.shape[0]
        if n > self.cap:
            raise ValueError(f"step over {n} observations exceeds act_cap {self.cap}")
        perturbed = self.param_noise is not None and apply_noise
        a = self.param_noise_actor if perturbed else self.actor
        with torch.cuda.device(self.device):
            x = self.graphs.home("act_obs", self.cap, (self.ob_dim,), torch.float32, self.device)[:n]
            x.copy_(torch.from_numpy(obs))

            def body():
                self._encode(a, x, n)
                a.forward(n)
                if compute_Q:
                    if perturbed:
                        self._encode(self.actor, x, n)
                        self.actor.forward(n)
                    self._encode(self.critic, x, n, act=self.actor.mu)
                    self.critic.forward(n)
                    mean, std = self._ret_norm()
                    ops.ddpg_denorm(self.critic.out, self.critic.ld_out, mean, std, self.q_act, n)
            self.graphs.run(("act", n, perturbed, bool(compute_Q)), body)
            action = a.mu[:n].cpu().numpy()
            q = self.q_act[:n].cpu().numpy().reshape(n, 1) if compute_Q else None
        if self.action_noise is not None and apply_noise:
            noise = self.action_noise()
            assert noise.shape == action[0].shape
            action = action + noise
        action = np.clip(action, self.action_range[0], self.action_range[1])
        return action, q, None, None

    def store_transition(self, obs0, action, reward, obs1, terminal1):
        reward = np.asarray(reward) * self.reward_scale
        with torch.cuda.device(self.device):
            pos0, n = self.memory.append_batch(obs0, action, reward, obs1, terminal1)
            if self.obs_rms is not None:
                ops.ddpg_obs_rms(self.memory.obs0, pos0, self.memory.limit, n, self.ob_dim, self.obs_rms.state,
                                 self.obs_rms.mean, self.obs_rms.std)

    def train_device(self, idxs=None):
        """One train step on device; -> the float32 device vector [critic_loss, actor_loss] (no synchronisation).
        idxs: the batch's item indices (default: drawn as the reference draws them)."""
        m, B = self.memory, self.batch_size
        if idxs is None:
            idxs = m.sample_indices(B)
        B = len(idxs)
        if B > self.cap:
            raise ValueError(f"batch {B} exceeds the agent's capacity {self.cap}")
        a, c, ta, tc = self.actor, self.critic, self.target_actor, self.target_critic
        with torch.cuda.device(self.device):
            sel = self.graphs.upload("sel", m.selection(idxs), self.cap + 1, (), torch.int64, self.device)
            self.actor_opt.begin_step(self.actor_lr)
            self.critic_opt.begin_step(self.critic_lr)

            def body():
                rmean, rstd = self._ret_norm()
                self._encode(ta, m.obs1, B, sel=sel)
                ta.forward(B)
                self._encode(tc, m.obs1, B, sel=sel, act=ta.mu)
                tc.forward(B)
                ops.ddpg_target(tc.out, tc.ld_out, sel, m.limit, m.rewards, m.terminals1, rmean, rstd, self.gamma,
                                self.y, B)
                if self.normalize_returns and self.enable_popart:
                    ops.ddpg_ret_rms(self.y, B, self.ret_rms.state, rmean, rstd,
                                     popart=(c.head.w.view(-1), c.head.b, tc.head.w.view(-1), tc.head.b))
                    c.refresh()
                    tc.refresh()
                self._encode(a, m.obs0, B, sel=sel)
                a.forward(B)
                self._critic_pass(m.obs0, B, sel, m.actions, True)
                ops.ddpg_loss(c.out, c.ld_out, self.y, rmean, rstd, B, c.dout, c.ld_out, self.losses)
                a.store.grads.zero_()
                c.store.grads.zero_()
                c.critic_backward(B, 1.0 / B)
                if self.critic_l2_reg > 0:
                    ops.ddpg_l2(c.store.params, c.store.grads, self.l2_segs, self.critic_l2_reg, self.losses[:1])
                ops.ddpg_actor_dz(c.dact, c.dact.shape[1], a.mu, B, self.nA, a.dout, a.ld_out)
                a.actor_backward(B, 1.0 / B)
                self.actor_opt.apply()
                self.critic_opt.apply()
                a.refresh()
                c.refresh()
            self.graphs.run(("train", B), body)
        return self.losses

    def train(self):
        """-> (critic_loss, actor_loss) of the step, as host floats (a synchronisation)."""
        cl, al = self.train_device().cpu().numpy()
        return cl, al

    def update_target_net(self):
        ta, tc = self.target_actor, self.target_critic

        def body():
            ops.soft_update(ta.store.params, self.actor.store.params, 1.0 - self.tau, self.tau, tc.store.params,
                            self.critic.store.params)
            ta.refresh()
            tc.refresh()
        with torch.cuda.device(self.device):
            self.graphs.run(("target",), body)

    def adapt_param_noise_device(self, idxs=None):
        """-> the float32 device scalar of the distance (no synchronisation); None without parameter noise."""
        if self.param_noise is None:
            return None
        m = self.memory
        if idxs is None:
            idxs = m.sample_indices(self.batch_size)
        B = len(idxs)
        a, ad = self.actor, self.adaptive_param_noise_actor
        with torch.cuda.device(self.device):
            sel = self.graphs.upload("sel", m.selection(idxs), self.cap + 1, (), torch.int64, self.device)

            def body():
                self._perturb(ad)
                self._encode(a, m.obs0, B, sel=sel)
                a.forward(B)
                self._encode(ad, m.obs0, B, sel=sel)
                ad.forward(B)
                ops.ddpg_pn_adapt(a.mu, ad.mu, B * self.nA, self.param_noise.desired_action_stddev, self.pn_stddev,
                                  self.pn_stddev32, self.pn_dist)
            self.graphs.run(("adapt", B), body)
        return self.pn_dist

    def adapt_param_noise(self):
        if self.param_noise is None:
            return 0.
        d = float(self.adapt_param_noise_device().item())
        self.param_noise.current_stddev = float(self.pn_stddev.item())
        return d

    def reset(self):
        if self.action_noise is not None:
            self.action_noise.reset()
        if self.param_noise is not None:
            with torch.cuda.device(self.device):
                self.graphs.run(("perturb",), lambda: self._perturb(self.param_noise_actor))

    def get_stats(self):
        m, B = self.memory, self.batch_size
        with torch.cuda.device(self.device):
            if self.stats_sample is None:
                # a fixed sample: the same inputs every time (:343-347)
                idxs = m.sample_indices(B)
                rows = torch.from_numpy((m.start + idxs) % m.limit).to(self.device)
                self.stats_sample = {'obs0': m.obs0.index_select(0, rows), 'actions': m.actions.index_select(0, rows)}
            obs, act = self.stats_sample['obs0'], self.stats_sample['actions']
            B = obs.shape[0]
            self._encode(self.actor, obs, B)
            self.actor.forward(B)
            self._critic_pass(obs, B, None, act, False)
            q = self.critic.out[:2 * B, 0].cpu().numpy()
            mu = self.actor.mu[:B].cpu().numpy()
            names, values = [], []
            if self.normalize_returns:
                rm, rs = self.ret_rms.mean.item(), self.ret_rms.std.item()
                names += ['ret_rms_mean', 'ret_rms_std']
                values += [np.float32(rm), np.float32(rs)]
                q = (q * np.float32(rs) + np.float32(rm)).astype(np.float32)
            if self.normalize_observations:
                names += ['obs_rms_mean', 'obs_rms_std']
                values += [np.mean(self.obs_rms.mean.cpu().numpy()), np.mean(self.obs_rms.std.cpu().numpy())]
            names += ['reference_Q_mean', 'reference_Q_std', 'reference_actor_Q_mean', 'reference_actor_Q_std',
                      'reference_action_mean', 'reference_action_std']
            values += [np.mean(q[:B]), np.std(q[:B]), np.mean(q[B:]), np.std(q[B:]), np.mean(mu), np.std(mu)]
            if self.param_noise is not None:
                pa = self.param_noise_actor
                self._encode(pa, obs, B)
                pa.forward(B)
                pmu = pa.mu[:B].cpu().numpy()
                names += ['reference_perturbed_action_mean', 'reference_perturbed_action_std']
                values += [np.mean(pmu), np.std(pmu)]
        stats = dict(zip(names, values))
        if self.param_noise is not None:
            self.param_noise.current_stddev = float(self.pn_stddev.item())
            stats = {**stats, **self.param_noise.get_stats()}
        return stats

    def get_variables(self):
        """Every variable under its TF name, in the reference's creation order."""
        out = OrderedDict()
        if self.obs_rms is not None:
            out.update(self.obs_rms.tf_variables('obs_rms'))
        if self.ret_rms is not None:
            out.update(self.ret_rms.tf_variables('ret_rms'))
        for net in (self.actor, self.critic, self.target_actor, self.target_critic, self.param_noise_actor,
                    self.adaptive_param_noise_actor):
            if net is not None:
                out.update(net.tf_variables())
        return out
