"""The HER agent (baselines/her/ddpg.py) on the device.

A train step is one fixed launch sequence, captured once per batch size and replayed (graphs.GraphCache).  The host
draws the sample (her_sampler.py) and uploads its (episode, t, future_t) rows through pinned buffers; Adam's step
sizes go to the device.  The sequence (csrc/her.cu, nn.py):
  sample + relabel + reward + preprocess + normalise + encode (one launch) -> target pi on [o_2 | g_2] -> target Q on
  [o_2 | g_2 | pi' / max_u] -> y = clip(r + gamma Q', -clip_return, 0 or inf) -> pi on [o | g] -> ONE Q pass over 2B
  rows [o | g | u / max_u] and [o | g | pi / max_u] -> Q_loss and the head gradients -> Q backward (weight gradients from
  the first B rows; the second B rows only carry d(-sum Q_pi) down to the action columns) -> pi's head gradient
  (through 1 / max_u, the action_l2 term and max_u tanh') -> pi backward -> Adam on each network.
Both gradients are taken at the parameters the step started from, as in the reference's single sess.run (:251-256).

When the environment's reward is not the goal-distance rule csrc/her.cu restates (experiment/config.py decides), the
step runs as two graph segments: the sample launch, which also writes ag_2, the relabelled g and info down to staging
buffers, then, after the host has called compute_reward and uploaded r, the rest.
"""
from collections import OrderedDict

import numpy as np
import torch

from .. import graphs, nn, ops
from .actor_critic import ActorCritic
from .normalizer import Normalizer
from .replay_buffer import ReplayBuffer


def dims_to_shapes(input_dims):
    return {key: tuple([val]) if val > 0 else tuple() for key, val in input_dims.items()}


def postprocess_actions(u, noise_eps, random_eps, max_u, dimu):
    """get_actions' host half (ddpg.py:145-153): Gaussian noise, clip, eps-random actions, from numpy's global
    stream."""
    noise = noise_eps * max_u * np.random.randn(*u.shape)
    u += noise
    u = np.clip(u, -max_u, max_u)
    pick = np.random.binomial(1, random_eps, u.shape[0]).reshape(-1, 1)
    u += pick * (np.random.uniform(low=-max_u, high=max_u, size=(u.shape[0], dimu)) - u)
    if u.shape[0] == 1:
        u = u[0]
    return u.copy()


class DDPG(object):
    def __init__(self, input_dims, buffer_size, hidden, layers, network_class, polyak, batch_size, Q_lr, pi_lr,
                 norm_eps, norm_clip, max_u, action_l2, clip_obs, scope, T, rollout_batch_size, subtract_goals,
                 relative_goals, clip_pos_returns, clip_return, bc_loss, q_filter, num_demo, demo_batch_size,
                 prm_loss_weight, aux_loss_weight, sample_transitions, gamma, reuse=False, seed=None, act_cap=None,
                 device=None, **kwargs):
        """The reference's arguments; seed: the stream of the Glorot initialisers (numpy's global stream is left
        alone, as TF's initialisers leave it).  act_cap: the most observations one get_actions call takes."""
        if bc_loss:
            raise NotImplementedError("her demonstrations (bc_loss / q_filter, demo_file) are not supported")
        self.input_dims, self.buffer_size, self.hidden, self.layers = input_dims, buffer_size, hidden, layers
        self.network_class, self.polyak, self.batch_size = network_class, float(polyak), int(batch_size)
        self.Q_lr, self.pi_lr, self.norm_eps, self.norm_clip = Q_lr, pi_lr, norm_eps, norm_clip
        self.max_u, self.action_l2, self.clip_obs, self.scope, self.T = max_u, float(action_l2), clip_obs, scope, T
        self.rollout_batch_size, self.subtract_goals, self.relative_goals = rollout_batch_size, subtract_goals, \
            bool(relative_goals)
        self.clip_pos_returns, self.clip_return = clip_pos_returns, clip_return
        self.bc_loss, self.q_filter, self.num_demo, self.demo_batch_size = bc_loss, q_filter, num_demo, demo_batch_size
        self.prm_loss_weight, self.aux_loss_weight = prm_loss_weight, aux_loss_weight
        self.sample_transitions, self.gamma, self.reuse = sample_transitions, gamma, reuse
        if self.clip_return is None:
            self.clip_return = np.inf
        if float(norm_clip) >= 65504:
            raise ValueError("norm_clip must be below fp16's range: normalised inputs are split into fp16 halves")
        self.dimo, self.dimg, self.dimu = input_dims['o'], input_dims['g'], input_dims['u']
        input_shapes = dims_to_shapes(self.input_dims)
        stage_shapes = OrderedDict()
        for key in sorted(self.input_dims.keys()):
            if key.startswith('info_'):
                continue
            stage_shapes[key] = (None, *input_shapes[key])
        for key in ['o', 'g']:
            stage_shapes[key + '_2'] = stage_shapes[key]
        stage_shapes['r'] = (None,)
        self.stage_shapes = stage_shapes

        dev = self.device = torch.device(device) if device is not None else \
            torch.device("cuda", torch.cuda.current_device())
        buffer_shapes = {key: (self.T - 1 if key != 'o' else self.T, *input_shapes[key])
                         for key, val in input_shapes.items()}
        buffer_shapes['g'] = (buffer_shapes['g'][0], self.dimg)
        buffer_shapes['ag'] = (self.T, self.dimg)
        buffer_size = (self.buffer_size // self.rollout_batch_size) * self.rollout_batch_size
        self.buffer = ReplayBuffer(buffer_shapes, buffer_size, self.T, self.sample_transitions, device=dev)

        self.cap = max(self.batch_size, int(act_cap or 0), int(rollout_batch_size))
        rng = np.random.RandomState(seed)
        with torch.cuda.device(dev):
            self.o_stats = Normalizer(self.dimo, self.norm_eps, self.norm_clip, device=dev)
            self.g_stats = Normalizer(self.dimg, self.norm_eps, self.norm_clip, device=dev)
            spec = ActorCritic(self.dimo, self.dimg, self.dimu, hidden, layers)
            self.main_pi, self.main_Q = spec.build(f'{scope}/main', self.cap, dev, rng)
            self.target_pi, self.target_Q = spec.build(f'{scope}/target', self.cap, dev, rng)
            mu = np.broadcast_to(np.asarray(self.max_u, np.float64), (self.dimu,)).astype(np.float32)
            self.max_u_dev = torch.from_numpy(mu.copy()).to(dev)
            self.Q_adam = nn.Optimizer(self.main_Q.store, eps=1e-8)
            self.pi_adam = nn.Optimizer(self.main_pi.store, eps=1e-8)
            f32 = dict(dtype=torch.float32, device=dev)
            cap = self.cap
            self.r = torch.zeros(cap, **f32)
            self.y = torch.zeros(cap, **f32)
            self.Q_loss = torch.zeros(1, **f32)
            self.Q_pi = torch.zeros(cap, **f32)
            self.pi_main = torch.zeros(cap, self.dimu, **f32)      # pi of the main actor's last pass
            self.pi_target = torch.zeros(cap, self.dimu, **f32)
            self._r_host = torch.zeros(cap, dtype=torch.float32).pin_memory()
            self._norm_host = self._norm_dev = None
            self._init_target_net()
        self.graphs = graphs.GraphCache()

    # ---- helpers ----------------------------------------------------------------------------------------------------
    def _upload_norm_sel(self, rows):
        """The normaliser's sample rows (rollout_batch_size * T of them) through a pinned buffer of their own."""
        n = len(rows)
        if self._norm_host is None or self._norm_host.shape[0] < n:
            self._norm_host = torch.zeros(n, 3, dtype=torch.int64).pin_memory()
            self._norm_dev = torch.zeros(n, 3, dtype=torch.int64, device=self.device)
        torch.cuda.current_stream().synchronize()            # the previous upload has been read
        self._norm_host[:n].copy_(torch.from_numpy(np.ascontiguousarray(rows, np.int64)))
        self._norm_dev[:n].copy_(self._norm_host[:n], non_blocking=True)
        return self._norm_dev[:n]

    def _preprocess_og(self, o, ag, g):
        if self.relative_goals:
            g_shape = g.shape
            g = g.reshape(-1, self.dimg)
            ag = ag.reshape(-1, self.dimg)
            g = self.subtract_goals(g, ag)
            g = g.reshape(*g_shape)
        o = np.clip(o, -self.clip_obs, self.clip_obs)
        g = np.clip(g, -self.clip_obs, self.clip_obs)
        return o, g

    def _reward_rule(self):
        rule = getattr(self.sample_transitions, 'device_reward', None)
        if rule is None:
            return 0, 0.0
        return {'sparse': 1, 'dense': 2}[rule[0]], float(rule[1])

    # ---- the reference's interface ----------------------------------------------------------------------------------
    def step(self, obs):
        actions = self.get_actions(obs['observation'], obs['achieved_goal'], obs['desired_goal'])
        return actions, None, None, None

    def get_actions(self, o, ag, g, noise_eps=0., random_eps=0., use_target_net=False, compute_Q=False):
        o, g = self._preprocess_og(o, ag, g)
        o = np.asarray(o, np.float32).reshape(-1, self.dimo)
        g = np.asarray(g, np.float32).reshape(-1, self.dimg)
        n = o.shape[0]
        if n > self.cap:
            raise ValueError(f"get_actions over {n} observations exceeds the agent's capacity {self.cap}")
        pi, Q = (self.target_pi, self.target_Q) if use_target_net else (self.main_pi, self.main_Q)
        with torch.cuda.device(self.device):
            x = self.graphs.home("act_o", self.cap, (self.dimo,), torch.float32, self.device)[:n]
            xg = self.graphs.home("act_g", self.cap, (self.dimg,), torch.float32, self.device)[:n]
            x.copy_(torch.from_numpy(o))
            xg.copy_(torch.from_numpy(g))
            out = self.pi_target if use_target_net else self.pi_main

            def body():
                om, os_, gm, gs = self.o_stats.mean, self.o_stats.std, self.g_stats.mean, self.g_stats.std
                ops.her_obs_encode(x, xg, n, om, os_, gm, gs, self.norm_clip, pi.x0, pi.in_pad,
                                   Q.x0 if compute_Q else None, Q.in_pad)
                pi.forward(n)
                ops.her_pi(pi.out, pi.ld_out, n, self.dimu, self.max_u_dev, out, Q.x0 if compute_Q else None,
                           Q.in_pad, self.dimo + self.dimg)
                if compute_Q:
                    Q.forward(n)
            self.graphs.run(("act", n, bool(use_target_net), bool(compute_Q)), body)
            u = out[:n].cpu().numpy()
            q = Q.out[:n, :1].cpu().numpy() if compute_Q else None
        ret = [postprocess_actions(u, noise_eps, random_eps, self.max_u, self.dimu)] + ([q] if compute_Q else [])
        return ret[0] if len(ret) == 1 else ret

    def store_episode(self, episode_batch, update_stats=True):
        """episode_batch: array of batch_size x (T or T+1) x dim_key; 'o' and 'ag' are of size T+1, others T."""
        dev = self.device
        with torch.cuda.device(dev):
            staged = {k: torch.from_numpy(np.asarray(v, np.float64)).to(dev) for k, v in episode_batch.items()
                      if k in self.buffer.buffers}
            self.buffer.store_episode(episode_batch, staged)
            if update_stats:
                # the sampler over the new episodes only (ddpg.py:225-240); o_2, ag_2 and the reward are not used
                n_ep, T = episode_batch['u'].shape[:2]
                num = n_ep * T
                ep, t, ft = self.sample_transitions.draw(n_ep, T, num)
                sel = self._upload_norm_sel(np.stack([ep, t, ft], axis=1))
                # numpy computes the statistics in the transitions' dtype
                f32_o = np.asarray(episode_batch['o']).dtype == np.float32
                gdt = np.result_type(episode_batch['g'], episode_batch['ag']) if self.relative_goals else \
                    np.asarray(episode_batch['g']).dtype
                f32_g = gdt == np.float32
                ops.her_norm(staged['o'], staged['ag'], staged['g'], sel, num, self.relative_goals, self.clip_obs,
                             f32_o, f32_g, self.o_stats.tensors, self.g_stats.tensors, self.norm_eps)

    def get_current_buffer_size(self):
        return self.buffer.get_current_size()

    def sample_batch(self):
        """The batch's (episode, t, future_t) rows, drawn from numpy's global stream as buffer.sample draws them."""
        return self.buffer.draw(self.batch_size)

    def stage_batch(self, batch=None):
        """Upload a batch (default: a new sample_batch()) for the next train(stage=False)."""
        if batch is None:
            batch = self.sample_batch()
        with torch.cuda.device(self.device):
            self._staged = self.graphs.upload("sel", batch, self.cap, (3,), torch.int64, self.device)

    def train_device(self, stage=True):
        """One train step on the device; -> (the float32 device scalar Q_loss, the device Q_pi [B]) without a
        synchronisation."""
        if stage:
            self.stage_batch()
        sel = self._staged
        B = sel.shape[0]
        if B > self.cap:
            raise ValueError(f"batch {B} exceeds the agent's capacity {self.cap}")
        pi, Q, tpi, tQ = self.main_pi, self.main_Q, self.target_pi, self.target_Q
        rtype, thr = self._reward_rule()
        ring = self.buffer.ring
        lo, hi = -self.clip_return, (0. if self.clip_pos_returns else np.inf)
        cols = self.dimo + self.dimg
        with torch.cuda.device(self.device):
            self.Q_adam.begin_step(self.Q_lr)
            self.pi_adam.begin_step(self.pi_lr)
            staging = None
            if rtype == 0:
                staging = [self.graphs.home(nm, self.cap, (d,), torch.float64, self.device)[:B]
                           for nm, d in (("ag2", self.dimg), ("g", self.dimg), ("info", max(1, ring[4].shape[2])))]

            def sample():
                ops.her_sample(ring, sel, B, self.relative_goals, self.clip_obs, self.o_stats.mean, self.o_stats.std,
                               self.g_stats.mean, self.g_stats.std, self.norm_clip, self.max_u_dev, rtype, thr, self.r,
                               pi.x0, tpi.x0, pi.in_pad, Q.x0, tQ.x0, Q.in_pad,
                               *(staging if staging is not None else (None, None, None)))

            def step():
                tpi.forward(B)
                ops.her_pi(tpi.out, tpi.ld_out, B, self.dimu, self.max_u_dev, self.pi_target, tQ.x0, tQ.in_pad, cols)
                tQ.forward(B)
                ops.her_target(tQ.out, tQ.ld_out, self.r, B, self.gamma, lo, hi, self.y)
                pi.forward(B)
                ops.her_pi(pi.out, pi.ld_out, B, self.dimu, self.max_u_dev, self.pi_main, Q.x0[B:2 * B], Q.in_pad,
                           cols)
                Q.forward(2 * B)
                ops.her_loss(Q.out, Q.ld_out, self.y, B, Q.dout, Q.ld_out, self.Q_loss, self.Q_pi)
                pi.store.grads.zero_()
                Q.store.grads.zero_()
                Q.backward(B, 1.0 / B, 2 * B)
                ops.her_actor_dz(Q.dact, Q.dact.shape[1], pi.out, pi.ld_out, self.pi_main, B, self.dimu,
                                 self.max_u_dev, self.action_l2, pi.dout, pi.ld_out)
                pi.backward(B, 1.0 / B, B)
                self.Q_adam.apply()
                self.pi_adam.apply()
                pi.refresh()
                Q.refresh()

            if rtype:
                def body():
                    sample()
                    step()
                self.graphs.run(("train", B), body)
            else:
                self.graphs.run(("sample", B), sample)
                self._host_reward(B, staging)
                self.graphs.run(("train_r", B), step)
        return self.Q_loss, self.Q_pi[:B]

    def _host_reward(self, B, staging):
        """r = env.compute_reward(ag_2, g, info) on the host for rewards the device does not restate."""
        ag2, g, info = (t.cpu().numpy() for t in staging)
        info_d = {k.replace('info_', ''): info[:, o:o + d].astype(np.float64)
                  for k, (o, d) in self.buffer.info_off.items()}
        r = np.asarray(self.sample_transitions.reward_fun(ag_2=ag2, g=g, info=info_d), np.float32).reshape(B)
        self._r_host[:B].copy_(torch.from_numpy(r))
        self.r[:B].copy_(self._r_host[:B], non_blocking=True)
        torch.cuda.current_stream().synchronize()

    def train(self, stage=True):
        """-> (critic_loss, Q_pi): the reference returns main.Q_pi_tf as its second value (:251-257)."""
        loss, q_pi = self.train_device(stage)
        return np.float32(loss.item()), q_pi.cpu().numpy().reshape(-1, 1)

    def _init_target_net(self):
        ops.soft_update(self.target_Q.store.params, self.main_Q.store.params, 0.0, 1.0, self.target_pi.store.params,
                        self.main_pi.store.params)
        self.target_pi.refresh()
        self.target_Q.refresh()

    def update_target_net(self):
        def body():
            ops.soft_update(self.target_Q.store.params, self.main_Q.store.params, self.polyak, 1.0 - self.polyak,
                            self.target_pi.store.params, self.main_pi.store.params)
            self.target_pi.refresh()
            self.target_Q.refresh()
        with torch.cuda.device(self.device):
            self.graphs.run(("target",), body)

    def clear_buffer(self):
        self.buffer.clear_buffer()

    def logs(self, prefix=''):
        logs = []
        logs += [('stats_o/mean', np.mean(self.o_stats.mean.cpu().numpy()))]
        logs += [('stats_o/std', np.mean(self.o_stats.std.cpu().numpy()))]
        logs += [('stats_g/mean', np.mean(self.g_stats.mean.cpu().numpy()))]
        logs += [('stats_g/std', np.mean(self.g_stats.std.cpu().numpy()))]
        if prefix != '' and not prefix.endswith('/'):
            return [(prefix + '/' + key, val) for key, val in logs]
        return logs

    def get_variables(self):
        """Every variable under its TF name, in the reference's creation order."""
        out = OrderedDict()
        out.update(self.o_stats.tf_variables(f'{self.scope}/o_stats'))
        out.update(self.g_stats.tf_variables(f'{self.scope}/g_stats'))
        for net in (self.main_pi, self.main_Q, self.target_pi, self.target_Q):
            out.update(net.tf_variables())
        return out

    def load_variables(self, values):
        with torch.cuda.device(self.device):
            self.o_stats.load_tf(values, f'{self.scope}/o_stats')
            self.g_stats.load_tf(values, f'{self.scope}/g_stats')
            for net in (self.main_pi, self.main_Q, self.target_pi, self.target_Q):
                net.load_tf(values)

    def save(self, save_path):
        """tf_util.save_variables: a joblib dict {tf_name: array}."""
        import os
        import joblib
        d = os.path.dirname(save_path)
        if d:
            os.makedirs(d, exist_ok=True)
        joblib.dump(self.get_variables(), save_path)

    def load(self, load_path):
        import os
        import joblib
        self.load_variables(joblib.load(os.path.expanduser(load_path)))

    def __getstate__(self):
        """Pickled policies carry the variables (the reference's state['tf']) and the arguments, not the buffer."""
        keep = ('input_dims', 'buffer_size', 'hidden', 'layers', 'network_class', 'polyak', 'batch_size', 'Q_lr',
                'pi_lr', 'norm_eps', 'norm_clip', 'max_u', 'action_l2', 'clip_obs', 'scope', 'T',
                'rollout_batch_size', 'relative_goals', 'clip_pos_returns', 'clip_return', 'gamma')
        state = {k: self.__dict__[k] for k in keep}
        state['tf'] = self.get_variables()
        return state

    def __setstate__(self, state):
        from .experiment.config import simple_goal_subtract
        from .her_sampler import make_sample_her_transitions
        tf = state.pop('tf')
        self.__init__(**state, subtract_goals=simple_goal_subtract, bc_loss=0, q_filter=0, num_demo=0,
                      demo_batch_size=0, prm_loss_weight=0, aux_loss_weight=0,
                      sample_transitions=make_sample_her_transitions('none', 0, None))
        self.load_variables(tf)
