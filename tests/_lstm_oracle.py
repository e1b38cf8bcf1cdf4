"""Recurrent PPO2 (networks `lstm`, `cnn_lstm`) restated on torch-CPU: test infrastructure, like oracle/nets.py, whose
primitives (nature_cnn, encode_observation, the distributions, the global-norm clip, TF-Adam) it reuses unchanged.

  init_recurrent_params   variable creation order of policies.py:126-177 with models.py lstm / cnn_lstm:
                          [c1..c3, fc1,] lstm/wx, lstm/wh (ortho_init(1.0), a2c/utils.py:89-91), lstm/b, pi, vf
  lstm_cell_seq           a2c/utils.py:84-97 lstm() over [nsteps] steps of [nenv] rows (batch_to_seq env-major)
  recurrent_forward       policies.py:41-64 on the recurrent latent, rows env-major (row e * nsteps + t)
  RecurrentPPO2Oracle     ppo2/model.py:133-158 train() with states and masks (ppo2.py:167-180 minibatches)
  lstm_steps              the cell over time-major rows from the input projection, keeping gates, c and masked h_{t-1}
  lstm_steps_backward     its BPTT (d loss / d pre-activation gates), as the sequence kernels of csrc/lstm.cu compute it

Gradients come from torch.autograd (the oracle only); float64 by default."""
import math
from collections import OrderedDict

import numpy as np
import torch

from oracle import nets


def init_recurrent_params(network, ob_shape, ac_kind, ac_dim, nlstm=128, seed=None, scope="ppo2_model", onehot_n=0):
    rng = np.random if seed is None else np.random.RandomState(seed)
    p = OrderedDict()
    pre = f"{scope}/pi"
    if network == "cnn_lstm":
        nin = nets._init_network(p, pre, "cnn", ob_shape, rng)
    elif network == "lstm":
        nin = onehot_n or int(np.prod(ob_shape))
    else:
        raise ValueError(network)
    p[f"{pre}/lstm/wx:0"] = nets.ortho_init_np((nin, 4 * nlstm), 1.0, rng)
    p[f"{pre}/lstm/wh:0"] = nets.ortho_init_np((nlstm, 4 * nlstm), 1.0, rng)
    p[f"{pre}/lstm/b:0"] = np.zeros((4 * nlstm,), np.float32)
    if nlstm != ac_dim:                                                  # _matching_fc distributions.py:351-355
        p[f"{scope}/pi/w:0"] = nets.ortho_init_np((nlstm, ac_dim), 0.01, rng)
        p[f"{scope}/pi/b:0"] = np.zeros((ac_dim,), np.float32)
    if ac_kind == "box":
        p[f"{scope}/pi/logstd:0"] = np.zeros((1, ac_dim), np.float32)
    p[f"{scope}/vf/w:0"] = nets.ortho_init_np((nlstm, 1), 1.0, rng)
    p[f"{scope}/vf/b:0"] = np.zeros((1,), np.float32)
    return p


def lstm_cell_seq(xs, ms, s, wx, wh, b):
    """a2c/utils.py:84-97.  xs [nenv, nsteps, nin], ms [nenv, nsteps] (done before step t), s [nenv, 2H] = [c | h].
    Returns (h [nenv, nsteps, H], final state [nenv, 2H])."""
    H = wh.shape[0]
    c, h = s[:, :H], s[:, H:]
    hs = []
    for t in range(xs.shape[1]):
        keep = (1.0 - ms[:, t])[:, None]
        c, h = c * keep, h * keep
        z = xs[:, t] @ wx + h @ wh + b
        i, f, o, u = torch.sigmoid(z[:, :H]), torch.sigmoid(z[:, H:2 * H]), torch.sigmoid(z[:, 2 * H:3 * H]), \
            torch.tanh(z[:, 3 * H:])
        c = f * c + i * u
        h = o * torch.tanh(c)
        hs.append(h)
    return torch.stack(hs, 1), torch.cat([c, h], 1)


def recurrent_forward(tp, network, obs, masks, states, nenv, onehot_n=0, scope="ppo2_model"):
    """policies.py:41-64 over nenv environments x nsteps (rows env-major).  Returns (pi, logstd or None, vf, state)."""
    pre = f"{scope}/pi"
    dtype = tp[f"{pre}/lstm/wx:0"].dtype
    obs = torch.as_tensor(obs)
    if network == "cnn_lstm":
        x = nets.nature_cnn(tp, pre, obs)
    else:
        x = nets.encode_observation(obs, dtype, onehot_n=onehot_n)
        x = x.reshape(x.shape[0], -1)
    nb = x.shape[0]
    xs = x.reshape(nenv, nb // nenv, -1)                                 # batch_to_seq: env-major rows
    ms = torch.as_tensor(np.asarray(masks), dtype=dtype).reshape(nenv, nb // nenv)
    hseq, snew = lstm_cell_seq(xs, ms, torch.as_tensor(np.asarray(states), dtype=dtype),
                               tp[f"{pre}/lstm/wx:0"], tp[f"{pre}/lstm/wh:0"], tp[f"{pre}/lstm/b:0"])
    lat = hseq.reshape(nb, -1)                                           # seq_to_batch
    pi = lat @ tp[f"{scope}/pi/w:0"] + tp[f"{scope}/pi/b:0"] if f"{scope}/pi/w:0" in tp else lat
    vf = (lat @ tp[f"{scope}/vf/w:0"] + tp[f"{scope}/vf/b:0"])[:, 0]
    return pi, tp.get(f"{scope}/pi/logstd:0"), vf, snew


class RecurrentPPO2Oracle(nets.PPO2Oracle):
    """ppo2/model.py:133-158 with states: the loss of ppo2/model.py:57-91 over the recurrent forward."""

    def __init__(self, params, network, ent_coef, vf_coef, max_grad_norm, nsteps, onehot_n=0, dtype=torch.float64):
        super().__init__(params, network, ent_coef, vf_coef, max_grad_norm, dtype=dtype)
        self.nsteps, self.onehot_n = nsteps, onehot_n

    def train(self, lr, cliprange, obs, returns, masks, actions, values, neglogpacs, states=None):
        dt = self.dtype
        advs = nets.normalize_advs(returns, values)
        for t in self.tp.values():
            t.requires_grad_(True)
        nenv = len(returns) // self.nsteps
        pi, logstd, vpred, _ = recurrent_forward(self.tp, self.network, obs, masks, states, nenv, self.onehot_n)
        act = torch.as_tensor(actions)
        if logstd is None:
            neglogpac, entropy = nets.cat_neglogp(pi, act), nets.cat_entropy(pi).mean()
        else:
            act = act.to(dt)
            neglogpac, entropy = nets.gauss_neglogp(pi, logstd, act), nets.gauss_entropy(pi, logstd).mean()
        f = lambda a: torch.as_tensor(np.asarray(a), dtype=dt)
        oldv, R, oldnlp, A = f(values), f(returns), f(neglogpacs), f(advs)
        vclip = oldv + torch.clamp(vpred - oldv, -cliprange, cliprange)
        vf_loss = 0.5 * torch.maximum((vpred - R) ** 2, (vclip - R) ** 2).mean()
        ratio = torch.exp(oldnlp - neglogpac)
        pg_loss = torch.maximum(-A * ratio, -A * torch.clamp(ratio, 1.0 - cliprange, 1.0 + cliprange)).mean()
        approxkl = 0.5 * ((neglogpac - oldnlp) ** 2).mean()
        clipfrac = ((ratio - 1.0).abs() > cliprange).to(dt).mean()
        loss = pg_loss - entropy * self.ent_coef + vf_loss * self.vf_coef
        grads = torch.autograd.grad(loss, list(self.tp.values()), allow_unused=True)
        grads = [g if g is not None else torch.zeros_like(p) for g, p in zip(grads, self.tp.values())]
        for t in self.tp.values():
            t.requires_grad_(False)
        self.last_grads = OrderedDict((k, g.numpy().copy()) for k, g in zip(self.tp.keys(), grads))
        if self.max_grad_norm is not None:
            grads, _ = nets.clip_by_global_norm(grads, self.max_grad_norm)
        self.t += 1
        for (k, p), g in zip(list(self.tp.items()), grads):
            self.tp[k], self.m[k], self.v[k] = nets.adam_tf(p, g, self.m[k], self.v[k], self.t, lr, eps=self.adam_eps)
        return [float(s) for s in (pg_loss, vf_loss, entropy, approxkl, clipfrac)]

    def value(self, obs, masks, states):
        with torch.no_grad():
            return recurrent_forward(self.tp, self.network, obs, masks, states, len(states), self.onehot_n)[2].numpy()


def lstm_numpy_loop(xs, ms, s, wx, wh, b):
    """Definition-level float64 loops of a2c/utils.py:84-97 (no vectorised matmul), for anchoring lstm_cell_seq."""
    nenv, T, nin = xs.shape
    H = wh.shape[0]
    c, h = s[:, :H].copy(), s[:, H:].copy()
    out = np.zeros((nenv, T, H))
    sig = lambda v: 1.0 / (1.0 + math.exp(-v))
    for e in range(nenv):
        for t in range(T):
            keep = 1.0 - ms[e, t]
            cp = [c[e, j] * keep for j in range(H)]
            hp = [h[e, j] * keep for j in range(H)]
            for j in range(H):
                z = [b[g * H + j] + sum(xs[e, t, k] * wx[k, g * H + j] for k in range(nin))
                     + sum(hp[k] * wh[k, g * H + j] for k in range(H)) for g in range(4)]
                c[e, j] = sig(z[1]) * cp[j] + sig(z[0]) * math.tanh(z[3])
                h[e, j] = sig(z[2]) * math.tanh(c[e, j])
                out[e, t, j] = h[e, j]
    return out, np.concatenate([c, h], 1)


def _sig(x):
    return 1.0 / (1.0 + np.exp(-x))


def lstm_steps(xg, wh, masks, s0, T, B, H, mistake=None):
    """a2c/utils.py lstm() over time-major rows (row t*B + b), numpy float64, with what a backward needs: returns
    (h, c, gates [i | f | o | u], masked h_{t-1}, final state [c | h]).  mistake: 'mask_after' (reset after the
    step), 'swap_fi'."""
    xg = xg.reshape(T, B, 4 * H)
    c, h = s0[:, :H].copy(), s0[:, H:].copy()
    hs, cs, gs, hps = [], [], [], []
    for t in range(T):
        keep = (1.0 - masks[t])[:, None]
        if mistake != "mask_after":
            c, h = c * keep, h * keep
        hps.append(h)
        z = xg[t] + h @ wh
        i, f, o, u = _sig(z[:, :H]), _sig(z[:, H:2 * H]), _sig(z[:, 2 * H:3 * H]), np.tanh(z[:, 3 * H:])
        if mistake == "swap_fi":
            i, f = f, i
        c = f * c + i * u
        h = o * np.tanh(c)
        if mistake == "mask_after":
            c, h = c * keep, h * keep
        hs.append(h), cs.append(c), gs.append(np.concatenate([i, f, o, u], 1))
    return (np.concatenate(hs), np.concatenate(cs), np.concatenate(gs), np.concatenate(hps),
            np.concatenate([c, h], 1))


def lstm_steps_backward(dh, gates, cs, masks, s0, wh, T, B, H, mistake=None):
    """BPTT of lstm_steps: dz [T*B, 4H].  mistake: 'no_carry' (drops the recurrent dh)."""
    dh, gates, cs = dh.reshape(T, B, H), gates.reshape(T, B, 4 * H), cs.reshape(T, B, H)
    dz = np.zeros((T, B, 4 * H))
    dc = np.zeros((B, H))
    carry = np.zeros((B, H))
    for t in reversed(range(T)):
        keep = (1.0 - masks[t])[:, None]
        i, f, o, u = (gates[t][:, k * H:(k + 1) * H] for k in range(4))
        cp = (cs[t - 1] if t > 0 else s0[:, :H]) * keep
        d = dh[t] + (0 if mistake == "no_carry" else carry)
        tc = np.tanh(cs[t])
        dc = dc + d * o * (1 - tc * tc)
        dz[t] = np.concatenate([dc * u * i * (1 - i), dc * cp * f * (1 - f), d * tc * o * (1 - o),
                                dc * i * (1 - u * u)], 1)
        carry = (dz[t] @ wh.T) * keep
        dc = dc * f * keep
    return dz.reshape(T * B, 4 * H)
