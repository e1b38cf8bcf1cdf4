"""CPU oracle of the MultiDiscrete and MultiBinary action heads (test infrastructure), restated from the reference's
definitions in common/distributions.py:

  MultiCategoricalPd (:76-94, 206-225): one CategoricalPd per component over the consecutive logit blocks of widths
    nvec; neglogp / entropy / kl are the components' sums, sample is the per-component Gumbel-max cast to int32.
  BernoulliPd (:115-128, 254-276): p = sigmoid(logits); neglogp = sum sigmoid_xent(logits, x);
    entropy = sum sigmoid_xent(logits, p); kl = sum sigmoid_xent(other, p) - sum sigmoid_xent(logits, p);
    sample = float(u < p).

and the MultiDiscrete observation encoding of common/input.py:58-61 (concatenated one-hots).  It builds on the
Categorical / Gaussian oracle in oracle/nets.py: same parameter dictionaries, forward pass and PPO2 loss arithmetic
(ppo2/model.py:57-91), with the distribution chosen by `pd` in {'cat', 'mcat', 'bern', 'gauss'}.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import nets


def _blocks(logits, nvec):
    return torch.split(logits, [int(n) for n in nvec], dim=-1)


# ------------------------------------------------------------------------------------------------ MultiCategorical
def mcat_neglogp(logits, actions, nvec):
    a = torch.as_tensor(actions).long().reshape(logits.shape[0], len(nvec))
    return sum(nets.cat_neglogp(l, a[:, i]) for i, l in enumerate(_blocks(logits, nvec)))


def mcat_entropy(logits, nvec):
    return sum(nets.cat_entropy(l) for l in _blocks(logits, nvec))


def mcat_kl(logits, other, nvec):
    return sum(nets.cat_kl(l, o) for l, o in zip(_blocks(logits, nvec), _blocks(other, nvec)))


def mcat_sample(logits, uniforms, nvec):
    """Per-component Gumbel-max with the injected uniforms (column j of `uniforms` perturbs logit column j)."""
    u = _blocks(torch.as_tensor(uniforms, dtype=logits.dtype), nvec)
    return torch.stack([nets.cat_sample(l, ui) for l, ui in zip(_blocks(logits, nvec), u)], dim=-1).to(torch.int32)


# ------------------------------------------------------------------------------------------------ Bernoulli
def sigmoid_xent(logits, labels):
    """tf.nn.sigmoid_cross_entropy_with_logits: max(l, 0) - l * y + log(1 + exp(-|l|))."""
    return torch.clamp(logits, min=0) - logits * labels + torch.log1p(torch.exp(-logits.abs()))


def bern_neglogp(logits, x):
    return sigmoid_xent(logits, torch.as_tensor(x, dtype=logits.dtype)).sum(dim=-1)


def bern_entropy(logits):
    return sigmoid_xent(logits, torch.sigmoid(logits)).sum(dim=-1)


def bern_kl(logits, other):
    ps = torch.sigmoid(logits)
    return sigmoid_xent(other, ps).sum(dim=-1) - sigmoid_xent(logits, ps).sum(dim=-1)


def bern_sample(logits, uniforms):
    return (torch.as_tensor(uniforms, dtype=logits.dtype) < torch.sigmoid(logits)).to(torch.float32)


# ------------------------------------------------------------------------------------------------ policy / loss
def encode_multidiscrete(obs, nvec, dtype=torch.float32):
    """common/input.py:58-61: concat_i one_hot(obs[..., i], nvec[i])."""
    o = torch.as_tensor(np.asarray(obs)).long()
    return torch.cat([F.one_hot(o[..., i], int(n)) for i, n in enumerate(nvec)], dim=-1).to(dtype)


def init_policy_params(network, ob_shape, pd, nvec_or_n, value_network=None, **kw):
    """Variables of policy_fn + PolicyWithValue for a MultiDiscrete (pd 'mcat', pi width sum(nvec)) or MultiBinary
    (pd 'bern', pi width n) action space: the Categorical creation order and draws, no logstd."""
    width = int(np.sum(nvec_or_n)) if pd == "mcat" else int(nvec_or_n)
    return nets.init_policy_params(network, ob_shape, "discrete", width, value_network=value_network, **kw)


def neglogp(pd, pi, logstd, actions, nvec=None):
    if pd == "cat":
        return nets.cat_neglogp(pi, actions)
    if pd == "mcat":
        return mcat_neglogp(pi, actions, nvec)
    if pd == "bern":
        return bern_neglogp(pi, actions)
    return nets.gauss_neglogp(pi, logstd, actions)


def entropy(pd, pi, logstd, nvec=None):
    if pd == "cat":
        return nets.cat_entropy(pi)
    if pd == "mcat":
        return mcat_entropy(pi, nvec)
    if pd == "bern":
        return bern_entropy(pi)
    return nets.gauss_entropy(pi, logstd)


def ppo_loss(tp, network, obs, actions, advs, returns, oldneglogp, oldvpred, cliprange, ent_coef, vf_coef,
             value_network=None, pd="cat", nvec=None):
    """ppo2/model.py:57-91 with the pd's neglogp / entropy."""
    pi, logstd, vpred = nets.policy_forward(tp, network, obs, value_network)
    neglogpac = neglogp(pd, pi, logstd, actions, nvec)
    ent = entropy(pd, pi, logstd, nvec).mean()
    vpredclipped = oldvpred + torch.clamp(vpred - oldvpred, -cliprange, cliprange)
    vf_loss = 0.5 * torch.maximum((vpred - returns) ** 2, (vpredclipped - returns) ** 2).mean()
    ratio = torch.exp(oldneglogp - neglogpac)
    pg_loss = torch.maximum(-advs * ratio, -advs * torch.clamp(ratio, 1.0 - cliprange, 1.0 + cliprange)).mean()
    approxkl = 0.5 * ((neglogpac - oldneglogp) ** 2).mean()
    clipfrac = ((ratio - 1.0).abs() > cliprange).to(ratio.dtype).mean()
    loss = pg_loss - ent * ent_coef + vf_loss * vf_coef
    return loss, [pg_loss, vf_loss, ent, approxkl, clipfrac]


def policy_step(params, network, obs, noise, value_network=None, pd="cat", nvec=None, dtype=torch.float32):
    """PolicyWithValue.step (policies.py:77-96) with injected noise: (actions, values, neglogp, pi)."""
    tp = nets.to_torch(params, dtype)
    with torch.no_grad():
        pi, logstd, vf = nets.policy_forward(tp, network, torch.as_tensor(obs), value_network)
        noise = torch.as_tensor(noise, dtype=dtype)
        if pd == "mcat":
            a = mcat_sample(pi, noise, nvec)
        elif pd == "bern":
            a = bern_sample(pi, noise)
        elif pd == "cat":
            a = nets.cat_sample(pi, noise)
        else:
            a = nets.gauss_sample(pi, logstd, noise)
        nlp = neglogp(pd, pi, logstd, a, nvec)
    return a.numpy(), vf.numpy(), nlp.numpy(), pi.numpy()


class PPO2Oracle(nets.PPO2Oracle):
    """nets.PPO2Oracle (ppo2/model.py Model.train) with the loss of `pd`."""

    def __init__(self, params, network, ent_coef, vf_coef, max_grad_norm, value_network=None, pd="cat", nvec=None,
                 dtype=torch.float32):
        super().__init__(params, network, ent_coef, vf_coef, max_grad_norm, value_network=value_network, dtype=dtype)
        self.pd, self.nvec = pd, nvec

    def grads(self, cliprange, obs, returns, actions, values, neglogpacs, advs=None):
        dt = self.dtype
        if advs is None:
            advs = nets.normalize_advs(returns, values)
        for t in self.tp.values():
            t.requires_grad_(True)
        act = torch.as_tensor(np.asarray(actions))
        if act.dtype.is_floating_point:
            act = act.to(dt)
        loss, stats = ppo_loss(self.tp, self.network, torch.as_tensor(obs), act, torch.as_tensor(advs, dtype=dt),
                               torch.as_tensor(returns, dtype=dt), torch.as_tensor(neglogpacs, dtype=dt),
                               torch.as_tensor(values, dtype=dt), cliprange, self.ent_coef, self.vf_coef,
                               self.value_network, self.pd, self.nvec)
        grads = torch.autograd.grad(loss, list(self.tp.values()), allow_unused=True)
        grads = [g if g is not None else torch.zeros_like(p) for g, p in zip(grads, self.tp.values())]
        for t in self.tp.values():
            t.requires_grad_(False)
        return [float(s) for s in stats], grads

    def step(self, obs, noise):
        return policy_step(self.params_np(), self.network, obs, noise, self.value_network, self.pd, self.nvec,
                           self.dtype)
