"""float64 torch-CPU mirror of one DDPG train step (baselines/ddpg/ddpg_learner.py:66-331, models.py,
common/mpi_running_mean_std.py, common/mpi_adam.py:30-42) and of the numpy pieces the kernels restate bit for bit.

Ordinary torch / numpy arithmetic on the host; nothing here calls a kernel of the project.  Variables are dicts keyed by
the reference's TF names ('actor/mlp_fc0/w:0', 'critic/output/kernel:0', 'actor/LayerNorm/gamma:0', ...).
"""
import math

import numpy as np
import torch

LN_EPS = 1e-12


def ln_scope(k):
    return "LayerNorm" if k == 0 else f"LayerNorm_{k}"


def _t(a):
    return torch.tensor(np.asarray(a, np.float64), dtype=torch.float64)


def mlp(x, P, scope, num_layers, layer_norm):
    h = x
    for i in range(num_layers):
        h = h @ P[f"{scope}/mlp_fc{i}/w:0"] + P[f"{scope}/mlp_fc{i}/b:0"]
        if layer_norm:
            m = h.mean(dim=1, keepdim=True)
            v = ((h - m) ** 2).mean(dim=1, keepdim=True)
            h = (h - m) / torch.sqrt(v + LN_EPS) * P[f"{scope}/{ln_scope(i)}/gamma:0"] + \
                P[f"{scope}/{ln_scope(i)}/beta:0"]
        h = torch.tanh(h)
    return h


def actor(x, P, scope, num_layers, layer_norm):
    return torch.tanh(mlp(x, P, scope, num_layers, layer_norm) @ P[f"{scope}/dense/kernel:0"] + P[f"{scope}/dense/bias:0"])


def critic(x, a, P, scope, num_layers, layer_norm):
    h = mlp(torch.cat([x, a], dim=1), P, scope, num_layers, layer_norm)
    return h @ P[f"{scope}/output/kernel:0"] + P[f"{scope}/output/bias:0"]


def normalize(x, mean, std):
    return (x - mean) / (std + 1e-8)


def rms_mean_std(state, D):
    """mpi_running_mean_std.py:29-30 in numpy float32 from the float64 [sum | sumsq | count] state."""
    s, q, c = state[:D], state[D:2 * D], state[2 * D]
    mean = (s / c).astype(np.float32)
    std = np.sqrt(np.maximum((q / c).astype(np.float32) - np.square(mean), np.float32(1e-2)))
    return mean, std


def obs_rms_rows(state, rows):
    """RunningMeanStd.update(np.array([row])) for every row in order (ddpg_learner.py:281-287), numpy float64."""
    state = np.array(state, np.float64)
    D = (state.size - 1) // 2
    for r in np.asarray(rows, np.float32).reshape(-1, D):
        x = r.astype(np.float64)[None]
        add = np.concatenate([x.sum(axis=0), np.square(x).sum(axis=0), [1.0]])
        state[:D] += add[:D]
        state[D:2 * D] += add[D:2 * D]
        state[2 * D] += add[2 * D]
    return state


def ret_rms_batch(state, y):
    """RunningMeanStd.update(target_Q.flatten()) with shape (): numpy's pairwise sums of the float64 batch."""
    state = np.array(state, np.float64)
    x = np.asarray(y, np.float32).reshape(-1).astype(np.float64)
    state[0] += x.sum(axis=0)
    state[1] += np.square(x).sum(axis=0)
    state[2] += float(len(x))
    return state


def adam(p, g, m, v, t, lr, eps=1e-8, b1=0.9, b2=0.999):
    """mpi_adam.py:30-42 in float64 -> (p, m, v)."""
    a = lr * math.sqrt(1 - b2 ** t) / (1 - b1 ** t)
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    return p - a * m / (np.sqrt(v) + eps), m, v


def train_step(P, batch, cfg, obs_mean=None, obs_std=None, ret_state=None, skip_target_popart=False,
               actor_at_target=False, no_done_mask=False, actor_leak=False):
    """One train() of ddpg_learner.py:289-331 up to the gradients, in float64.

    P: TF name -> array of every variable (actor/, critic/, target_actor/, target_critic/).  batch: obs0, obs1, actions,
    rewards [B], terminals1 [B].  cfg: num_layers, layer_norm, gamma, normalize_returns, popart, critic_l2_reg.
    The keyword flags build the mistakes the GPU tests must tell apart from the right step.
    Returns dict(critic_grads, actor_grads, critic_loss, actor_loss, P (after Pop-Art), ret_state, y)."""
    L, ln = cfg["num_layers"], cfg["layer_norm"]
    T = {k: _t(v) for k, v in P.items()}
    B = len(batch["rewards"])

    def nobs(x):
        x = _t(x)
        if obs_mean is not None:
            x = normalize(x, _t(obs_mean), _t(obs_std))
        return torch.clamp(x, -5.0, 5.0)

    o0, o1 = nobs(batch["obs0"]), nobs(batch["obs1"])
    rmean = rstd = None
    if cfg["normalize_returns"]:
        m_, s_ = rms_mean_std(ret_state, 1)
        rmean, rstd = float(m_[0]), float(s_[0])
    with torch.no_grad():
        q1 = critic(o1, actor(o1, T, "target_actor", L, ln), T, "target_critic", L, ln)[:, 0]
        if rmean is not None:
            q1 = q1 * rstd + rmean
        d = _t(batch["terminals1"])
        y = _t(batch["rewards"]) + (1.0 if no_done_mask else (1.0 - d)) * cfg["gamma"] * q1
    new_state = ret_state
    if cfg["normalize_returns"] and cfg["popart"]:
        new_state = ret_rms_batch(ret_state, y.numpy().astype(np.float32))
        nm_, ns_ = rms_mean_std(new_state, 1)
        nm, ns = float(nm_[0]), float(ns_[0])
        for sc in (("critic",) if skip_target_popart else ("critic", "target_critic")):
            T[f"{sc}/output/kernel:0"] = T[f"{sc}/output/kernel:0"] * rstd / ns
            T[f"{sc}/output/bias:0"] = (T[f"{sc}/output/bias:0"] * rstd + rmean - nm) / ns
        rmean, rstd = nm, ns
    cvars = [k for k in T if k.startswith("critic/")]
    avars = [k for k in T if k.startswith("actor/")]
    for k in cvars + avars:
        T[k] = T[k].clone().requires_grad_(True)
    q = critic(o0, _t(batch["actions"]), T, "critic", L, ln)[:, 0]
    yn = y if rmean is None else normalize(y, rmean, rstd)
    critic_loss = ((q - yn) ** 2).mean()
    reg = cfg.get("critic_l2_reg", 0.0)
    if reg > 0:
        names = [k for k in cvars if k.endswith("/w:0") and "output" not in k]
        critic_loss = critic_loss + sum(reg * (T[k] ** 2).sum() / 2 for k in names)
    asc = "target_actor" if actor_at_target else "actor"
    if actor_at_target:
        for k in list(T):
            if k.startswith("target_actor/"):
                T[k] = T[k].clone().requires_grad_(True)
    qa = critic(o0, actor(o0, T, asc, L, ln), T, "critic", L, ln)[:, 0]
    if rmean is not None:
        qa = qa * rstd + rmean
    actor_loss = -qa.mean()
    cg = torch.autograd.grad(critic_loss + (actor_loss if actor_leak else 0.0), [T[k] for k in cvars],
                             retain_graph=True)
    agvars = avars if not actor_at_target else [k.replace("actor/", "target_actor/", 1) for k in avars]
    ag = torch.autograd.grad(actor_loss, [T[k] for k in agvars])
    return dict(critic_grads={k: g.numpy() for k, g in zip(cvars, cg)},
                actor_grads={k: g.numpy() for k, g in zip(avars, ag)},
                critic_loss=critic_loss.item(), actor_loss=actor_loss.item(),
                P={k: v.detach().numpy() for k, v in T.items()}, ret_state=new_state, y=y.numpy())


def clip_by_norm(g, c):
    n = np.sqrt((np.asarray(g, np.float64) ** 2).sum())
    return g * c / max(n, c) if c is not None else g


def polyak(t, s, tau):
    """target <- (1 - tau) target + tau online with float32 constants and float32 arithmetic, unfused."""
    t, s = np.asarray(t, np.float32), np.asarray(s, np.float32)
    return (np.float32(1.0 - tau) * t + np.float32(tau) * s).astype(np.float32)
