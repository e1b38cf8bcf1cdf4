"""Float64 mirror of ACER's loss head (acer/acer.py:103-178), RMSProp + moving average (:181-188), and a whole train
step of an mlp ACER network built on tests/_net_refs.py.  Plain numpy / torch float64; never calls a kernel."""
import types

import numpy as np
import torch

import _net_refs as NR

EPS = 1e-6


def softmax(l):
    l = np.asarray(l, np.float64)
    e = np.exp(l - l.max(axis=-1, keepdims=True))
    return e / e.sum(axis=-1, keepdims=True)


def retrace(R, D, q_i, v, rho_i, nenv, nsteps, gamma):
    """q_retrace (acer.py:25-51): R, D, q_i, rho_i [nenv, nsteps], v [nenv, nsteps + 1] -> qret [nenv, nsteps]."""
    qret = v[:, -1].copy()
    out = np.zeros((nenv, nsteps))
    for i in range(nsteps - 1, -1, -1):
        qret = R[:, i] + gamma * qret * (1.0 - D[:, i])
        out[:, i] = qret
        qret = np.minimum(1.0, rho_i[:, i]) * (qret - q_i[:, i]) + v[:, i]
    return out


def head(pi, q, pol, actions, rewards, dones, mus, nenv, nsteps, gamma=0.99, c=10.0, delta=1.0, q_coef=0.5,
         ent_coef=0.01, trust_region=True, entropy_logits=False, bc_drop_f=False, bc_drop_eps=False,
         shift_dones=False, no_adj_max=False):
    """The loss head in float64.  pi, q, pol: [nenv * (nsteps + 1), nA] rows e * (nsteps + 1) + t; actions, rewards,
    dones [nenv * nsteps]; mus [nenv * nsteps, nA].  Returns dpi, dq (N * d loss / d logits, q; zero on each env's last
    row), qret, v, f and the 12 statistics of ops.acer_loss.  The keyword mutants restate tempting mistakes."""
    T, N = nsteps, nenv * nsteps
    nA = pi.shape[1]
    F = softmax(pi).reshape(nenv, T + 1, nA)
    FP = softmax(pol).reshape(nenv, T + 1, nA)
    Q = np.asarray(q, np.float64).reshape(nenv, T + 1, nA)
    V = (F * Q).sum(-1)
    A = np.asarray(actions).reshape(nenv, T)
    MU = np.asarray(mus, np.float64).reshape(nenv, T, nA)
    f, fp, qq = F[:, :T], FP[:, :T], Q[:, :T]
    take = lambda x: np.take_along_axis(x, A[..., None], -1)[..., 0]
    f_i, q_i = take(f), take(qq)
    rho = f / (MU + EPS)
    rho_i = take(rho)
    D = np.asarray(dones, np.float64).reshape(nenv, T)
    if shift_dones:
        D = np.concatenate([np.zeros((nenv, 1)), D[:, :-1]], axis=1)
    qret = retrace(np.asarray(rewards, np.float64).reshape(nenv, T), D, q_i, V, rho_i, nenv, T, gamma)
    v = V[:, :T]
    Af = (qret - v) * np.minimum(c, rho_i)
    loss_f = -np.mean(np.log(f_i + EPS) * Af)
    w = np.maximum(0.0, 1.0 - c / (rho + (0.0 if bc_drop_eps else EPS)))
    Bm = (qq - v[..., None]) * w * (1.0 if bc_drop_f else f)
    loss_bc = -np.mean((np.log(f + EPS) * Bm).sum(-1))
    if entropy_logits:
        lg = np.asarray(pi, np.float64).reshape(nenv, T + 1, nA)[:, :T]
        lse = np.log(np.exp(lg - lg.max(-1, keepdims=True)).sum(-1, keepdims=True)) + lg.max(-1, keepdims=True)
        H = -(f * (lg - lse)).sum(-1)
        dH = -(np.log(f) + 1.0)
    else:
        H = -(f * np.log(f + 1e-6)).sum(-1)
        dH = -(np.log(f + 1e-6) + f / (f + 1e-6))
    entropy = H.mean()
    loss_policy = loss_f + loss_bc
    loss_q = np.mean(0.5 * (qret - q_i) ** 2)
    loss = loss_policy + q_coef * loss_q - ent_coef * entropy
    onehot = np.eye(nA)[A]
    g = onehot * (Af / (f_i + EPS))[..., None] + Bm / (f + EPS) + ent_coef * dH
    k = -fp / (f + EPS)
    kg = (k * g).sum(-1)
    raw = (kg - delta) / ((k * k).sum(-1) + EPS)
    adj = (raw if no_adj_max else np.maximum(0.0, raw)) if trust_region else np.zeros_like(kg)
    gp = g - adj[..., None] * k
    dl = f * ((f * gp).sum(-1, keepdims=True) - gp)
    dpi = np.zeros((nenv, T + 1, nA))
    dpi[:, :T] = dl
    dqv = np.zeros((nenv, T + 1, nA))
    dqv[:, :T] = onehot * (-q_coef * (qret - q_i))[..., None]
    d = qret - q_i
    ev = 1.0 - d.var() / qret.var()
    norm = lambda x: np.sqrt((x * x).sum(-1)).mean()
    stats = np.array([loss, loss_q, entropy, loss_policy, loss_f, loss_bc, ev, norm(k), norm(g), np.abs(kg).mean(),
                      np.abs(adj).mean(), norm(gp)])
    return types.SimpleNamespace(dpi=dpi.reshape(-1, nA), dq=dqv.reshape(-1, nA), qret=qret.reshape(-1),
                                 v=V.reshape(-1), f=F.reshape(-1, nA), stats=stats, adj=adj)


def rmsprop_ema(p, g, ms, shadow, lr, clip, decay=0.99, eps=1e-5, alpha=0.99, eps_outside=False, ema_first=False):
    """tf.clip_by_global_norm + RMSPropOptimizer(decay, eps, momentum 0) + ExponentialMovingAverage(alpha), float64."""
    p, g, ms, shadow = (np.asarray(a, np.float64).copy() for a in (p, g, ms, shadow))
    if clip:
        g = g * (clip / max(np.sqrt((g * g).sum()), clip))
    if ema_first:
        shadow -= (shadow - p) * (1 - alpha)
    ms += (g * g - ms) * (1 - decay)
    p -= lr * g / ((np.sqrt(ms) + eps) if eps_outside else np.sqrt(ms + eps))
    if not ema_first:
        shadow -= (shadow - p) * (1 - alpha)
    return p, ms, shadow


def acer_net(params, copy, x, num_layers=2, scope="acer_model", dev="cpu", kind="mlp"):
    """The ACER network in float64 with autograd leaves: (pi logits, q, leaves, first convs).  kind 'cnn' takes
    uint8 images [B, 84, 84, C]."""
    first = NR._first_convs(kind, [f"{scope}/pi"] + ([f"{scope}/vf"] if copy else []))
    net = NR._Net(False, None, False, None, ())
    leaves = NR._leaves(dict(params), first, False, False, dev)
    xt = NR._t(x, dev)
    tw = dict(num_layers=num_layers, ob_shape=tuple(np.shape(x)[1:]) if kind == "cnn" else None)
    lat = NR._tower(leaves, net, f"{scope}/pi", kind, xt, **tw)
    vlat = NR._tower(leaves, net, f"{scope}/vf", kind, xt, **tw) if copy else lat
    pi = lat @ leaves[f"{scope}/pi/w:0"] + leaves[f"{scope}/pi/b:0"]
    q = vlat @ leaves[f"{scope}/q/w:0"] + leaves[f"{scope}/q/b:0"]
    return pi, q, leaves, first


def train_step(params, shadow, ms, x, actions, rewards, dones, mus, nenv, nsteps, lr, copy, max_grad_norm=10.0,
               trust_region=True, names=None, **head_kw):
    """One whole mlp train call in float64: the head gradients from `head`, the network gradient, the global norm and
    the two partial norms, then clip + RMSProp + moving average.  params / shadow / ms: TF name -> array; names:
    the order of the flat update (every variable is updated elementwise, so any order gives the same result).
    Returns (new params, new ms, new shadow, the 15 statistics in the reference's order)."""
    pi, q, leaves, first = acer_net(params, copy, x)
    with torch.no_grad():
        pol, _, _, _ = acer_net(shadow, copy, x)
    N = nenv * nsteps
    h = head(pi.detach().numpy(), q.detach().numpy(), pol.numpy(), actions, rewards, dones, mus, nenv, nsteps,
             trust_region=trust_region, **head_kw)
    tdp, tdq = torch.from_numpy(h.dpi / N), torch.from_numpy(h.dq / N)

    def grads(a, b):
        gs = torch.autograd.grad((pi * tdp * a).sum() + (q * tdq * b).sum(), list(leaves.values()),
                                 allow_unused=True, retain_graph=True)
        return {k: torch.zeros_like(p) if g is None else g for (k, p), g in zip(leaves.items(), gs)}
    G = grads(1.0, 1.0)
    gn = lambda G: np.sqrt(sum(float((G[k].double() ** 2).sum()) for k in G))
    norm, norm_pol, norm_q = gn(G), gn(grads(1.0, 0.0)), gn(grads(0.0, 1.0))
    names = list(G) if names is None else names
    flat = lambda d, g=False: np.concatenate([np.asarray(d[k].detach().numpy() if g else d[k], np.float64).ravel()
                                              for k in names])
    p1, ms1, sh1 = rmsprop_ema(flat(params), flat(G, True), flat(ms), flat(shadow), lr, max_grad_norm)
    out = []
    for arr in (p1, ms1, sh1):
        d, o = {}, 0
        for k in names:
            n = int(np.prod(np.shape(params[k])))
            d[k] = arr[o:o + n].reshape(np.shape(params[k]))
            o += n
        out.append(d)
    s = h.stats
    stats = list(s[:7]) + [norm, norm_q, norm_pol, s[11], s[7], s[8], s[9], s[10]]
    return out[0], out[1], out[2], np.array(stats), h


def stack_obs(enc_obs, dones, nsteps):
    """The stacking rule of _stack_obs (buffer.py:124-140) restated: block i of row t is frame t + i, multiplied (in the
    frames' dtype) by the 0/1 mask of the dones among the nstack - 1 - i steps before t.  Pinned to the reference's own
    outputs by tests/golden/acer_buffer.npz."""
    nenv, nstack = enc_obs.shape[0], enc_obs.shape[1] - nsteps
    nc = enc_obs.shape[-1]
    out = np.zeros((nenv, nsteps + 1) + enc_obs.shape[2:-1] + (nc * nstack,), dtype=enc_obs.dtype)
    notdone = np.ones((nenv, nsteps + 1), dtype=enc_obs.dtype)
    notdone[:, 1:] = 1 - np.asarray(dones, dtype=enc_obs.dtype)
    for i in range(nstack):
        blk = enc_obs[:, i:i + nsteps + 1]
        if i < nstack - 1:
            keep = np.ones((nenv, nsteps + 1), dtype=enc_obs.dtype)
            for j in range(nstack - 1 - i):
                keep[:, j:] *= notdone[:, :nsteps + 1 - j]
            blk = blk * keep.reshape(keep.shape + (1,) * (enc_obs.ndim - 2))
        out[..., i * nc:(i + 1) * nc] = blk
    return out
