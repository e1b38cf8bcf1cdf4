"""Plain float64 references for the kernels between the last GEMM of an update and the parameter write: the PPO2 loss
heads (Categorical, MultiCategorical, Bernoulli, DiagGaussian), the advantage moments, the DQN TD / Huber step and
TF-Adam, plus the device buffers of the three head layouts the kernels must handle.

Everything here is ordinary torch / numpy arithmetic in float64 on the CPU; nothing calls a kernel of the project.

The PPO2 loss is ppo2/model.py:57-91 in "sum" scaling (the kernels leave the 1/M of tf.reduce_mean to the weight
gradient epilogues), with the distributions of tests/_action_oracle.py and oracle/nets.py.  tf.maximum sends the
gradient of a tie to its first argument; torch.maximum would split it, so the references use torch.where.  A `mutant`
builds the same reference with one plausible kernel mistake, for the self-check of a tolerance (tests/_refs.py).
"""
import types

import numpy as np
import torch

import _action_oracle as ao

LAYOUTS = ("fused", "copy", "scalar")
F16_G = 1e-6                 # absolute part of the fp16 gradient bound: |got - ref| <= 2^-11 |ref| + 1e-6


def pad(n, m):
    return (n + m - 1) // m * m


# ------------------------------------------------------------------------------------------------ head buffers
def head_bufs(nout, B, layout, rows=None):
    """Device buffers of a head's outputs (fp32) and gradients (fp16) in the layouts PolicyNet and the kernels use:

      fused  : [pi | vf] in one row (value in column nout), gradient row [dpi | dv] with a pitch that is a multiple of 8
               (16-byte vector stores; dv is column nout of the gradient row);
      copy   : value_network='copy': separate value and dv buffers, gradient pitch a multiple of 8;
      scalar : fused rows, but the gradient view starts one column into an odd-pitch buffer, so the kernels must take
               their one-element store path.

    Gradient buffers have `rows` (>= B) rows and start as NaN: what a kernel must not write keeps the NaN.
    Returns a namespace with ho, ld, vo, ldv (inputs), g, ld_g, dv, ld_dv (outputs), zero_cols (columns of a written
    gradient row the kernel stores as exact zeros) and keep_cols (columns of a written row that must stay NaN)."""
    rows = B if rows is None else rows
    nan = float("nan")
    if layout == "fused":
        ld, ld_g = pad(nout + 1, 16), pad(nout + 1, 64)
        ho = torch.zeros(B, ld, device="cuda")
        g = torch.full((rows, ld_g), nan, dtype=torch.float16, device="cuda")
        vo, ldv, dv, ld_dv = ho[:, nout:], ld, g[:, nout:], ld_g
        written = set(range(nout + 1)) | set(range(nout, pad(nout, 8)))
        zero = set(range(nout + 1, pad(nout, 8)))
    elif layout == "copy":
        ld, ld_g = pad(nout, 16), pad(nout, 64)
        ho = torch.zeros(B, ld, device="cuda")
        g = torch.full((rows, ld_g), nan, dtype=torch.float16, device="cuda")
        vo, ldv = torch.zeros(B, 16, device="cuda"), 16
        dv, ld_dv = torch.full((rows, 8), nan, dtype=torch.float16, device="cuda"), 8
        written = set(range(pad(nout, 8)))
        zero = set(range(nout, pad(nout, 8)))
    else:
        assert layout == "scalar", layout
        ld = pad(nout + 1, 16) + 3                            # odd input pitch too
        ho = torch.zeros(B, ld, device="cuda")[:, 1:]
        ld_g = pad(nout + 2, 8) + 1                           # odd pitch, and the view starts 2 bytes into the buffer
        g = torch.full((rows, ld_g), nan, dtype=torch.float16, device="cuda")[:, 1:]
        assert g.data_ptr() % 16 == 2
        vo, ldv, dv, ld_dv = ho[:, nout:], ld, g[:, nout:], ld_g
        written, zero = set(range(nout + 1)), set()
    keep = sorted(set(range(g.shape[1])) - written)
    return types.SimpleNamespace(ho=ho, ld=ld, vo=vo, ldv=ldv, g=g, ld_g=ld_g, dv=dv, ld_dv=ld_dv,
                                 zero_cols=sorted(zero), keep_cols=keep, rows=rows, layout=layout)


def check_untouched(bufs, B, nout):
    """Rows past B keep their NaN; in written rows the padding the vector store covers is exactly 0 and every other
    column outside the head keeps its NaN."""
    g = bufs.g.float().cpu()
    assert bool(torch.isnan(g[B:]).all()), "the kernel wrote gradient rows past B"
    if bufs.zero_cols:
        assert float(g[:B, bufs.zero_cols].abs().max()) == 0.0, "padding of the last 8-column store group is not 0"
    if bufs.keep_cols:
        assert bool(torch.isnan(g[:B, bufs.keep_cols]).all()), "the kernel wrote columns outside the head"
    if bufs.layout == "copy":
        d = bufs.dv.float().cpu()
        assert bool(torch.isnan(d[B:]).all()) and bool(torch.isnan(d[:B, 1:]).all())


# ------------------------------------------------------------------------------------------------ PPO2 loss
def _tf_max(a, b):
    """tf.maximum: value max(a, b), gradient to the first argument on ties."""
    return torch.where(a >= b, a, b)


def ppo_ref(pd, head, v, acts, R, oldv, oldnlp, adv, clip, ent_coef, vf_coef, nvec=None, logstd=None, mutant=None):
    """float64 per-row PPO2 loss of ppo2/model.py:57-91 and its gradients, sum scaling.

    pd: 'cat' / 'mcat' / 'bern' / 'gauss'; head [B, nout] logits or means; v [B]; acts rows as the kernel reads them;
    adv the normalised advantages (float32 values, as the kernel rounds them).  logstd [d] for 'gauss'.
    mutant: None, 'no_entropy' (-ent_coef * H dropped), 'pg_clip_passes' (the clipped surrogate passes gradient outside
    [1 - clip, 1 + clip]), 'vf_clip_passes' (the clipped value passes gradient outside its interval), 'vf_wrong_branch'
    (the value gradient of the smaller of the two losses), 'drop_last_entropy' (MultiCategorical: the last segment's
    entropy missing).
    Returns a namespace: dhead [B, nout], dv [B], dlogstd_rows [B, d] (gauss: per-row dL/dlogstd), rows5 [B, 5]
    (per-row pg loss, value loss, entropy, approxkl, clipfrac), stats [5] (their sums), nlp, ratio, near (rows within
    fp32 rounding of a branch boundary, where the kernel may legitimately take the other branch), zones (dict of
    per-row branch masks)."""
    f64 = lambda x: torch.as_tensor(np.asarray(x), dtype=torch.float64)
    l = f64(head).clone().requires_grad_(True)
    vv = f64(v).clone().requires_grad_(True)
    B = l.shape[0]
    ls = None
    if pd == "gauss":
        ls = f64(logstd)[None].repeat(B, 1).requires_grad_(True)
        a = f64(acts)
        nlp = ao.neglogp("gauss", l, ls, a)
        H = ao.entropy("gauss", l, ls)
    else:
        a = f64(acts) if pd == "bern" else torch.as_tensor(np.asarray(acts))
        nlp = ao.neglogp(pd, l, None, a, nvec)
        if mutant == "drop_last_entropy":
            H = ao.mcat_entropy(l, nvec) - ao.mcat_entropy(l[:, sum(nvec[:-1]):], nvec[-1:])
        else:
            H = ao.entropy(pd, l, None, nvec)
    R, oldv, oldnlp, adv = (f64(x) for x in (R, oldv, oldnlp, adv))
    ratio = torch.exp(oldnlp - nlp)
    rc = torch.clamp(ratio, 1 - clip, 1 + clip)
    if mutant == "pg_clip_passes":
        rc = ratio + (rc - ratio).detach()
    p1, p2 = -adv * ratio, -adv * rc
    pg = _tf_max(p1, p2)
    dvv = vv - oldv
    vcl = oldv + torch.clamp(dvv, -clip, clip)
    if mutant == "vf_clip_passes":
        vcl = vv + (vcl - vv).detach()
    l1, l2 = (vv - R) ** 2, (vcl - R) ** 2
    vl = 0.5 * _tf_max(l1, l2)
    if mutant == "vf_wrong_branch":
        lo = torch.where(l1 >= l2, l2, l1)
        vl = vl.detach() + 0.5 * (lo - lo.detach())
    ent_term = 0.0 if mutant == "no_entropy" else ent_coef * H
    loss = (pg - ent_term + vf_coef * vl).sum()
    grads = torch.autograd.grad(loss, [l, vv] + ([ls] if ls is not None else []))
    kl = 0.5 * (nlp - oldnlp) ** 2
    cf = ((ratio - 1).abs() > clip).double()
    rows5 = torch.stack([pg, vl, H, kl, cf], 1).detach()
    r, d, L1, L2 = ratio.detach(), dvv.detach(), l1.detach(), l2.detach()
    vclipped = d.abs() > clip
    near = ((r - (1 - clip)).abs() <= 1e-4 * r) | ((r - (1 + clip)).abs() <= 1e-4 * r)
    near |= (d.abs() - clip).abs() <= 1e-5 * (1 + vv.detach().abs() + oldv.abs())
    near |= vclipped & ((L1 - L2).abs() <= 1e-5 * (L1 + L2))
    zones = {"ratio_below": r < 1 - clip, "ratio_inside": (r >= 1 - clip) & (r <= 1 + clip),
             "ratio_above": r > 1 + clip, "adv_pos": adv > 0, "adv_neg": adv < 0,
             "v_unclipped": ~vclipped, "v_low": d < -clip, "v_high": d > clip, "l1_ge_l2": L1 >= L2, "l1_lt_l2": L1 < L2}
    return types.SimpleNamespace(
        dhead=grads[0].numpy(), dv=grads[1].numpy(), dlogstd_rows=grads[2].numpy() if ls is not None else None,
        rows5=rows5.numpy(), stats=rows5.sum(0).numpy(), nlp=nlp.detach().numpy(), ratio=r.numpy(),
        near=near.numpy(), zones={k: z.numpy() for k, z in zones.items()})


def gumbel_clear(l32, u, nvec, gap=1e-4):
    """Rows whose Gumbel-max sample (scores l - log(-log u)) has a top-2 gap above `gap` in every segment: there the
    fp32 kernel and a float64 reference must pick the same action."""
    sc = l32.astype(np.float64) - np.log(-np.log(u.astype(np.float64)))
    clear = np.ones(l32.shape[0], bool)
    for blk in np.split(sc, np.cumsum(nvec)[:-1], axis=1):
        if blk.shape[1] > 1:
            top2 = np.sort(blk, 1)[:, -2:]
            clear &= (top2[:, 1] - top2[:, 0]) > gap
    return clear


def adv_normalise(R, oldv, mean, std):
    """The kernels' normalised advantage: the fp32 difference, centred and scaled in float64, rounded to fp32
    (ppo2/model.py:136-139 with the moments of adv_stats)."""
    d = (np.asarray(R, np.float32) - np.asarray(oldv, np.float32)).astype(np.float64)
    return ((d - mean) / (std + 1e-8)).astype(np.float32)


# ------------------------------------------------------------------------------------------------ advantage moments
def adv_moments(R, V):
    """Two-pass float64 mean and population std of the fp32 differences R - V (numpy's np.std, ddof = 0)."""
    d = (np.asarray(R, np.float32) - np.asarray(V, np.float32)).astype(np.float64)
    mean = d.sum() / d.size
    return mean, float(np.sqrt(((d - mean) ** 2).sum() / d.size))


def gamma_k(k, u=2.0 ** -53):
    """Higham's gamma_k = k u / (1 - k u): the relative error bound of k floating-point additions in a row."""
    return k * u / (1 - k * u)


# ------------------------------------------------------------------------------------------------ DQN TD step
def dueling_q(a, s):
    """deepq/models.py:38-40: q = s + (a - mean(a)); s None: q = a."""
    return a if s is None else s[:, None] + (a - a.mean(1, keepdim=True))


def dqn_ref(qt_a, qt_s, on_a, on_s, tg_a, tg_s, actions, rewards, dones, weights, gamma, double_q, mutant=None):
    """float64 TD error, sum_b w_b huber(td_b) and its gradients w.r.t. the raw q(s) head outputs (build_graph.py:
    388-413, tf_util.py:39-45).  All row arrays are per batch row (already gathered).  double_q: the online argmax
    (first index of the max wins, as tf.argmax); mutant 'last_max' lets the last one win.
    Returns a namespace: td, d_a [B, nA], d_s [B] (None without dueling), loss, gap (top-2 gap of the online q, inf
    when nA == 1)."""
    f64 = lambda x: None if x is None else torch.as_tensor(np.asarray(x), dtype=torch.float64)
    a = f64(qt_a).clone().requires_grad_(True)
    s = None if qt_s is None else f64(qt_s).clone().requires_grad_(True)
    q = dueling_q(a, s)
    q_tg = dueling_q(f64(tg_a), f64(tg_s))
    nA = a.shape[1]
    if double_q:
        q_on = dueling_q(f64(on_a), f64(on_s))
        arg = torch.argmax(q_on, 1) if mutant != "last_max" else nA - 1 - torch.argmax(q_on.flip(1), 1)
        best = q_tg.gather(1, arg[:, None])[:, 0]
        top2 = torch.sort(q_on, 1).values
        gap = (top2[:, -1] - top2[:, -2]) if nA > 1 else torch.full((a.shape[0],), float("inf"), dtype=torch.float64)
    else:
        best = q_tg.max(1).values
        gap = torch.full((a.shape[0],), float("inf"), dtype=torch.float64)
    target = f64(rewards) + gamma * (1.0 - f64(dones)) * best
    td = q.gather(1, torch.as_tensor(np.asarray(actions)).long()[:, None])[:, 0] - target
    x = td.abs()
    hub = torch.where(x < 1.0, 0.5 * td * td, x - 0.5)
    loss = (f64(weights) * hub).sum()
    grads = torch.autograd.grad(loss, [a] + ([s] if s is not None else []))
    return types.SimpleNamespace(td=td.detach().numpy(), d_a=grads[0].numpy(),
                                 d_s=grads[1].numpy() if s is not None else None, loss=float(loss.detach()),
                                 rows_loss=(f64(weights) * hub).detach().numpy(), gap=gap.numpy())


# ------------------------------------------------------------------------------------------------ TF-Adam
def adam_tf(p, g, m, v, lr_t, beta1, beta2, eps):
    """One TF-Adam step in the order of mpi_adam.py:37-42 with the step size lr_t = lr sqrt(1 - b2^t) / (1 - b1^t)
    already formed: m = b1 m + (1 - b1) g; v = b2 v + (1 - b2) g^2; p = p - lr_t m / (sqrt(v) + eps)."""
    m = beta1 * m + (1 - beta1) * g
    v = beta2 * v + (1 - beta2) * g * g
    return p - lr_t * m / (np.sqrt(v) + eps), m, v


def clip_scale(sumsq, clip):
    """tf.clip_by_global_norm / tf.clip_by_norm factor clip / max(||g||, clip); 1 when clip <= 0."""
    return 1.0 if clip <= 0 else clip / max(float(np.sqrt(sumsq)), clip)


# ------------------------------------------------------------------------------------------------ sampler streams
_M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(seed, rows, ctr, stream):
    """The acting samplers' Philox4x32-10 (csrc/policy_heads.cu philox4) on the host: counter (row lo, row hi, ctr,
    stream), key = seed.  rows: int array; returns uint32 [len(rows), 4]."""
    r = np.asarray(rows, np.uint64)
    c = [r & _M32, r >> np.uint64(32), np.full_like(r, ctr), np.full_like(r, stream)]
    k0, k1 = np.uint64(seed & 0xFFFFFFFF), np.uint64((seed >> 32) & 0xFFFFFFFF)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c[0], np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _M32]
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & _M32, (k1 + np.uint64(0xBB67AE85)) & _M32
    return np.stack(c, 1).astype(np.uint32)


def philox_uniforms(seed, B, n, offset):
    """float32 [B, n]: uniform j of row b of an acting pass at stream position `offset` -- word j % 4 of counter j // 4,
    mapped to the open interval as u01_open does (fp32 arithmetic, as on the device)."""
    out = np.empty((B, n), np.float32)
    for c in range(-(-n // 4)):
        w = philox4x32_10(seed, np.arange(B), c, offset)
        for i in range(4):
            if 4 * c + i < n:
                out[:, 4 * c + i] = ((w[:, i] >> 8).astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -24)
    return out


def dqn_act_draws(seed, step, B, nA):
    """The DQN act kernel's splitmix64 draws (csrc/replay.cu dqn_act_kernel) for rows 0..B-1 at `step`: (u float32 in
    (0, 1), the random action in [0, nA))."""
    m = (1 << 64) - 1
    us, rs = np.empty(B, np.float32), np.empty(B, np.int64)
    for b in range(B):
        x = (seed + 0x9E3779B97F4A7C15 * ((step * 1315423911 + b + 1) & m)) & m
        x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & m
        x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & m
        x ^= x >> 31
        us[b] = (np.float32(x >> 40) + np.float32(0.5)) * np.float32(2.0 ** -24)
        rs[b] = (x & 0xFFFFFF) % nA
    return us, rs
