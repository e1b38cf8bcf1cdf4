"""Restatements for the HER tests: the sample-and-encode launch and the normaliser (exact, numpy in the reference's
dtypes), and a float64 mirror of the train step (baselines/her/ddpg.py:355-390, actor_critic.py)."""
import numpy as np


def halves(v):
    """The fp16 [hi | lo] pair of float32 values: hi = fp16(v), lo = fp16(v - hi)."""
    v = np.asarray(v, np.float32)
    hi = v.astype(np.float16)
    return hi, (v - hi.astype(np.float32)).astype(np.float16)


def normalize(x, mean, std, clip):
    """normalizer.py:77 in float32."""
    x = np.asarray(x, np.float32)
    return np.clip((x - mean) / std, np.float32(-clip), np.float32(clip)).astype(np.float32)


def sample(ring, sel, relative, clip_obs, stats, norm_clip, max_u, reward=None, relabel_at=None):
    """her_sampler + _preprocess_og + staging + normalize on float64 ring arrays.  relabel_at (a tempting mistake):
    'ag_t' or 'ag_t1' take the replacement goal from ag[t] or ag[t+1].  -> dict of float32 network inputs and r."""
    o, ag, g, u = ring
    ep, t, ft = sel[:, 0], sel[:, 1], sel[:, 2]
    gs = g[ep, t].copy()
    her = ft >= 0
    src = {None: ft, 'ag_t': t, 'ag_t1': t + 1}[relabel_at]
    gs[her] = ag[ep[her], src[her]]
    ag0, ag1 = ag[ep, t], ag[ep, t + 1]
    out = {}
    if reward is not None:
        rtype, thr = reward
        d = np.linalg.norm(ag1 - gs, axis=-1)
        out['r'] = (-(d > thr).astype(np.float32) if rtype == 'sparse' else -d).astype(np.float32)
    g0 = gs - ag0 if relative else gs
    g1 = gs - ag1 if relative else gs
    c = lambda x: np.clip(x, -clip_obs, clip_obs).astype(np.float32)
    (om, os_), (gm, gsd) = stats
    on, o2n = normalize(c(o[ep, t]), om, os_, norm_clip), normalize(c(o[ep, t + 1]), om, os_, norm_clip)
    gn, g2n = normalize(c(g0), gm, gsd, norm_clip), normalize(c(g1), gm, gsd, norm_clip)
    out.update(o=on, g=gn, o_2=o2n, g_2=g2n, u_in=(u[ep, t].astype(np.float32) / max_u).astype(np.float32),
               ag_2=ag1, g_relabelled=gs)
    return out


def norm_update(state, mean, std, episode, sel, relative, clip_obs, eps, count0=None):
    """Normalizer.update over the sampled transitions of one stored episode batch (numpy in the batch's dtypes),
    then recompute_stats in float32.  state: float32 [sum | sumsq | count].  count0 (a tempting mistake): override the
    count before the update.  -> (state, mean, std)."""
    ep, t, ft = sel[:, 0], sel[:, 1], sel[:, 2]
    o, ag, g = episode['o'][ep, t], episode['ag'][ep, t], episode['g'][ep, t].copy()
    her = ft >= 0
    g[her] = episode['ag'][ep[her], ft[her]]
    if relative:
        g = g - ag
    o, g = np.clip(o, -clip_obs, clip_obs), np.clip(g, -clip_obs, clip_obs)
    out = []
    for v, (st, D) in ((o, (state[0], o.shape[1])), (g, (state[1], g.shape[1]))):
        st = st.copy()
        if count0 is not None:
            st[2 * D] = count0
        local_sum, local_sumsq, local_count = np.zeros(D, np.float32), np.zeros(D, np.float32), np.zeros(1, np.float32)
        local_sum += v.sum(axis=0)
        local_sumsq += (np.square(v)).sum(axis=0)
        local_count[0] += v.shape[0]
        count = (st[2 * D:] + local_count).astype(np.float32)
        s = (st[:D] + local_sum).astype(np.float32)
        sq = (st[D:2 * D] + local_sumsq).astype(np.float32)
        m = (s / count).astype(np.float32)
        e2 = np.float32(eps) * np.float32(eps)
        sd = np.sqrt(np.maximum(e2, sq / count - np.square(s / count))).astype(np.float32)
        out.append((np.concatenate([s, sq, count]), m, sd))
    return out


# ---- the float64 mirror ---------------------------------------------------------------------------------------------
def _fwd(P, scope, x, L, masks=None):
    """masks: per hidden layer, the device's ReLU decisions (bool [B, N]), taken where the float64 pre-activation is
    within fp16 resolution of zero (|z| < 1e-2 of its row's largest): there either sign is a correct rounding."""
    h, hs = x, [x]
    for i in range(L + 1):
        z = h @ P[f'{scope}/_{i}/kernel:0'] + P[f'{scope}/_{i}/bias:0']
        if i < L:
            h = np.maximum(z, 0.0)
            if masks is not None:
                amb = np.abs(z) < 1e-2 * np.abs(z).max(axis=1, keepdims=True)
                h = np.where(amb, np.where(masks[i], z, 0.0), h)
            hs.append(h)
    return z, hs


def _bwd(P, scope, hs, dz, L):
    """d loss / d z of the last layer -> ({tf name: gradient}, d loss / d input)."""
    G = {}
    for i in reversed(range(L + 1)):
        W = P[f'{scope}/_{i}/kernel:0']
        G[f'{scope}/_{i}/kernel:0'] = hs[i].T @ dz
        G[f'{scope}/_{i}/bias:0'] = dz.sum(axis=0)
        dx = dz @ W.T
        dz = dx * (hs[i] > 0) if i > 0 else dx
    return G, dx


def ambiguous_units(P, scope, x, L, masks):
    """How many hidden units the device's ReLU decisions settle (see _fwd), and whether every other decision agrees."""
    h, n, agree = np.asarray(x, np.float64), 0, True
    for i in range(L):
        z = h @ P[f'{scope}/_{i}/kernel:0'] + P[f'{scope}/_{i}/bias:0']
        amb = np.abs(z) < 1e-2 * np.abs(z).max(axis=1, keepdims=True)
        n += int(amb.sum())
        agree &= bool(np.array_equal((z > 0)[~amb], masks[i][~amb]))
        h = np.maximum(z, 0.0)
    return n, agree


def train_step(P, inp, cfg, variant=None, pi_masks=None):
    """One HER step in float64 from the float32 network inputs.  P: {tf name: array} of main and target; inp: sample()'s
    dict plus r; cfg: dimo, dimg, dimu, layers, max_u, gamma, clip_return, clip_pos_returns, action_l2.  variant (the
    tempting mistakes): 'l2_over_B', 'no_upper_clip', 'u_not_scaled'.  pi_masks: the device's ReLU decisions of the
    main actor's hidden layers (see _fwd).  -> dict of gradients, loss, y, q_pi."""
    f = lambda a: np.asarray(a, np.float64)
    L, mu, s = cfg['layers'], f(cfg['max_u']), cfg['scope']
    o, g, o2, g2, r = f(inp['o']), f(inp['g']), f(inp['o_2']), f(inp['g_2']), f(inp['r'])
    u_in = f(inp['u_in']) if variant != 'u_not_scaled' else f(inp['u_in']) * mu
    B, dimu = o.shape[0], cfg['dimu']
    P = {k: f(v) for k, v in P.items()}
    zt, _ = _fwd(P, f'{s}/target/pi', np.concatenate([o2, g2], 1), L)
    pit = mu * np.tanh(zt)
    qt, _ = _fwd(P, f'{s}/target/Q', np.concatenate([o2, g2, pit / mu], 1), L)
    hi = 0. if cfg['clip_pos_returns'] and variant != 'no_upper_clip' else np.inf
    y = np.clip(r + cfg['gamma'] * qt[:, 0], -cfg['clip_return'], hi)
    z, hpi = _fwd(P, f'{s}/main/pi', np.concatenate([o, g], 1), L, pi_masks)
    pi = mu * np.tanh(z)
    q, hq = _fwd(P, f'{s}/main/Q', np.concatenate([o, g, u_in], 1), L)
    qpi, hqpi = _fwd(P, f'{s}/main/Q', np.concatenate([o, g, pi / mu], 1), L)
    loss = np.mean((y - q[:, 0]) ** 2)
    GQ, _ = _bwd(P, f'{s}/main/Q', hq, (-2.0 * (y - q[:, 0]) / B)[:, None], L)
    _, dx = _bwd(P, f'{s}/main/Q', hqpi, np.full((B, 1), -1.0 / B), L)
    n_l2 = B if variant == 'l2_over_B' else B * dimu
    dpi = dx[:, -dimu:] / mu + cfg['action_l2'] * 2.0 * (pi / mu) / mu / n_l2
    dz = dpi * mu * (1.0 - np.tanh(z) ** 2)
    Gpi, _ = _bwd(P, f'{s}/main/pi', hpi, dz, L)
    pi_loss = -np.mean(qpi) + cfg['action_l2'] * np.mean((pi / mu) ** 2)
    return dict(Q_grads=GQ, pi_grads=Gpi, loss=loss, pi_loss=pi_loss, y=y, q_pi=qpi[:, 0])
