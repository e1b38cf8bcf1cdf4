"""Plain float64 mirror of the networks an update runs through: the PPO2 policy / value network (common/policies.py
PolicyNet over nn.Tower) and the DQN Q network (deepq/build_graph.py QNet), with their gradients.

Everything here is ordinary torch arithmetic in float64; it runs on the CPU or the GPU and never calls a kernel of the
project.  Parameters come in the TF naming and layouts of `ParamStore.export_tf` (conv HWIO, fc [in, out]).

`policy_ref` / `q_ref` evaluate the network on the observations and return the head outputs, every pre-activation and
d(sum(out * seed)) / d(param) for each TF variable.  The frozen identity head of PolicyNet (latent width == nout) has
no TF variable; for it the gradient of the internal `head_pi/w`, `head_pi/b` is returned.

rnd=True evaluates what the kernels evaluate:
  * weights rounded to fp16 (the first conv's with 1/255 folded in first, as nn.Conv's in_scale does); biases fp32;
  * every stored activation rounded to fp16, straight-through for the gradient;
  * tanh' taken as 1 - s^2 from the stored fp16 activation s;
  * every stored pre-activation gradient (the data-gradient GEMMs' fp16 outputs) rounded to fp16 in the backward;
  * ReLU decisions taken from `masks` (name -> 0/1 tensor shaped like the pre-activation) where the caller supplies
    them, e.g. from the kernels' own stored activations; for a tanh layer `masks[name]` is the stored activation itself,
    which replaces the mirror's in the forward (the backward keeps the mirror's 1 - s^2);
  * a ReLU layer's stored activation taken from `stored` (name -> the kernels' fp16 values) where the caller supplies
    it, as the forward value only (straight-through): the kernels round an fp32 sum and the mirror a float64 one, so
    the two can differ by one fp16 rounding, and under a recurrence (cnn_lstm's latent into the cell) such a flip
    carries into every later step.  The caller checks that both agree within that rounding first;
  * mlp observations kept in float32: the encoder's fp16 hi/lo split loses at most max(2^-22 |v|, 2^-25);
  * LayerNorm: z stays fp32 (exact here), the output activation y is stored fp16, d loss / d z is stored fp16;
  * LSTM: Wx and Wh fp16; xg, c and the gates fp32 (exact here); h and the masked h_{t-1} stored fp16; dz rounded to
    fp16 where the weight-gradient / data-gradient GEMMs read it, unrounded in the recurrent carry.

absolute=True evaluates the same network on |x|, |W|, |b| and |seed| with the ReLU masks and stored tanh activations of
a signed run (`ref_acts`): a tanh layer outputs |s| and passes the gradient through |1 - s^2|; a LayerNorm outputs
|gamma| (|xhat| + |J| z) + |beta| (its size plus the error z carries into it) and passes the gradient through |J|^T, the
magnitudes of its Jacobian's terms.  The LSTM cell's forward outputs |h| of the signed run only: it does not carry the
size of |x| |Wx| + |h_{t-1}| |Wh| into h, so the cell's forward rounding error is not in S and the fitted per-tensor
factor g of the GPU tests absorbs it; its backward takes every factor of the BPTT by magnitude.  Outputs and gradients
are the scale S of the error bound (tests/_refs.py), the network analogue of |A| @ |B|.
"""
import collections
import types

import numpy as np
import torch

import _layer_norm_refs as LN
import _lstm_oracle as LO
import _refs as R

NATURE_CONVS = (("c1", 32, 8, 4), ("c2", 64, 4, 2), ("c3", 64, 3, 1))   # common/models.py:21-24


# ------------------------------------------------------------------------------------------------ conv stack
def conv_geometry(ob_shape, convs, same):
    """Per conv layer (stride, (pad_top, pad_left), OH, OW) of a stack over (H, W, C) inputs (VALID or TF SAME)."""
    H, W, _ = ob_shape
    out = []
    for _nm, _nf, rf, st in convs:
        if same:
            OH, OW = -(-H // st), -(-W // st)
            pads = (max((OH - 1) * st + rf - H, 0) // 2, max((OW - 1) * st + rf - W, 0) // 2)
        else:
            OH, OW, pads = (H - rf) // st + 1, (W - rf) // st + 1, (0, 0)
        out.append((st, pads, OH, OW))
        H, W = OH, OW
    return out


def conv_stack(x, Ws, bs, geometry, act):
    """The conv layers of a tower in float64: pre_i = conv(a_(i-1), W_i) + b_i with W_i HWIO, a_i = act(i, pre_i).
    Returns the last activation and every pre-activation."""
    a, pres = x, []
    for i, (W, b, (st, pads, OH, OW)) in enumerate(zip(Ws, bs, geometry)):
        pre = R.conv2d(a, W, (st, st), pads, OH, OW) + b.reshape(-1)
        pres.append(pre)
        a = act(i, pre)
    return a, pres


def kernel_act(tower, i, B, start=0):
    """NHWC [B, OH, OW, nf] view of the kernels' stored activation of conv i of an nn.Tower, samples start .. start+B.
    Every layout stores a sample's activations as one run of OH * OW * nf elements."""
    c = tower.convs[i]
    h = tower.hconv[i]
    if tower.shift_mode and i + 1 < len(tower.convs) and tower.convs[i + 1].stride > 1:
        s = tower.convs[i + 1].stride
        return R.depth_to_space(h[start:start + B].view(B, c.OH // s, c.OW // s, s * s * c.nf), s)
    return h.reshape(-1)[start * c.P * c.nf:(start + B) * c.P * c.nf].view(B, c.OH, c.OW, c.nf)


def reference(tower, imgs, Ws, bs, masks, dlat, B, rnd=True):
    """float64 forward through the conv stack (+ fc1) of an nn.Tower with the given weights and ReLU masks; returns the
    last layer's pre-activation and the pre-activations of every conv.  Backward: d(sum(pre_last * dlat) / B)."""
    nconv = len(tower.convs)

    def act(i, pre):
        if i + 1 == nconv and not tower.fcs:
            return pre
        a = pre * masks[i]
        return a + (a.half().double() - a).detach() if rnd else a     # the kernels store activations in fp16
    c0 = tower.convs[0]
    geom = conv_geometry((c0.H, c0.W, c0.C), [(c.name, c.nf, c.rf, c.stride) for c in tower.convs], c0.same)
    a, pres = conv_stack(imgs, Ws[:nconv], bs[:nconv], geom, act)
    if not tower.fcs:
        return a.reshape(B, -1), pres
    return a.reshape(B, -1) @ Ws[nconv] + bs[nconv], pres


# ------------------------------------------------------------------------------------------------ activations
class _StoredTanh(torch.autograd.Function):
    """s = tanh(z) (rounded to fp16 when rnd); backward g * (1 - s^2) from the stored s (g alone when no_dact)."""

    @staticmethod
    def forward(ctx, z, rnd, no_dact):
        s = torch.tanh(z)
        if rnd:
            s = s.half().double()
        ctx.save_for_backward(s)
        ctx.no_dact = no_dact
        return s

    @staticmethod
    def backward(ctx, g):
        s, = ctx.saved_tensors
        return (g if ctx.no_dact else g * (1.0 - s * s)), None, None


class _GradRound(torch.autograd.Function):
    """Identity forward; the backward rounds the incoming gradient to fp16 (a data gradient the kernels store)."""

    @staticmethod
    def forward(ctx, z):
        return z.view_as(z)

    @staticmethod
    def backward(ctx, g):
        return g.half().double()


class _AbsLayerNorm(torch.autograd.Function):
    """Absolute mode of a LayerNorm at the signed run's xhat and rstd, with |J| the magnitudes of the terms of
    J = rstd (I - 1/N - xhat xhat^T / N): u = |gamma| (|xhat| + |J| z) + |beta| for the absolute run's z (the size of
    xhat plus the error z carries into it); the backward passes |J|^T (|gamma| g) to z, and g (|xhat| + |J| z), g to
    gamma and beta."""

    @staticmethod
    def forward(ctx, z, gamma, beta, xhat, rstd):
        ax = xhat.abs()
        scale = ax + rstd * (z + z.mean(1, keepdim=True) + ax * (ax * z).mean(1, keepdim=True))
        ctx.save_for_backward(gamma, ax, rstd, scale)
        return gamma * scale + beta

    @staticmethod
    def backward(ctx, g):
        gamma, ax, rstd, scale = ctx.saved_tensors
        gg = gamma * g
        dz = rstd * (gg + gg.mean(1, keepdim=True) + ax * (gg * ax).mean(1, keepdim=True))
        return dz, (g * scale).sum(0), g.sum(0), None, None


class _LSTMSeq(torch.autograd.Function):
    """h rows [T*E, H] of the cell (tests/_lstm_oracle.py lstm_steps) from the input projection xg [T*E, 4H], Wh, masks
    [T, E] and start states [E, 2H]; the backward is lstm_steps_backward.  The recurrent carry keeps dz unrounded (the
    kernel holds it in fp32); with rnd the gradients of xg (-> Wx, b, x) and Wh take dz rounded to fp16 and Wh's takes
    the stored fp16 masked h_{t-1}, as the weight-gradient GEMMs read them.  With ref (the signed run's gates, c,
    masked h_{t-1}) the absolute network: |h| of the signed run forward (see the module docstring), every factor of
    the BPTT taken by magnitude.  unmasked_dwh
    (mutant): dWh from h_{t-1} before the mask."""

    @staticmethod
    def forward(ctx, xg, wh, masks, s0, rnd, ref, unmasked_dwh):
        T, E = masks.shape
        H = wh.shape[0]
        np_ = lambda t: t.detach().cpu().numpy()
        if ref is None:
            h, cs, gates, hps, _ = LO.lstm_steps(np_(xg), np_(wh), masks, s0, T, E, H)
            prev = np.concatenate([s0[None, :, H:], h.reshape(T, E, H)[:-1]]).reshape(T * E, H)
        else:
            h, cs, gates, hps, prev = ref
            h, cs, gates = np.abs(h), np.abs(cs), gates.copy()
            gates[:, 3 * H:] = np.abs(gates[:, 3 * H:])
            s0 = np.abs(s0)
        ctx.saved = (gates, cs, hps, prev, masks, s0, np_(wh), rnd, ref is not None, unmasked_dwh)
        ctx.dev = xg.device
        ctx.record = (h, cs, gates, hps, prev)
        return torch.as_tensor(h, device=xg.device)

    @staticmethod
    def backward(ctx, dh):
        gates, cs, hps, prev, masks, s0, wh, rnd, absolute, unmasked_dwh = ctx.saved
        T, E = masks.shape
        H = wh.shape[0]
        dhn = dh.detach().cpu().numpy()
        dz = LO.lstm_steps_backward(np.abs(dhn) if absolute else dhn, gates, cs, masks, s0, wh, T, E, H)
        a = np.abs(prev if unmasked_dwh else hps) if absolute else (prev if unmasked_dwh else hps)
        if rnd:
            dz, a = _f16(dz), _f16(a)
        t = lambda v: torch.as_tensor(v, device=ctx.dev)
        return t(dz), t(a.T @ dz), None, None, None, None, None


def _f16(a):
    return np.asarray(a).astype(np.float16).astype(np.float64)


class _Net:
    """Evaluation state of one mirror run: rounding, masks, the signed run's activations (absolute mode), records."""

    def __init__(self, rnd, masks, absolute, ref_acts, no_dact, stored=None):
        self.rnd, self.masks, self.absolute, self.stored = rnd, masks or {}, absolute, stored or {}
        self.ref_acts, self.no_dact = ref_acts or {}, set(no_dact or ())
        self.pres, self.acts = collections.OrderedDict(), collections.OrderedDict()

    def act(self, name, pre, kind):
        """kind 'relu' / 'tanh' / None (no activation, not stored)."""
        self.pres[name] = pre.detach()
        if kind is None:
            return pre
        if self.rnd:
            pre = _GradRound.apply(pre)
        if self.absolute:
            ra = self.ref_acts[name]
            if kind == "relu":
                return pre * ra
            return ra.abs() + (pre - pre.detach()) * (1.0 - ra * ra).abs()
        if kind == "relu":
            m = self.masks.get(name)
            m = (pre > 0).double() if m is None else m.double()
            self.acts[name] = m
            a = pre * m
            if name in self.no_dact:                    # mutant: the mask's derivative left out of the backward
                a = pre + (a - pre).detach()
            a = a + (a.half().double() - a).detach() if self.rnd else a
            st = self.stored.get(name)
            return a if st is None else a + (st.double() - a).detach()
        s = _StoredTanh.apply(pre, self.rnd, name in self.no_dact)
        m = self.masks.get(name)
        if m is not None:                               # the kernels' stored activation (forward value only)
            s = s + (m.double() - s).detach()
        self.acts[name] = s.detach()
        return s

    def ln(self, scope, z, gamma, beta):
        """LayerNorm `scope` over a fully connected layer's fp32 pre-activation z: u = gamma * xhat + beta
        (_layer_norm_refs.ln_torch).  With rnd the kernels' stored d loss / d z is fp16; z itself stays fp32 (exact
        here).  The caller passes u to act(), which rounds the stored activation and d loss / d u."""
        if self.rnd:
            z = _GradRound.apply(z)
        if self.absolute:
            return _AbsLayerNorm.apply(z, gamma, beta, *self.ref_acts[scope])
        zd = z.detach()
        mean = zd.mean(1, keepdim=True)
        rstd = 1.0 / torch.sqrt(((zd - mean) ** 2).mean(1, keepdim=True) + LN.EPS)
        self.acts[scope] = ((zd - mean) * rstd, rstd)
        return LN.ln_torch(z, gamma, beta)

    def lstm(self, name, xg, wh, seq, unmasked_dwh=False):
        """The LSTM cell over the time-major rows of xg = x.wx + b (seq = (masks [T, E], start states [E, 2H]), numpy
        float64).  With rnd h is stored fp16 and the heads' d loss / d h arrives in fp16."""
        masks, s0 = seq
        h = _LSTMSeq.apply(xg, wh, masks, s0, self.rnd, self.ref_acts.get(name) if self.absolute else None,
                           unmasked_dwh)
        if not self.absolute:
            self.acts[name] = h.grad_fn.record if h.grad_fn is not None else None
        if self.rnd:
            h = _GradRound.apply(h)
            h = h + (h.half().double() - h).detach()
        return h


def _leaves(params, first_convs, rnd, absolute, dev):
    """float64 leaf tensors of the TF variables the kernels use: fp16-rounded weights (c1 scaled by 1/255 first)."""
    out = collections.OrderedDict()
    scale1 = torch.tensor(1.0 / 255.0, dtype=torch.float32)
    for k, v in params.items():
        t = torch.as_tensor(np.asarray(v))
        is_w = k.endswith(("/w:0", "/weights:0", "/lstm/wx:0", "/lstm/wh:0"))
        if k in first_convs:
            t = (t.float() * scale1).half().double() if rnd else t.double() / 255.0
        elif is_w and rnd:
            t = t.float().half().double()
        else:
            t = t.double()
        t = t.to(dev)
        out[k] = (t.abs() if absolute else t).requires_grad_(True)
    return out


def _tower(P, net, prefix, kind, x, convs=NATURE_CONVS, same=False, num_layers=2, contrib=False, ob_shape=None,
           seq=None, unmasked_dwh=False):
    """Latent of one nn.Tower: cnn / conv_only convs over uint8 images [B, H, W, C] (as float64), the tanh mlp over
    encoded observation rows [B, in_dim] (layer-normalised where P holds the norms), or the LSTM cell of lstm /
    cnn_lstm over time-major rows (seq: see policy_ref)."""
    B = x.shape[0]
    if kind in ("lstm", "cnn_lstm"):
        # models.py lstm: the encoded observation straight into the cell; cnn_lstm: the NatureCNN latent
        lat = x if kind == "lstm" else _tower(P, net, prefix, "cnn", x, ob_shape=ob_shape)
        xg = lat @ P[f"{prefix}/lstm/wx:0"] + P[f"{prefix}/lstm/b:0"]
        return net.lstm(f"{prefix}/lstm", xg, P[f"{prefix}/lstm/wh:0"], seq, unmasked_dwh=unmasked_dwh)
    if kind in ("cnn", "conv_only"):
        if contrib:
            names = [f"{prefix}/convnet/{'Conv' if i == 0 else f'Conv_{i}'}" for i in range(len(convs))]
            wk, bk = "weights:0", "biases:0"
        else:
            names = [f"{prefix}/{nm}" for nm, _nf, _rf, _st in convs]
            wk, bk = "w:0", "b:0"
        a, _ = conv_stack(x, [P[f"{n}/{wk}"] for n in names], [P[f"{n}/{bk}"] for n in names],
                          conv_geometry(ob_shape, convs, same), lambda i, pre: net.act(names[i], pre, "relu"))
        flat = a.reshape(B, -1)
        if kind == "conv_only":
            return flat
        return net.act(f"{prefix}/fc1", flat @ P[f"{prefix}/fc1/w:0"] + P[f"{prefix}/fc1/b:0"], "relu")
    h = x
    for i in range(num_layers):
        z = h @ P[f"{prefix}/mlp_fc{i}/w:0"] + P[f"{prefix}/mlp_fc{i}/b:0"]
        ln = f"{prefix}/{LN.ln_scope(i)}"
        if f"{ln}/gamma:0" in P:                                        # mlp(layer_norm=True), models.py:97-98
            z = net.ln(ln, z, P[f"{ln}/gamma:0"], P[f"{ln}/beta:0"])
        h = net.act(f"{prefix}/mlp_fc{i}", z, "tanh")
    return h


def _first_convs(kind, prefixes, contrib=False):
    """TF names of the first conv weights (the ones that carry models.py:19's 1/255)."""
    if kind not in ("cnn", "conv_only", "cnn_lstm"):
        return set()
    return {f"{p}/convnet/Conv/weights:0" if contrib else f"{p}/c1/w:0" for p in prefixes}


def _grads(loss, P, first_convs):
    gs = torch.autograd.grad(loss, list(P.values()), allow_unused=True)
    out = collections.OrderedDict()
    for (k, p), g in zip(P.items(), gs):
        g = torch.zeros_like(p) if g is None else g
        out[k] = g / 255.0 if k in first_convs else g         # d/d(w) of the unscaled master weight
    return out


def _t(a, dev):
    return torch.as_tensor(np.asarray(a) if not torch.is_tensor(a) else a).to(dev).double()


# ------------------------------------------------------------------------------------------------ PPO2 policy
def policy_ref(params, cfg, obs, seed_pi, seed_v, rnd=False, masks=None, absolute=False, ref_acts=None, no_dact=(),
               identity=False, seq=None, unmasked_dwh=False, stored=None, dev="cpu"):
    """PolicyNet's forward (towers, [pi | vf] heads) and d(sum(pi * seed_pi) + sum(v * seed_v)) / d(param).

    cfg: dict(kind='mlp' | 'cnn' | 'lstm' | 'cnn_lstm', copy=value_network == 'copy', num_layers, ob_shape, scope).
    obs: uint8 images (cnn, cnn_lstm) or encoded observation rows (mlp, lstm, see `encode_obs`); the recurrent networks
    take T*E time-major rows (row t*E + e) with seq = (masks [T, E] "done before step t", start states [E, 2H]), numpy
    float64.  identity: the frozen identity head (no 'pi/w', 'pi/b').  The norms of mlp(layer_norm=True) are used
    wherever params holds them.  unmasked_dwh (mutant): the LSTM's dWh from h_{t-1} before the mask.  stored: ReLU
    layers' stored activations to use as forward values (module docstring).
    Returns a namespace: pi [B, nout], v [B], pres (name -> pre-activation), acts (ReLU masks / stored tanh
    activations, for an absolute run), grads (TF name -> gradient; 'head_pi/w', 'head_pi/b' for the identity head)."""
    scope = cfg.get("scope", "ppo2_model")
    kind, copy = cfg["kind"], cfg.get("copy", False)
    P = dict(params)
    P.pop(f"{scope}/pi/logstd:0", None)                          # the loss kernel's own gradient (not the network's)
    first = _first_convs(kind, [f"{scope}/pi"] + ([f"{scope}/vf"] if copy else []))
    net = _Net(rnd, masks, absolute, ref_acts, no_dact, stored)
    leaves = _leaves(P, first, rnd, absolute, dev)
    x = _t(obs, dev)
    if absolute:
        x = x.abs()
    tw = dict(num_layers=cfg.get("num_layers", 2), ob_shape=cfg.get("ob_shape"), seq=seq, unmasked_dwh=unmasked_dwh)
    lat = _tower(leaves, net, f"{scope}/pi", kind, x, **tw)
    vlat = _tower(leaves, net, f"{scope}/vf", kind, x, **tw) if copy else lat
    if identity:
        L = lat.shape[1]
        leaves["head_pi/w"] = torch.eye(L, dtype=torch.float64, device=dev).requires_grad_(True)
        leaves["head_pi/b"] = torch.zeros(L, dtype=torch.float64, device=dev).requires_grad_(True)
        wk, bk = "head_pi/w", "head_pi/b"
    else:
        wk, bk = f"{scope}/pi/w:0", f"{scope}/pi/b:0"
    pi = net.act("pi", lat @ leaves[wk] + leaves[bk], None)
    v = net.act("vf", vlat @ leaves[f"{scope}/vf/w:0"] + leaves[f"{scope}/vf/b:0"], None)[:, 0]
    sp, sv = _t(seed_pi, dev), _t(seed_v, dev)
    if absolute:
        sp, sv = sp.abs(), sv.abs()
    g = _grads((pi * sp).sum() + (v * sv).sum(), leaves, first)
    return types.SimpleNamespace(pi=pi.detach(), v=v.detach(), pres=net.pres, acts=net.acts, grads=g)


def policy_ref_sliced(params, cfg, obs, seed_pi, seed_v, rows, masks=None, each=None, identity=False, dev="cpu"):
    """policy_ref (rnd=True) and its absolute network, the error scale S, over consecutive slices of `rows` samples:
    the float64 activations of a whole benchmark minibatch do not fit in memory at once.  Every term of a gradient
    belongs to one row (fixed ReLU decisions, per-element roundings), so the slices' gradients add up to the unsliced
    ones to float64 rounding.
    obs, seed_pi, seed_v: as policy_ref, sliced here (obs may stay uint8: each slice is widened on its own).  masks:
    None (the mirror's own ReLU decisions) or masks(s, e) -> the decisions of rows s .. e-1, built per slice.  each:
    each(s, e, ref, S) with both runs of every slice, for per-row checks.
    Returns a namespace: pi, v (every row), grads and S (TF name -> float64 sums over the slices)."""
    n = obs.shape[0]
    pis, vs, grads, S = [], [], None, None
    for s in range(0, n, rows):
        e = min(s + rows, n)
        m = None if masks is None else masks(s, e)
        ref = policy_ref(params, cfg, obs[s:e], seed_pi[s:e], seed_v[s:e], rnd=True, masks=m, identity=identity,
                         dev=dev)
        ab = policy_ref(params, cfg, obs[s:e], seed_pi[s:e], seed_v[s:e], absolute=True, ref_acts=ref.acts,
                        identity=identity, dev=dev)
        if each is not None:
            each(s, e, ref, ab)
        pis.append(ref.pi)
        vs.append(ref.v)
        if grads is None:
            grads, S = ref.grads, ab.grads
        else:
            for k in grads:
                grads[k] += ref.grads[k]
                S[k] += ab.grads[k]
    return types.SimpleNamespace(pi=torch.cat(pis), v=torch.cat(vs), grads=grads, S=S)


def encode_obs(obs, onehot_n=0, nvec=None, mean=None, inv_std=None, clip=(-5.0, 5.0)):
    """The observation encoder (csrc/obs_encode.cu) in float32: Discrete -> one-hot, MultiDiscrete -> concatenated
    one-hots, Box -> the float32 rows, normalised as clip((x - mean) * inv_std, lo, hi) with float32 operations when
    mean / inv_std (float32 arrays) are given.  Returns float64 [B, in_dim]."""
    obs = np.asarray(obs)
    B = obs.shape[0]
    if nvec:
        cols = [np.eye(n)[obs.reshape(B, -1)[:, i].astype(np.int64)] for i, n in enumerate(nvec)]
        return np.concatenate(cols, 1)
    if onehot_n:
        return np.eye(onehot_n)[obs.reshape(-1).astype(np.int64)]
    x = obs.reshape(B, -1).astype(np.float32)
    if mean is not None:
        x = np.minimum(np.maximum((x - mean.astype(np.float32)) * inv_std.astype(np.float32),
                                  np.float32(clip[0])), np.float32(clip[1]))
    return x.astype(np.float64)


# ------------------------------------------------------------------------------------------------ DQN Q network
def _fc_name(j):
    return "fully_connected" if j == 0 else f"fully_connected_{j}"


def q_ref(params, cfg, obs, seed_a, seed_s=None, rnd=False, masks=None, absolute=False, ref_acts=None, no_dact=(),
          detach_state_stream=False, dev="cpu"):
    """QNet's forward (trunk, action_value / state_value streams) and d(sum(A * seed_a) + sum(S * seed_s)) / d(param).

    cfg: dict(kind='mlp' | 'cnn' | 'conv_only', hiddens, dueling, num_layers, ob_shape, scope).  A [B, nA] are the raw
    action scores, S [B] the state score (dueling); q = S + A - mean(A) is formed by the TD step, not here.
    detach_state_stream (mutant): the state stream's gradient does not reach the trunk."""
    scope = cfg.get("scope", "deepq/q_func")
    kind, hiddens, dueling = cfg["kind"], tuple(cfg["hiddens"]), cfg.get("dueling", True)
    contrib = kind == "conv_only"
    first = _first_convs(kind, [scope], contrib)
    net = _Net(rnd, masks, absolute, ref_acts, no_dact)
    leaves = _leaves(params, first, rnd, absolute, dev)
    x = _t(obs, dev)
    if absolute:
        x = x.abs()
    lat = _tower(leaves, net, scope, kind, x, same=contrib, contrib=contrib, num_layers=cfg.get("num_layers", 2),
                 ob_shape=cfg.get("ob_shape"))
    outs = []
    for sname in ["action_value"] + (["state_value"] if dueling else []):
        h = lat.detach() if (detach_state_stream and sname == "state_value") else lat
        for j in range(len(hiddens) + 1):
            pfx = f"{scope}/{sname}/{_fc_name(j)}"
            z = h @ leaves[pfx + "/weights:0"] + leaves[pfx + "/biases:0"]
            ln = f"{scope}/{sname}/{LN.ln_scope(j)}"
            if j < len(hiddens) and f"{ln}/gamma:0" in leaves:        # layer_norm=True, deepq/models.py:24-25,34-35
                z = net.ln(ln, z, leaves[f"{ln}/gamma:0"], leaves[f"{ln}/beta:0"])
            h = net.act(pfx, z, "relu" if j < len(hiddens) else None)
        outs.append(h)
    A = outs[0]
    S = outs[1][:, 0] if dueling else None
    sa = _t(seed_a, dev)
    loss = (A * (sa.abs() if absolute else sa)).sum()
    if dueling:
        ss = _t(seed_s, dev)
        loss = loss + (S * (ss.abs() if absolute else ss)).sum()
    g = _grads(loss, leaves, first)
    return types.SimpleNamespace(A=A.detach(), S=None if S is None else S.detach(), pres=net.pres, acts=net.acts,
                                 grads=g)


# ------------------------------------------------------------------------------------------------ configurations
# PPO2 networks of tests/test_update_composition_gpu.py: observation space ('box', shape) uint8 for cnn / float32 for
# mlp, ('discrete', n) or ('mdisc', nvec); action space ('cat', n), ('gauss', d), ('mcat', nvec) or ('bern', n).
PPO_CONFIGS = {
    "cnn84_cat6_shared": dict(kind="cnn", ob=("box", (84, 84, 4)), ac=("cat", 6)),
    "cnn84_cat6_copy": dict(kind="cnn", ob=("box", (84, 84, 4)), ac=("cat", 6), copy=True),
    "cnn64_cat6_shared": dict(kind="cnn", ob=("box", (64, 64, 4)), ac=("cat", 6)),
    "mlp376_gauss17_copy_h64": dict(kind="mlp", ob=("box", (376,)), ac=("gauss", 17), copy=True),
    "mlp11_gauss3_copy_h256": dict(kind="mlp", ob=("box", (11,)), ac=("gauss", 3), copy=True, num_hidden=256),
    "mlp11_gauss3_copy_l1_h32": dict(kind="mlp", ob=("box", (11,)), ac=("gauss", 3), copy=True, num_layers=1,
                                     num_hidden=32),
    "mlp13_cat15_l3_h20": dict(kind="mlp", ob=("box", (13,)), ac=("cat", 15), num_layers=3, num_hidden=20),
    "mlp_disc10_cat4": dict(kind="mlp", ob=("discrete", 10), ac=("cat", 4)),
    "mlp_mdisc33_mcat33": dict(kind="mlp", ob=("mdisc", (3, 3)), ac=("mcat", (3, 3))),
    "mlp5_gauss32_copy_identity": dict(kind="mlp", ob=("box", (5,)), ac=("gauss", 32), copy=True, num_hidden=32),
    "mlp11_bern5_normalized": dict(kind="mlp", ob=("box", (11,)), ac=("bern", 5), normalize=True),
}

# DQN networks: trunk, stream hidden widths, dueling, double-Q, observation space
DQN_CONFIGS = {
    "mlp_dueling_h64_32_double": dict(kind="mlp", ob=("box", (8,)), hiddens=(64, 32), dueling=True, double_q=True),
    "mlp_plain_h20_max": dict(kind="mlp", ob=("box", (8,)), hiddens=(20,), dueling=False, double_q=False),
    "mlp_dueling_h20_double": dict(kind="mlp", ob=("box", (8,)), hiddens=(20,), dueling=True, double_q=True),
    "cnn_dueling_h256": dict(kind="cnn", ob=("box", (84, 84, 4)), hiddens=(256,), dueling=True, double_q=True),
    "conv_only_dueling_h256": dict(kind="conv_only", ob=("box", (84, 84, 4)), hiddens=(256,), dueling=True,
                                   double_q=True),
    "mlp_disc7_dueling_h64": dict(kind="mlp", ob=("discrete", 7), hiddens=(64,), dueling=True, double_q=True),
}

# The layer-normalised and recurrent networks of tests/test_update_composition_rnn_ln_gpu.py.  Recurrent minibatches
# are E whole environments of T steps (nlstm: the cell width).
PPO_RNN_LN_CONFIGS = {
    "mlp376_gauss17_copy_ln": dict(kind="mlp", ob=("box", (376,)), ac=("gauss", 17), copy=True, layer_norm=True),
    "mlp11_cat4_shared_ln": dict(kind="mlp", ob=("box", (11,)), ac=("cat", 4), layer_norm=True),
    "lstm_box7_gauss3_h128": dict(kind="lstm", ob=("box", (7,)), ac=("gauss", 3), nlstm=128),
    "lstm_disc5_cat3_h64": dict(kind="lstm", ob=("discrete", 5), ac=("cat", 3), nlstm=64),
    "cnn_lstm_cat6_h64": dict(kind="cnn_lstm", ob=("box", (84, 84, 4)), ac=("cat", 6), nlstm=64),
    "cnn_lstm_cat6_h128": dict(kind="cnn_lstm", ob=("box", (84, 84, 4)), ac=("cat", 6), nlstm=128),
}

DQN_LN_CONFIGS = {
    "mlp_dueling_h64_32_double_ln": dict(kind="mlp", ob=("box", (8,)), hiddens=(64, 32), dueling=True, double_q=True,
                                         layer_norm=True),
    "mlp_plain_h32_32_ln": dict(kind="mlp", ob=("box", (8,)), hiddens=(32, 32), dueling=False, double_q=False,
                                layer_norm=True),
    "conv_only_dueling_h256_ln": dict(kind="conv_only", ob=("box", (84, 84, 4)), hiddens=(256,), dueling=True,
                                      double_q=True, layer_norm=True),
}


def in_dim(ob):
    """Width of the encoded observation rows (mlp) or the image shape (cnn)."""
    kind, arg = ob
    return arg if kind == "box" else ((arg,) if kind == "discrete" else (sum(arg),))


def ppo_nout(ac):
    kind, arg = ac
    return sum(arg) if kind == "mcat" else arg


def ppo_mirror_cfg(cfg):
    return dict(kind=cfg["kind"], copy=cfg.get("copy", False), num_layers=cfg.get("num_layers", 2),
                ob_shape=in_dim(cfg["ob"]) if cfg["kind"] != "mlp" else None)


def ppo_identity(cfg):
    if cfg["kind"] in ("lstm", "cnn_lstm"):
        return cfg["nlstm"] == ppo_nout(cfg["ac"])
    return cfg["kind"] == "mlp" and cfg.get("num_hidden", 64) == ppo_nout(cfg["ac"])


def dqn_mirror_cfg(cfg):
    return dict(kind=cfg["kind"], hiddens=cfg["hiddens"], dueling=cfg["dueling"],
                ob_shape=in_dim(cfg["ob"]) if cfg["kind"] != "mlp" else None)
