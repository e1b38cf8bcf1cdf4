"""DDPG's actor and critic (baselines/ddpg/models.py) on the device.

Actor: mlp over the normalised observation, then `dense` (nb_actions, kernel U(-3e-3, 3e-3), zero bias), then tanh.
Critic: mlp over the concatenation [normalised observation | action] (models.py:43), then `output` (1, kernel U(-3e-3,
3e-3), zero bias).  Both are float32 parameter stores (nn.ParamStore) with fp16 operand copies; the towers' first layer
reads the fp16 [hi | lo] rows csrc/ddpg.cu's encoder writes, so an action reaches the critic at float32 precision.

Only network='mlp' applies: the critic concatenates the observation with the action, which an image tower cannot take.
"""
import numpy as np
import torch

from .. import nn, ops


class Model:
    """The (network, kwargs) of a network the agent builds (models.py:5-20)."""

    def __init__(self, name, network='mlp', num_layers=2, num_hidden=64, layer_norm=False, **network_kwargs):
        if network != 'mlp':
            raise NotImplementedError(f"ddpg network={network!r}: only 'mlp' is implemented (the critic concatenates the "
                                      "observation with the action, ddpg/models.py:43)")
        if network_kwargs:
            raise TypeError(f"unsupported mlp arguments for ddpg: {sorted(network_kwargs)}")
        if int(num_layers) < 1:
            raise NotImplementedError("ddpg mlp towers need num_layers >= 1")
        self.name, self.network = name, network
        self.num_layers, self.num_hidden, self.layer_norm = int(num_layers), int(num_hidden), bool(layer_norm)


class Actor(Model):
    def __init__(self, nb_actions, name='actor', network='mlp', **network_kwargs):
        super().__init__(name, network, **network_kwargs)
        self.nb_actions = nb_actions


class Critic(Model):
    def __init__(self, name='critic', network='mlp', **network_kwargs):
        super().__init__(name, network, **network_kwargs)


def _uniform(urng, shape):
    # tf.random_uniform_initializer(-3e-3, 3e-3); TF's own stream is not reproduced, the values come from urng
    return urng.uniform(-3e-3, 3e-3, size=shape).astype(np.float32)


class Net:
    """One network copy: tower + head, workspaces for `cap` rows.  kind 'actor': head `dense` (nA) with the float32 tanh
    output mu; kind 'critic': input [obs | action], head `output` (1)."""

    def __init__(self, spec, kind, scope, ob_dim, nA, cap, device, rng, urng):
        self.kind, self.scope, self.ob_dim, self.nA, self.cap = kind, scope, int(ob_dim), int(nA), int(cap)
        self.device = device
        store = self.store = nn.ParamStore(device)
        nin = self.ob_dim + (self.nA if kind == 'critic' else 0)
        self.tower = nn.Tower(store, 'mlp', (nin,), 'tower', scope, rng, cap, init='ortho', num_layers=spec.num_layers,
                              num_hidden=spec.num_hidden, layer_norm=spec.layer_norm)
        L, nout = self.tower.latent_dim, (self.nA if kind == 'actor' else 1)
        hname = 'dense' if kind == 'actor' else 'output'
        self.head = nn.Linear(store, hname, L, nout, None, _uniform(urng, (L, nout)), tf_w=f'{scope}/{hname}/kernel:0',
                              tf_b=f'{scope}/{hname}/bias:0')
        store.finalize()
        self.tower.materialize()
        self.head.materialize()
        f32, f16 = dict(dtype=torch.float32, device=device), dict(dtype=torch.float16, device=device)
        self.in_pad = self.tower.in_pad
        self.x0 = self.tower.x0                           # [cap, 2 * in_pad] encoded input rows
        self.ld_out = nn._pad8(nout)
        self.out = torch.zeros(cap, self.ld_out, **f32)   # head output (actor: pre-tanh z; critic: Q)
        self.dout = torch.zeros(cap, self.ld_out, **f16)  # head gradient (sum scaling)
        if kind == 'actor':
            self.mu = torch.zeros(cap, self.nA, **f32)
        else:
            self.dact = torch.zeros(cap, nn._pad8(self.nA), **f32)       # d Q / d action columns
            N = spec.num_hidden
            self.ln_scratch = torch.zeros(2, N, **f32)                   # the actor rows' LayerNorm parameter gradients
        self.cast_plan = ops.CastPlan(self.tower.cast_jobs() + self.head.cast_jobs(), device)
        self.refresh()
        # TF name -> internal name, in creation order
        self.tf_names = list(store.tf_map.keys())

    def refresh(self):
        self.cast_plan.run()

    def forward(self, B):
        """The head over B rows of x0; the actor also writes mu = tanh(z)."""
        h, ldh = self.tower.forward(None, B, encoded=self.x0)
        self.head.forward(h, ldh, B, self.out, self.ld_out, mode=ops.MODE_F32_STORE, act=ops.ACT_NONE)
        if self.kind == 'actor':
            ops.ddpg_tanh(self.out, self.ld_out, self.mu, B, self.nA)

    def actor_backward(self, B, alpha):
        """self.dout (d loss / d z, sum scaling) -> every variable's gradient, scaled by alpha."""
        tw = self.tower
        h, ldh = tw.hfc[-1], tw.ld_hfc[-1]
        self.head.wgrad(h, ldh, self.dout, self.ld_out, B, alpha)
        self.head.dgrad(self.dout, self.ld_out, B, tw.dlatent, tw.ld_dlatent, saved=h, ld_saved=ldh, act=tw.latent_act)
        tw.backward(B, alpha)

    def critic_backward(self, B, alpha):
        """self.dout rows [0, B): d critic_loss / d Q, rows [B, 2B): d actor_loss / d Q(s, mu(s)) (sum scaling).  The
        weight gradients (scaled by alpha) come from the first B rows only; the second B rows are carried down to the
        action columns of the input: self.dact[:B] = d actor_loss / d mu (sum scaling)."""
        tw, M = self.tower, 2 * B
        fcs, lns = tw.fcs, tw.lns
        h, ldh = tw.hfc[-1], tw.ld_hfc[-1]
        self.head.wgrad(h, ldh, self.dout, self.ld_out, B, alpha)
        self.head.dgrad(self.dout, self.ld_out, M, tw.dzfc[-1], tw.ld_hfc[-1], saved=h, ld_saved=ldh, act=tw.latent_act)
        dz, lddz = tw.dzfc[-1], tw.ld_hfc[-1]
        for i in reversed(range(len(fcs))):
            l, ln = fcs[i], lns[i]
            if ln is not None:
                ops.ln_bwd(dz, lddz, ln.z, ln.ldz, ln.gamma, dz, lddz, ln.ggamma, ln.gbeta, B, ln.N, alpha, nn.LN_EPS)
                ops.ln_bwd(dz[B:], lddz, ln.z[B:], ln.ldz, ln.gamma, dz[B:], lddz, self.ln_scratch[0],
                           self.ln_scratch[1], B, ln.N, alpha, nn.LN_EPS)
            if i > 0:
                xin, ldx = tw.hfc[i - 1], tw.ld_hfc[i - 1]
                l.wgrad(xin, ldx, dz, lddz, B, alpha)
                l.dgrad(dz, lddz, M, tw.dzfc[i - 1], tw.ld_hfc[i - 1], saved=xin, ld_saved=ldx, act=fcs[i - 1].act)
                dz, lddz = tw.dzfc[i - 1], tw.ld_hfc[i - 1]
            else:
                l.wgrad(self.x0, 2 * self.in_pad, dz, lddz, B, alpha)
                # the action rows of mlp_fc0/w: d/d a = dz W[ob_dim:ob_dim + nA, :]^T, float32
                ops.gemm(dz[B:], l.w_bwd[self.ob_dim:], self.dact, M=B, N=self.nA, K=l.N, lda=lddz, ldb=l.Np,
                         ldc=self.dact.shape[1], mode=ops.MODE_F32_STORE, act=ops.ACT_NONE, tag="dgrad.ddpg_action")

    def tf_variables(self):
        return self.store.export_tf()

    def tf_internal(self, tf_name):
        return self.store.tf_map[tf_name][0]

    def segments(self, pred):
        """(offset, length) of the variables whose TF name satisfies pred, in creation order."""
        out = []
        for k in self.tf_names:
            if pred(k):
                internal = self.tf_internal(k)
                shape = self.store.tf_map[k][2]
                out.append((self.store.offsets[internal], int(np.prod(shape))))
        return out
