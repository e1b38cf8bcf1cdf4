"""actor_critic.py: the HER actor and critic on the device.

pi = max_u * tanh(nn([o | g], [hidden] * layers + [dimu])) and Q = nn([o | g | u / max_u], [hidden] * layers + [1]),
with o and g normalised (normalizer.py:72-77).  nn (util.py:49-62) is a stack of dense layers `_0` .. `_layers`, ReLU
between them and none after the last, Glorot-uniform kernels and zero biases.  Q is evaluated twice on one set of
weights: on pi / max_u (Q_pi) and on the stored u / max_u (Q); the train step runs both as one pass over 2B rows.

Each network is a float32 parameter store (nn.ParamStore) with fp16 operand copies; its first layer reads the fp16
[hi | lo] rows csrc/her.cu writes, so inputs reach it at float32 precision.
"""
import numpy as np
import torch

from .. import nn, ops


class ActorCritic:
    """The network spec (actor_critic.py:5-46): what create_actor_critic builds, per scope."""

    def __init__(self, dimo, dimg, dimu, hidden, layers, **kwargs):
        if int(layers) < 1:
            raise NotImplementedError("her networks need layers >= 1")
        self.dimo, self.dimg, self.dimu = int(dimo), int(dimg), int(dimu)
        self.hidden, self.layers = int(hidden), int(layers)

    def build(self, scope, cap, device, rng):
        """-> (pi, Q) networks named {scope}/pi/_k and {scope}/Q/_k, pi's variables drawn first."""
        sizes = [self.hidden] * self.layers
        pi = MLP(f'{scope}/pi', self.dimo + self.dimg, sizes + [self.dimu], cap, device, rng)
        q = MLP(f'{scope}/Q', self.dimo + self.dimg + self.dimu, sizes + [1], 2 * cap, device, rng,
                act_cols=(self.dimo + self.dimg, self.dimu))
        return pi, q


class MLP:
    """nn() over `cap` rows of encoded input.  act_cols (critic): (first column, count) of the action inputs whose
    data gradient the backward carries out of the second half of the rows."""

    def __init__(self, scope, nin, sizes, cap, device, rng, act_cols=None):
        self.scope, self.nin, self.cap, self.device = scope, int(nin), int(cap), device
        store = self.store = nn.ParamStore(device)
        self.layers = []
        K = self.nin
        for i, n in enumerate(sizes):
            last = i == len(sizes) - 1
            self.layers.append(nn.Linear(store, f'{scope}/_{i}', K, n, None if last else 'relu',
                                         nn.xavier_uniform((K, n), rng), tf_w=f'{scope}/_{i}/kernel:0',
                                         tf_b=f'{scope}/_{i}/bias:0', split_in=(i == 0)))
            K = n
        store.finalize()
        for l in self.layers:
            l.materialize()
        self.hidden, self.head = self.layers[:-1], self.layers[-1]
        f16, f32 = dict(dtype=torch.float16, device=device), dict(dtype=torch.float32, device=device)
        self.in_pad = nn._pad8(self.nin)
        self.x0 = torch.zeros(cap, 2 * self.in_pad, **f16)
        self.h = [torch.zeros(cap, l.Np, **f16) for l in self.hidden]
        self.dz = [torch.zeros(cap, l.Np, **f16) for l in self.hidden]
        self.nout = sizes[-1]
        self.ld_out = nn._pad8(self.nout)
        self.out = torch.zeros(cap, self.ld_out, **f32)     # pi: pre-tanh z; Q: the value
        self.dout = torch.zeros(cap, self.ld_out, **f16)    # head gradient (sum scaling)
        self.act_cols = act_cols
        if act_cols is not None:
            self.dact = torch.zeros(cap, nn._pad8(act_cols[1]), **f32)
        self.cast_plan = ops.CastPlan([j for l in self.layers for j in l.cast_jobs()], device)
        self.refresh()
        self.tf_names = list(store.tf_map.keys())

    def refresh(self):
        self.cast_plan.run()

    def forward(self, B):
        h, ldh = self.x0, 2 * self.in_pad
        for l, out in zip(self.hidden, self.h):
            l.forward(h, ldh, B, out, l.Np)
            h, ldh = out, l.Np
        self.head.forward(h, ldh, B, self.out, self.ld_out, mode=ops.MODE_F32_STORE, act=ops.ACT_NONE)

    def backward(self, B, alpha, M):
        """self.dout rows [0, M) (sum scaling) -> every variable's gradient (alpha times that of rows [0, B)).  With
        M = 2B (the critic) rows [B, 2B) are carried down to the action columns: self.dact[:B]."""
        lw = self.layers
        dz, lddz = self.dout, self.ld_out
        for i in reversed(range(len(lw))):
            l = lw[i]
            if i > 0:
                xin, ldx = self.h[i - 1], lw[i - 1].Np
                l.wgrad(xin, ldx, dz, lddz, B, alpha)
                l.dgrad(dz, lddz, M, self.dz[i - 1], ldx, saved=xin, ld_saved=ldx, act=lw[i - 1].act)
                dz, lddz = self.dz[i - 1], ldx
            else:
                l.wgrad(self.x0, 2 * self.in_pad, dz, lddz, B, alpha)
                if M > B:
                    c0, n = self.act_cols
                    ops.gemm(dz[B:], l.w_bwd[c0:], self.dact, M=B, N=n, K=l.N, lda=lddz, ldb=l.Np,
                             ldc=self.dact.shape[1], mode=ops.MODE_F32_STORE, act=ops.ACT_NONE, tag="dgrad.her_action")

    def tf_variables(self):
        return self.store.export_tf()

    def load_tf(self, values):
        self.store.import_tf(values)
        self.refresh()
