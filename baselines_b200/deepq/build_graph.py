"""DQN act / train / update_target on the H100 kernels.

Behavioural mirror of baselines/deepq/build_graph.py (build_act :146-199, build_train :317-449) and
baselines/deepq/models.py (build_q_func :5-45): the same (act, train, update_target, debug) callables, built on a
`QNet` (conv / mlp trunk + dueling streams) instead of a TF graph.

train(obs_t, action, reward, obs_tp1, done, weight) -> td_error, doing: q(s), double-Q target from the online
argmax and the target network (:399-408), Huber loss (tf_util.py:39-45) weighted by the importance weights
(:413), per-variable clip_by_norm(10) (:416-421), Adam (eps 1e-8, deepq.py:205).
"""

import numpy as np
import torch

from .. import graphs, nn, ops


def _fc_name(j):
    return "fully_connected" if j == 0 else f"fully_connected_{j}"


class QNet:
    """Trunk + (dueling) streams with workspaces for `cap` samples.  Variables are created in the order
    trunk, action_value stream, state_value stream with the same RandomState, so the oracle's
    init_q_params(seed) reproduces them."""

    def __init__(self, ob_shape, num_actions, network, cap, device, rng, scope="deepq/q_func", hiddens=(256,),
                 dueling=True, layer_norm=False, **network_kwargs):
        if layer_norm:
            raise NotImplementedError("layer_norm is outside the hot-path scope")
        self.device, self.cap, self.nA, self.dueling = device, cap, int(num_actions), bool(dueling)
        self.hiddens = tuple(hiddens)
        store = self.store = nn.ParamStore(device)
        kind = network
        if kind == "cnn":
            self.trunk = nn.Tower(store, "cnn", ob_shape, "trunk", scope, rng, cap, init="ortho", **network_kwargs)
        elif kind == "conv_only":
            self.trunk = nn.Tower(store, "conv_only", ob_shape, "trunk", scope, rng, cap, init="xavier", same_pad=True,
                                  tf_style="contrib", **network_kwargs)
        elif kind == "mlp":
            self.trunk = nn.Tower(store, "mlp", ob_shape, "trunk", scope, rng, cap, init="ortho", **network_kwargs)
        elif kind in ("lstm", "cnn_lstm", "lnlstm", "cnn_lnlstm"):
            raise NotImplementedError(f"network={kind!r}: recurrent Q networks are not implemented (deepq acts on "
                                      "single observations)")
        else:
            raise ValueError(f"unknown network {kind!r}")
        L = self.trunk.latent_dim
        self.streams = []
        for sname, nout in [("action_value", self.nA)] + ([("state_value", 1)] if self.dueling else []):
            layers, nin = [], L
            for j, h in enumerate(self.hiddens):
                layers.append(nn.Linear(store, f"{sname}/{j}", nin, h, "relu", nn.xavier_uniform((nin, h), rng),
                                        tf_w=f"{scope}/{sname}/{_fc_name(j)}/weights:0",
                                        tf_b=f"{scope}/{sname}/{_fc_name(j)}/biases:0"))
                nin = h
            j = len(self.hiddens)
            layers.append(nn.Linear(store, f"{sname}/{j}", nin, nout, None, nn.xavier_uniform((nin, nout), rng),
                                    tf_w=f"{scope}/{sname}/{_fc_name(j)}/weights:0",
                                    tf_b=f"{scope}/{sname}/{_fc_name(j)}/biases:0"))
            self.streams.append(layers)
        store.finalize()
        self._materialize()
        self.refresh()

    def _materialize(self):
        dev, cap = self.device, self.cap
        f16 = dict(dtype=torch.float16, device=dev)
        self.trunk.materialize()
        L = self.trunk.latent_dim
        for layers in self.streams:
            for l in layers:
                l.materialize()
        ns = len(self.streams)
        self.first_widths = [layers[0].N for layers in self.streams]
        self.cat_w = sum(nn._pad8(w) for w in self.first_widths)
        self.cat_off = np.cumsum([0] + [nn._pad8(w) for w in self.first_widths])[:-1].tolist()
        # activations / gradients of the first stream layers live side by side (K-concatenated dgrad into the trunk)
        self.h_cat = torch.zeros(cap, self.cat_w, **f16)
        self.dz_cat = torch.zeros(cap, self.cat_w, **f16)
        self.w_cat_bwd = torch.zeros(L, self.cat_w, **f16)
        self.hid = [[torch.zeros(cap, l.Np, **f16) for l in layers[1:-1]] for layers in self.streams]
        self.dhid = [[torch.zeros(cap, l.Np, **f16) for l in layers[1:-1]] for layers in self.streams]
        self.ld_out = 16 * ((self.nA + 1 + 15) // 16)
        self.out = torch.zeros(cap, self.ld_out, dtype=torch.float32, device=dev)    # [A scores | S] per row
        self.s_col = nn._pad8(self.nA)               # dS lives at a 16-byte aligned column of dout
        self.ld_dout = 64 * ((self.s_col + 1 + 63) // 64)
        self.dout = torch.zeros(cap, self.ld_dout, **f16)

    def refresh(self):
        """fp16 operand copies of every layer in one batched launch (ops.CastPlan)."""
        if getattr(self, "_cast_plan", None) is None:
            self._cast_plan = ops.CastPlan(self._refresh_layers, self.device)
        else:
            for c in self.trunk.convs:
                if c.wdg is not None:
                    ops.dgrad_weights(c.w, c.wdg, c.rf, c.rf, c.C, c.nf, c.stride, c.ld_wdg)
        self._cast_plan.run()

    def _refresh_layers(self):
        self.trunk.refresh()
        for si, layers in enumerate(self.streams):
            for l in layers:
                l.refresh()
            l0 = layers[0]
            ops.cast_transpose(l0.w, l0.K, l0.N, self.w_cat_bwd[:, self.cat_off[si]:], self.cat_w, None, 0)

    def encode(self, obs, idx=None):
        """-> (x, src_idx) in the trunk's input format."""
        if self.trunk.in_u8:
            return obs, idx
        # vector observations stay float32 rows; the trunk's encode kernel gathers them through idx and splits
        # them into fp16 [hi | lo] operand rows (no narrowing of the stored observation, common/input.py:56-57)
        x = obs.reshape(obs.shape[0], -1)
        if x.dtype != torch.float32:
            x = x.to(torch.float32)
        return x.contiguous(), idx

    def forward(self, obs, B, idx=None, out=None):
        """q head outputs for B samples: out[:, :nA] action scores, out[:, nA] state score (dueling)."""
        x, src = self.encode(obs, idx)
        lat, ldl = self.trunk.forward(x, B, src)
        self._lat, self._ld_lat = lat, ldl
        out = self.out if out is None else out
        for si, layers in enumerate(self.streams):
            h, ldh = lat, ldl
            nl = len(layers)
            for j, l in enumerate(layers):
                if j == nl - 1:
                    col = 0 if si == 0 else self.nA
                    l.forward(h, ldh, B, out[:, col:], self.ld_out, mode=ops.MODE_F32_STORE)
                elif j == 0:
                    dst = self.h_cat[:, self.cat_off[si]:]
                    l.forward(h, ldh, B, dst, self.cat_w)
                    h, ldh = dst, self.cat_w
                else:
                    l.forward(h, ldh, B, self.hid[si][j - 1], l.Np)
                    h, ldh = self.hid[si][j - 1], l.Np
        return out

    def backward(self, B, inv_B):
        """Consumes self.dout ([dA | dS] in sum scaling); fills store.grads with the MEAN-loss gradient."""
        tr = self.trunk
        direct = len(self.streams[0]) == 1             # no hidden layers: streams read the latent directly
        for si, layers in enumerate(self.streams):
            nl = len(layers)
            col = 0 if si == 0 else self.s_col
            dz, lddz = self.dout[:, col:], self.ld_dout
            for j in reversed(range(nl)):
                l = layers[j]
                if j == 0:
                    xin, ldx = self._lat, self._ld_lat
                elif j == 1:
                    xin, ldx = self.h_cat[:, self.cat_off[si]:], self.cat_w
                else:
                    xin, ldx = self.hid[si][j - 2], layers[j - 1].Np
                l.wgrad(xin, ldx, dz, lddz, B, inv_B)
                if j == 0:
                    break
                if j == 1:
                    out, ldo = self.dz_cat[:, self.cat_off[si]:], self.cat_w
                else:
                    out, ldo = self.dhid[si][j - 2], layers[j - 1].Np
                l.dgrad(dz, lddz, B, out, ldo, saved=xin, ld_saved=ldx, act=ops.ACT_RELU)
                dz, lddz = out, ldo
        # d latent = [dz_A | dz_S] [W_A | W_S]^T  * act'(latent): ONE K-concatenated GEMM into the trunk
        if direct:
            raise NotImplementedError("hiddens=[] (streams without a hidden layer)")
        ops.gemm(self.dz_cat, self.w_cat_bwd, tr.dlatent, M=B, N=tr.latent_dim, K=self.cat_w, lda=self.cat_w,
                 ldb=self.cat_w, ldc=tr.ld_dlatent, saved=self._lat, ld_saved=self._ld_lat, mode=ops.MODE_F16_DACT,
                 act=tr.latent_act, tag="dgrad.streams")
        tr.backward(B, inv_B)


class DQNModel:
    """Online + target QNet, optimiser and the train step."""

    def __init__(self, ob_space, num_actions, network, lr, gamma=1.0, grad_norm_clipping=None, double_q=True,
                 batch_cap=512, device=None, seed=None, adam_eps=1e-8, **network_kwargs):
        if not torch.cuda.is_available():
            raise RuntimeError("baselines_b200.deepq needs a CUDA device: no CPU fallback on the hot path")
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.nA, self.gamma, self.double_q, self.lr = int(num_actions), float(gamma), bool(double_q), lr
        rng = np.random.RandomState(seed) if seed is not None else np.random
        ob_shape = tuple(ob_space.shape)
        if hasattr(ob_space, "n") and not hasattr(ob_space, "nvec"):          # Discrete obs: one-hot (common/input.py:54-55)
            network_kwargs = dict(network_kwargs, onehot_n=int(ob_space.n))
        with torch.cuda.device(self.device):
            self.q = QNet(ob_shape, num_actions, network, batch_cap, self.device, rng, "deepq/q_func", **network_kwargs)
            self.qt = QNet(ob_shape, num_actions, network, batch_cap, self.device, np.random.RandomState(0),
                           "deepq/target_q_func", **network_kwargs)
            self.opt = nn.Optimizer(self.q.store, eps=adam_eps, max_grad_norm=grad_norm_clipping,
                                    per_variable=grad_norm_clipping is not None)
            dev = self.device
            self.on_out = torch.zeros_like(self.q.out)                 # online q(s') kept aside
            self.td = torch.zeros(batch_cap, dtype=torch.float32, device=dev)
            self.loss = torch.zeros(1, dtype=torch.float64, device=dev)
            self._act = torch.zeros(batch_cap, dtype=torch.int64, device=dev)
            # fixed homes for per-step inputs and scalars, so that a step is a replayable launch sequence (graphs.py)
            self._idx_buf = torch.zeros(batch_cap, dtype=torch.int64, device=dev)
            self._w_buf = torch.zeros(batch_cap, dtype=torch.float32, device=dev)
            self._eps_dev = torch.zeros(1, dtype=torch.float32, device=dev)
            self._step_dev = torch.zeros(1, dtype=torch.int64, device=dev)
            self._act_obs = None
        self.graphs = graphs.GraphCache()
        self.batch_cap = batch_cap
        self.eps = 0.0
        self._seed = int(np.random.randint(0, 2 ** 31 - 1))
        self.update_target()

    def update_target(self):
        """build_graph.py:426-430: assign every q_func variable to target_q_func."""
        self.qt.store.params.copy_(self.q.store.params)
        self.qt.refresh()

    def act_device(self, obs_dev, B, eps):
        """build_graph.py:184-192 on B observations.  The observations are staged in a fixed buffer, eps and the
        random-stream position live on the device, so the pass is captured once per B and replayed."""
        if B > self.batch_cap:
            raise ValueError(f"act batch {B} exceeds batch_cap {self.batch_cap}")
        if self._act_obs is None or self._act_obs.shape[1:] != obs_dev.shape[1:] or self._act_obs.dtype != obs_dev.dtype:
            self._act_obs = torch.zeros((self.batch_cap,) + tuple(obs_dev.shape[1:]), dtype=obs_dev.dtype,
                                        device=self.device)
            self.graphs.clear()
        self._act_obs[:B].copy_(obs_dev)
        ops.set_scalars(self._eps_dev, eps)
        x = self._act_obs[:B]

        def body():
            out = self.q.forward(x, B)
            S = out[:, self.nA:] if self.q.dueling else None
            ops.dqn_act(out, self.q.ld_out, S, self.q.ld_out, self.nA, 0.0, self._seed, 0, self._act, B,
                        eps_dev=self._eps_dev, step_dev=self._step_dev)
            ops.counter_add(self._step_dev, 1)
        self.graphs.run(("act", B), body)
        return self._act[:B]

    def q_values(self, obs):
        with torch.cuda.device(self.device):
            x = torch.as_tensor(np.ascontiguousarray(obs)).to(self.device)
            B = x.shape[0]
            out = self.q.forward(x, B)[:B].clone()
            A = out[:, :self.nA]
            if self.q.dueling:
                out = (out[:, self.nA:self.nA + 1] + (A - A.mean(dim=1, keepdim=True))).cpu().numpy()
            else:
                out = A.cpu().numpy()
            self.q.trunk.check_obs_range()
            return out

    def train_device(self, obs_t, obs_tp1, actions, rewards, dones, weights, idx, B, lr=None):
        """One step of build_graph.py:380-444 on device-resident arrays.  obs_* / actions / rewards / dones are the
        replay storage (gathered through idx) or already-gathered batches (idx None).  Returns td_error[B].
        With idx (the resident replay path) the step is a fixed launch sequence: indices and weights are copied into
        fixed buffers, Adam's step size goes to the device, and the sequence is captured once and replayed."""
        q, qt, nA = self.q, self.qt, self.nA
        with torch.cuda.device(self.device):
            self.opt.begin_step(self.lr if lr is None else lr)
            replay = idx is not None
            if replay:
                self._idx_buf[:B].copy_(idx)
                self._w_buf[:B].copy_(weights)
                idx, weights = self._idx_buf[:B], self._w_buf[:B]
            ld = q.ld_out
            sp = (lambda o: o[:, nA:]) if q.dueling else (lambda o: None)

            def body():
                if self.double_q:
                    q.forward(obs_tp1, B, idx, out=self.on_out)        # online q(s')  (first: it reuses q's workspace)
                qt.forward(obs_tp1, B, idx)                            # target q(s')
                q.forward(obs_t, B, idx)                               # online q(s)   (last: activations kept for bwd)
                q.store.grads.zero_()
                self.loss.zero_()
                ops.dqn_td(q.out, ld, sp(q.out), ld, self.on_out, ld, sp(self.on_out), ld, qt.out, ld, sp(qt.out), ld,
                           nA, idx, actions, rewards, dones, weights, self.gamma, self.double_q, self.td, q.dout,
                           q.ld_dout, q.dout[:, q.s_col:] if q.dueling else None, q.ld_dout, self.loss, B)
                q.backward(B, 1.0 / B)
                self.opt.apply()
                q.refresh()
            if replay:
                self.graphs.run(("train", B, obs_t.data_ptr(), obs_tp1.data_ptr(), actions.data_ptr(),
                                 rewards.data_ptr(), dones.data_ptr()), body)
            else:
                body()
            return self.td[:B]


def build_act(model):
    """act(ob, stochastic=True, update_eps=-1) -> actions (build_graph.py:146-199 semantics: eps is sticky and is
    updated when update_eps >= 0; stochastic=False gives the greedy action)."""
    def act(ob, stochastic=True, update_eps=-1):
        if update_eps >= 0:
            model.eps = float(update_eps)
        with torch.cuda.device(model.device):
            x = torch.as_tensor(np.ascontiguousarray(ob)).to(model.device)
            a = model.act_device(x, x.shape[0], model.eps if stochastic else 0.0).cpu().numpy()
            model.q.trunk.check_obs_range()
            return a
    return act


def build_train(make_obs_ph=None, q_func=None, num_actions=None, optimizer=None, grad_norm_clipping=None, gamma=1.0,
                double_q=True, scope="deepq", reuse=None, param_noise=False, param_noise_filter_func=None, *,
                ob_space=None, network="mlp", lr=5e-4, batch_cap=512, seed=None, **network_kwargs):
    """Same return value as the reference's build_train (build_graph.py:317-449):
    (act, train, update_target, debug).  `make_obs_ph` / `q_func` / `optimizer` are TF objects in the reference and
    are ignored here; the architecture comes from (ob_space, network, **network_kwargs)."""
    if param_noise:
        raise NotImplementedError("param_noise is outside the hot-path scope")
    model = DQNModel(ob_space, num_actions, network, lr, gamma=gamma, grad_norm_clipping=grad_norm_clipping,
                     double_q=double_q, batch_cap=batch_cap, seed=seed, **network_kwargs)
    act = build_act(model)

    def train(obs_t, action, reward, obs_tp1, done, weight):
        dev = model.device
        f = lambda z, dt: torch.as_tensor(np.ascontiguousarray(z)).to(dev, dt)
        B = len(action)
        ot, o1 = torch.as_tensor(np.ascontiguousarray(obs_t)).to(dev), torch.as_tensor(np.ascontiguousarray(obs_tp1)).to(dev)
        td = model.train_device(ot, o1, f(action, torch.int64), f(reward, torch.float32), f(done, torch.float32),
                                f(weight, torch.float32), None, B)
        return td.cpu().numpy()

    return act, train, model.update_target, {"q_values": model.q_values, "model": model}
