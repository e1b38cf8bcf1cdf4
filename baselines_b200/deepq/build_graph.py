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
    init_q_params(seed) reproduces them.  layer_norm (deepq/models.py:5,24-25,34-35): a LayerNorm between every hidden
    fully_connected of the streams and its ReLU; build_q_func consumes the argument, so the trunk never sees it."""

    def __init__(self, ob_shape, num_actions, network, cap, device, rng, scope="deepq/q_func", hiddens=(256,),
                 dueling=True, layer_norm=False, **network_kwargs):
        self.device, self.cap, self.nA, self.dueling = device, cap, int(num_actions), bool(dueling)
        self.scope = scope
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
        self.streams, self.stream_lns = [], []          # stream_lns[si][j]: the norm of hidden layer j, or None
        for sname, nout in [("action_value", self.nA)] + ([("state_value", 1)] if self.dueling else []):
            layers, lns, nin = [], [], L
            for j, h in enumerate(self.hiddens):
                layers.append(nn.Linear(store, f"{sname}/{j}", nin, h, "relu", nn.xavier_uniform((nin, h), rng),
                                        tf_w=f"{scope}/{sname}/{_fc_name(j)}/weights:0",
                                        tf_b=f"{scope}/{sname}/{_fc_name(j)}/biases:0"))
                lns.append(nn.LayerNorm(store, f"{sname}/ln{j}", h, "relu", f"{scope}/{sname}/{nn.ln_scope(j)}", cap)
                           if layer_norm else None)
                nin = h
            j = len(self.hiddens)
            layers.append(nn.Linear(store, f"{sname}/{j}", nin, nout, None, nn.xavier_uniform((nin, nout), rng),
                                    tf_w=f"{scope}/{sname}/{_fc_name(j)}/weights:0",
                                    tf_b=f"{scope}/{sname}/{_fc_name(j)}/biases:0"))
            self.streams.append(layers)
            self.stream_lns.append(lns)
        store.finalize()
        self._materialize()
        # built once: refresh() runs inside captured graphs
        self._operand_launches = self.trunk.operand_launches()
        self.cast_plan = ops.CastPlan(self.cast_jobs(), device)
        self.refresh()

    def _materialize(self):
        dev, cap = self.device, self.cap
        f16 = dict(dtype=torch.float16, device=dev)
        self.trunk.materialize()
        L = self.trunk.latent_dim
        for layers, lns in zip(self.streams, self.stream_lns):
            for l in layers + [n for n in lns if n is not None]:
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

    def cast_jobs(self):
        """The casts of every fp16 operand: the trunk's, then per stream its layers' and its block of w_cat_bwd."""
        jobs = self.trunk.cast_jobs()
        for si, layers in enumerate(self.streams):
            jobs += [j for l in layers for j in l.cast_jobs()]
            l0 = layers[0]
            jobs.append(ops.CastJob(l0.w, l0.K, l0.N, self.w_cat_bwd[:, self.cat_off[si]:], self.cat_w, None, 0, 1.0))
        return jobs

    def refresh(self):
        """fp16 operand copies of every layer: the trunk's operand kernels that are not plain casts, then one batched
        launch (ops.CastPlan) for every cast."""
        for f in self._operand_launches:
            f()
        self.cast_plan.run()

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
        self.trunk_forward(obs, B, idx)
        return self.streams_forward(B, self.out if out is None else out)

    def trunk_forward(self, obs, B, idx=None):
        x, src = self.encode(obs, idx)
        self._lat, self._ld_lat = self.trunk.forward(x, B, src)

    def streams_forward(self, B, out, streams=None):
        """The streams over the latent trunk_forward left.  streams: the layers to run (default: this network's own; a
        perturbed copy's for parameter-space noise, through the same workspaces and norms)."""
        lat, ldl = self._lat, self._ld_lat
        for si, layers in enumerate(self.streams if streams is None else streams):
            h, ldh = lat, ldl
            nl = len(layers)
            for j, l in enumerate(layers):
                if j == nl - 1:
                    col = 0 if si == 0 else self.nA
                    l.forward(h, ldh, B, out[:, col:], self.ld_out, mode=ops.MODE_F32_STORE)
                elif j == 0:
                    dst = self.h_cat[:, self.cat_off[si]:]
                    nn.linear_ln_forward(l, self.stream_lns[si][j], h, ldh, B, dst, self.cat_w)
                    h, ldh = dst, self.cat_w
                else:
                    nn.linear_ln_forward(l, self.stream_lns[si][j], h, ldh, B, self.hid[si][j - 1], l.Np)
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
                if j < nl - 1 and self.stream_lns[si][j] is not None:
                    self.stream_lns[si][j].backward(B, dz, lddz, inv_B)
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


class StreamCopy:
    """A perturbed copy of a QNet's stream `fully_connected` variables (build_graph.py:254,277 `perturbed_q_func`,
    `adaptive_q_func`): compact fp32 weights and biases, their fp16 forward operands and the head outputs.  Only these
    variables differ from q_func (default_param_noise_filter :131-143), so the trunk, the norms and the workspaces are
    q_func's."""

    def __init__(self, q, scope):
        import copy
        self.scope, dev = scope, q.device
        self.tf_names, self.jobs, off = {}, [], 0              # tf name -> (offset, shape); (src, dst, len, perturb)
        by_internal = {v[0]: k for k, v in q.store.tf_map.items()}
        for layers in q.streams:
            for l in layers:
                for part, shape in (("/w", (l.K, l.N)), ("/b", (l.N,))):
                    n = int(np.prod(shape))
                    self.jobs.append((q.store.offsets[l.name + part], off, n, 1))
                    self.tf_names[by_internal[l.name + part].replace(q.scope, scope, 1)] = (off, shape)
                    off += (n + 3) // 4 * 4
        self.numel = off
        self.params = torch.zeros(off, dtype=torch.float32, device=dev)
        self.streams, k = [], 0
        for layers in q.streams:
            mine = []
            for l in layers:
                c = copy.copy(l)
                (ow, sw), (ob, sb) = [(j[1], j[2]) for j in self.jobs[k:k + 2]]
                k += 2
                c.w, c.b = self.params[ow:ow + sw].view(l.K, l.N), self.params[ob:ob + sb]
                c.w_fwd = torch.zeros(l.N, l.Kf, dtype=torch.float16, device=dev)
                mine.append(c)
            self.streams.append(mine)
        self.out = torch.zeros_like(q.out)
        self.cast = ops.CastPlan(self.cast_jobs(), dev)

    def cast_jobs(self):
        """The casts of the copy's fp16 operands: the forward operands w_fwd (the copy has no backward)."""
        return [ops.CastJob(c.w, c.K, c.N, None, 0, c.w_fwd, c.Kf, 1.0) for layers in self.streams for c in layers]

    def export_tf(self):
        host = self.params.cpu().numpy()
        return {k: host[o:o + int(np.prod(sh))].reshape(sh).copy() for k, (o, sh) in self.tf_names.items()}

    def import_tf(self, values):
        for k, (o, sh) in self.tf_names.items():
            if k in values:
                a = np.ascontiguousarray(values[k], dtype=np.float32).reshape(-1)
                self.params[o:o + a.size].copy_(torch.from_numpy(a).to(self.params.device))
        self.cast.run()


class ParamNoise:
    """State of parameter-space noise (build_graph.py:246-287): the perturbed and the adaptive stream copies, the noise
    scale (0.01), the KL threshold (0.05) and the last mean_kl as float32 device scalars, and the Philox position."""

    def __init__(self, q, seed):
        dev = q.device
        self.q, self.seed = q, int(seed)
        self.perturbed = StreamCopy(q, "deepq/perturbed_q_func")
        self.adaptive = StreamCopy(q, "deepq/adaptive_q_func")
        jobs = self.perturbed.jobs
        self.jobs = torch.tensor(jobs, dtype=torch.int64, device=dev)
        self.njobs, self.max_len = len(jobs), max(j[2] for j in jobs)
        self.scale = torch.full((1,), 0.01, dtype=torch.float32, device=dev)
        self.threshold = torch.full((1,), 0.05, dtype=torch.float32, device=dev)
        self.mean_kl = torch.zeros(1, dtype=torch.float32, device=dev)
        self.ctr = torch.zeros(1, dtype=torch.int64, device=dev)
        self.normals = None                      # tests: float32 [numel] noise used instead of the Philox stream
        for c in (self.perturbed, self.adaptive):           # until the first reset a copy is q_func
            for s, d, n, _ in jobs:
                c.params[d:d + n].copy_(q.store.params[s:s + n])
            c.cast.run()

    def perturb(self, copy_):
        """perturb_vars (:258-272): copy_ <- q_func + N(0, scale^2), then its fp16 operands (one launch each)."""
        ops.param_perturb(self.q.store.params, copy_.params, self.jobs, self.njobs, self.max_len, self.scale, self.seed,
                          self.ctr, normals=self.normals)
        ops.counter_add(self.ctr, 1)
        copy_.cast.run()

    def export_tf(self):
        d = {"deepq/param_noise_scale:0": np.float32(self.scale.item()),
             "deepq/param_noise_threshold:0": np.float32(self.threshold.item())}
        d.update(self.perturbed.export_tf())
        d.update(self.adaptive.export_tf())
        return d

    def import_tf(self, d):
        """Files written without these keys leave the state as it is."""
        if "deepq/param_noise_scale:0" in d:
            self.scale.fill_(float(d["deepq/param_noise_scale:0"]))
        if "deepq/param_noise_threshold:0" in d:
            self.threshold.fill_(float(d["deepq/param_noise_threshold:0"]))
        self.perturbed.import_tf(d)
        self.adaptive.import_tf(d)


class DQNModel:
    """Online + target QNet, optimiser and the train step."""

    def __init__(self, ob_space, num_actions, network, lr, gamma=1.0, grad_norm_clipping=None, double_q=True,
                 batch_cap=512, device=None, seed=None, adam_eps=1e-8, param_noise=False, **network_kwargs):
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
        self.graphs = graphs.GraphCache()
        self.batch_cap = batch_cap
        self.eps = 0.0
        self._seed = int(np.random.randint(0, 2 ** 31 - 1))
        with torch.cuda.device(self.device):
            self.pn = ParamNoise(self.q, self._seed) if param_noise else None
        self.update_target()

    def update_target(self):
        """build_graph.py:426-430: assign every q_func variable to target_q_func."""
        self.qt.store.params.copy_(self.q.store.params)
        self.qt.refresh()

    def _stage_act(self, obs_dev, B, eps):
        """The inputs of an acting pass over B observations: the observations go to a fixed buffer (graphs.home) and
        eps to the device, so the pass is a replayable launch sequence.  Returns the staged observations."""
        if B > self.batch_cap:
            raise ValueError(f"act batch {B} exceeds batch_cap {self.batch_cap}")
        x = self.graphs.home("act_obs", self.batch_cap, obs_dev.shape[1:], obs_dev.dtype, self.device)[:B]
        x.copy_(obs_dev)
        ops.set_scalars(self._eps_dev, eps)
        return x

    def act_device(self, obs_dev, B, eps):
        """build_graph.py:184-192 on B observations.  The observations are staged in a fixed buffer, eps and the
        random-stream position live on the device, so the pass is captured once per B and replayed."""
        x = self._stage_act(obs_dev, B, eps)

        def body():
            out = self.q.forward(x, B)
            S = out[:, self.nA:] if self.q.dueling else None
            ops.dqn_act(out, self.q.ld_out, S, self.q.ld_out, self.nA, 0.0, self._seed, 0, self._act, B,
                        eps_dev=self._eps_dev, step_dev=self._step_dev)
            ops.counter_add(self._step_dev, 1)
        self.graphs.run(("act", B), body)
        return self._act[:B]

    def act_device_param_noise(self, obs_dev, B, eps, reset, update_scale):
        """build_graph.py:290-313 on B observations, in this order: (1) eps (and the threshold, by the caller) are set;
        (2) reset: perturbed <- q_func + N(0, scale^2) with the scale as it is before this call's update; (3)
        update_scale: adaptive <- q_func + N(0, scale^2), the streams of q_func and of the adaptive copy, mean_kl and the
        scale update; (4) epsilon-greedy over the PERTURBED scores.  (The reference's graph leaves the order of (2) and
        (3) to the TF runtime.)  One trunk forward serves all three networks; the sequence is captured per
        (B, reset, update_scale)."""
        pn, q = self.pn, self.q
        x = self._stage_act(obs_dev, B, eps)

        def body():
            q.trunk_forward(x, B)
            if reset:
                pn.perturb(pn.perturbed)
            if update_scale:
                pn.perturb(pn.adaptive)
                q.streams_forward(B, q.out)
                q.streams_forward(B, pn.adaptive.out, pn.adaptive.streams)
                ops.dqn_param_noise_adapt(q.out, pn.adaptive.out, q.ld_out, self.nA, q.dueling, B, pn.scale,
                                          pn.threshold, pn.mean_kl)
            out = q.streams_forward(B, pn.perturbed.out, pn.perturbed.streams)
            S = out[:, self.nA:] if q.dueling else None
            ops.dqn_act(out, q.ld_out, S, q.ld_out, self.nA, 0.0, self._seed, 0, self._act, B,
                        eps_dev=self._eps_dev, step_dev=self._step_dev)
            ops.counter_add(self._step_dev, 1)
        # injected noise (tests) is a different pointer set: keep it out of the captured sequences
        if pn.normals is None:
            self.graphs.run(("act_pn", B, bool(reset), bool(update_scale)), body)
        else:
            body()
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
    updated when update_eps >= 0; stochastic=False gives the greedy action).  A model built with param_noise=True gets
    build_act_with_param_noise's act (:290-313) instead."""
    if model.pn is not None:
        return build_act_with_param_noise(model)

    def act(ob, stochastic=True, update_eps=-1):
        if update_eps >= 0:
            model.eps = float(update_eps)
        with torch.cuda.device(model.device):
            x = torch.as_tensor(np.ascontiguousarray(ob)).to(model.device)
            a = model.act_device(x, x.shape[0], model.eps if stochastic else 0.0).cpu().numpy()
            model.q.trunk.check_obs_range()
            return a
    return act


def build_act_with_param_noise(model):
    """act(ob, reset=False, update_param_noise_threshold=False, update_param_noise_scale=False, stochastic=True,
    update_eps=-1) with the reference's sticky values (build_graph.py:290-313): eps is replaced when update_eps >= 0,
    the threshold when update_param_noise_threshold >= 0 -- so the default False (== 0.0) sets it to 0, as the
    reference's givens do.  Actions are epsilon-greedy over the perturbed network (DQNModel.act_device_param_noise)."""
    def act(ob, reset=False, update_param_noise_threshold=False, update_param_noise_scale=False, stochastic=True,
            update_eps=-1):
        if update_eps >= 0:
            model.eps = float(update_eps)
        with torch.cuda.device(model.device):
            if update_param_noise_threshold >= 0:
                ops.set_scalars(model.pn.threshold, float(update_param_noise_threshold))
            x = torch.as_tensor(np.ascontiguousarray(ob)).to(model.device)
            a = model.act_device_param_noise(x, x.shape[0], model.eps if stochastic else 0.0, bool(reset),
                                             bool(update_param_noise_scale)).cpu().numpy()
            model.q.trunk.check_obs_range()
            return a
    return act


def build_train(make_obs_ph=None, q_func=None, num_actions=None, optimizer=None, grad_norm_clipping=None, gamma=1.0,
                double_q=True, scope="deepq", reuse=None, param_noise=False, param_noise_filter_func=None, *,
                ob_space=None, network="mlp", lr=5e-4, batch_cap=512, seed=None, **network_kwargs):
    """Same return value as the reference's build_train (build_graph.py:317-449):
    (act, train, update_target, debug).  `make_obs_ph` / `q_func` / `optimizer` are TF objects in the reference and
    are ignored here; the architecture comes from (ob_space, network, **network_kwargs)."""
    if param_noise_filter_func is not None:
        raise NotImplementedError("param_noise_filter_func is a predicate over TF variables; the default filter "
                                  "(the fully_connected variables, build_graph.py:131-143) is the one implemented")
    model = DQNModel(ob_space, num_actions, network, lr, gamma=gamma, grad_norm_clipping=grad_norm_clipping,
                     double_q=double_q, batch_cap=batch_cap, seed=seed, param_noise=param_noise, **network_kwargs)
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
