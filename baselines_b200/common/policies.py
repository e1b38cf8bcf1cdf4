"""Policy / value network for the PPO2 learner on the H100 kernels.

Behavioural mirror of the reference's common/policies.py (build_policy :121-179, PolicyWithValue
:13-119), common/distributions.py (CategoricalPd :153-204, MultiCategoricalPd :206-225, DiagGaussianPd :227-251,
BernoulliPd :254-276) and common/input.py:43-63.  The object protocol (step / value) is kept; the TF graph is
replaced by an explicit sequence of libb200rl kernel launches.
"""
import numpy as np
import torch

from .. import _lib, nn, ops
from . import spaces


RECURRENT_NETWORKS = ("lstm", "cnn_lstm")


class PolicyBuilder:
    """What `build_policy(env, network, **kwargs)` returns (reference: a `policy_fn` closure,
    policies.py:126).  Carries the architecture; `Model` instantiates it on a device."""

    def __init__(self, ob_space, ac_space, network, value_network=None, normalize_observations=False,
                 estimate_q=False, **network_kwargs):
        if callable(network) and not isinstance(network, str):
            raise NotImplementedError("custom network callables build TF graphs in the reference; this learner "
                                      "supports the registry names 'cnn', 'mlp', 'conv_only', 'lstm', 'cnn_lstm'")
        if network in ("lnlstm", "cnn_lnlstm") or (network in RECURRENT_NETWORKS and network_kwargs.get("layer_norm")):
            raise NotImplementedError(f"network={network!r}: layer-normalised LSTMs are not implemented "
                                      "(supported recurrent networks: 'lstm', 'cnn_lstm' without layer_norm)")
        if network in ("impala_cnn", "impala_cnn_lstm"):
            raise NotImplementedError(f"network={network!r}: the IMPALA residual tower is not implemented")
        if value_network not in (None, "shared", "copy"):
            raise NotImplementedError("value_network must be None/'shared'/'copy' (policies.py:154-166)")
        if value_network == "copy" and network in RECURRENT_NETWORKS:
            # the reference leaves this a TODO (policies.py:165): the copied value tower would need its own state
            raise NotImplementedError("value_network='copy' is not supported with recurrent networks")
        self.ob_space, self.ac_space = ob_space, ac_space
        self.network = network
        self.value_network = "copy" if value_network == "copy" else None
        self.normalize_observations = bool(normalize_observations)
        # policies.py:58-61: ACER's policy replaces the scalar value head 'vf' by a Q head 'q' of width nA
        if estimate_q and not spaces.is_discrete(ac_space):
            raise NotImplementedError("estimate_q=True needs a Discrete action space (policies.py:59)")
        self.estimate_q = bool(estimate_q)
        self.network_kwargs = network_kwargs


def build_policy(env, policy_network, value_network=None, normalize_observations=False, estimate_q=False,
                 **policy_kwargs):
    """Same call signature as the reference's build_policy (policies.py:121)."""
    return PolicyBuilder(env.observation_space, env.action_space, policy_network, value_network,
                         normalize_observations, estimate_q, **policy_kwargs)


def _pad(n, m):
    return (n + m - 1) // m * m


class PolicyNet:
    """Towers + heads + workspaces for at most `cap` samples per launch sequence."""

    def __init__(self, builder, cap, device, rng=np.random, scope="ppo2_model"):
        self.device, self.cap = device, cap
        ob_space, ac_space = builder.ob_space, builder.ac_space
        self.ob_shape = tuple(ob_space.shape)
        # common/input.py:54-61: Discrete(n) / MultiDiscrete(nvec) observations are fed one-hot (MultiBinary ones are
        # rejected there too)
        self.ob_nvec = None
        if spaces.is_multi_discrete(ob_space):
            self.ob_nvec = [int(v) for v in np.asarray(ob_space.nvec).reshape(-1)]
        if spaces.is_multi_binary(ob_space):
            raise NotImplementedError("MultiBinary observations have no encoding in common/input.py:43-63")
        self.ob_onehot = int(ob_space.n) if spaces.is_discrete(ob_space) else 0
        if (self.ob_onehot or self.ob_nvec) and builder.network not in ("mlp", "lstm"):
            raise NotImplementedError("Discrete / MultiDiscrete observations need a vector network ('mlp', 'lstm')")
        # the action distribution (distributions.py:278-290 make_pdtype): 'cat' Categorical (Discrete), 'mcat'
        # MultiCategorical (MultiDiscrete), 'bern' Bernoulli (MultiBinary), 'gauss' DiagGaussian (Box)
        self.nvec = None
        if spaces.is_multi_discrete(ac_space):
            self.pd = "mcat"
            self.nvec = [int(v) for v in np.asarray(ac_space.nvec).reshape(-1)]
            if not self.nvec or min(self.nvec) < 1:                            # distributions.py:79
                raise ValueError(f"MultiDiscrete action nvec entries must be >= 1, got {self.nvec}")
            self.nout, self.act_dim = sum(self.nvec), len(self.nvec)
        elif spaces.is_multi_binary(ac_space):
            self.pd = "bern"
            self.nout = self.act_dim = int(ac_space.n)
        elif spaces.is_discrete(ac_space):
            self.pd = "cat"
            self.nout, self.act_dim = int(ac_space.n), 0
        elif spaces.is_box(ac_space):
            self.pd = "gauss"
            assert len(ac_space.shape) == 1                                    # distributions.py:281
            self.nout = self.act_dim = int(ac_space.shape[0])
        else:
            raise NotImplementedError("action spaces: Discrete, MultiDiscrete, MultiBinary and Box "
                                      "(distributions.py:278-290)")
        kind = builder.network
        self.kind = kind
        self.copy_vf = builder.value_network == "copy"
        store = self.store = nn.ParamStore(device)
        kw = dict(builder.network_kwargs)
        if self.ob_onehot:
            kw["onehot_n"] = self.ob_onehot
        if self.ob_nvec:
            kw["onehot_nvec"] = self.ob_nvec
        # creation order == the reference's variable creation order (it fixes the ortho_init RNG stream)
        self.tower_pi = nn.Tower(store, kind, self.ob_shape, "pi", f"{scope}/pi", rng, cap, **kw)
        self.tower_vf = nn.Tower(store, kind, self.ob_shape, "vf", f"{scope}/vf", rng, cap, **kw) if self.copy_vf else None
        # recurrent networks (models.py lstm / cnn_lstm): the state is [nenv, 2 * nlstm] = [c | h] (utils.py:96)
        self.recurrent = self.tower_pi.lstm is not None
        self.nlstm = self.tower_pi.lstm.H if self.recurrent else 0
        L = self.tower_pi.latent_dim
        # distributions.py:351-355 (_matching_fc): when the latent is already nout wide the 'pi' layer is skipped and
        # the latent IS the logits / mean.  Here the head keeps a frozen identity block (its gradient is zeroed before
        # the norm / Adam, `freeze_identity`), so logits = latent exactly and d latent flows through the same kernels;
        # no 'pi/w', 'pi/b' variables exist (and no ortho_init draw is consumed), like the reference.
        self.pi_identity = (L == self.nout)
        w_pi = np.eye(L, dtype=np.float32) if self.pi_identity else nn.ortho_init((L, self.nout), 0.01, rng)  # policies.py:49
        if self.pd == "gauss":
            store.add("pi/logstd", np.zeros((1, self.nout), np.float32))         # distributions.py:104
            store.map_tf(f"{scope}/pi/logstd:0", "pi/logstd", (1, self.nout))
        Lv = self.tower_vf.latent_dim if self.copy_vf else L
        # the value head: 'vf' [Lv, 1] (policies.py:63), or with estimate_q the Q head 'q' [Lv, nA] (:60); both fc()
        # with init_scale 1, created after the 'pi' head
        self.nv = self.nout if builder.estimate_q else 1
        vname = "q" if builder.estimate_q else "vf"
        w_vf = nn.ortho_init((Lv, self.nv), 1.0, rng)
        nv = self.nv
        if self.copy_vf:
            self.head_pi = nn.Linear(store, "head_pi", L, self.nout, None, w_pi,
                                     tf_w=None if self.pi_identity else f"{scope}/pi/w:0",
                                     tf_b=None if self.pi_identity else f"{scope}/pi/b:0")
            self.head_vf = nn.Linear(store, "head_vf", Lv, nv, None, w_vf,
                                     tf_w=f"{scope}/{vname}/w:0", tf_b=f"{scope}/{vname}/b:0")
            self.head = None
        else:
            # fused [pi | vf] head: one skinny GEMM; TF variables are column slices of it
            n = self.nout
            self.head = nn.Linear(store, "head", L, n + nv, None, np.concatenate([w_pi, w_vf], axis=1))
            if not self.pi_identity:
                store.map_tf(f"{scope}/pi/w:0", "head/w", (L, n), col_slice=slice(0, n))
                store.map_tf(f"{scope}/pi/b:0", "head/b", (n,), col_slice=slice(0, n))
            store.map_tf(f"{scope}/{vname}/w:0", "head/w", (L, nv), col_slice=slice(n, n + nv))
            store.map_tf(f"{scope}/{vname}/b:0", "head/b", (nv,), col_slice=slice(n, n + nv))
        # policies.py:133-137,182-185: float observations pass through clip((x - mean) / std, -5, 5) of a
        # RunningMeanStd (mpi_running_mean_std.py:11-33: float64 sum / sumsq / count variables, epsilon 1e-2).  Nothing
        # in ppo2 ever updates those statistics, so they stay at their initial values (mean 0, std 1) unless a
        # checkpoint provides others; they are kept, saved and loaded under the reference's variable names.
        self.obs_rms = None
        if builder.normalize_observations and not self.tower_pi.in_u8 and not self.ob_onehot and not self.ob_nvec:
            d = self.tower_pi.raw_dim
            self.obs_rms = {"runningsum": np.zeros(self.ob_shape, np.float64),
                            "runningsumsq": np.full(self.ob_shape, 1e-2, np.float64),
                            "count": np.float64(1e-2)}
            self.rms_names = {k: f"{scope}/{k}:0" for k in self.obs_rms}
        store.finalize()
        self._materialize()
        # read from the final operand tensors (fuse0 re-points the first layers' w_fwd); built here, never in refresh(),
        # which runs inside captured graphs
        self._operand_launches = [f for t in (self.tower_pi, self.tower_vf) if t for f in t.operand_launches()]
        self.cast_plan = ops.CastPlan(self.cast_jobs(), device)
        self.set_obs_rms()
        self.refresh()

    # ------------------------------------------------------------------------------------------
    def _materialize(self):
        dev, cap = self.device, self.cap
        self.tower_pi.materialize()
        if self.tower_vf:
            self.tower_vf.materialize()
        f32 = dict(dtype=torch.float32, device=dev)
        f16 = dict(dtype=torch.float16, device=dev)
        # value_network='copy' with mlp towers: both first layers read the same encoded observations, by far the largest
        # operand of the network (cfg-3: 403 MB per chunk against 34 MB of hidden activations).  They run as ONE GEMM
        # with N = 2 * hidden (forward) and ONE weight-gradient GEMM: the two Linear objects keep their own fp32
        # parameters (checkpoint names / layouts unchanged); their fp16 forward operands, outputs and output gradients
        # are the two halves of shared buffers.
        tp, tv = self.tower_pi, self.tower_vf
        # With layer_norm the first layers write fp32 pre-activations into their norms' workspaces and run apart.
        self.fuse0 = bool(tv is not None and tp.kind == "mlp" and tp.lns[0] is None and tp.fcs[0].N == tv.fcs[0].N and
                          tp.fcs[0].K == tv.fcs[0].K and tp.fcs[0].act == tv.fcs[0].act and
                          2 * tp.fcs[0].N in (64, 128, 256))
        if self.fuse0:
            a, b = tp.fcs[0], tv.fcs[0]
            N = a.N
            self.w0cat = torch.zeros(2 * N, a.Kf, **f16)
            a.w_fwd, b.w_fwd = self.w0cat[:N], self.w0cat[N:]
            self.h0cat = torch.empty(cap, 2 * N, **f16)
            self.dz0cat = torch.empty(cap, 2 * N, **f16)
            for t, c0 in ((tp, 0), (tv, N)):
                t.hfc[0], t.dzfc[0], t.ld_hfc[0] = self.h0cat[:, c0:c0 + N], self.dz0cat[:, c0:c0 + N], 2 * N
                if len(t.fcs) == 1:
                    t.dlatent, t.ld_dlatent = t.dzfc[0], 2 * N
            self.b0cat = torch.zeros(2 * N, **f32)
            self.g0cat = torch.zeros(a.K, 2 * N, **f32)
        if self.head is not None:
            self.head.materialize()
            self.ld_ho = _pad(self.nout + self.nv, 16)
            self.headout = torch.zeros(cap, self.ld_ho, **f32)
            self.pi_out, self.ld_pi = self.headout, self.ld_ho
            self.v_out, self.ld_v = self.headout[:, self.nout:], self.ld_ho
            self.ld_dh = _pad(self.nout + self.nv, 64)
            self.dhead = torch.zeros(cap, self.ld_dh, **f16)                  # padding columns stay zero
            self.dpi, self.ld_dpi = self.dhead, self.ld_dh
            self.dv, self.ld_dv = self.dhead[:, self.nout:], self.ld_dh
        else:
            self.head_pi.materialize()
            self.head_vf.materialize()
            self.ld_pi = _pad(self.nout, 16)
            self.pi_out = torch.zeros(cap, self.ld_pi, **f32)
            self.ld_v = _pad(self.nv, 16)
            self.v_out = torch.zeros(cap, self.ld_v, **f32)
            self.ld_dpi = _pad(self.nout, 64)
            self.dpi = torch.zeros(cap, self.ld_dpi, **f16)
            self.ld_dv = _pad(self.nv, 64)
            self.dv = torch.zeros(cap, self.ld_dv, **f16)
        if self.pd == "gauss":
            self.logstd = self.store.views["pi/logstd"].view(-1)
            self.g_logstd = self.store.gviews["pi/logstd"].view(-1)
        # MultiDiscrete: offsets of the components' logit blocks, allocated once (captured launch sequences read it)
        self.seg_off = ops.segment_table(self.nvec, dev) if self.pd == "mcat" else None
        self.adv_st = torch.zeros(2, dtype=torch.float64, device=dev)
        self.stats = torch.zeros(5, dtype=torch.float64, device=dev)
        self.clip_dev = torch.zeros(1, dtype=torch.float32, device=dev)      # clip range of the current update
        self.rng_ctr = torch.zeros(1, dtype=torch.int64, device=dev)         # sampler stream position (Philox offset)

    def action_shape(self, *lead):
        """Device action rows: int64 [*] (Discrete), int64 [*, k] (MultiDiscrete), float32 [*, n] (MultiBinary),
        float32 [*, d] (Box)."""
        return tuple(lead) if self.pd == "cat" else tuple(lead) + (self.act_dim,)

    @property
    def action_dtype(self):
        return torch.int64 if self.pd in ("cat", "mcat") else torch.float32

    def actions_to_numpy(self, a):
        """Device actions -> what the reference's pd.sample() hands out: int32 for MultiDiscrete
        (distributions.py:222), float32 for MultiBinary (:273), int64 / float32 as before otherwise."""
        out = a.cpu().numpy()
        return out.astype(np.int32) if self.pd == "mcat" else out

    def set_obs_rms(self, values=None):
        """Install RunningMeanStd variables (mpi_running_mean_std.py:29-30: mean = sum/count,
        std = sqrt(max(sumsq/count - mean^2, 1e-2)), both float32) into the observation encoder."""
        if self.obs_rms is None:
            return
        if values:
            for k in self.obs_rms:
                if k in values:
                    self.obs_rms[k] = np.asarray(values[k], np.float64).reshape(np.shape(self.obs_rms[k]))
        r = self.obs_rms
        mean = (r["runningsum"] / r["count"]).astype(np.float32)
        std = np.sqrt(np.maximum((r["runningsumsq"] / r["count"]).astype(np.float32) - np.square(mean), np.float32(1e-2)))
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a.reshape(-1), dtype=np.float32)).to(self.device)
        norm = (t(mean), t(np.float32(1.0) / std), -5.0, 5.0)
        self.tower_pi.obs_norm = norm
        if self.tower_vf:
            self.tower_vf.obs_norm = norm

    def freeze_identity(self):
        """Zero the gradient of the frozen identity 'pi' block (see pi_identity) before the norm and Adam."""
        if not self.pi_identity:
            return
        if self.head is not None:
            self.head.gw[:, :self.nout].zero_()
            self.head.gb[:self.nout].zero_()
        else:
            self.head_pi.gw.zero_()
            self.head_pi.gb.zero_()

    def cast_jobs(self):
        """The casts of every fp16 operand: the towers', then the heads'.  With fuse0 the first layers' w_fwd are the
        halves of w0cat."""
        heads = [self.head_pi, self.head_vf] if self.tower_vf else [self.head]
        return [j for m in [self.tower_pi, self.tower_vf] + heads if m for j in m.cast_jobs()]

    def refresh(self):
        """Re-derive the fp16 operand copies from the fp32 master weights (after init / Adam / load): the few operand
        kernels that are not plain casts, then one batched launch (ops.CastPlan) for every cast / transpose."""
        for f in self._operand_launches:
            f()
        self.cast_plan.run()
        if self.fuse0:                                     # the fused first layer's bias operand [b_pi | b_vf]
            N = self.tower_pi.fcs[0].N
            self.b0cat[:N].copy_(self.tower_pi.fcs[0].b)
            self.b0cat[N:].copy_(self.tower_vf.fcs[0].b)

    # ------------------------------------------------------------------------------------------
    def encode_obs(self, obs_host_or_dev):
        """Stage observations on the device in the format the first kernel reads.  Box uint8 images stay uint8 (the
        cast of models.py:19 is fused into the first conv's load); vector observations stay float32 rows
        [B, raw_dim] -- the reference never narrows them (common/input.py:56-57 tf.to_float) -- and a Discrete
        observation is its integer stored as float32 (one-hot happens in the encode kernel, input.py:54-55)."""
        t = obs_host_or_dev if torch.is_tensor(obs_host_or_dev) else torch.from_numpy(np.ascontiguousarray(obs_host_or_dev))
        if self.tower_pi.in_u8:
            if t.dtype != torch.uint8:
                raise NotImplementedError("cnn towers take uint8 images (common/models.py:19)")
            return t.to(self.device, non_blocking=True).contiguous()
        B = t.shape[0]
        return t.reshape(B, -1).to(torch.float32).to(self.device, non_blocking=True).contiguous()

    def check_obs_range(self, flag=None):
        """ValueError if an observation encoded since the last check was beyond fp16 (nn.Tower.check_obs_range)."""
        self.tower_pi.check_obs_range(flag)

    def forward(self, x, B, src_idx=None, masks=True, seq=None):
        """Towers + heads for B samples of x (optionally gathered through src_idx); masks=False: no backward follows.
        seq (recurrent networks): how the B rows form sequences (nn.Seq)."""
        if self.fuse0:
            tp, tv = self.tower_pi, self.tower_vf
            a = tp.fcs[0]
            enc = tp.encode(x, B, src_idx)
            ops.gemm(enc, self.w0cat, self.h0cat, M=B, N=2 * a.N, K=a.Kp + a.K, lda=2 * tp.in_pad, ldb=a.Kf,
                     ldc=2 * a.N, bias=self.b0cat, mode=ops.MODE_F16_ACT, act=a.act, tag="fwd.pi+vf/mlp_fc0")
            lat, ldl = tp.forward(x, B, src_idx, encoded=enc, skip_first=True)
            latv, ldlv = tv.forward(x, B, src_idx, encoded=enc, skip_first=True)
            self._lat_pi, self._ld_lat_pi, self._lat_vf, self._ld_lat_vf = lat, ldl, latv, ldlv
            self.head_pi.forward(lat, ldl, B, self.pi_out, self.ld_pi, mode=ops.MODE_F32_STORE)
            self.head_vf.forward(latv, ldlv, B, self.v_out, self.ld_v, mode=ops.MODE_F32_STORE)
            return
        lat, ldl = self.tower_pi.forward(x, B, src_idx, masks=masks, seq=seq)
        self._lat_pi, self._ld_lat_pi = lat, ldl
        if self.head is not None:
            self.head.forward(lat, ldl, B, self.headout, self.ld_ho, mode=ops.MODE_F32_STORE)
        else:
            # the value tower of value_network='copy' reads the same observations: encode them once
            enc = self.tower_pi.x0 if self.tower_pi.kind == "mlp" else None
            latv, ldlv = self.tower_vf.forward(x, B, src_idx, encoded=enc, masks=masks)
            self._lat_vf, self._ld_lat_vf = latv, ldlv
            self.head_pi.forward(lat, ldl, B, self.pi_out, self.ld_pi, mode=ops.MODE_F32_STORE)
            self.head_vf.forward(latv, ldlv, B, self.v_out, self.ld_v, mode=ops.MODE_F32_STORE)

    def act(self, x, B, actions, values, neglogp, noise=None, seed=0, seq=None):
        """PolicyWithValue.step (policies.py:77-96) into caller-provided device tensors.  The sampler's stream position
        is a device counter advanced after every pass, so the sequence can be replayed from a CUDA graph."""
        _lib.phase = "@act"
        self.forward(x, B, masks=False, seq=seq)
        if self.pd in ("cat", "mcat"):
            ops.cat_step(self.pi_out, self.ld_pi, self.nout, self.v_out, self.ld_v, actions, values, neglogp, B,
                         uniforms=noise, seed=seed, offset_dev=self.rng_ctr, seg_off=self.seg_off)
        elif self.pd == "bern":
            ops.bern_step(self.pi_out, self.ld_pi, self.nout, self.v_out, self.ld_v, actions, values, neglogp, B,
                          uniforms=noise, seed=seed, offset_dev=self.rng_ctr)
        else:
            ops.gauss_step(self.pi_out, self.ld_pi, self.logstd, self.nout, self.v_out, self.ld_v, actions, values,
                           neglogp, B, normals=noise, seed=seed, offset_dev=self.rng_ctr)
        ops.counter_add(self.rng_ctr, 1)

    def _fused_first_wgrad(self, B, alpha):
        """[gW_pi | gW_vf] += alpha * x^T [dz_pi | dz_vf]: the encoded observations are read once (twice with the lo half)
        instead of once per tower; the result is split into the two parameters' gradient views."""
        tp, tv = self.tower_pi, self.tower_vf
        a, b = tp.fcs[0], tv.fcs[0]
        N2, x, ldx = 2 * a.N, tp._mlp_in, 2 * tp.in_pad
        bn = 256 if N2 == 256 else (128 if N2 > 64 else 64)
        tiles = -(-a.K // 128) * -(-N2 // bn)
        kb = -(-B // 64)
        split = max(1, min(kb // 2 if kb >= 2 else 1, -(-2 * ops.num_sms() // tiles)))
        self.g0cat.zero_()
        for xs in ((x, x[:, a.Kp:]) if a.split_in else (x,)):
            ops.gemm(xs, self.dz0cat, self.g0cat, M=a.K, N=N2, K=B, lda=ldx, ldb=N2, ldc=N2, mn_major=True,
                     mode=ops.MODE_F32_ATOMIC, alpha=alpha * a.in_scale, split_k=split, tag="wgrad.pi+vf/mlp_fc0")
        a.gw.add_(self.g0cat[:, :a.N])
        b.gw.add_(self.g0cat[:, a.N:])
        ops.colsum(tp.dzfc[0], a.gb, B, a.N, N2, alpha=alpha)
        ops.colsum(tv.dzfc[0], b.gb, B, b.N, N2, alpha=alpha)

    def loss_backward(self, x, B, src_idx, actions, returns, old_values, old_neglogp, cliprange, ent_coef, vf_coef,
                      inv_M, seq=None):
        """One chunk of ppo2/model.py:57-114: forward, loss statistics, full backward into store.grads
        (gradients of the MEAN loss: every wgrad carries alpha = 1/M).  cliprange None: read it from `clip_dev`
        (written with ops.set_scalars by the caller) -- the form a captured launch sequence uses."""
        clip_dev = self.clip_dev if cliprange is None else None
        cliprange = 0.0 if cliprange is None else cliprange
        _lib.phase = "@train"
        self.forward(x, B, src_idx, seq=seq)
        if self.pd in ("cat", "mcat"):
            ops.cat_loss(self.pi_out, self.ld_pi, self.nout, self.v_out, self.ld_v, actions, src_idx, returns,
                         old_values, old_neglogp, self.adv_st, cliprange, ent_coef, vf_coef, self.dpi, self.ld_dpi,
                         self.dv, self.ld_dv, self.stats, B, cliprange_dev=clip_dev, seg_off=self.seg_off)
        elif self.pd == "bern":
            ops.bern_loss(self.pi_out, self.ld_pi, self.nout, self.v_out, self.ld_v, actions, src_idx, returns,
                          old_values, old_neglogp, self.adv_st, cliprange, ent_coef, vf_coef, self.dpi, self.ld_dpi,
                          self.dv, self.ld_dv, self.stats, B, cliprange_dev=clip_dev)
        else:
            ops.gauss_loss(self.pi_out, self.ld_pi, self.logstd, self.nout, self.v_out, self.ld_v, actions, src_idx,
                           returns, old_values, old_neglogp, self.adv_st, cliprange, ent_coef, vf_coef, self.dpi,
                           self.ld_dpi, self.dv, self.ld_dv, self.g_logstd, inv_M, self.stats, B,
                           cliprange_dev=clip_dev)
        self.backward(B, inv_M)

    def backward(self, B, alpha):
        """Backward of the last forward from the head-output gradients in dpi / dv: every weight gradient accumulates
        alpha * (its gradient of the sum over the B rows) into store.grads."""
        tp = self.tower_pi
        if self.head is not None:
            self.head.wgrad(self._lat_pi, self._ld_lat_pi, self.dhead, self.ld_dh, B, alpha)
            self.head.dgrad(self.dhead, self.ld_dh, B, tp.dlatent, tp.ld_dlatent, saved=self._lat_pi,
                            ld_saved=self._ld_lat_pi, act=tp.latent_act)
            tp.backward(B, alpha)
        else:
            tv = self.tower_vf
            self.head_pi.wgrad(self._lat_pi, self._ld_lat_pi, self.dpi, self.ld_dpi, B, alpha)
            self.head_pi.dgrad(self.dpi, self.ld_dpi, B, tp.dlatent, tp.ld_dlatent, saved=self._lat_pi,
                               ld_saved=self._ld_lat_pi, act=tp.latent_act)
            tp.backward(B, alpha, skip_first_wgrad=self.fuse0)
            self.head_vf.wgrad(self._lat_vf, self._ld_lat_vf, self.dv, self.ld_dv, B, alpha)
            self.head_vf.dgrad(self.dv, self.ld_dv, B, tv.dlatent, tv.ld_dlatent, saved=self._lat_vf,
                               ld_saved=self._ld_lat_vf, act=tv.latent_act)
            tv.backward(B, alpha, skip_first_wgrad=self.fuse0)
            if self.fuse0:
                self._fused_first_wgrad(B, alpha)
