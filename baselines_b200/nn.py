"""Host-side executor for the policy / Q networks: owns the flat fp32 parameter + Adam buffers, the fp16
operand copies, per-layer activation workspaces, and sequences the libb200rl kernels.

Mirrors (by behaviour, not by code) the layer primitives of the reference:
  conv / fc / ortho_init            baselines/a2c/utils.py:20-63
  nature_cnn / mlp / conv_only      baselines/common/models.py:15-26, 74-103, 221-249
All math runs in hand-written CUDA (ops.*); torch here only allocates memory and provides streams.
"""
import functools
import math
from collections import OrderedDict, namedtuple

import numpy as np
import torch

from . import ops

NATURE_CONVS = (("c1", 32, 8, 4), ("c2", 64, 4, 2), ("c3", 64, 3, 1))   # common/models.py:21-24


def _pad8(n):
    return (n + 7) // 8 * 8


def ortho_init(shape, scale, rng=np.random):
    """Orthogonal init used by every PPO2 layer (a2c/utils.py:20-35): SVD of a gaussian matrix drawn from
    the (globally seeded) numpy RandomState; host-side, done once."""
    shape = tuple(shape)
    flat = shape if len(shape) == 2 else (int(np.prod(shape[:-1])), shape[-1])
    a = rng.normal(0.0, 1.0, flat)
    u, _, v = np.linalg.svd(a, full_matrices=False)
    q = (u if u.shape == flat else v).reshape(shape)
    return (scale * q[:shape[0], :shape[1]]).astype(np.float32)


def xavier_uniform(shape, rng):
    """tf.contrib.layers default initializer (deepq/models.py:23-37, common/models.py:241)."""
    if len(shape) == 2:
        fan_in, fan_out = shape
    else:
        rf = int(np.prod(shape[:-2]))
        fan_in, fan_out = shape[-2] * rf, shape[-1] * rf
    lim = math.sqrt(6.0 / (fan_in + fan_out))
    return rng.uniform(-lim, lim, size=shape).astype(np.float32)


class ParamStore:
    """One flat fp32 buffer each for parameters, gradients and the two Adam slots (28 B/param per step),
    with named views.  `tf_names` maps the reference's TF variable names (tf_util.py:345-355 checkpoint
    keys) onto (possibly strided) views so checkpoints round-trip."""

    def __init__(self, device):
        self.device = device
        self._specs = []          # (name, shape, init ndarray)
        self.views = OrderedDict()
        self.gviews = OrderedDict()
        self.offsets = OrderedDict()
        self.tf_map = OrderedDict()   # tf name -> (internal name, slicer or None, tf shape)
        self.row_perms = {}
        self.params = self.grads = self.m = self.v = None

    def add(self, name, init):
        init = np.ascontiguousarray(init, dtype=np.float32)
        assert name not in [s[0] for s in self._specs], name
        self._specs.append((name, init.shape, init))
        return name

    def map_tf(self, tf_name, internal, tf_shape, col_slice=None, row_perm=None):
        """row_perm[i] = row of the TF-layout [K, N] matrix stored at internal row i."""
        self.tf_map[tf_name] = (internal, col_slice, tuple(tf_shape))
        if row_perm is not None:
            self.row_perms[tf_name] = np.asarray(row_perm, dtype=np.int64)

    def finalize(self):
        off = 0
        for name, shape, _ in self._specs:
            self.offsets[name] = off
            off += (int(np.prod(shape)) + 3) // 4 * 4
        self.numel = off
        dev = self.device
        self.params = torch.zeros(off, dtype=torch.float32, device=dev)
        self.grads = torch.zeros(off, dtype=torch.float32, device=dev)
        self.m = torch.zeros(off, dtype=torch.float32, device=dev)
        self.v = torch.zeros(off, dtype=torch.float32, device=dev)
        host = np.zeros(off, np.float32)
        for name, shape, init in self._specs:
            o, n = self.offsets[name], int(np.prod(shape))
            host[o:o + n] = init.ravel()
            self.views[name] = self.params[o:o + n].view(*shape)
            self.gviews[name] = self.grads[o:o + n].view(*shape)
        self.params.copy_(torch.from_numpy(host))
        self.n_true = sum(int(np.prod(s)) for _, s, _ in self._specs)
        return self

    def segment_offsets(self):
        """[nseg+1] element offsets of every variable (for per-variable tf.clip_by_norm)."""
        offs = [self.offsets[n] for n, _, _ in self._specs] + [self.numel]
        return np.asarray(offs, dtype=np.int64)

    # ---- checkpoint-format access (TF names / layouts) -------------------------------------------
    def _tf_view(self, buf_views, tf_name):
        internal, sl, shape = self.tf_map[tf_name]
        v = buf_views[internal]
        if sl is not None:
            v = v[..., sl]
        return v, shape

    def _views_of(self, flat):
        out = {}
        for name, shape, _ in self._specs:
            o, n = self.offsets[name], int(np.prod(shape))
            out[name] = flat[o:o + n].view(*shape)
        return out

    def export_tf(self, which="params"):
        flat = {"params": self.params, "grads": self.grads, "m": self.m, "v": self.v}[which]
        views = self._views_of(flat)
        out = OrderedDict()
        for tf_name in self.tf_map:
            v, shape = self._tf_view(views, tf_name)
            a = v.detach().cpu().numpy()
            if tf_name in self.row_perms:
                b = np.empty_like(a)
                b[self.row_perms[tf_name]] = a
                a = b
            out[tf_name] = a.reshape(shape).copy()
        return out

    def import_tf(self, values, which="params"):
        flat = {"params": self.params, "grads": self.grads, "m": self.m, "v": self.v}[which]
        views = self._views_of(flat)
        for tf_name, arr in values.items():
            if tf_name not in self.tf_map:
                continue
            v, shape = self._tf_view(views, tf_name)
            a = np.ascontiguousarray(arr, dtype=np.float32).reshape(v.shape)
            if tf_name in self.row_perms:
                a = np.ascontiguousarray(a[self.row_perms[tf_name]])
            v.copy_(torch.from_numpy(a).to(self.device))


class Linear:
    """y = act(x W + b) with W [K, N] fp32 master (TF [in, out] layout) and two fp16 operand copies:
    w_fwd [N, Kp] (= W^T, forward B operand) and w_bwd [K, Np] (dgrad B operand)."""

    def __init__(self, store, name, K, N, act, w_init, b_init=None, in_scale=1.0, w_shape=None, b_shape=None,
                 tf_w=None, tf_b=None, row_perm=None, split_in=False):
        self.store, self.name, self.K, self.N, self.act = store, name, K, N, ops.ACT_CODES[act]
        self.in_scale = float(in_scale)
        self.Kp, self.Np = _pad8(K), _pad8(N)
        # split_in: the input rows are fp16 [hi | lo] pairs of float32 values (csrc/obs_encode.cu); the forward
        # operand is W^T stacked twice along K, the weight gradient is the sum of the hi and lo contributions
        self.split_in = bool(split_in)
        self.Kf = 2 * self.Kp if self.split_in else self.Kp
        w_init = np.asarray(w_init, np.float32).reshape(K, N)
        if row_perm is not None:
            w_init = w_init[np.asarray(row_perm)]
        store.add(name + "/w", w_init)
        store.add(name + "/b", np.zeros(N, np.float32) if b_init is None else np.asarray(b_init, np.float32).reshape(N))
        if tf_w:
            store.map_tf(tf_w, name + "/w", w_shape or (K, N), row_perm=row_perm)
        if tf_b:
            store.map_tf(tf_b, name + "/b", b_shape or (N,))
        self.w_fwd = self.w_bwd = None

    def materialize(self):
        dev = self.store.device
        self.w = self.store.views[self.name + "/w"]
        self.b = self.store.views[self.name + "/b"]
        self.gw = self.store.gviews[self.name + "/w"]
        self.gb = self.store.gviews[self.name + "/b"]
        self.w_fwd = torch.zeros(self.N, self.Kf, dtype=torch.float16, device=dev)
        self.w_bwd = torch.zeros(self.K, self.Np, dtype=torch.float16, device=dev)

    def cast_jobs(self):
        """The casts that derive w_bwd and w_fwd (both halves of a split_in one) from the fp32 master weight."""
        jobs = [ops.CastJob(self.w, self.K, self.N, self.w_bwd, self.Np, self.w_fwd, self.Kf, self.in_scale)]
        if self.split_in:
            jobs.append(ops.CastJob(self.w, self.K, self.N, None, 0, self.w_fwd[:, self.Kp:], self.Kf, self.in_scale))
        return jobs

    def forward(self, x, ldx, M, out, ldo, mode=ops.MODE_F16_ACT, act=None):
        K = self.Kp + self.K if self.split_in else self.K
        ops.gemm(x, self.w_fwd, out, M=M, N=self.N, K=K, lda=ldx, ldb=self.Kf, ldc=ldo, bias=self.b,
                 mode=mode, act=self.act if act is None else act, tag="fwd." + self.name)

    def wgrad(self, x, ldx, dz, lddz, M, alpha):
        """gW += alpha * x^T dz (fp32 atomics, split-K over the batch rows); gb += alpha * colsum(dz)."""
        bn = 256 if (self.N > 128 and self.N % 256 == 0) else (128 if self.N > 64 else 64)   # b200rl_gemm_f16's N tile
        tiles = -(-self.K // 128) * -(-self.N // bn)
        kb = -(-M // 64)
        split = max(1, min(kb // 2 if kb >= 2 else 1, -(-2 * ops.num_sms() // tiles)))
        ops.gemm(x, dz, self.gw, M=self.K, N=self.N, K=M, lda=ldx, ldb=lddz, ldc=self.N, mn_major=True,
                 mode=ops.MODE_F32_ATOMIC, alpha=alpha * self.in_scale, split_k=split, tag="wgrad." + self.name)
        if self.split_in:                                  # + lo^T dz
            ops.gemm(x[:, self.Kp:], dz, self.gw, M=self.K, N=self.N, K=M, lda=ldx, ldb=lddz, ldc=self.N,
                     mn_major=True, mode=ops.MODE_F32_ATOMIC, alpha=alpha * self.in_scale, split_k=split,
                     tag="wgrad." + self.name)
        ops.colsum(dz, self.gb, M, self.N, lddz, alpha=alpha)

    def dgrad(self, dz, lddz, M, out, ldo, saved=None, ld_saved=0, act=ops.ACT_NONE, remap=(0, 0, 0), saved_bits=None):
        """out[M, K] = (dz W^T) * act'(saved); saved_bits: the ReLU mask as 1 bit per element instead of `saved`."""
        if saved_bits is not None and act == ops.ACT_RELU:
            ops.gemm(dz, self.w_bwd, out, M=M, N=self.K, K=self.N, lda=lddz, ldb=self.Np, ldc=ldo, saved_bits=saved_bits,
                     ld_saved=ld_saved, mode=ops.MODE_F16_DACT, act=act, tag="dgrad." + self.name, remap=remap)
        elif saved is None or act == ops.ACT_NONE:
            ops.gemm(dz, self.w_bwd, out, M=M, N=self.K, K=self.N, lda=lddz, ldb=self.Np, ldc=ldo,
                     mode=ops.MODE_F16_ACT, act=ops.ACT_NONE, tag="dgrad." + self.name, remap=remap)
        else:
            ops.gemm(dz, self.w_bwd, out, M=M, N=self.K, K=self.N, lda=lddz, ldb=self.Np, ldc=ldo, saved=saved,
                     ld_saved=ld_saved, mode=ops.MODE_F16_DACT, act=act, tag="dgrad." + self.name, remap=remap)


LN_EPS = 1e-12      # variance_epsilon of tf.contrib.layers.layer_norm (tf.nn.batch_normalization inside it)


def ln_scope(k):
    """Name tf.contrib.layers.layer_norm gives its k-th use inside one variable scope."""
    return "LayerNorm" if k == 0 else f"LayerNorm_{k}"


class LayerNorm:
    """y = act(gamma * (z - mean) / sqrt(var + LN_EPS) + beta) over each row of a layer's fp32 pre-activation z
    (tf.contrib.layers.layer_norm(center=True, scale=True), common/models.py:97-98, deepq/models.py:24-25).  Variables
    beta (zeros) then gamma (ones), [N] each, `<tf_scope>/{beta,gamma}:0`; neither draws from the RNG.  They stay fp32:
    the operand refresh has nothing to cast."""

    def __init__(self, store, name, N, act, tf_scope, cap):
        self.store, self.name, self.N, self.act, self.cap = store, name, N, ops.ACT_CODES[act], cap
        store.add(name + "/beta", np.zeros(N, np.float32))
        store.add(name + "/gamma", np.ones(N, np.float32))
        store.map_tf(f"{tf_scope}/beta:0", name + "/beta", (N,))
        store.map_tf(f"{tf_scope}/gamma:0", name + "/gamma", (N,))

    def materialize(self):
        v, g = self.store.views, self.store.gviews
        self.beta, self.gamma = v[self.name + "/beta"], v[self.name + "/gamma"]
        self.gbeta, self.ggamma = g[self.name + "/beta"], g[self.name + "/gamma"]
        # the layer's pre-activation: written by its GEMM (MODE_F32_STORE), read again by the backward
        self.z = torch.empty(self.cap, _pad8(self.N), dtype=torch.float32, device=self.store.device)
        self.ldz = _pad8(self.N)

    def forward(self, M, y, ldy):
        ops.ln_fwd(self.z, self.ldz, self.gamma, self.beta, y, ldy, M, self.N, self.act, LN_EPS)

    def backward(self, M, du, lddu, alpha):
        """du: d loss / d (gamma * xhat + beta), replaced in place by d loss / d z; the norm's gradients accumulate."""
        ops.ln_bwd(du, lddu, self.z, self.ldz, self.gamma, du, lddu, self.ggamma, self.gbeta, M, self.N, alpha, LN_EPS)


def linear_ln_forward(l, ln, x, ldx, M, out, ldo):
    """out = l's activation of x: act(x W + b), or with a norm act(LN(x W + b)) through the norm's fp32 workspace."""
    if ln is None:
        l.forward(x, ldx, M, out, ldo)
    else:
        l.forward(x, ldx, M, ln.z, ln.ldz, mode=ops.MODE_F32_STORE, act=ops.ACT_NONE)
        ln.forward(M, out, ldo)


class Conv(Linear):
    """NHWC convolution lowered to im2col + wgmma GEMM (a2c/utils.py:37-56)."""

    def __init__(self, store, name, H, W, C, nf, rf, stride, act, w_init, plan, same_pad=False, in_scale=1.0,
                 tf_w=None, tf_b=None, b_shape=None):
        """plan: this layer's ConvLayerPlan (plan_conv_stack)."""
        self.H, self.W, self.C, self.nf, self.rf, self.stride, self.same = H, W, C, nf, rf, stride, same_pad
        self.OH, self.OW = ops._conv_out(H, W, rf, stride, same_pad)
        self.P = self.OH * self.OW
        self.s2d, self.geom, self.implicit_dgrad = plan.s2d, plan.geom, plan.implicit_dgrad
        self.implicit = plan.path == "implicit"
        # space-to-depth view: stride-s conv, filter k*s  ->  stride-1 conv, filter k, over s*s*C channels.  The fp32
        # master weight is stored with its K rows in (a, b, dy, dx, c) order; row_perm maps them back to the
        # reference's HWIO (ky, kx, c) order for checkpoints.
        row_perm = None
        if self.s2d:
            s_, k = stride, rf // stride
            idx = np.empty(rf * rf * C, dtype=np.int64)
            i = 0
            for a in range(k):
                for b in range(k):
                    for dy in range(s_):
                        for dx in range(s_):
                            for c in range(C):
                                idx[i] = ((a * s_ + dy) * rf + (b * s_ + dx)) * C + c
                                i += 1
            row_perm = idx
        super().__init__(store, name, rf * rf * C, nf, act, w_init, in_scale=in_scale, w_shape=(rf, rf, C, nf),
                         b_shape=b_shape or (1, nf, 1, 1), tf_w=tf_w, tf_b=tf_b, row_perm=row_perm)

    def im2col(self, x, cols, B, src_idx=None):
        ops.im2col(x, cols, B, self.H, self.W, self.C, self.rf, self.stride, self.same, src_idx=src_idx, tag=self.name)

    def col2im(self, dcols, saved, dx, B, act):
        ops.col2im(dcols, saved, dx, B, self.H, self.W, self.C, self.rf, self.stride, self.same, act=act, tag=self.name)

    # ---- implicit-GEMM path (TMA im2col through self.geom): no cols / dcols buffers -----------------------------
    def materialize(self):
        super().materialize()
        self.wdg = None
        if self.implicit_dgrad:
            An = -(-self.rf // self.stride)
            self.An, self.ld_wdg = An, An * An * self.nf
            self.wdg = torch.zeros(self.stride * self.stride * self.C, self.ld_wdg, dtype=torch.float16,
                                   device=self.store.device)

    def operand_launches(self):
        """The operand kernels that are not casts, as calls without arguments: the pixel-shuffle data-gradient weights
        wdg."""
        if self.wdg is None:
            return []
        return [functools.partial(ops.dgrad_weights, self.w, self.wdg, self.rf, self.rf, self.C, self.nf, self.stride,
                                  self.ld_wdg)]

    def fwd_implicit(self, x, B, out):
        H, W, C, R, S, sh, sw, pt, pl = self.geom
        ops.conv_gemm(x, B, H, W, C, R, S, sh, sw, pt, pl, self.OH, self.OW, self.w_fwd, self.Kp, out, self.nf,
                      self.nf, 0, ops.MODE_F16_ACT, act=self.act, bias=self.b, tag="fwd." + self.name)

    def wgrad_implicit(self, x, dz, B, alpha):
        H, W, C, R, S, sh, sw, pt, pl = self.geom
        tiles = -(-self.K // 128)
        rows = B * self.P
        split = max(1, min((rows // 64) // 2 if rows >= 128 else 1, -(-2 * ops.num_sms() // tiles)))
        ops.conv_gemm(x, B, H, W, C, R, S, sh, sw, pt, pl, self.OH, self.OW, dz, self.nf, self.gw, self.nf, self.nf, 1,
                      ops.MODE_F32_ATOMIC, alpha=alpha * self.in_scale, split_k=split, tag="wgrad." + self.name)
        ops.colsum(dz, self.gb, rows, self.nf, self.nf, alpha=alpha)

    def dgrad_implicit(self, dz, B, saved_in, dx, act):
        """dx[B,H,W,C] = conv_transpose(dz) * act'(saved_in): one implicit GEMM over dz with the pixel-shuffle
        epilogue.  (VALID padding only.)"""
        s, An = self.stride, self.An
        G_h, G_w = -(-self.H // s), -(-self.W // s)
        ops.conv_gemm(dz, B, self.OH, self.OW, self.nf, An, An, 1, 1, An - 1, An - 1, G_h, G_w, self.wdg, self.ld_wdg,
                      dx, 0, s * s * self.C, 0, ops.MODE_F16_SHUFFLE, act=act, saved=saved_in,
                      shuffle=(self.H, self.W, self.C, s), tag="dgrad." + self.name)


LSTM_SIZES = (64, 128)     # nlstm instances of csrc/lstm.cu

Seq = namedtuple("Seq", "T B masks mask_idx state state_idx state_out")
Seq.__doc__ = """How the rows of one LSTM pass form sequences: T time-major steps of B environments (row t*B + b); masks
uint8 "done before step t" of row r at masks[mask_idx[r]] (mask_idx None: masks[r]); environment b starts from row
state_idx[b] (None: b) of the float32 [*, 2H] state; state_out: where the final state goes (None: not kept)."""


class LSTM:
    """The cell of a2c/utils.py:84-97 lstm() over a sequence: the input projection x.wx + b is one GEMM over all rows (a
    Linear, MODE_F32_STORE), the recurrence csrc/lstm.cu.  Variables wx [nin, 4H], wh [H, 4H], b [4H] under
    `<tf_prefix>/lstm/` in the reference's [i | f | o | u] gate layout; wx and wh take ortho_init(1.0) in that order
    (utils.py:89-91)."""

    def __init__(self, store, prefix, tf_prefix, nin, H, winit, split_in=False):
        if H not in LSTM_SIZES:
            raise NotImplementedError(f"nlstm={H}: the LSTM sequence kernels are built for nlstm in {LSTM_SIZES}")
        self.store, self.H, self.nin = store, H, nin
        w_x = winit((nin, 4 * H), 1.0)
        w_h = winit((H, 4 * H), 1.0)
        self.wx = Linear(store, f"{prefix}/lstm/wx", nin, 4 * H, None, w_x, tf_w=f"{tf_prefix}/lstm/wx:0",
                         tf_b=f"{tf_prefix}/lstm/b:0", split_in=split_in)
        self.wh_name = store.add(f"{prefix}/lstm/wh", w_h)
        store.map_tf(f"{tf_prefix}/lstm/wh:0", self.wh_name, (H, 4 * H))

    def materialize(self, cap):
        dev, H = self.store.device, self.H
        self.wx.materialize()
        self.wh = self.store.views[self.wh_name]
        self.gwh = self.store.gviews[self.wh_name]
        f16, f32 = dict(dtype=torch.float16, device=dev), dict(dtype=torch.float32, device=dev)
        self.wh16 = torch.zeros(H, 4 * H, **f16)          # forward operand (Wh)
        self.whT16 = torch.zeros(4 * H, H, **f16)         # backward operand (Wh^T)
        self.xg = torch.zeros(cap, 4 * H, **f32)          # x.wx + b, overwritten in place by the gate activations
        self.c = torch.zeros(cap, H, **f32)
        self.h = torch.zeros(cap, H, **f16)               # the latent
        self.hprev = torch.zeros(cap, H, **f16)           # masked h_{t-1}: the A operand of dWh
        self.dh = torch.zeros(cap, H, **f16)              # d loss / d h_t, written by the heads' data gradient
        self.dz = torch.zeros(cap, 4 * H, **f16)

    def cast_jobs(self):
        """wx's casts, then wh16 = fp16(wh) and whT16 = fp16(wh^T)."""
        return self.wx.cast_jobs() + [ops.CastJob(self.wh, self.H, 4 * self.H, self.wh16, 4 * self.H, self.whT16, self.H,
                                                  1.0)]

    def refresh(self):
        """Eager operand refresh, one launch per cast."""
        for j in self.cast_jobs():
            ops.cast_transpose(*j)

    def forward(self, x, ldx, seq, train=True):
        """x: [T*B, *] fp16 input rows (time-major).  train=False: only h and the state (acting / value passes)."""
        H, rows = self.H, seq.T * seq.B
        self.wx.forward(x, ldx, rows, self.xg, 4 * H, mode=ops.MODE_F32_STORE, act=ops.ACT_NONE)
        ops.lstm_seq_fwd(self.xg, 4 * H, self.wh16, seq.masks, seq.state, self.h, H, seq.T, seq.B, H,
                         mask_idx=seq.mask_idx, state_idx=seq.state_idx, state_out=seq.state_out,
                         hprev_out=self.hprev if train else None, gates_out=self.xg if train else None,
                         c_out=self.c if train else None)
        self._x, self._ldx, self._seq = x, ldx, seq
        return self.h, H

    def backward(self, alpha, dx=None, ldo=0, saved=None, ld_saved=0, act=ops.ACT_NONE):
        """self.dh -> dz; dWh += alpha hprev^T dz, dWx += alpha x^T dz, db += alpha colsum(dz); dx = (dz Wx^T) act'(saved)
        when dx is given."""
        H, seq = self.H, self._seq
        rows = seq.T * seq.B
        ops.lstm_seq_bwd(self.dh, H, self.xg, self.c, seq.masks, seq.state, self.whT16, self.dz, 4 * H, seq.T, seq.B, H,
                         mask_idx=seq.mask_idx, state_idx=seq.state_idx)
        tiles = -(-H // 128) * -(-4 * H // 256)
        kb = -(-rows // 64)
        split = max(1, min(kb // 2 if kb >= 2 else 1, -(-2 * ops.num_sms() // tiles)))
        ops.gemm(self.hprev, self.dz, self.gwh, M=H, N=4 * H, K=rows, lda=H, ldb=4 * H, ldc=4 * H, mn_major=True,
                 mode=ops.MODE_F32_ATOMIC, alpha=alpha, split_k=split, tag="wgrad.lstm/wh")
        self.wx.wgrad(self._x, self._ldx, self.dz, 4 * H, rows, alpha)
        if dx is not None:
            self.wx.dgrad(self.dz, 4 * H, rows, dx, ldo, saved=saved, ld_saved=ld_saved, act=act)


ConvLayerPlan = namedtuple("ConvLayerPlan", "path s2d geom implicit_dgrad kx")
ConvLayerPlan.__doc__ = """How one conv layer runs.  path: "shift" (csrc/conv_shift.cu), "implicit" (TMA im2col GEMM over the
input viewed as geom = (H, W, C, R, S, stride_h, stride_w, pad_t, pad_l)) or "explicit" (im2col + GEMM).  s2d: the
layer reads its input space-to-depth'ed (and its master weight rows are stored in that order).  implicit_dgrad: the
data gradient is one implicit GEMM with the pixel-shuffle epilogue instead of GEMM + col2im.  kx: taps per filter row
the shift-GEMM weight gradient folds into one pass."""
ConvStackPlan = namedtuple("ConvStackPlan", "shift fused_u8 layers")
ConvStackPlan.__doc__ = """shift: every layer runs as shift-GEMM, and every layer writes its 1-bit ReLU mask, which the next
data gradient (or fc1's) reads.  fused_u8: the first shift layer reads the uint8 frames itself."""

# (k, nf, Cg) instances of the x-folded shift-GEMM weight gradient (csrc/conv_shift.cu conv_shift_wgrad_kernel)
_XFOLD_WGRAD = ((2, 32, 64), (2, 64, 64), (2, 64, 128), (3, 64, 64))


def _shift_stack_ok(ob_shape, convs):
    """Every layer of a VALID conv stack passes the host checks of csrc/conv_shift.cu on its space-to-depth view: its
    forward and weight gradient, and the data gradient that writes its input gradient."""
    H, W, C = ob_shape
    for i, (_nm, nf, rf, st) in enumerate(convs):
        if rf % st or H % st or W % st:                 # space-to-depth view: a stride-1 k x k conv
            return False
        k, Hg, Wg, Cg = rf // st, H // st, W // st, C * st * st
        span = (k - 1) * Wg + (k - 1)                    # rows between the first and the last tap
        # b200rl_conv_shift_fwd: C = 64 or 128, 1..16 taps, grid >= 2 x 2; b200rl_conv_shift_wgrad: N = 32 or 64
        if Cg not in (64, 128) or k * k > 16 or Hg < 2 or Wg < 2 or nf not in (32, 64):
            return False
        # b200rl_conv_shift_fwd: span <= 32 rows for C = 64, <= 16 for C = 128 (sh_arows); resident weights
        # taps * C/64 * N * 128 B <= 80 KB for C = 64, <= 64 KB for C = 128 (sh_wres_bytes)
        if span > (32 if Cg == 64 else 16) or k * k * (Cg // 64) * nf * 128 > (80 if Cg == 64 else 64) * 1024:
            return False
        # the data gradient of layer i > 0 is b200rl_conv_shift_fwd with C = nf: 64
        if i > 0 and nf != 64:
            return False
        OH, OW = ops._conv_out(H, W, rf, st, False)
        if i + 1 < len(convs):
            nrf, nst = convs[i + 1][2], convs[i + 1][3]
            if OH % nst or OW % nst:                     # layer i writes its output space-to-depth'ed for layer i+1
                return False
            # the data gradient of layer i+1 writes N = s^2 * nf outputs (b200rl_conv_shift_fwd: N = 64 or 128 here, C =
            # 64, resident weights taps * N * 128 B <= 80 KB)
            kn = nrf // nst
            if nf * nst * nst not in (64, 128) or kn * kn * nf * nst * nst * 128 > 80 * 1024:
                return False
        H, W, C = OH, OW, nf
    return True


def _implicit_geom(H, W, C, rf, st, same_pad, s2d):
    """The input as TMA im2col sees it, or None.  b200rl_conv_gemm: 16, 32 or 64 channels per tap; a layer with few
    channels is viewed through "super-pixels" of 16 consecutive (x, c) elements when the stride allows it."""
    if s2d:
        return (H // st, W // st, C * st * st, rf // st, rf // st, 1, 1, 0, 0)
    pad_t = pad_l = 0
    if same_pad:
        OH, OW = ops._conv_out(H, W, rf, st, True)
        pad_t, pad_l = max((OH - 1) * st + rf - H, 0) // 2, max((OW - 1) * st + rf - W, 0) // 2
    m = 64 // C if C in (16, 32) else 1
    if m > 1 and W % m == 0 and rf % m == 0 and st % m == 0 and pad_l % m == 0:
        # merge m horizontally adjacent pixels into one 64-channel "pixel": same memory, same K order,
        # but full 128-byte TMA rows and m x fewer taps
        return (H, W // m, C * m, rf, rf // m, st, st // m, pad_t, pad_l // m)
    if C in (16, 32, 64):
        return (H, W, C, rf, rf, st, st, pad_t, pad_l)
    if 16 % C == 0 and (W * C) % 16 == 0 and (rf * C) % 16 == 0 and (st * C) % 16 == 0 and (pad_l * C) % 16 == 0:
        k = 16 // C
        return (H, W // k, 16, rf, rf // k, st, st // k, pad_t, pad_l // k)
    return None


def plan_conv_stack(ob_shape, convs, same_pad, has_fc):
    """The convolution path of every layer of a conv stack over uint8 (H, W, C) observations, from the shapes alone.
    convs: (name, filters, filter size, stride) per layer; has_fc: an fc layer follows the stack.  Returns a
    ConvStackPlan.  A stack that passes the shift-GEMM checks runs as shift-GEMM; any other one layer by layer on the
    implicit GEMM where its geometry allows, else on im2col + GEMM."""
    if not same_pad and _shift_stack_ok(ob_shape, convs):
        if not has_fc:
            raise NotImplementedError("shift-mode conv_only towers")
        H, W, C = ob_shape
        layers = []
        for _nm, nf, rf, st in convs:
            k, Cg = rf // st, C * st * st
            OH, OW = ops._conv_out(H, W, rf, st, False)
            assert (OH * OW * nf) % 16 == 0                  # the 1-bit mask is written in 16-element words
            layers.append(ConvLayerPlan("shift", st > 1, None, False, k if (k, nf, Cg) in _XFOLD_WGRAD else 1))
            H, W, C = OH, OW, nf
        _nm, nf0, rf0, st0 = convs[0]
        # b200rl_conv_shift_fwd / b200rl_conv_shift_wgrad, uint8 source: s = 4, s*C = 16, N = 32, resident weights
        # taps * N * 128 B <= 16 KB (SH_U8_WRES_BYTES)
        fused_u8 = st0 == 4 and ob_shape[2] == 4 and nf0 == 32 and (rf0 // st0) ** 2 * nf0 * 128 <= 16 * 1024
        return ConvStackPlan(True, fused_u8, layers)
    H, W, C = ob_shape
    layers = []
    for i, (_nm, nf, rf, st) in enumerate(convs):
        # first layer: space-to-depth'ed by b200rl_s2d_gather (H, W multiples of s; s*C, W*C multiples of 8) into the
        # 16 / 32 / 64 channels per tap of b200rl_conv_gemm
        s2d = (i == 0 and st > 1 and not same_pad and rf % st == 0 and H % st == 0 and W % st == 0 and
               C * st * st in (16, 32, 64) and (st * C) % 8 == 0 and (W * C) % 8 == 0)
        geom = _implicit_geom(H, W, C, rf, st, same_pad, s2d)
        # pixel-shuffle data gradient (b200rl_conv_gemm over dz: 16 / 32 / 64 channels per tap; shuffle epilogue:
        # C % 16 == 0; VALID padding only)
        implicit_dgrad = i > 0 and geom is not None and not same_pad and nf in (16, 32, 64) and C % 16 == 0
        layers.append(ConvLayerPlan("explicit" if geom is None else "implicit", s2d, geom, implicit_dgrad, 1))
        H, W = ops._conv_out(H, W, rf, st, same_pad)
        C = nf
    return ConvStackPlan(False, False, layers)


class Tower:
    """A latent network (conv stack + fc, or mlp) with its activation workspace for `cap` samples."""

    def __init__(self, store, kind, ob_shape, prefix, tf_prefix, rng, cap, init="ortho", num_layers=2,
                 num_hidden=64, convs=NATURE_CONVS, same_pad=False, fc_hidden=512, tf_style="a2c", onehot_n=0,
                 onehot_nvec=None, nlstm=128, layer_norm=False):
        """kind: cnn, conv_only, mlp, or the recurrent lstm (the observation encoding of mlp, then an LSTM; models.py
        lstm) and cnn_lstm (cnn, then an LSTM; models.py cnn_lstm).  The recurrent towers' forward and backward take
        the rows as sequences (Seq)."""
        if layer_norm and kind != "mlp":
            raise NotImplementedError("layer_norm is an argument of 'mlp' (common/models.py:75); layer-normalised LSTMs "
                                      "(lnlstm, cnn_lnlstm) are not implemented")
        self.kind, self.cap, self.store = kind, cap, store
        self.base = {"lstm": "mlp", "cnn_lstm": "cnn"}.get(kind, kind)      # the tower below the LSTM
        if kind == "lstm":
            num_layers = 0                              # models.py lstm: flatten(X) straight into the cell
        self.convs, self.fcs = [], []
        self.lns = []                                   # per fc layer: its LayerNorm or None
        self.lstm = None
        winit = (lambda shape, scale: ortho_init(shape, scale, rng)) if init == "ortho" else \
                (lambda shape, scale: xavier_uniform(shape, rng))
        if self.base in ("cnn", "conv_only"):
            H, W, C = ob_shape
            self.in_u8 = True
            scale_in = 1.0 / 255.0                                           # models.py:19 folded into c1 weights
            self.plan = plan_conv_stack(ob_shape, convs, same_pad, self.base == "cnn")
            self.shift_mode = self.plan.shift
            for i, ((nm, nf, rf, stride), lp) in enumerate(zip(convs, self.plan.layers)):
                if tf_style == "a2c":
                    tfw, tfb, bshape = f"{tf_prefix}/{nm}/w:0", f"{tf_prefix}/{nm}/b:0", (1, nf, 1, 1)
                else:
                    cn = "Conv" if i == 0 else f"Conv_{i}"
                    tfw, tfb, bshape = f"{tf_prefix}/convnet/{cn}/weights:0", f"{tf_prefix}/convnet/{cn}/biases:0", (nf,)
                conv = Conv(store, f"{prefix}/{nm}", H, W, C, nf, rf, stride, "relu",
                            winit((rf, rf, C, nf), math.sqrt(2)), lp, same_pad=same_pad,
                            in_scale=scale_in if i == 0 else 1.0, tf_w=tfw, tf_b=tfb, b_shape=bshape)
                self.convs.append(conv)
                H, W, C = conv.OH, conv.OW, nf
            self.flat = H * W * C
            if self.base == "cnn":
                self.fcs.append(Linear(store, f"{prefix}/fc1", self.flat, fc_hidden, "relu",
                                       winit((self.flat, fc_hidden), math.sqrt(2)),
                                       tf_w=f"{tf_prefix}/fc1/w:0", tf_b=f"{tf_prefix}/fc1/b:0"))
                self.latent_dim, self.latent_act = fc_hidden, ops.ACT_RELU
            else:
                self.latent_dim, self.latent_act = self.flat, ops.ACT_RELU
            self.in_dim = None
        elif self.base == "mlp":
            self.in_u8 = False
            self.shift_mode = False
            # Discrete(n) observations are one-hot encoded (common/input.py:54-55): raw rows hold the integer;
            # MultiDiscrete(nvec) ones are the concatenated one-hots of their components (:58-61): raw rows hold the
            # len(nvec) integers
            self.onehot_nvec = None if onehot_nvec is None else [int(v) for v in onehot_nvec]
            if self.onehot_nvec:
                self.onehot_n, self.raw_dim = sum(self.onehot_nvec), len(self.onehot_nvec)
            else:
                self.onehot_n = int(onehot_n)
                self.raw_dim = 1 if self.onehot_n else int(np.prod(ob_shape))
            nin = self.onehot_n if self.onehot_n else self.raw_dim
            self.in_dim, self.in_pad = nin, _pad8(nin)
            self.obs_norm = None                   # (mean, inv_std, lo, hi) float32 device tensors, policies.py:182-185
            for i in range(num_layers):                                       # models.py:94-99 (tanh)
                self.fcs.append(Linear(store, f"{prefix}/mlp_fc{i}", nin, num_hidden, "tanh",
                                       winit((nin, num_hidden), math.sqrt(2)),
                                       tf_w=f"{tf_prefix}/mlp_fc{i}/w:0", tf_b=f"{tf_prefix}/mlp_fc{i}/b:0",
                                       split_in=(i == 0)))
                if layer_norm:                                                # models.py:97-98
                    self.lns.append(LayerNorm(store, f"{prefix}/mlp_ln{i}", num_hidden, "tanh",
                                              f"{tf_prefix}/{ln_scope(i)}", cap))
                nin = num_hidden
            self.latent_dim, self.latent_act = nin, ops.ACT_TANH
        else:
            raise ValueError(f"unknown network type {kind!r} (supported: cnn, conv_only, mlp, lstm, cnn_lstm)")
        self.layers = self.convs + self.fcs
        self.lns = self.lns or [None] * len(self.fcs)
        if kind in ("lstm", "cnn_lstm"):
            # utils.py:89-91: wx and wh take ortho_init(1.0) after the layers below them (it fixes the RNG stream)
            self.lstm = LSTM(store, prefix, tf_prefix, self.latent_dim, nlstm,
                             lambda shape, scale: ortho_init(shape, scale, rng), split_in=self.base == "mlp")
            self.latent_dim, self.latent_act = nlstm, ops.ACT_NONE

    def materialize(self):
        self._materialize_layers()
        if self.lstm is not None:
            self.lstm.materialize(self.cap)
            self.dlatent, self.ld_dlatent = self.lstm.dh, self.lstm.H

    def _materialize_layers(self):
        dev, cap = self.store.device, self.cap
        f16 = dict(dtype=torch.float16, device=dev)
        for l in self.layers + [n for n in self.lns if n is not None]:
            l.materialize()
        if self.convs and self.shift_mode:
            self._materialize_shift(f16)
            self.hfc = [torch.empty(cap, l.Np, **f16) for l in self.fcs]
            self.dzfc = [torch.empty(cap, l.Np, **f16) for l in self.fcs]
            self.ld_hfc = [l.Np for l in self.fcs]     # row pitch of hfc[i] / dzfc[i]
            self.dlatent, self.ld_dlatent = self.dzfc[-1], self.fcs[-1].Np
            return
        self.cols = [None if c.implicit else torch.empty(cap * c.P, c.K, **f16) for c in self.convs]
        self.hconv = [torch.empty(cap * c.P, c.nf, **f16) for c in self.convs]
        self.dcols = [None] + [None if c.implicit_dgrad else torch.empty(cap * c.P, c.K, **f16)
                               for c in self.convs[1:]]
        self.dzconv = [torch.zeros(cap * c.P, c.nf, **f16) for c in self.convs]
        if self.convs and self.convs[0].implicit and self.in_u8:
            c0 = self.convs[0]
            self.x16 = torch.empty(cap, c0.H * c0.W * c0.C, **f16)     # gathered uint8 -> fp16 observations
        self.hfc = [torch.empty(cap, l.Np, **f16) for l in self.fcs]
        self.dzfc = [torch.empty(cap, l.Np, **f16) for l in self.fcs]
        self.ld_hfc = [l.Np for l in self.fcs]         # row pitch of hfc[i] / dzfc[i] (a fused first layer widens [0])
        if self.base == "mlp":
            self.x0 = torch.zeros(cap, 2 * self.in_pad, **f16)      # [hi | lo] operand rows of the float32 observations
            # set by the encoder when an observation value is beyond fp16 (|v| >= 65520); see check_obs_range
            self.obs_overflow = torch.zeros(1, dtype=torch.int32, device=dev)
            self.ob_seg = ops.segment_table(self.onehot_nvec, dev) if self.onehot_nvec else None
        # where the heads write d(loss)/d(latent pre-activation)
        if self.fcs:
            self.dlatent, self.ld_dlatent = self.dzfc[-1], self.fcs[-1].Np
        elif self.convs:
            self.dlatent, self.ld_dlatent = self.dzconv[-1], self.flat

    # ---- shift-GEMM conv stack ---------------------------------------------------------------------------------
    def _materialize_shift(self, f16):
        cap, cv = self.cap, self.convs
        self.sg = []                                   # per layer: dict(Hg, Wg, Cg, k, s, kx, shifts, yshifts)
        for c, lp in zip(cv, self.plan.layers):
            s_, k = c.stride, c.rf // c.stride
            Hg, Wg, Cg = c.H // s_, c.W // s_, c.C * s_ * s_
            # x-fold (weight gradient): the kx horizontally adjacent taps of a filter row are walked as taps shifted by
            # one more grid row each, from the filter row's shift in yshifts
            self.sg.append(dict(Hg=Hg, Wg=Wg, Cg=Cg, k=k, s=s_, kx=lp.kx,
                                shifts=[a * Wg + b for a in range(k) for b in range(k)],
                                yshifts=[a * Wg for a in range(k)]))
        g0 = self.sg[0]
        # first layer straight from the uint8 images (producer warps gather + cast + space-to-depth in smem)
        self.fused_u8 = self.plan.fused_u8
        self.x16 = None if self.fused_u8 else torch.empty(cap, g0["Hg"] * g0["Wg"] * g0["Cg"], **f16)
        # activations: layer i's output is stored space-to-depth'ed for layer i+1 (compact after the last conv)
        self.hconv = [torch.empty(cap, c.OH * c.OW * c.nf, **f16) for c in cv]
        # 1 bit per element "activation > 0" of every conv output: the ReLU mask of the next layer's data gradient (the
        # last conv's serves the fc1 data gradient)
        self.hbits = [torch.zeros(cap * (c.OH * c.OW * c.nf // 16), dtype=torch.int16, device=self.hconv[i].device)
                      for i, c in enumerate(cv)]
        # gradients w.r.t. conv outputs live zero-bordered on the conv's INPUT grid
        self.dY = [torch.zeros(cap, g["Hg"] * g["Wg"] * c.nf, **f16) for c, g in zip(cv, self.sg)]
        # data-gradient weight operands [N' = Cg, taps * nf] (tap blocks of the master weight side by side)
        self.wd = [None] + [torch.zeros(g["Cg"], g["k"] * g["k"] * c.nf, **f16) for c, g in zip(cv[1:], self.sg[1:])]
        self.flat = cv[-1].OH * cv[-1].OW * cv[-1].nf

    def _forward_shift(self, x, B, src_idx, masks=True):
        cv, sg = self.convs, self.sg
        c0 = cv[0]
        if self.fused_u8:
            self._u8 = (x, src_idx, c0.H, c0.W, c0.C, c0.stride)
            cur = None
        else:
            self._u8 = None
            ops.s2d_gather(x, self.x16, B, c0.H, c0.W, c0.C, c0.stride, src_idx=src_idx)
            cur = self.x16
        for i, (c, g) in enumerate(zip(cv, sg)):
            if i + 1 < len(cv) and cv[i + 1].stride > 1:
                sn = cv[i + 1].stride
                Hn, Wn, Cn = c.OH // sn, c.OW // sn, c.nf * sn * sn
                omap = (2, Hn * Wn * Cn, Wn * Cn, Cn, c.nf, sn)
            else:
                omap = (0, c.OH * c.OW * c.nf, c.OW * c.nf, c.nf, 0, 0)
            ops.conv_shift_fwd(cur, B, g["Hg"], g["Wg"], g["Cg"], c.w_fwd, c.Kp, c.nf, g["shifts"], c.OH, c.OW,
                               self.hconv[i], omap, bias=c.b, act=c.act, tag="fwd." + c.name,
                               u8=self._u8 if i == 0 else None, bits_out=self.hbits[i] if masks else None,
                               useful_rows=B * c.OH * c.OW)
            cur = self.hconv[i]
        return cur, self.flat

    def _backward_shift(self, B, alpha):
        """self.dY[-1] holds d loss / d (last conv pre-activation) on its grid (written by the fc dgrad)."""
        cv, sg = self.convs, self.sg
        for i in reversed(range(len(cv))):
            c, g = cv[i], sg[i]
            rows = B * g["Hg"] * g["Wg"]
            xin = self.x16 if i == 0 else self.hconv[i - 1]
            ops.conv_shift_wgrad(xin, rows, g["Cg"], self.dY[i], c.nf, g["yshifts"] if g["kx"] > 1 else g["shifts"],
                                 c.gw, c.nf, alpha=alpha * c.in_scale, tag="wgrad." + c.name, gbias=c.gb,
                                 alpha_b=alpha, u8=self._u8 if i == 0 else None, useful_rows=B * c.OH * c.OW,
                                 kx=g["kx"])
            if i == 0:
                break
            # dX_i (= dY_{i-1} after the ReLU mask) as a shift-GEMM over dY_i with negative shifts
            cp, gp = cv[i - 1], sg[i - 1]
            omap = (1, gp["Hg"] * gp["Wg"] * cp.nf, gp["Wg"] * cp.nf, cp.nf, cp.nf, g["s"])
            smap = (0, g["Hg"] * g["Wg"] * g["Cg"], g["Wg"] * g["Cg"], g["Cg"], 0, 0)
            ops.conv_shift_fwd(self.dY[i], B, g["Hg"], g["Wg"], c.nf, self.wd[i], g["k"] * g["k"] * c.nf, g["Cg"],
                               [-sft for sft in g["shifts"]], g["Hg"], g["Wg"], self.dY[i - 1], omap,
                               smap=smap, act=ops.ACT_RELU, dact=True, tag="dgrad." + c.name,
                               saved_bits=self.hbits[i - 1], useful_rows=B * c.OH * c.OW)

    def cast_jobs(self):
        """The casts of the tower's fp16 operands: its layers', the shift-GEMM data-gradient tap blocks wd, the LSTM's.
        They read the operand tensors as they are when called."""
        jobs = [j for l in self.layers for j in l.cast_jobs()]
        if self.convs and self.shift_mode:
            for c, g, wd in zip(self.convs[1:], self.sg[1:], self.wd[1:]):
                taps, Cg, nf = g["k"] * g["k"], g["Cg"], c.nf
                # wd[:, t*nf:(t+1)*nf] = fp16(W[t*Cg:(t+1)*Cg, :])
                jobs += [ops.CastJob(c.w[t * Cg:(t + 1) * Cg], Cg, nf, wd[:, t * nf:], taps * nf, None, 0, 1.0)
                         for t in range(taps)]
        if self.lstm is not None:
            jobs += self.lstm.cast_jobs()
        return jobs

    def operand_launches(self):
        """The convs' operand kernels that are not casts (Conv.operand_launches)."""
        return [f for c in self.convs for f in c.operand_launches()]

    def refresh(self):
        """Eager operand refresh: the launches a network's refresh makes for this tower, with one launch per cast."""
        for f in self.operand_launches():
            f()
        for j in self.cast_jobs():
            ops.cast_transpose(*j)

    # x: uint8 [*,H,W,C] images (cnn) or fp16 [*, in_pad] rows (mlp); src_idx gathers samples from it
    def encode(self, x, B, src_idx=None):
        """mlp: float32 rows (optionally gathered through src_idx) -> encoded fp16 [hi | lo] operand rows in x0."""
        nm = self.obs_norm
        ops.obs_encode(x, self.x0, B, self.raw_dim, self.in_dim, self.in_pad, src_idx=src_idx,
                       mean=nm[0] if nm else None, inv_std=nm[1] if nm else None,
                       clip=(nm[2], nm[3]) if nm else (0.0, 0.0), onehot_n=self.onehot_n, seg_off=self.ob_seg,
                       overflow=self.obs_overflow)
        return self.x0

    def check_obs_range(self, flag=None):
        """Raise ValueError when an encoded observation value was beyond fp16 since the last check: its hi/lo pair is
        +-inf and the network output NaN.  Reads the device flag (a synchronisation) unless the caller passes a host
        copy of it; clears the flag before raising."""
        if self.base != "mlp":
            return
        if flag is None:
            flag = int(self.obs_overflow.item())
        if flag:
            self.obs_overflow.zero_()
            raise ValueError("observation values must satisfy |v| < 65520 after normalisation: the encoder splits "
                             "each float32 value into two fp16 halves, and fp16 ends at 65504")

    def forward(self, x, B, src_idx=None, encoded=None, masks=True, skip_first=False, seq=None):
        """encoded (mlp only): operand rows another tower already produced from the same observations.
        masks=False (acting passes: no backward follows): the convs skip their 1-bit ReLU mask output, the LSTM its
        saved gates.  skip_first (mlp only): hfc[0] was already produced by a fused first layer (common/policies.py).
        seq (lstm, cnn_lstm): how the B rows form sequences (Seq, seq.T * seq.B == B)."""
        assert B <= self.cap
        if self.convs and self.shift_mode:
            h, ldh = self._forward_shift(x, B, src_idx, masks)
        elif self.convs:
            cur = x
            for i, c in enumerate(self.convs):
                if c.implicit:
                    if i == 0 and self.in_u8:
                        # fused minibatch gather + uint8->fp16 cast (models.py:19, ppo2.py:165): 84 B/elem of traffic
                        if c.s2d:
                            ops.s2d_gather(cur, self.x16, B, c.H, c.W, c.C, c.stride, src_idx=src_idx)
                        else:
                            n_el = c.H * c.W * c.C
                            ops.im2col(cur, self.x16, B, 1, 1, n_el, 1, 1, False, src_idx=src_idx, tag="gather_cast")
                        cur = self.x16
                    elif i == 0 and src_idx is not None:
                        raise NotImplementedError("gather of fp16 image inputs")
                    c.fwd_implicit(cur, B, self.hconv[i])
                else:
                    c.im2col(cur, self.cols[i], B, src_idx=src_idx if i == 0 else None)
                    c.forward(self.cols[i], c.K, B * c.P, self.hconv[i], c.nf)
                cur = self.hconv[i]
            self._conv_in0 = self.x16 if (self.convs[0].implicit and self.in_u8) else x
            h, ldh = cur, self.flat                      # [B, OH*OW*C] view of the NHWC activation (H,W,C order)
        else:
            # float32 rows (optionally gathered through src_idx) -> encoded fp16 [hi | lo] operand rows
            if encoded is None:
                encoded = self.encode(x, B, src_idx)
            h, ldh = encoded, 2 * self.in_pad
            self._mlp_in = h
        for i, l in enumerate(self.fcs):
            if not (skip_first and i == 0):
                linear_ln_forward(l, self.lns[i], h, ldh, B, self.hfc[i], self.ld_hfc[i])
            h, ldh = self.hfc[i], self.ld_hfc[i]
        if self.lstm is not None:
            assert seq is not None and seq.T * seq.B == B, "recurrent towers take their rows as sequences"
            h, ldh = self.lstm.forward(h, ldh, seq, train=masks)
        return h, ldh                                    # latent [B, latent_dim] fp16, row pitch ldh

    # consumes self.dlatent: fp16 [B, ld_dlatent] gradient w.r.t. the latent PRE-activation (with a norm: w.r.t. the
    # normalised, scaled and shifted value the activation reads)
    def backward(self, B, alpha, skip_first_wgrad=False):
        """skip_first_wgrad (mlp): the caller computes the first layer's weight gradient (fused over two towers)."""
        nfc = len(self.fcs)
        dz, lddz = self.dlatent, self.ld_dlatent
        if self.lstm is not None:
            if not self.fcs:                            # lstm: the input is the encoded observation
                self.lstm.backward(alpha)
                return
            l = self.fcs[-1]                            # cnn_lstm: dx is fc1's output gradient through its ReLU
            self.lstm.backward(alpha, dx=self.dzfc[-1], ldo=self.ld_hfc[-1], saved=self.hfc[-1],
                               ld_saved=self.ld_hfc[-1], act=l.act)
            dz, lddz = self.dzfc[-1], self.ld_hfc[-1]
        for i in reversed(range(nfc)):
            l = self.fcs[i]
            if self.lns[i] is not None:
                self.lns[i].backward(B, dz, lddz, alpha)
            if i == 0 and skip_first_wgrad and not self.convs:
                return
            if i > 0:
                xin, ldx, act_in = self.hfc[i - 1], self.ld_hfc[i - 1], self.fcs[i - 1].act
            elif self.convs:
                xin, ldx, act_in = self.hconv[-1], self.flat, ops.ACT_RELU
            else:
                xin, ldx, act_in = self._mlp_in, 2 * self.in_pad, None
            l.wgrad(xin, ldx, dz, lddz, B, alpha)
            if act_in is None:
                return
            if i > 0:
                out, ldo = self.dzfc[i - 1], self.ld_hfc[i - 1]
                l.dgrad(dz, lddz, B, out, ldo, saved=xin, ld_saved=ldx, act=act_in)
            elif self.shift_mode:
                cL, gL = self.convs[-1], self.sg[-1]
                out, ldo = self.dY[-1], gL["Hg"] * gL["Wg"] * cL.nf      # scatter into the zero-bordered grid
                l.dgrad(dz, lddz, B, out, ldo, saved=xin, ld_saved=ldx, act=act_in, remap=(cL.nf, cL.OW, gL["Wg"]),
                        saved_bits=self.hbits[-1])
            else:
                out, ldo = self.dzconv[-1], self.flat
                l.dgrad(dz, lddz, B, out, ldo, saved=xin, ld_saved=ldx, act=act_in)
            dz, lddz = out, ldo
        if self.convs and self.shift_mode:
            self._backward_shift(B, alpha)
            return
        for i in reversed(range(len(self.convs))):
            c = self.convs[i]
            dzc = self.dzconv[i]
            if c.implicit:
                c.wgrad_implicit(self._conv_in0 if i == 0 else self.hconv[i - 1], dzc, B, alpha)
            else:
                c.wgrad(self.cols[i], c.K, dzc, c.nf, B * c.P, alpha)
            if i == 0:
                break
            if c.implicit_dgrad:
                c.dgrad_implicit(dzc, B, self.hconv[i - 1], self.dzconv[i - 1], ops.ACT_RELU)
            else:
                if self.dcols[i] is None:
                    raise RuntimeError("explicit dgrad workspace missing")
                c.dgrad(dzc, c.nf, B * c.P, self.dcols[i], c.K)
                c.col2im(self.dcols[i], self.hconv[i - 1], self.dzconv[i - 1], B, act=ops.ACT_RELU)


class Optimizer:
    """Global-norm clip + TF-Adam on the flat buffers (ppo2/model.py:100-114), or per-variable
    clip_by_norm (deepq/build_graph.py:416-421).  No host synchronisation."""

    def __init__(self, store, eps, max_grad_norm=None, per_variable=False, beta1=0.9, beta2=0.999):
        self.store, self.eps, self.clip, self.per_variable = store, eps, max_grad_norm, per_variable
        self.beta1, self.beta2, self.t = beta1, beta2, 0
        nseg = len(store._specs) if per_variable else 1
        self.nseg = nseg
        self.sumsq = torch.zeros(nseg, dtype=torch.float64, device=store.device)
        self.seg_off = torch.from_numpy(store.segment_offsets()).to(store.device) if per_variable else None
        self.lr_dev = torch.zeros(1, dtype=torch.float32, device=store.device)    # lr_t of the current step

    def begin_step(self, lr):
        """Host half of a step: advance t and hand the bias-corrected step size lr*sqrt(1-b2^t)/(1-b1^t)
        (mpi_adam.py:37) to the device.  Separate from `apply` so that `apply` is a fixed launch sequence."""
        self.t += 1
        lr_t = lr * math.sqrt(1.0 - self.beta2 ** self.t) / (1.0 - self.beta1 ** self.t)
        ops.set_scalars(self.lr_dev, lr_t)
        return lr_t

    def apply(self, clip=True):
        """Device half: norm(s) + clip + Adam, reading the step size written by begin_step."""
        s = self.store
        clip = self.clip if (self.clip is not None and clip) else 0.0
        if clip > 0:
            if self.per_variable:
                ops.seg_sumsq(s.grads, self.seg_off, self.nseg, self.sumsq)
            else:
                ops.sumsq(s.grads, self.sumsq)
        ops.clip_adam(s.params, s.grads, s.m, s.v, 0.0, self.beta1, self.beta2, self.eps, clip,
                      self.sumsq if clip > 0 else None, self.seg_off if (clip > 0 and self.per_variable) else None,
                      self.nseg if self.per_variable else 0, lr_t_dev=self.lr_dev)

    def step(self, lr, clip=True):
        """clip=False: the gradient buffer already holds clipped gradients (MicrobatchedModel)."""
        self.begin_step(lr)
        self.apply(clip)
