"""float64 references for layer normalisation (tf.contrib.layers.layer_norm(center=True, scale=True) after a fully
connected layer: common/models.py:97-98, deepq/models.py:24-25,34-35) and for the networks that use it.

Ordinary numpy / torch-CPU arithmetic; nothing here calls a kernel of the project.  The network references build on
oracle/nets.py: its PPO2Oracle and DQNOracle run unchanged while `nets.mlp` / `nets.q_forward` are swapped for the
versions below, which normalise wherever the parameter dict holds LayerNorm variables and are the originals where it
does not.
"""
import contextlib
import math
from collections import OrderedDict

import numpy as np
import torch

from oracle import nets

EPS = 1e-12                 # tf.contrib.layers.layer_norm's variance_epsilon (baselines_b200.nn.LN_EPS)
ACTS = {0: lambda v: v, 1: lambda v: np.maximum(v, 0.0), 2: np.tanh}


def ln_scope(k):
    return "LayerNorm" if k == 0 else f"LayerNorm_{k}"


# ---------------------------------------------------------------------------------------------- one layer, numpy
def ln_forward(z, gamma, beta, act=0, eps=EPS):
    """-> (y, u, xhat, rstd) in float64: biased variance over each row (tf.nn.moments)."""
    z, gamma, beta = (np.asarray(a, np.float64) for a in (z, gamma, beta))
    mean = z.mean(axis=1, keepdims=True)
    var = ((z - mean) ** 2).mean(axis=1, keepdims=True)
    rstd = 1.0 / np.sqrt(var + eps)
    xhat = (z - mean) * rstd
    u = gamma * xhat + beta
    return ACTS[act](u), u, xhat, rstd


def ln_forward_one_pass(z, gamma, beta, act=0, eps=EPS):
    """The plausible mistake: var = E[x^2] - E[x]^2 in float32, which cancels for rows with a large mean."""
    z = np.asarray(z, np.float32)
    mean = z.mean(axis=1, keepdims=True, dtype=np.float32)
    var = np.maximum((z * z).mean(axis=1, keepdims=True, dtype=np.float32) - mean * mean, np.float32(0))
    xhat = (z - mean).astype(np.float64) / np.sqrt(var.astype(np.float64) + eps)
    return ACTS[act](np.asarray(gamma, np.float64) * xhat + np.asarray(beta, np.float64))


def ln_backward(du, z, gamma, eps=EPS):
    """du = d loss / d u  ->  (dz, dgamma, dbeta) in float64."""
    du, gamma = np.asarray(du, np.float64), np.asarray(gamma, np.float64)
    _, _, xhat, rstd = ln_forward(z, gamma, np.zeros_like(gamma), 0, eps)
    g = gamma * du
    dz = rstd * (g - g.mean(axis=1, keepdims=True) - xhat * (g * xhat).mean(axis=1, keepdims=True))
    return dz, (du * xhat).sum(axis=0), du.sum(axis=0)


def ln_forward_loops(z, gamma, beta, eps=EPS):
    """The definition, element by element (python floats are float64)."""
    rows, N = np.shape(z)
    u = np.zeros((rows, N))
    for r in range(rows):
        mean = sum(float(z[r][c]) for c in range(N)) / N
        var = sum((float(z[r][c]) - mean) ** 2 for c in range(N)) / N
        for c in range(N):
            u[r, c] = float(gamma[c]) * (float(z[r][c]) - mean) / math.sqrt(var + eps) + float(beta[c])
    return u


def dbeta_in_kernel_order(du16, alpha, lanes_per_row):
    """dbeta of csrc/layer_norm.cu bit for bit, from the fp16 du: float32 sums over each 128-row slice by lane group
    (group t of 256 / lanes_per_row takes rows t, t + groups, ... in order), the groups in order, times alpha; then
    sum_partials (csrc/gemm_wgmma.cu): slice p goes to accumulator p % 8, the 8 accumulators are added in order."""
    du = np.asarray(du16, np.float16).astype(np.float32)
    rows, N = du.shape
    groups = 256 // lanes_per_row
    parts = []
    for r0 in range(0, rows, 128):
        sl = du[r0:r0 + 128]
        s = np.zeros(N, np.float32)
        for t in range(groups):
            a = np.zeros(N, np.float32)
            for r in range(t, sl.shape[0], groups):
                a = a + sl[r]
            s = s + a
        parts.append(np.float32(alpha) * s)
    acc = [np.zeros(N, np.float32) for _ in range(8)]
    for p, v in enumerate(parts):
        acc[p % 8] = acc[p % 8] + v
    out = np.zeros(N, np.float32)
    for a in acc:
        out = out + a
    return out


# ---------------------------------------------------------------------------------------------- networks, torch
def ln_torch(z, gamma, beta, eps=EPS):
    mean = z.mean(dim=1, keepdim=True)
    var = ((z - mean) ** 2).mean(dim=1, keepdim=True)
    return gamma * ((z - mean) / torch.sqrt(var + eps)) + beta


def _maybe_ln(tp, scope, z):
    if f"{scope}/gamma:0" in tp:
        return ln_torch(z, tp[f"{scope}/gamma:0"], tp[f"{scope}/beta:0"])
    return z


_MLP, _Q_FORWARD = nets.mlp, nets.q_forward


def mlp(tp, prefix, obs, num_layers=2):
    """models.py:93-101 with layer_norm: fc -> layer_norm -> tanh."""
    dtype = tp[f"{prefix}/mlp_fc0/w:0"].dtype
    h = obs.to(dtype).reshape(obs.shape[0], -1)
    for i in range(num_layers):
        z = h @ tp[f"{prefix}/mlp_fc{i}/w:0"] + tp[f"{prefix}/mlp_fc{i}/b:0"]
        h = torch.tanh(_maybe_ln(tp, f"{prefix}/{ln_scope(i)}", z))
    return h


def q_forward(tp, network, obs, scope, n_hidden=1, dueling=True):
    """deepq/models.py:10-43 with layer_norm in the streams; the trunks are oracle/nets.py's."""
    if network == "cnn":
        lat = nets.nature_cnn(tp, scope, obs)
    elif network == "mlp":
        lat = _MLP(tp, scope, obs)
    else:                                                           # conv_only, models.py:221-249
        h = obs.to(tp[f"{scope}/convnet/Conv/weights:0"].dtype) / 255.0
        for i, (_n, _nf, _rf, stride) in enumerate(nets.NATURE_CONVS):
            nm = "Conv" if i == 0 else f"Conv_{i}"
            h = torch.relu(nets._conv_nhwc(h, tp[f"{scope}/convnet/{nm}/weights:0"],
                                           tp[f"{scope}/convnet/{nm}/biases:0"], stride, pad="SAME"))
        lat = h.reshape(h.shape[0], -1)

    def stream(sname):
        x = lat
        for j in range(n_hidden):
            z = x @ tp[f"{scope}/{sname}/{nets._fc_name(j)}/weights:0"] + tp[f"{scope}/{sname}/{nets._fc_name(j)}/biases:0"]
            x = torch.relu(_maybe_ln(tp, f"{scope}/{sname}/{ln_scope(j)}", z))
        return x @ tp[f"{scope}/{sname}/{nets._fc_name(n_hidden)}/weights:0"] \
            + tp[f"{scope}/{sname}/{nets._fc_name(n_hidden)}/biases:0"]

    a = stream("action_value")
    if not dueling:
        return a
    return stream("state_value") + (a - a.mean(dim=1, keepdim=True))


@contextlib.contextmanager
def layer_norm_nets():
    """oracle/nets.py with its mlp and q_forward replaced by the layer-normalised ones above."""
    nets.mlp, nets.q_forward = mlp, q_forward
    try:
        yield
    finally:
        nets.mlp, nets.q_forward = _MLP, _Q_FORWARD


def with_policy_norms(params, scope="ppo2_model", num_layers=2):
    """init_policy_params' dict with beta (zeros) and gamma (ones) after every mlp_fc{i}/b, in creation order."""
    out = OrderedDict()
    for k, v in params.items():
        out[k] = v
        for i in range(num_layers):
            for tower in ("pi", "vf"):
                if k == f"{scope}/{tower}/mlp_fc{i}/b:0":
                    out[f"{scope}/{tower}/{ln_scope(i)}/beta:0"] = np.zeros(v.shape, np.float32)
                    out[f"{scope}/{tower}/{ln_scope(i)}/gamma:0"] = np.ones(v.shape, np.float32)
    return out


def with_q_norms(params, n_hidden=1, scope="deepq/q_func"):
    """init_q_params' dict with the norms of the streams' hidden layers (not of the trunk: build_q_func consumes
    layer_norm, deepq/models.py:5)."""
    out = OrderedDict()
    for k, v in params.items():
        out[k] = v
        for sname in ("action_value", "state_value"):
            for j in range(n_hidden):
                if k == f"{scope}/{sname}/{nets._fc_name(j)}/biases:0":
                    out[f"{scope}/{sname}/{ln_scope(j)}/beta:0"] = np.zeros(v.shape, np.float32)
                    out[f"{scope}/{sname}/{ln_scope(j)}/gamma:0"] = np.ones(v.shape, np.float32)
    return out


def randomise_norms(params, rng):
    """gamma = 1, beta = 0 would leave a network blind to both (and to a norm credited to its neighbour): gamma drawn
    from U(0.5, 1.5), beta from N(0, 0.3^2), in place and in key order, as float32."""
    for k in params:
        if k.endswith("gamma:0"):
            params[k] = rng.uniform(0.5, 1.5, np.shape(params[k])).astype(np.float32)
        elif k.endswith("beta:0") and "LayerNorm" in k:
            params[k] = (rng.randn(*np.shape(params[k])) * 0.3).astype(np.float32)
    return params


# ---------------------------------------------------------------------------------------------- parameter-space noise
class ParamNoiseState:
    """The act-call state machine of deepq/build_graph.py:290-313 in float32: sticky eps and threshold, and the scale
    that grows by 1.01 when the measured mean_kl is under the threshold and shrinks by 1.01 otherwise.  The order inside
    a call is the one baselines_b200 fixes: eps and threshold first, then the reset perturbation (with the scale before
    this call's update), then the scale update."""

    def __init__(self):
        self.eps, self.scale, self.threshold = np.float32(0.0), np.float32(0.01), np.float32(0.05)
        self.reset_scale = None                  # the scale the last reset perturbed with

    def call(self, mean_kl, reset=False, update_param_noise_threshold=False, update_param_noise_scale=False,
             update_eps=-1):
        if update_eps >= 0:
            self.eps = np.float32(update_eps)
        if update_param_noise_threshold >= 0:                       # False == 0.0 replaces it too, as in the reference
            self.threshold = np.float32(update_param_noise_threshold)
        if reset:
            self.reset_scale = self.scale
        if update_param_noise_scale:
            up = np.float32(mean_kl) < self.threshold
            self.scale = np.float32(self.scale * np.float32(1.01)) if up else np.float32(self.scale / np.float32(1.01))


def mean_kl(q, q_adapt):
    """build_graph.py:279-280 in float64: mean over rows of sum_a softmax(q) (log softmax(q) - log softmax(q_adapt))."""
    def logsm(v):
        v = np.asarray(v, np.float64)
        v = v - v.max(axis=1, keepdims=True)
        return v - np.log(np.exp(v).sum(axis=1, keepdims=True))
    lp, lr = logsm(q), logsm(q_adapt)
    return float((np.exp(lp) * (lp - lr)).sum(axis=1).mean())


def philox_normals(seed, offset, idx):
    """Normal number e (for e in idx) of a parameter perturbation at stream position `offset`, in float64 from the
    device's float32 uniforms: Box-Muller over words (2p, 2p + 1), p = (e & 3) >> 1, of Philox block e >> 2; cos for
    even e, sin for odd e (csrc/param_noise.cu)."""
    from _loss_refs import philox4x32_10
    idx = np.asarray(idx, np.int64)
    w = philox4x32_10(seed, idx >> 2, 0, offset)
    u = ((w >> 8).astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -24)
    p = (idx & 3) >> 1
    u1 = u[np.arange(len(idx)), 2 * p].astype(np.float64)
    u2 = u[np.arange(len(idx)), 2 * p + 1].astype(np.float64)
    r = np.sqrt(-2.0 * np.log(u1))
    return np.where(idx & 1, r * np.sin(2 * np.pi * u2), r * np.cos(2 * np.pi * u2))
