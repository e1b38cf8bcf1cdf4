"""GPU: whole PPO2 and DQN updates, every parameter's gradient and Adam step, against the float64 network mirror.

The kernels of an update are tested one family at a time elsewhere (GEMM / conv boundaries, conv paths, loss heads,
optimiser).  This file tests the layer that composes them: PolicyNet (fused [pi | vf] head and its TF column slices,
value_network='copy', the fused first mlp layer with its shared w0cat / b0cat / h0cat / dz0cat and the g0cat split,
the frozen identity head), nn.Tower (hi/lo first layer, tanh, depth, padded widths), QNet (dueling streams, the
K-concatenated data gradient into the trunk, cat_off padding, hidden layers) and the Optimizer wiring (lr_t and t,
global vs per-variable clip, the operand refresh after the step, inside a captured graph).

Each configuration builds the real Model / DQNModel and runs three minibatches through the public path (train_rollout
eagerly and graph-captured with src_idx; train_device without and with replay idx), checking after each one:
  a. the fp16 head-gradient rows the head GEMMs consume equal the float64 loss gradient (tests/_loss_refs.py) at the
     kernels' own head outputs, within one fp16 rounding (+1e-6), rows at a branch boundary excluded;
  b. every TF variable's gradient equals the mirror (tests/_net_refs.py, kernel rounding on) seeded with those rows,
     ReLU decisions taken from the kernels' stored activations: |got - ref| <= g * S + 2^-23 |ref|, S the mirror's
     absolute network, g per tensor.  Each bound must reject "one sample dropped" (the row with the largest gradient
     of each head) and a composition mistake named for the configuration;
  c. params / m / v after the step equal float64 TF-Adam applied to the exported pre-step state and the kernels' own
     gradients (global clip for PPO2, per-variable for DQN), within 16 fp32 roundings; the bound rejects lr_t of step
     t + 1 and, where clipping is active, the clip factor left out.  The frozen identity block stays bit-for-bit;
  d. later minibatches' gradients equal the mirror at the parameters the step before wrote.  On the graph paths the
     first call with a launch sequence runs eagerly (graphs.GraphCache), the second is captured and replayed, the
     third replays: the third step's forward reads the fp16 operands the replayed refresh() of the second wrote, so
     an operand copy (w0cat, b0cat, w_cat_bwd, wdg, the shift-GEMM wd) that goes stale under replay fails here;
  e. a NatureCNN update gathered through src_idx in three uneven chunks: each chunk's rows are bit-identical to the
     unchunked run's, and the accumulated gradient meets (b) against the same reference.

Tolerances: every g is 3.5x the maximum observed on an H100 80GB HBM3 (700 W power limit), floor 1e-8; the observed
values are listed next to the constants.  Each run prints its own [observed] lines.
"""
import math

import numpy as np
import pytest
import torch

import _loss_refs as lr
import _net_refs as N
import _refs as R
from baselines_b200 import _lib
from test_update_path_gpu import G_DLOGSTD, G_STATS, _gauss_nscale, _stats_check, _within_f16

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
U32 = 2.0 ** -24
ADAM_G = 16 * U32                  # as test_update_path_gpu.py::test_clip_adam_three_step_trajectory_vs_float64_tf_adam
G_MASK = 1e-6                      # |pre| / S where a kernel ReLU decision may differ from float64

# g per configuration and TF variable (short names): 3.5x the maximum observed on an H100 80GB HBM3 (700 W power
# limit) over two to seven runs, each with the eager and graph paths and every step (and the chunked run of
# cnn84_cat6_shared), floor 1e-8.  The observed value of a tensor varies between runs by up to ~10x: it is set by
# whether some stored fp16 data gradient lands on the other side of a rounding tie than its float64 value, and the
# second step starts from parameters that differ between runs in the last bits (split-K fp32 atomics).
_OBSERVED = {
    "cnn84_cat6_shared": {"pi/c1/w": 5.57e-08, "pi/c1/b": 2.32e-08, "pi/c2/w": 3.47e-07, "pi/c2/b": 9.00e-07,
                          "pi/c3/w": 3.51e-07, "pi/c3/b": 1.36e-06, "pi/fc1/w": 1.23e-06, "pi/fc1/b": 9.17e-05,
                          "pi/w": 6.45e-09, "pi/b": 1.24e-08, "vf/w": 6.45e-09, "vf/b": 2.29e-09},
    "cnn84_cat6_copy": {"pi/c1/w": 1.34e-07, "pi/c1/b": 6.21e-08, "pi/c2/w": 4.82e-07, "pi/c2/b": 1.09e-07,
                        "pi/c3/w": 2.59e-07, "pi/c3/b": 1.39e-07, "pi/fc1/w": 1.18e-06, "pi/fc1/b": 3.91e-06,
                        "vf/c1/w": 2.48e-07, "vf/c1/b": 1.29e-07, "vf/c2/w": 2.96e-07, "vf/c2/b": 2.35e-07,
                        "vf/c3/w": 1.40e-07, "vf/c3/b": 1.13e-06, "vf/fc1/w": 1.17e-06, "vf/fc1/b": 5.08e-08,
                        "pi/w": 6.12e-09, "pi/b": 8.53e-09, "vf/w": 4.50e-09, "vf/b": 8.06e-10},
    "cnn64_cat6_shared": {"pi/c1/w": 2.88e-08, "pi/c1/b": 1.38e-08, "pi/c2/w": 9.80e-07, "pi/c2/b": 1.01e-06,
                          "pi/c3/w": 6.46e-07, "pi/c3/b": 2.33e-06, "pi/fc1/w": 1.18e-06, "pi/fc1/b": 8.88e-06,
                          "pi/w": 1.05e-08, "pi/b": 1.77e-08, "vf/w": 1.19e-08, "vf/b": 3.72e-10},
    "mlp376_gauss17_copy_h64": {"pi/mlp_fc0/w": 2.17e-05, "pi/mlp_fc0/b": 6.72e-06, "pi/mlp_fc1/w": 2.34e-05,
                                "pi/mlp_fc1/b": 1.74e-05, "vf/mlp_fc0/w": 9.55e-05, "vf/mlp_fc0/b": 2.90e-05,
                                "vf/mlp_fc1/w": 2.39e-05, "vf/mlp_fc1/b": 1.87e-05, "pi/w": 4.12e-05, "pi/b": 7.49e-09,
                                "vf/w": 1.10e-05, "vf/b": 8.69e-11},
    "mlp11_gauss3_copy_h256": {"pi/mlp_fc0/w": 4.47e-06, "pi/mlp_fc0/b": 2.08e-06, "pi/mlp_fc1/w": 4.71e-05,
                               "pi/mlp_fc1/b": 1.98e-05, "vf/mlp_fc0/w": 1.11e-05, "vf/mlp_fc0/b": 3.78e-06,
                               "vf/mlp_fc1/w": 4.03e-05, "vf/mlp_fc1/b": 1.89e-05, "pi/w": 2.40e-05, "pi/b": 2.66e-09,
                               "vf/w": 1.31e-05, "vf/b": 0.00e+00},
    "mlp11_gauss3_copy_l1_h32": {"pi/mlp_fc0/w": 6.21e-05, "pi/mlp_fc0/b": 1.55e-05, "vf/mlp_fc0/w": 1.65e-06,
                                 "vf/mlp_fc0/b": 7.75e-07, "pi/w": 8.11e-06, "pi/b": 4.25e-09, "vf/w": 5.38e-07,
                                 "vf/b": 1.50e-09},
    "mlp13_cat15_l3_h20": {"pi/mlp_fc0/w": 5.46e-06, "pi/mlp_fc0/b": 1.65e-06, "pi/mlp_fc1/w": 5.26e-06,
                           "pi/mlp_fc1/b": 4.22e-06, "pi/mlp_fc2/w": 1.07e-05, "pi/mlp_fc2/b": 7.14e-06,
                           "pi/w": 3.98e-05, "pi/b": 1.76e-08, "vf/w": 5.28e-06, "vf/b": 5.27e-10},
    "mlp_disc10_cat4": {"pi/mlp_fc0/w": 1.73e-05, "pi/mlp_fc0/b": 1.52e-06, "pi/mlp_fc1/w": 1.63e-05,
                        "pi/mlp_fc1/b": 5.23e-06, "pi/w": 1.06e-06, "pi/b": 6.45e-09, "vf/w": 7.81e-07,
                        "vf/b": 1.39e-09},
    "mlp_mdisc33_mcat33": {"pi/mlp_fc0/w": 9.22e-06, "pi/mlp_fc0/b": 2.64e-06, "pi/mlp_fc1/w": 8.09e-06,
                           "pi/mlp_fc1/b": 3.57e-06, "pi/w": 2.15e-05, "pi/b": 8.90e-09, "vf/w": 8.72e-06,
                           "vf/b": 1.23e-09},
    "mlp5_gauss32_copy_identity": {"pi/mlp_fc0/w": 1.66e-05, "pi/mlp_fc0/b": 6.75e-06, "pi/mlp_fc1/w": 2.96e-05,
                                   "pi/mlp_fc1/b": 1.86e-05, "vf/mlp_fc0/w": 4.57e-06, "vf/mlp_fc0/b": 1.06e-06,
                                   "vf/mlp_fc1/w": 3.34e-06, "vf/mlp_fc1/b": 1.98e-06, "vf/w": 2.49e-06,
                                   "vf/b": 0.00e+00},
    "mlp11_bern5_normalized": {"pi/mlp_fc0/w": 1.17e-05, "pi/mlp_fc0/b": 4.56e-06, "pi/mlp_fc1/w": 1.99e-05,
                               "pi/mlp_fc1/b": 8.99e-06, "pi/w": 4.95e-06, "pi/b": 5.21e-09, "vf/w": 6.59e-06,
                               "vf/b": 7.11e-10},
    "mlp_dueling_h64_32_double": {"mlp_fc0/w": 1.39e-07, "mlp_fc0/b": 7.51e-08, "mlp_fc1/w": 1.09e-06,
                                  "mlp_fc1/b": 5.76e-07, "action_value/fully_connected/weights": 2.27e-06,
                                  "action_value/fully_connected/biases": 5.82e-07,
                                  "action_value/fully_connected_1/weights": 9.81e-06,
                                  "action_value/fully_connected_1/biases": 3.39e-09,
                                  "action_value/fully_connected_2/weights": 5.31e-06,
                                  "action_value/fully_connected_2/biases": 4.54e-09,
                                  "state_value/fully_connected/weights": 5.87e-06,
                                  "state_value/fully_connected/biases": 3.15e-06,
                                  "state_value/fully_connected_1/weights": 1.78e-05,
                                  "state_value/fully_connected_1/biases": 9.07e-09,
                                  "state_value/fully_connected_2/weights": 5.12e-07,
                                  "state_value/fully_connected_2/biases": 1.02e-09},
    "mlp_plain_h20_max": {"mlp_fc0/w": 2.54e-06, "mlp_fc0/b": 7.73e-07, "mlp_fc1/w": 9.27e-06, "mlp_fc1/b": 4.88e-06,
                          "action_value/fully_connected/weights": 2.19e-05,
                          "action_value/fully_connected/biases": 5.29e-09,
                          "action_value/fully_connected_1/weights": 1.06e-05,
                          "action_value/fully_connected_1/biases": 2.57e-09},
    "cnn_dueling_h256": {"c1/w": 4.11e-09, "c1/b": 1.92e-09, "c2/w": 1.90e-08, "c2/b": 1.46e-08, "c3/w": 2.00e-08,
                         "c3/b": 1.69e-07, "fc1/w": 1.30e-07, "fc1/b": 4.80e-06,
                         "action_value/fully_connected/weights": 3.26e-08,
                         "action_value/fully_connected/biases": 2.81e-06,
                         "action_value/fully_connected_1/weights": 1.09e-09,
                         "action_value/fully_connected_1/biases": 6.73e-09,
                         "state_value/fully_connected/weights": 4.20e-08,
                         "state_value/fully_connected/biases": 2.75e-08,
                         "state_value/fully_connected_1/weights": 8.66e-10,
                         "state_value/fully_connected_1/biases": 0.00e+00},
    "mlp_disc7_dueling_h64": {"mlp_fc0/w": 1.09e-06, "mlp_fc0/b": 1.48e-07, "mlp_fc1/w": 1.92e-06,
                              "mlp_fc1/b": 6.42e-07, "action_value/fully_connected/weights": 3.40e-07,
                              "action_value/fully_connected/biases": 6.45e-09,
                              "action_value/fully_connected_1/weights": 3.39e-08,
                              "action_value/fully_connected_1/biases": 6.98e-09,
                              "state_value/fully_connected/weights": 1.57e-06,
                              "state_value/fully_connected/biases": 1.48e-08,
                              "state_value/fully_connected_1/weights": 1.57e-07,
                              "state_value/fully_connected_1/biases": 0.00e+00},
    "mlp_dueling_h20_double": {"mlp_fc0/w": 7.18e-07, "mlp_fc0/b": 3.08e-07, "mlp_fc1/w": 3.92e-06,
                               "mlp_fc1/b": 2.29e-06, "action_value/fully_connected/weights": 7.70e-06,
                               "action_value/fully_connected/biases": 3.03e-09,
                               "action_value/fully_connected_1/weights": 2.35e-06,
                               "action_value/fully_connected_1/biases": 3.73e-10,
                               "state_value/fully_connected/weights": 8.43e-06,
                               "state_value/fully_connected/biases": 0.00e+00,
                               "state_value/fully_connected_1/weights": 9.71e-07,
                               "state_value/fully_connected_1/biases": 0.00e+00},
    "conv_only_dueling_h256": {"convnet/Conv/weights": 5.50e-07, "convnet/Conv/biases": 1.21e-07,
                               "convnet/Conv_1/weights": 2.71e-07, "convnet/Conv_1/biases": 3.83e-07,
                               "convnet/Conv_2/weights": 1.29e-07, "convnet/Conv_2/biases": 1.28e-07,
                               "action_value/fully_connected/weights": 1.33e-06,
                               "action_value/fully_connected/biases": 8.24e-06,
                               "action_value/fully_connected_1/weights": 2.04e-09,
                               "action_value/fully_connected_1/biases": 3.20e-09,
                               "state_value/fully_connected/weights": 1.53e-06,
                               "state_value/fully_connected/biases": 9.37e-09,
                               "state_value/fully_connected_1/weights": 1.47e-09,
                               "state_value/fully_connected_1/biases": 0.00e+00},
}
G = {(c, t): 3.5 * max(v, 1e-8) for c, per in _OBSERVED.items() for t, v in per.items()}


def _report(what, seen, g):
    print(f"[observed] {what}: g = {seen:.3e} (allowed {g:.3e})")


def _f32(x):
    return float(np.float32(x))


# ================================================================================================ PPO2
# max_grad_norm per configuration: a small one clips every step, a large one never does
PPO_CLIP = {"cnn84_cat6_shared": 0.05, "mlp376_gauss17_copy_h64": 0.05, "mlp13_cat15_l3_h20": 0.05,
            "mlp11_bern5_normalized": 0.05}
PPO_LR = 3e-4
CLIPRANGE, ENT, VFC = 0.2, 0.01, 0.5


def _spaces(cfg):
    from baselines_b200.common import spaces
    ok, oa = cfg["ob"]
    if ok == "box":
        ob = spaces.Box(0, 255, oa, np.uint8) if cfg["kind"] == "cnn" else spaces.Box(-10, 10, oa, np.float32)
    elif ok == "discrete":
        ob = spaces.Discrete(oa)
    else:
        ob = spaces.MultiDiscrete(list(oa))
    ak, aa = cfg["ac"]
    ac = {"cat": lambda: spaces.Discrete(aa), "gauss": lambda: spaces.Box(-1, 1, (aa,), np.float32),
          "mcat": lambda: spaces.MultiDiscrete(list(aa)), "bern": lambda: spaces.MultiBinary(aa)}[ak]()
    return ob, ac


def _ppo_model(name, M, chunk=None, seed=0):
    from baselines_b200.common.policies import PolicyBuilder
    from baselines_b200.ppo2.model import Model
    cfg = N.PPO_CONFIGS[name]
    ob, ac = _spaces(cfg)
    kw = dict(num_layers=cfg.get("num_layers", 2), num_hidden=cfg.get("num_hidden", 64)) if cfg["kind"] == "mlp" else {}
    np.random.seed(seed)
    pol = PolicyBuilder(ob, ac, cfg["kind"], value_network="copy" if cfg.get("copy") else None,
                        normalize_observations=cfg.get("normalize", False), **kw)
    model = Model(policy=pol, ob_space=ob, ac_space=ac, nbatch_act=8, nbatch_train=M, nsteps=1, ent_coef=ENT,
                  vf_coef=VFC, max_grad_norm=PPO_CLIP.get(name, 1e3), comm=False, train_chunk=chunk or M)
    net = model.net
    rng = _move_off_zero(model, seed)
    if cfg.get("normalize"):
        # statistics with |(x - mean) / std| beyond 5 for a good share of the observations: the clip is active
        d = N.in_dim(cfg["ob"])[0]
        net.set_obs_rms(dict(runningsum=rng.randn(d) * 5.0, runningsumsq=rng.rand(d) * 20.0 + 30.0, count=10.0))
        assert net.obs_rms is not None
    assert net.pi_identity == N.ppo_identity(cfg)
    return model


def _move_off_zero(model, seed):
    """Biases away from zero, so that a missing bias term or a stale bias operand shows, and a non-zero Gaussian
    logstd.  Returns the random stream, for further settings."""
    net = model.net
    rng = np.random.RandomState(seed + 100)
    p = net.store.export_tf("params")
    for k in p:
        if k.endswith("/b:0") and not k.endswith("logstd:0"):
            p[k] = (p[k] + 0.05 * rng.randn(*p[k].shape)).astype(np.float32)
    if net.pd == "gauss":
        p["ppo2_model/pi/logstd:0"] = (0.2 * rng.randn(1, net.nout)).astype(np.float32)
    model.set_params(p)
    return rng


def _norm_arrays(net):
    if net.obs_rms is None:
        return None, None
    r = net.obs_rms
    mean = (r["runningsum"] / r["count"]).astype(np.float32)
    std = np.sqrt(np.maximum((r["runningsumsq"] / r["count"]).astype(np.float32) - np.square(mean), np.float32(1e-2)))
    return mean, np.float32(1.0) / std


def _encode(net, cfg, raw):
    """The mirror's input rows for raw observation rows: images as float64, or the encoder's float32 values."""
    if cfg["kind"] == "cnn":
        return torch.as_tensor(raw).to(DEV).double()
    ok, oa = cfg["ob"]
    mean, inv_std = _norm_arrays(net)
    x = N.encode_obs(raw, onehot_n=oa if ok == "discrete" else 0, nvec=list(oa) if ok == "mdisc" else None,
                     mean=mean, inv_std=inv_std)
    return torch.as_tensor(x).to(DEV)


def _raw_obs(rng, cfg, n):
    ok, oa = cfg["ob"]
    if cfg["kind"] == "cnn":
        return rng.randint(0, 256, (n,) + oa).astype(np.uint8)
    if ok == "discrete":
        return rng.randint(0, oa, (n, 1)).astype(np.float32)
    if ok == "mdisc":
        return np.stack([rng.randint(0, k, n) for k in oa], 1).astype(np.float32)
    return (rng.randn(n, *oa) * 3.0).astype(np.float32)


def _ppo_rollout(model, cfg, rng, n):
    """Rollout buffers of n rows: observations, actions, returns, old values and old neglogp near the current policy."""
    net = model.net
    pd, nout = cfg["ac"][0], net.nout
    raw = _raw_obs(rng, cfg, n)
    P = net.store.export_tf("params")
    z = np.zeros(n)
    head = N.policy_ref(P, N.ppo_mirror_cfg(cfg), _encode(net, cfg, raw), np.zeros((n, nout)), z,
                        identity=net.pi_identity, dev=DEV)
    mu, v = head.pi.cpu().numpy(), head.v.cpu().numpy()
    nvec = list(cfg["ac"][1]) if pd == "mcat" else None
    ls = P.get("ppo2_model/pi/logstd:0")
    if pd == "cat":
        acts = rng.randint(0, nout, n).astype(np.int64)
    elif pd == "mcat":
        acts = np.stack([rng.randint(0, k, n) for k in nvec], 1).astype(np.int64)
    elif pd == "bern":
        acts = (rng.rand(n, nout) < 0.5).astype(np.float32)
    else:
        acts = (mu + np.exp(ls) * rng.randn(n, nout)).astype(np.float32)
    nlp = lr.ppo_ref(pd, mu, v, acts, z, z, z, z, 0.2, 0.0, 0.0, nvec=nvec,
                     logstd=None if ls is None else ls[0]).nlp
    old_nlp = (nlp + 0.15 * rng.randn(n)).astype(np.float32)
    old_v = (v + 0.3 * rng.randn(n)).astype(np.float32)
    ret = (old_v + rng.randn(n)).astype(np.float32)
    dev = lambda a, dt=None: torch.as_tensor(a if dt is None else a.astype(dt)).to(DEV).contiguous()
    obs = dev(raw) if cfg["kind"] == "cnn" else dev(raw.reshape(n, -1))
    return dict(raw=raw, obs=obs, acts=dev(acts), acts_np=acts, ret=dev(ret), oldv=dev(old_v), oldnlp=dev(old_nlp),
                np=dict(ret=ret, oldv=old_v, oldnlp=old_nlp))


def _flat_state(store):
    return {k: getattr(store, k).detach().double().cpu().numpy().copy() for k in ("params", "m", "v")}


def _ppo_step(model, roll, rows, graph, lr_=PPO_LR, cliprange=CLIPRANGE):
    """One train_rollout on rows `rows` of the rollout: gathered through src_idx (graph-captured) or as contiguous
    M-row buffers (eager).  Returns the pre-step flat state and exported parameters."""
    before = _flat_state(model.net.store)
    params = model.net.store.export_tf("params")
    if graph:
        model.train_rollout(lr_, cliprange, roll["obs"], roll["acts"], roll["ret"], roll["oldv"], roll["oldnlp"],
                            torch.as_tensor(rows).to(DEV))
    else:
        r = torch.as_tensor(rows).to(DEV)
        sel = lambda t: t.index_select(0, r).contiguous()
        model.train_rollout(lr_, cliprange, sel(roll["obs"]), sel(roll["acts"]), sel(roll["ret"]),
                            sel(roll["oldv"]), sel(roll["oldnlp"]), None)
    torch.cuda.synchronize()
    return before, params


def _ppo_heads(net, B):
    """The kernels' head outputs and fp16 head-gradient rows (layout the head GEMMs read) of the last chunk."""
    nout = net.nout
    return (net.pi_out[:B, :nout].double().cpu(), net.v_out[:B, 0].double().cpu(),
            net.dpi[:B, :nout].double().cpu(), net.dv[:B, 0].double().cpu())


def _check_ppo_heads(name, cfg, net, roll, rows, M, params, clip=CLIPRANGE, ent=ENT, vfc=VFC, stats=None,
                     g_dlogstd=G_DLOGSTD, dlogstd_drop=1):
    """(a) head-gradient rows against _loss_refs.ppo_ref at the kernels' own head outputs; with `stats` (the kernels'
    five loss-statistic sums) those too, against the same reference's per-row terms.  A Gaussian's dL/dlogstd is
    within g_dlogstd of its absolute row sum, a bound that rejects the first dlogstd_drop rows dropped."""
    pd = cfg["ac"][0]
    pi, v, dpi, dv = _ppo_heads(net, M)
    nvec = list(cfg["ac"][1]) if pd == "mcat" else None
    mean, std = net.adv_st.cpu().numpy()
    R_, oldv, oldnlp = (roll["np"][k][rows] for k in ("ret", "oldv", "oldnlp"))
    adv = lr.adv_normalise(R_, oldv, mean, std)
    acts = roll["acts_np"][rows]
    ls = params["ppo2_model/pi/logstd:0"].reshape(-1) if pd == "gauss" else None      # the pre-step logstd
    pi32, v32 = pi.numpy().astype(np.float32), v.numpy().astype(np.float32)
    args = (pd, pi32, v32, acts, R_, oldv, oldnlp, adv, clip, ent, vfc)
    ref = lr.ppo_ref(*args, nvec=nvec, logstd=ls)
    ok = ~ref.near
    assert ok.mean() > 0.95
    nb = lr.ppo_ref(pd, pi32, v32, np.roll(acts, 1, 0), *args[4:], nvec=nvec, logstd=ls)
    nscale = _gauss_nscale(acts, pi32, ls, oldnlp)[ok] if pd == "gauss" else None
    _within_f16(dpi.numpy()[ok], ref.dhead[ok], {"actions of the neighbouring row": nb.dhead[ok]},
                f"{name} dpi", nscale)
    vm = lr.ppo_ref(*args, nvec=nvec, logstd=ls, mutant="vf_clip_passes")
    _within_f16(dv.numpy()[ok], ref.dv[ok], {"value clip passing gradient": vm.dv[ok]}, f"{name} dv")
    if pd == "gauss":                         # pi/logstd's gradient: the loss kernel's row sum times 1/M
        rws = ref.dlogstd_rows / M
        want = rws.sum(0)
        got = net.store.export_tf("grads")["ppo2_model/pi/logstd:0"].reshape(-1).astype(np.float64)
        S = np.abs(rws).sum(0) + np.abs(want)
        t = lambda a: torch.as_tensor(np.asarray(a, np.float64))
        muts = {"row 0 dropped" if dlogstd_drop == 1 else f"rows 0..{dlogstd_drop - 1} dropped":
                t(want - rws[:dlogstd_drop].sum(0))}
        if ent:                                   # without an entropy bonus the mutant is the reference itself
            muts["-ent_coef term dropped"] = t(lr.ppo_ref(*args, nvec=nvec, logstd=ls,
                                                          mutant="no_entropy").dlogstd_rows.sum(0) / M)
        for mn, mv in muts.items():
            print(f"[mutant] {name} pi/logstd {mn}: g = {R.excess(mv, t(want), t(S), 0.0):.3e}")
        seen = R.assert_within(t(got), t(want), t(S), g_dlogstd, 0.0, muts, f"{name} pi/logstd")
        _report(f"{name} pi/logstd", seen, g_dlogstd)
    if stats is not None:
        seen = _stats_check(stats, ref, pd, pi32, acts, oldnlp, adv, ls, M, name)
        _report(f"{name} loss statistics", seen, G_STATS)
    return dpi, dv


def _ppo_masks(net, M, start=0):
    """ReLU decisions of the kernels' stored activations of rows start .. start+M, keyed like the mirror's layers."""
    masks = {}
    towers = [("pi", net.tower_pi)] + ([("vf", net.tower_vf)] if net.tower_vf is not None else [])
    for nm, t in towers:
        if t.kind != "cnn":
            continue
        for i, c in enumerate(t.convs):
            masks[f"ppo2_model/{nm}/{c.name.split('/')[-1]}"] = (N.kernel_act(t, i, M, start) > 0).double()
        masks[f"ppo2_model/{nm}/fc1"] = (t.hfc[0][start:start + M, :t.fcs[0].N] > 0).double()
    return masks


def _short(k):
    return k.replace("ppo2_model/", "").replace("deepq/q_func/", "").replace(":0", "")


def _check_masks(what, ref, S, masks, report=True, g_mask=G_MASK):
    """Every kernel ReLU decision that differs from the mirror's lies within g_mask * S of zero.  Returns name ->
    (worst |pre| / S, decisions that differ)."""
    out = {}
    for k, m in masks.items():
        p, pa = ref.pres[k], S.pres[k]
        off = m != (p > 0).double()
        worst = float((p.abs()[off] / pa[off]).max()) if bool(off.any()) else 0.0
        out[k] = (worst, int(off.sum()))
        if report:
            _report(f"{what} {_short(k)} ReLU decisions ({int(off.sum())} differ) |pre|/S", worst, g_mask)
        assert worst <= g_mask, (what, k, worst)
    return out


def _assert_grads(what, table_key, got, ref_g, S_g, mutants, names, alpha, g_table=None):
    """(b): every TF variable in `names` within its bound, each bound rejecting its mutants.  mutants: name ->
    (grads dict, target tensors or None for all).  g_table: (table_key, short name) -> g, G by default."""
    g_table = G if g_table is None else g_table
    for k in names:
        gt = torch.as_tensor(got[k]).to(DEV).double().reshape(ref_g[k].shape)
        ref, S, g = ref_g[k] * alpha, S_g[k] * alpha, g_table[(table_key, _short(k))]
        muts = {mn: mg[k] * alpha for mn, (mg, targets) in mutants.items() if targets is None or k in targets}
        for mn, mg in muts.items():
            print(f"[mutant] {what} {_short(k)} {mn}: g = {R.excess(mg, ref, S, R.R_F32):.3e}")
        seen = R.assert_within(gt, ref, S, g, R.R_F32, muts, what=f"{what} {k}")
        _report(f"{what} {_short(k)}", seen, g)


def _ppo_mutants(cfg, params, x, seeds, masks, ident, mcfg, ref):
    """Mutated mirror gradients: one sample dropped, plus the composition mistakes this configuration can make."""
    dpi, dv = seeds
    run = lambda sp, sv, xx=x, **kw: N.policy_ref(params, mcfg, xx, sp, sv, rnd=True, masks=masks, identity=ident,
                                                  dev=DEV, **kw).grads
    # each head loses the one row with its largest gradient (a row may carry none for one head, e.g. a clipped value;
    # two dropped rows of one head could cancel)
    d0pi, d0v = dpi.clone(), dv.clone()
    d0pi[int(dpi.abs().sum(1).argmax())] = 0.0
    d0v[int(dv.abs().argmax())] = 0.0
    out = {"one sample dropped": (run(d0pi, d0v), None)}
    sc = "ppo2_model"
    vf_tensors = {k for k in params if k.startswith(f"{sc}/vf/")}
    out["vf head gradient taken from the pi column"] = (run(dpi, dpi[:, 0]), vf_tensors if cfg.get("copy") else
                                                         {f"{sc}/vf/w:0", f"{sc}/vf/b:0"})
    if cfg.get("copy") and cfg["kind"] == "mlp":
        a, b = f"{sc}/pi/mlp_fc0/w:0", f"{sc}/vf/mlp_fc0/w:0"
        sw = dict(ref.grads)
        sw[a], sw[b] = ref.grads[b], ref.grads[a]
        out["g0cat halves swapped"] = (sw, {a, b})
    if cfg.get("num_layers", 2) >= 3:
        out["second hidden layer's activation derivative omitted"] = (
            run(dpi, dv, no_dact={f"{sc}/pi/mlp_fc1"}), {f"{sc}/pi/mlp_fc{i}/{p}:0" for i in (0, 1) for p in "wb"})
    if cfg["ob"][0] != "box" or cfg.get("normalize"):
        out["observation of the neighbouring row"] = (run(dpi, dv, xx=torch.roll(x, 1, 0)), {f"{sc}/pi/mlp_fc0/w:0"})
    if cfg["kind"] == "cnn":
        out["fc1 ReLU derivative omitted"] = (run(dpi, dv, no_dact={f"{sc}/pi/fc1"}),
                                              {k for k in params if k.startswith(f"{sc}/pi/c")} | {f"{sc}/pi/fc1/w:0"})
    return out


def _check_ppo_grads(what, name, cfg, net, params, x, dpi, dv, masks, M):
    """(b) for the gradient in the store against the mirror at `params`, seeded with (dpi, dv)."""
    mcfg = N.ppo_mirror_cfg(cfg)
    ident = net.pi_identity
    dpi, dv = dpi.to(DEV), dv.to(DEV)
    ref = N.policy_ref(params, mcfg, x, dpi, dv, rnd=True, masks=masks, identity=ident, dev=DEV)
    S = N.policy_ref(params, mcfg, x, dpi, dv, rnd=False, absolute=True, ref_acts=ref.acts, identity=ident, dev=DEV)
    _check_masks(what, ref, S, masks)
    got = net.store.export_tf("grads")
    names = [k for k in got if not k.endswith("logstd:0")]
    muts = _ppo_mutants(cfg, params, x, (dpi, dv), masks, ident, mcfg, ref)
    _assert_grads(what, name, got, ref.grads, S.grads, muts, names, 1.0 / M)


def _check_adam(what, store, before, g_flat, lr_t_of, t, eps, seg_scale, clipped_mutant):
    """(c): params / m / v after the step against float64 TF-Adam from the exported pre-step state and the kernels'
    gradients times the clip factor per element (seg_scale)."""
    b1, b2, feps = _f32(0.9), _f32(0.999), _f32(eps)
    after = {k: torch.as_tensor(v) for k, v in _flat_state(store).items()}
    p0, m0, v0 = before["params"], before["m"], before["v"]
    g = g_flat * seg_scale
    P, Mm, V = lr.adam_tf(p0, g, m0, v0, lr_t_of(t), b1, b2, feps)
    P_next = lr.adam_tf(p0, g, m0, v0, lr_t_of(t + 1), b1, b2, feps)[0]
    Sm = b1 * np.abs(m0) + (1 - b1) * np.abs(g)
    Sp = np.abs(p0) + lr_t_of(t) * Sm / (np.sqrt(V) + feps)
    P, Mm, V, Sm, Sp, P_next = (torch.as_tensor(a) for a in (P, Mm, V, Sm, Sp, P_next))
    pm = {"lr_t of step t + 1": P_next}
    if clipped_mutant:
        unclipped = lr.adam_tf(p0, g_flat, m0, v0, lr_t_of(t), b1, b2, feps)
        pm["clip factor left out"] = torch.as_tensor(unclipped[0])
        mm = {"clip factor left out": torch.as_tensor(unclipped[1])}
        R.assert_within(after["m"], Mm, Sm, ADAM_G, 0.0, mm, f"{what} adam m")
    else:
        assert R.within(after["m"], Mm, Sm, ADAM_G, 0.0), f"{what} adam m"
    assert R.within(after["v"], V, V, ADAM_G, 0.0), f"{what} adam v"
    seen = R.assert_within(after["params"], P, Sp, ADAM_G, 0.0, pm, f"{what} adam p")
    _report(f"{what} adam p", seen, ADAM_G)
    return after


def _lr_t(lr_):
    return lambda t: _f32(lr_ * math.sqrt(1.0 - 0.999 ** t) / (1.0 - 0.9 ** t))


def _ppo_adam(what, name, model, before, M, lr_=PPO_LR, clipped=None):
    """(c) for a PPO2 step with learning rate lr_; clipped: whether the global clip scales this step (by default
    whether the configuration is in PPO_CLIP)."""
    store, net = model.net.store, model.net
    g_flat = store.grads.detach().double().cpu().numpy()
    clip = model.max_grad_norm
    sc = lr.clip_scale(math.fsum(g_flat * g_flat), clip)
    clipped = name in PPO_CLIP if clipped is None else clipped
    assert (sc < 1.0) == clipped, (name, sc)                     # which case this run is in
    _check_adam(what, store, before, g_flat, _lr_t(lr_), model.opt.t, 1e-5, sc, sc < 1.0)
    if net.pi_identity:                                          # the frozen identity block: bit-for-bit unchanged
        h = net.head_pi if net.head is None else net.head
        hw, gw = (h.w, h.gw) if net.head is None else (h.w[:, :net.nout], h.gw[:, :net.nout])
        assert torch.equal(hw.detach().cpu(), torch.eye(net.nout)), "identity head moved"
        assert float(gw.abs().max()) == 0.0, "identity head gradient not frozen"


PPO_M = 301
STEPS = 3                          # minibatches per run: eager, captured + replayed, replayed on the graph paths


def _assert_replayed(what, n_replays, expected):
    """A graph-path step after the first is a replay of the captured launch sequence; every other step runs eagerly."""
    assert n_replays == (1 if expected else 0), (what, n_replays)


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "src_idx_graph"])
@pytest.mark.parametrize("name", list(N.PPO_CONFIGS))
def test_ppo_update_composition_vs_float64(name, graph):
    cfg = N.PPO_CONFIGS[name]
    M = PPO_M
    model = _ppo_model(name, M)
    net = model.net
    if cfg.get("copy") and cfg["kind"] == "mlp":
        assert net.fuse0 == (2 * cfg.get("num_hidden", 64) <= 256), (name, net.fuse0)
    rng = np.random.RandomState(7)
    n = STEPS * M + 37
    roll = _ppo_rollout(model, cfg, rng, n)
    perm = rng.permutation(n)
    for step in range(STEPS):
        rows = perm[step * M:(step + 1) * M]
        what = f"{name} {'graph' if graph else 'eager'} step {step + 1}"
        replays = _lib.REPLAYS
        before, params = _ppo_step(model, roll, rows, graph)
        _assert_replayed(what, _lib.REPLAYS - replays, graph and step > 0)
        dpi, dv = _check_ppo_heads(what, cfg, net, roll, rows, M, params)
        x = _encode(net, cfg, roll["raw"][rows])
        _check_ppo_grads(what, name, cfg, net, params, x, dpi, dv, _ppo_masks(net, M), M)
        _ppo_adam(what, name, model, before, M)


def test_ppo_chunked_gathered_nature_cnn_update():
    """(e): the benchmarked path in miniature -- NatureCNN, a rollout gathered through src_idx, three uneven chunks
    (128, 128, 45 rows), graph-captured.  Per-row head outputs, head gradients and activations do not depend on the
    chunking (the last chunk's rows are bit-identical to the unchunked run's), so the accumulated gradient is checked
    against the mirror seeded with the unchunked run's rows.  Before each step the unchunked model takes the chunked
    one's state and refreshes its operands eagerly; the chunked model's operands come only from its own refresh(),
    replayed from the graph from the second step on."""
    name, M, chunk = "cnn84_cat6_shared", PPO_M, 128
    cfg = N.PPO_CONFIGS[name]
    full, chunked = _ppo_model(name, M), _ppo_model(name, M, chunk=chunk)
    assert chunked.chunk == chunk and full.chunk == M
    rng = np.random.RandomState(8)
    n = STEPS * M + 37
    roll = _ppo_rollout(full, cfg, rng, n)
    perm = rng.permutation(n)
    for step in range(STEPS):
        rows = perm[step * M:(step + 1) * M]
        what = f"{name} chunked step {step + 1}"
        for k in ("params", "m", "v"):                           # both models start the step from the same state
            getattr(full.net.store, k).copy_(getattr(chunked.net.store, k))
        full.net.refresh()
        _, params = _ppo_step(full, roll, rows, True)
        replays = _lib.REPLAYS
        before, params_c = _ppo_step(chunked, roll, rows, True)
        _assert_replayed(what, _lib.REPLAYS - replays, step > 0)
        assert all(np.array_equal(params[k], params_c[k]) for k in params)
        last = M - 2 * chunk
        for a, b in zip(_ppo_heads(full.net, M), _ppo_heads(chunked.net, last)):
            assert torch.equal(a[2 * chunk:], b), "per-row head outputs / gradients depend on the chunking"
        tf, tc = full.net.tower_pi, chunked.net.tower_pi
        assert torch.equal(tf.hfc[0][2 * chunk:M], tc.hfc[0][:last])
        dpi, dv = _check_ppo_heads(what + " (unchunked)", cfg, full.net, roll, rows, M, params)
        x = _encode(full.net, cfg, roll["raw"][rows])
        _check_ppo_grads(what, name, cfg, chunked.net, params, x, dpi, dv, _ppo_masks(full.net, M), M)
        _ppo_adam(what, name, chunked, before, M)


# ================================================================================================ DQN
DQN_NA, DQN_B, DQN_LR, GAMMA = 6, 301, 1e-3, 0.99
# grad_norm_clipping per configuration, the scale of the importance weights, and which variables the clip scales in the
# first update: "mixed" (some clipped, some not), "none" (the clip is on, no variable reaches it) or "off"
DQN_CLIP = {"mlp_dueling_h64_32_double": 10.0, "mlp_plain_h20_max": None, "mlp_dueling_h20_double": None,
            "cnn_dueling_h256": 10.0, "conv_only_dueling_h256": 10.0, "mlp_disc7_dueling_h64": None}
DQN_W_SCALE = {"mlp_dueling_h64_32_double": 40.0, "cnn_dueling_h256": 40.0, "conv_only_dueling_h256": 200.0}
DQN_CLIP_CASE = {"mlp_dueling_h64_32_double": "none", "mlp_plain_h20_max": "off", "mlp_dueling_h20_double": "off",
                 "cnn_dueling_h256": "mixed", "conv_only_dueling_h256": "mixed", "mlp_disc7_dueling_h64": "off"}


def _dqn_model(name, seed=3, B=DQN_B, lr_=DQN_LR, clip=None):
    """The DQNModel of configuration `name` (learning rate lr_, batch B, grad_norm_clipping clip), biases away from
    zero and a target network that differs from the online one."""
    from baselines_b200.common import spaces
    from baselines_b200.deepq.build_graph import DQNModel
    cfg = N.DQN_CONFIGS[name]
    ok, oa = cfg["ob"]
    if ok == "discrete":
        ob = spaces.Discrete(oa)
    else:
        ob = spaces.Box(0, 255, oa, np.uint8) if cfg["kind"] != "mlp" else spaces.Box(-5, 5, oa, np.float32)
    model = DQNModel(ob, DQN_NA, cfg["kind"], lr=lr_, gamma=GAMMA, grad_norm_clipping=clip,
                     double_q=cfg["double_q"], batch_cap=B, seed=seed, hiddens=cfg["hiddens"],
                     dueling=cfg["dueling"])
    rng = np.random.RandomState(seed + 100)
    p = model.q.store.export_tf("params")
    for k in p:
        if "biases" in k or k.endswith("/b:0"):
            p[k] = (p[k] + 0.05 * rng.randn(*p[k].shape)).astype(np.float32)
    model.q.store.import_tf(p, "params")
    model.q.refresh()
    model.update_target()
    # the target network a step behind: it differs from the online one
    p2 = {k: (v + 0.01 * rng.randn(*v.shape)).astype(np.float32) for k, v in p.items()}
    model.qt.store.import_tf({k.replace("q_func", "target_q_func", 1): v for k, v in p2.items()}, "params")
    model.qt.refresh()
    return model


def _dqn_batch(rng, cfg, n):
    if cfg["kind"] != "mlp":
        o = lambda: rng.randint(0, 256, (n,) + cfg["ob"][1]).astype(np.uint8)
    elif cfg["ob"][0] == "discrete":
        o = lambda: rng.randint(0, cfg["ob"][1], (n, 1)).astype(np.float32)
    else:
        o = lambda: (rng.randn(n, *cfg["ob"][1]) * 2.0).astype(np.float32)
    return dict(o_t=o(), o_1=o(), act=rng.randint(0, DQN_NA, n).astype(np.int64),
                rew=(rng.randn(n) * 2).astype(np.float32), done=(rng.rand(n) < 0.1).astype(np.float32))


def _dqn_x(cfg, raw):
    if cfg["kind"] != "mlp":
        return torch.as_tensor(raw).to(DEV).double()
    ok, oa = cfg["ob"]
    return torch.as_tensor(N.encode_obs(raw, onehot_n=oa if ok == "discrete" else 0)).to(DEV)


def _dqn_masks(q, B):
    masks = {}
    tr = q.trunk
    sc = "deepq/q_func"
    for i, c in enumerate(tr.convs):
        nm = ("Conv" if i == 0 else f"Conv_{i}") if tr.kind == "conv_only" else c.name.split("/")[-1]
        key = f"{sc}/convnet/{nm}" if tr.kind == "conv_only" else f"{sc}/{nm}"
        masks[key] = (N.kernel_act(tr, i, B) > 0).double()
    if tr.kind == "cnn":
        masks[f"{sc}/fc1"] = (tr.hfc[0][:B, :tr.fcs[0].N] > 0).double()
    for si, (sname, layers) in enumerate(zip(["action_value", "state_value"], q.streams)):
        for j, l in enumerate(layers[:-1]):
            h = q.h_cat[:B, q.cat_off[si]:q.cat_off[si] + l.N] if j == 0 else q.hid[si][j - 1][:B, :l.N]
            masks[f"{sc}/{sname}/{N._fc_name(j)}"] = (h > 0).double()
    return masks


def _check_dqn_heads(what, model, cfg, b, rows, w, B):
    q, nA = model.q, DQN_NA
    out, on, tg = (t[:B].double().cpu().numpy() for t in (q.out, model.on_out, model.qt.out))
    s = (lambda h: h[:, nA]) if cfg["dueling"] else (lambda h: None)
    args = (out[:, :nA], s(out), on[:, :nA], s(on), tg[:, :nA], s(tg), b["act"][rows], b["rew"][rows],
            b["done"][rows])
    ref = lr.dqn_ref(*args, w, GAMMA, cfg["double_q"])
    nb = lr.dqn_ref(*args, np.roll(w, 1), GAMMA, cfg["double_q"])
    ok = (ref.gap > 1e-5) & (np.abs(np.abs(ref.td) - 1.0) > 1e-5)
    assert ok.mean() > 0.95
    da = q.dout[:B, :nA].double().cpu()
    ds = q.dout[:B, q.s_col].double().cpu() if cfg["dueling"] else None
    _within_f16(da.numpy()[ok], ref.d_a[ok], {"importance weight of the neighbouring row": nb.d_a[ok]}, f"{what} dA")
    if cfg["dueling"]:
        _within_f16(ds.numpy()[ok], ref.d_s[ok], {"importance weight of the neighbouring row": nb.d_s[ok]},
                    f"{what} dS")
    return da, ds


def _dqn_mutants(cfg, params, x, da, ds, masks, mcfg, names, block=None):
    """block: (k, short names): for those tensors, whose bound cannot see one sample, k consecutive rows dropped from
    the row with the largest TD gradient on."""
    run = lambda a, s, xx=x, **kw: N.q_ref(params, mcfg, xx, a, s, rnd=True, masks=masks, dev=DEV, **kw).grads
    # the row with the largest TD gradient: both streams' seeds of a row come from the same d loss / dq
    i = int(da.abs().sum(1).argmax() if ds is None else ds.abs().argmax())

    def drop(k):
        r = slice(min(i, len(da) - k), min(i, len(da) - k) + k)
        a0 = da.clone()
        a0[r] = 0.0
        s0 = None
        if ds is not None:
            s0 = ds.clone()
            s0[r] = 0.0
        return run(a0, s0)
    weak = set() if block is None else {k for k in names if _short(k) in block[1]}
    out = {"one sample dropped": (drop(1), None if block is None else set(names) - weak)}
    if block is not None:
        out[f"{block[0]} consecutive rows dropped"] = (drop(block[0]), weak)
    sc = "deepq/q_func"
    trunk = {k for k in names if "_value/" not in k}
    if cfg["dueling"]:
        out["state stream left out of the trunk's data gradient"] = (run(da, ds, detach_state_stream=True), trunk)
    if len(cfg["hiddens"]) > 1:
        out["second hidden layer's activation derivative omitted"] = (
            run(da, ds, no_dact={f"{sc}/action_value/fully_connected_1", f"{sc}/state_value/fully_connected_1"}),
            {k for k in names if "/fully_connected/" in k or "/fully_connected_1/" in k} | trunk)
    else:
        out["hidden activation derivative omitted"] = (
            run(da, ds, no_dact={f"{sc}/action_value/fully_connected", f"{sc}/state_value/fully_connected"}),
            {k for k in names if "/fully_connected/" in k} | trunk)
    if cfg["ob"][0] == "discrete":
        out["observation of the neighbouring row"] = (run(da, ds, xx=torch.roll(x, 1, 0)), {f"{sc}/mlp_fc0/w:0"})
    return out


@pytest.mark.parametrize("replay", [False, True], ids=["gathered", "replay_idx"])
@pytest.mark.parametrize("name", list(N.DQN_CONFIGS))
def test_dqn_update_composition_vs_float64(name, replay):
    _dqn_update_run(name, replay, clip=DQN_CLIP[name], w_scale=DQN_W_SCALE.get(name, 1.0), case=DQN_CLIP_CASE[name])


def _dqn_update_run(name, replay, B=DQN_B, lr_=DQN_LR, clip=None, w_scale=1.0, case="off", g_table=None,
                    table_key=None, block=None):
    """Three DQN updates of configuration `name` at batch B, learning rate lr_ and grad_norm_clipping clip, checked
    (a) to (d).  w_scale: the scale of the importance weights; case: which variables the clip scales in the first
    update ("mixed", "none" or "off"); g_table / table_key: the gradient bounds (G and name by default); block: see
    _dqn_mutants."""
    cfg = N.DQN_CONFIGS[name]
    model = _dqn_model(name, B=B, lr_=lr_, clip=clip)
    q = model.q
    if cfg["dueling"] and q.first_widths[0] % 8:                 # the state stream starts past padding columns
        assert q.cat_off[1] == -(-q.first_widths[0] // 8) * 8 > q.first_widths[0], q.cat_off
    rng = np.random.RandomState(9)
    n = STEPS * B + 41
    b = _dqn_batch(rng, cfg, n)
    dev = lambda a: torch.as_tensor(a).to(DEV).contiguous()
    store = {k: dev(v) for k, v in b.items()}
    perm = rng.permutation(n)
    mcfg = N.dqn_mirror_cfg(cfg)
    for step in range(STEPS):
        rows = perm[step * B:(step + 1) * B]
        what = f"{name} {'replay' if replay else 'gathered'} step {step + 1}"
        replays = _lib.REPLAYS
        w = ((rng.rand(B) * 0.9 + 0.1) * w_scale).astype(np.float32)
        before = _flat_state(q.store)
        params = q.store.export_tf("params")
        if replay:
            model.train_device(store["o_t"], store["o_1"], store["act"], store["rew"], store["done"], dev(w),
                               dev(rows.astype(np.int64)), B)
        else:
            r = dev(rows.astype(np.int64))
            sel = lambda t: t.index_select(0, r).contiguous()
            model.train_device(sel(store["o_t"]), sel(store["o_1"]), sel(store["act"]), sel(store["rew"]),
                               sel(store["done"]), dev(w), None, B)
        torch.cuda.synchronize()
        _assert_replayed(what, _lib.REPLAYS - replays, replay and step > 0)
        da, ds = _check_dqn_heads(what, model, cfg, b, rows, w, B)
        x = _dqn_x(cfg, b["o_t"][rows])
        masks = _dqn_masks(q, B)
        ref = N.q_ref(params, mcfg, x, da.to(DEV), None if ds is None else ds.to(DEV), rnd=True, masks=masks, dev=DEV)
        S = N.q_ref(params, mcfg, x, da.to(DEV), None if ds is None else ds.to(DEV), absolute=True,
                    ref_acts=ref.acts, dev=DEV)
        _check_masks(what, ref, S, masks)
        got = q.store.export_tf("grads")
        names = list(got)
        muts = _dqn_mutants(cfg, params, x, da.to(DEV), None if ds is None else ds.to(DEV), masks, mcfg, names, block)
        _assert_grads(what, table_key or name, got, ref.grads, S.grads, muts, names, 1.0 / B, g_table)
        # (c) per-variable clip_by_norm, then Adam
        g_flat = q.store.grads.detach().double().cpu().numpy()
        off = q.store.segment_offsets()
        scale = np.ones_like(g_flat)
        facs = []
        for s0, s1 in zip(off[:-1], off[1:]):
            seg = g_flat[s0:s1]
            f = lr.clip_scale(math.fsum(seg * seg), clip) if clip else 1.0
            scale[s0:s1] = f
            facs.append(f)
        print(f"[observed] {what} per-variable clip factors: {np.round(facs, 3).tolist()}")
        now = case if step == 0 else ("off" if clip is None else "any")           # which case this run is in
        if now == "mixed":
            assert min(facs) < 1.0 and max(facs) == 1.0, (name, facs)
        elif now != "any":
            assert all(f == 1.0 for f in facs) and (clip is None) == (now == "off"), (name, facs)
        _check_adam(what, q.store, before, g_flat, _lr_t(lr_), model.opt.t, 1e-8, scale, min(facs) < 1.0)
