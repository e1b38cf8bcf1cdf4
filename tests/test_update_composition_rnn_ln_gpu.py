"""GPU: whole PPO2 and DQN updates of the layer-normalised and recurrent networks, every parameter's gradient and Adam
step, against the float64 network mirror (tests/_net_refs.py).

The checks are (a)-(d) of tests/test_update_composition_gpu.py, with its helpers, on the networks that file does not
build: PPO2 mlp(layer_norm=True) (LayerNorm between every fc and its tanh, fp32 pre-activations in the norms'
workspaces), PPO2 lstm and cnn_lstm through train_rollout_seq (time-major rows gathered through mask_idx, start states
through state_idx, the LSTM sequence kernels, dWh from the stored masked h_{t-1}), and deepq layer_norm=True (norms
in the streams, per-variable clip segments of the norms' variables).  On the graph paths the third step's forward and
backward read the fp16 operands (w_fwd, w_bwd, wh16, whT16) the replayed refresh of the second wrote.  The chunked
recurrent run also checks (e): two environment chunks accumulate into one minibatch, and each chunk's rows are
bit-identical to the unchunked run's.

Each bound must reject "one sample dropped" (one row; for the recurrent networks one whose step does not begin with a
reset) and a mistake named for the configuration: for the LSTM the start states read from rows
0..E-1 instead of through state_idx, the reset applied one step late, and dWh taken from h_{t-1} before the mask; for
the norms alpha (the 1/M of the mean loss) left out of dgamma / dbeta, and dgamma / dbeta credited to the neighbouring
LayerNorm.  Under a cnn_lstm's cell the mirror reads the kernels' stored fc1 latent, once it is shown equal to the
mirror's own within one fp16 rounding (_check_grads).

Tolerances: every g is 3.5x the maximum observed on an H100 80GB HBM3 (700 W power limit), floor 1e-8; the observed
values are listed next to the constants.  Each run prints its own [observed] lines.
"""
import math

import numpy as np
import pytest
import torch

import _layer_norm_refs as L
import _loss_refs as lr
import _net_refs as N
import test_update_composition_gpu as C
from baselines_b200 import _lib

pytestmark = pytest.mark.gpu

DEV = C.DEV
STEPS = C.STEPS

# g per configuration and TF variable (short names): 3.5x the maximum observed on an H100 80GB HBM3 (700 W power
# limit) over the eager and graph paths and every step (and the chunked run of lstm_box7_gauss3_h128), floor 1e-8
_OBSERVED = {
    "mlp376_gauss17_copy_ln": {"pi/mlp_fc0/w": 2.07e-06, "pi/mlp_fc0/b": 7.19e-07, "pi/LayerNorm/beta": 7.02e-07,
                               "pi/LayerNorm/gamma": 9.69e-09, "pi/mlp_fc1/w": 6.74e-06, "pi/mlp_fc1/b": 3.00e-06,
                               "pi/LayerNorm_1/beta": 5.73e-06, "pi/LayerNorm_1/gamma": 4.23e-07,
                               "vf/mlp_fc0/w": 9.26e-06, "vf/mlp_fc0/b": 3.05e-06, "vf/LayerNorm/beta": 3.94e-06,
                               "vf/LayerNorm/gamma": 6.25e-08, "vf/mlp_fc1/w": 1.59e-05, "vf/mlp_fc1/b": 5.67e-06,
                               "vf/LayerNorm_1/beta": 1.20e-05, "vf/LayerNorm_1/gamma": 1.34e-06, "pi/w": 2.04e-05,
                               "pi/b": 1.01e-08, "vf/w": 8.55e-06, "vf/b": 2.39e-10},
    "mlp11_cat4_shared_ln": {"pi/mlp_fc0/w": 1.69e-06, "pi/mlp_fc0/b": 1.10e-06, "pi/LayerNorm/beta": 1.72e-06,
                             "pi/LayerNorm/gamma": 9.94e-08, "pi/mlp_fc1/w": 7.27e-06, "pi/mlp_fc1/b": 3.91e-06,
                             "pi/LayerNorm_1/beta": 9.32e-06, "pi/LayerNorm_1/gamma": 3.51e-07, "pi/w": 1.07e-05,
                             "pi/b": 4.53e-09, "vf/w": 6.26e-06, "vf/b": 0.00e+00},
    "lstm_box7_gauss3_h128": {"pi/lstm/wx": 1.06e-05, "pi/lstm/b": 4.82e-06, "pi/lstm/wh": 1.73e-05, "pi/w": 2.97e-05,
                              "pi/b": 1.89e-09, "vf/w": 1.53e-05, "vf/b": 0.00e+00},
    "lstm_disc5_cat3_h64": {"pi/lstm/wx": 4.11e-05, "pi/lstm/b": 3.42e-06, "pi/lstm/wh": 1.02e-05, "pi/w": 6.46e-05,
                            "pi/b": 8.56e-09, "vf/w": 4.54e-05, "vf/b": 0.00e+00},
    "cnn_lstm_cat6_h64": {"pi/c1/w": 2.48e-09, "pi/c1/b": 1.25e-09, "pi/c2/w": 4.32e-08, "pi/c2/b": 1.15e-07,
                          "pi/c3/w": 8.82e-08, "pi/c3/b": 3.24e-06, "pi/fc1/w": 2.70e-07, "pi/fc1/b": 6.71e-06,
                          "pi/lstm/wx": 9.83e-09, "pi/lstm/b": 7.87e-06, "pi/lstm/wh": 4.68e-05, "pi/w": 5.72e-05,
                          "pi/b": 2.42e-08, "vf/w": 1.90e-05, "vf/b": 0.00e+00},
    "cnn_lstm_cat6_h128": {"pi/c1/w": 6.15e-09, "pi/c1/b": 1.00e-09, "pi/c2/w": 6.25e-08, "pi/c2/b": 6.15e-08,
                           "pi/c3/w": 5.18e-08, "pi/c3/b": 7.68e-07, "pi/fc1/w": 1.58e-07, "pi/fc1/b": 2.80e-05,
                           "pi/lstm/wx": 4.35e-08, "pi/lstm/b": 7.89e-06, "pi/lstm/wh": 2.28e-05, "pi/w": 8.62e-05,
                           "pi/b": 1.17e-08, "vf/w": 2.73e-05, "vf/b": 0.00e+00},
    "mlp_dueling_h64_32_double_ln": {"mlp_fc0/w": 5.20e-08, "mlp_fc0/b": 2.65e-08, "mlp_fc1/w": 1.60e-07,
                                     "mlp_fc1/b": 1.03e-07, "action_value/fully_connected/weights": 1.73e-06,
                                     "action_value/fully_connected/biases": 1.19e-06,
                                     "action_value/LayerNorm/beta": 1.27e-06, "action_value/LayerNorm/gamma": 7.50e-08,
                                     "action_value/fully_connected_1/weights": 8.26e-07,
                                     "action_value/fully_connected_1/biases": 1.80e-06,
                                     "action_value/LayerNorm_1/beta": 1.31e-06,
                                     "action_value/LayerNorm_1/gamma": 1.25e-08,
                                     "action_value/fully_connected_2/weights": 5.94e-08,
                                     "action_value/fully_connected_2/biases": 4.09e-09,
                                     "state_value/fully_connected/weights": 2.63e-06,
                                     "state_value/fully_connected/biases": 1.70e-06,
                                     "state_value/LayerNorm/beta": 2.44e-06, "state_value/LayerNorm/gamma": 1.74e-07,
                                     "state_value/fully_connected_1/weights": 1.78e-06,
                                     "state_value/fully_connected_1/biases": 5.26e-06,
                                     "state_value/LayerNorm_1/beta": 9.13e-09,
                                     "state_value/LayerNorm_1/gamma": 6.40e-08,
                                     "state_value/fully_connected_2/weights": 6.83e-08,
                                     "state_value/fully_connected_2/biases": 0.00e+00},
    "mlp_plain_h32_32_ln": {"mlp_fc0/w": 9.50e-08, "mlp_fc0/b": 6.40e-08, "mlp_fc1/w": 3.74e-07, "mlp_fc1/b": 2.02e-07,
                            "action_value/fully_connected/weights": 1.66e-06,
                            "action_value/fully_connected/biases": 7.98e-07, "action_value/LayerNorm/beta": 1.97e-06,
                            "action_value/LayerNorm/gamma": 9.48e-08,
                            "action_value/fully_connected_1/weights": 1.19e-06,
                            "action_value/fully_connected_1/biases": 3.34e-06,
                            "action_value/LayerNorm_1/beta": 1.92e-08, "action_value/LayerNorm_1/gamma": 7.49e-08,
                            "action_value/fully_connected_2/weights": 5.68e-07,
                            "action_value/fully_connected_2/biases": 2.43e-09},
    "conv_only_dueling_h256_ln": {"convnet/Conv/weights": 1.24e-07, "convnet/Conv/biases": 4.35e-08,
                                  "convnet/Conv_1/weights": 1.12e-07, "convnet/Conv_1/biases": 9.59e-08,
                                  "convnet/Conv_2/weights": 1.10e-07, "convnet/Conv_2/biases": 2.23e-06,
                                  "action_value/fully_connected/weights": 1.49e-07,
                                  "action_value/fully_connected/biases": 6.92e-06,
                                  "action_value/LayerNorm/beta": 7.82e-07, "action_value/LayerNorm/gamma": 2.17e-10,
                                  "action_value/fully_connected_1/weights": 6.79e-10,
                                  "action_value/fully_connected_1/biases": 7.42e-10,
                                  "state_value/fully_connected/weights": 2.20e-07,
                                  "state_value/fully_connected/biases": 1.89e-05,
                                  "state_value/LayerNorm/beta": 1.38e-08, "state_value/LayerNorm/gamma": 2.38e-10,
                                  "state_value/fully_connected_1/weights": 1.41e-09,
                                  "state_value/fully_connected_1/biases": 0.00e+00},
}
# these configurations' bounds join the table of test_update_composition_gpu.py, whose _assert_grads reads them
C.G.update({(c, t): 3.5 * max(v, 1e-8) for c, per in _OBSERVED.items() for t, v in per.items()})


def _shares(what, ref_g):
    """Each tensor's share of the global gradient norm: what a single relative-L2 check over all tensors cannot see."""
    tot = math.sqrt(sum(float((g * g).sum()) for g in ref_g.values()))
    sh = {C._short(k): math.sqrt(float((g * g).sum())) / tot for k, g in ref_g.items()}
    k = min(sh, key=sh.get)
    print(f"[share] {what}: smallest {k} {sh[k]:.2e}; " + ", ".join(f"{n} {v:.1e}" for n, v in sh.items()))


def _norm_mutants(params, ref_grads, M):
    """alpha left out of dgamma / dbeta (the norms' sums not scaled by 1/M), and each norm's dgamma / dbeta credited to
    the neighbouring LayerNorm of the same width."""
    norms = [k for k in params if "LayerNorm" in k]
    out = {}
    if not norms:
        return out
    noalpha = dict(ref_grads)
    for k in norms:
        noalpha[k] = ref_grads[k] * M
    out["alpha left out of dgamma / dbeta"] = (noalpha, set(norms))
    swapped, targets = dict(ref_grads), set()
    for k in norms:
        same = [o for o in norms if o != k and o.rsplit("/", 1)[1] == k.rsplit("/", 1)[1]
                and tuple(np.shape(params[o])) == tuple(np.shape(params[k]))]
        if same:
            swapped[k] = ref_grads[same[0]]
            targets.add(k)
    if targets:
        out["dgamma / dbeta credited to the neighbouring LayerNorm"] = (swapped, targets)
    return out


# ================================================================================================ PPO2
PPO_CLIP = {"mlp376_gauss17_copy_ln": 0.05, "lstm_disc5_cat3_h64": 0.05, "cnn_lstm_cat6_h128": 0.05}
C.PPO_CLIP.update(PPO_CLIP)                 # which case C._ppo_adam expects
RNN_T, RNN_E, RNN_NENV = 8, 12, 64     # steps per environment, environments per minibatch, environments in the rollout


def _ppo_model(name, M, nsteps=1, chunk=None, seed=0):
    from baselines_b200.common.policies import PolicyBuilder
    from baselines_b200.ppo2.model import Model
    cfg = N.PPO_RNN_LN_CONFIGS[name]
    ob, ac = C._spaces(dict(cfg, kind="cnn" if cfg["kind"] == "cnn_lstm" else "mlp"))
    kw = dict(layer_norm=True) if cfg.get("layer_norm") else {}
    if "nlstm" in cfg:
        kw["nlstm"] = cfg["nlstm"]
    np.random.seed(seed)
    pol = PolicyBuilder(ob, ac, cfg["kind"], value_network="copy" if cfg.get("copy") else None, **kw)
    model = Model(policy=pol, ob_space=ob, ac_space=ac, nbatch_act=8, nbatch_train=M, nsteps=nsteps, ent_coef=C.ENT,
                  vf_coef=C.VFC, max_grad_norm=PPO_CLIP.get(name, 1e3), comm=False, train_chunk=chunk or M)
    net = model.net
    rng = np.random.RandomState(seed + 100)
    p = net.store.export_tf("params")
    for k in p:
        if k.endswith("/b:0") and not k.endswith("logstd:0"):
            p[k] = (p[k] + 0.05 * rng.randn(*p[k].shape)).astype(np.float32)
    L.randomise_norms(p, rng)
    if net.pd == "gauss":
        p["ppo2_model/pi/logstd:0"] = (0.2 * rng.randn(1, net.nout)).astype(np.float32)
    model.set_params(p)
    assert net.pi_identity == N.ppo_identity(cfg) and not getattr(net, "fuse0", False)
    assert sum("LayerNorm" in k for k in p) == (4 * (2 if cfg.get("copy") else 1) if cfg.get("layer_norm") else 0)
    return model


def _x(net, cfg, raw):
    if cfg["kind"] == "cnn_lstm":
        return torch.as_tensor(raw).to(DEV).double()
    return C._encode(net, dict(cfg, kind="mlp"), raw)


def _masks(net, M):
    """ReLU decisions of the stored conv / fc1 activations below a cnn_lstm's cell (C._ppo_masks for the cnn base)."""
    t, masks = net.tower_pi, {}
    if t.base == "cnn":
        for i, c in enumerate(t.convs):
            masks[f"ppo2_model/pi/{c.name.split('/')[-1]}"] = (N.kernel_act(t, i, M) > 0).double()
        masks["ppo2_model/pi/fc1"] = (t.hfc[0][:M, :t.fcs[0].N] > 0).double()
    return masks


def _rollout(model, cfg, rng, n, seq=None):
    """C._ppo_rollout for these networks: the old policy's outputs from the mirror (over the whole rollout as one
    sequence for the recurrent ones)."""
    net = model.net
    pd, nout = cfg["ac"][0], net.nout
    raw = C._raw_obs(rng, dict(cfg, kind="cnn" if cfg["kind"] == "cnn_lstm" else "mlp"), n)
    P = net.store.export_tf("params")
    z = np.zeros(n)
    head = N.policy_ref(P, N.ppo_mirror_cfg(cfg), _x(net, cfg, raw), np.zeros((n, nout)), z, identity=net.pi_identity,
                        seq=seq, dev=DEV)
    mu, v = head.pi.cpu().numpy(), head.v.cpu().numpy()
    ls = P.get("ppo2_model/pi/logstd:0")
    acts = rng.randint(0, nout, n).astype(np.int64) if pd == "cat" else \
        (mu + np.exp(ls) * rng.randn(n, nout)).astype(np.float32)
    nlp = lr.ppo_ref(pd, mu, v, acts, z, z, z, z, 0.2, 0.0, 0.0, logstd=None if ls is None else ls[0]).nlp
    old_nlp = (nlp + 0.15 * rng.randn(n)).astype(np.float32)
    old_v = (v + 0.3 * rng.randn(n)).astype(np.float32)
    ret = (old_v + rng.randn(n)).astype(np.float32)
    dev = lambda a: torch.as_tensor(a).to(DEV).contiguous()
    obs = dev(raw) if cfg["kind"] == "cnn_lstm" else dev(raw.reshape(n, -1))
    return dict(raw=raw, obs=obs, acts=dev(acts), acts_np=acts, ret=dev(ret), oldv=dev(old_v), oldnlp=dev(old_nlp),
                np=dict(ret=ret, oldv=old_v, oldnlp=old_nlp))


FC1 = "ppo2_model/pi/fc1"


def _check_latent(what, ref, S, masks, latent):
    """cnn_lstm: the kernels' stored fc1 latent equals the mirror's within one fp16 rounding (the kernel rounds an fp32
    sum, the mirror a float64 one) plus G_MASK times the pre-activation's scale S.  The bound rejects the latent of the
    neighbouring row; a stale fc1 operand moves the latent by ~1% and fails it too."""
    mine = (ref.pres[FC1] * masks[FC1]).half().double()
    tol = 2.0 ** -10 * mine.abs() + C.G_MASK * S.pres[FC1]
    ratio = lambda v: float(((v.double() - mine).abs() / tol).max())
    worst = ratio(latent)
    C._report(f"{what} fc1 latent ({int((latent.double() != mine).sum())} of {mine.numel()} differ) |kernel - mirror| "
              "/ (one fp16 rounding + G_MASK S)", worst, 1.0)
    assert worst <= 1.0, (what, worst)
    assert ratio(torch.roll(latent, 1, 0)) > 1.0, "the latent bound does not reject the neighbouring row's"


def _check_grads(what, name, cfg, net, params, x, dpi, dv, masks, M, seq=None, seq_mutants=None):
    """(b) against the mirror seeded with the kernels' head-gradient rows.  Under a cnn_lstm's cell the mirror reads
    the kernels' stored fc1 latent once _check_latent has shown it equal to its own within one fp16 rounding: a
    rounding flip of that latent (values up to ~4, so a 2^-9 step) moves a whole row of the cell's input projection,
    and the recurrence carries it into every later step's h and dz."""
    mcfg, ident = N.ppo_mirror_cfg(cfg), net.pi_identity
    dpi, dv = dpi.to(DEV), dv.to(DEV)
    stored = None
    if FC1 in masks:
        t = net.tower_pi
        plain = N.policy_ref(params, mcfg, x, dpi, dv, rnd=True, masks=masks, identity=ident, seq=seq, dev=DEV)
        Sp = N.policy_ref(params, mcfg, x, dpi, dv, absolute=True, ref_acts=plain.acts, identity=ident, seq=seq,
                          dev=DEV)
        stored = {FC1: t.hfc[0][:M, :t.fcs[0].N]}
        _check_latent(what, plain, Sp, masks, stored[FC1])
    run = lambda sp, sv, **kw: N.policy_ref(params, mcfg, x, sp, sv, rnd=True, masks=masks, identity=ident, dev=DEV,
                                            stored=stored, **dict(dict(seq=seq), **kw))
    ref = run(dpi, dv)
    S = N.policy_ref(params, mcfg, x, dpi, dv, absolute=True, ref_acts=ref.acts, identity=ident, seq=seq, dev=DEV)
    C._check_masks(what, ref, S, masks)
    got = net.store.export_tf("grads")
    names = [k for k in got if not k.endswith("logstd:0")]
    _shares(what, {k: ref.grads[k] for k in names})
    # each head loses the one row with its largest gradient; for a recurrent network among the rows whose step does
    # not begin with a reset: a reset zeroes the row's h_{t-1} (its term of dWh = hprev^T dz) and cuts its carry to
    # the steps before, so dropping such a row can leave dWh unchanged
    live = torch.ones(len(dv), dtype=torch.bool, device=DEV) if seq is None else \
        torch.as_tensor(seq[0].reshape(-1) == 0, device=DEV)
    d0pi, d0v = dpi.clone(), dv.clone()
    d0pi[int(torch.where(live, dpi.abs().sum(1), -1.0).argmax())] = 0.0
    d0v[int(torch.where(live, dv.abs(), -1.0).argmax())] = 0.0
    muts = {"one sample dropped": (run(d0pi, d0v).grads, None)}
    muts.update(_norm_mutants(params, ref.grads, M))
    if seq is not None:
        for mn, (kw, targets) in seq_mutants.items():
            muts[mn] = (run(dpi, dv, **kw).grads, {k for k in names if any(t in k for t in targets)})
    C._assert_grads(what, name, got, ref.grads, S.grads, muts, names, 1.0 / M)


LN_PPO = [n for n, c in N.PPO_RNN_LN_CONFIGS.items() if c.get("layer_norm")]
RNN_PPO = [n for n, c in N.PPO_RNN_LN_CONFIGS.items() if "nlstm" in c]


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "src_idx_graph"])
@pytest.mark.parametrize("name", LN_PPO)
def test_ppo_layer_norm_update_composition_vs_float64(name, graph):
    cfg = N.PPO_RNN_LN_CONFIGS[name]
    M = C.PPO_M
    model = _ppo_model(name, M)
    net = model.net
    rng = np.random.RandomState(7)
    n = STEPS * M + 37
    roll = _rollout(model, cfg, rng, n)
    perm = rng.permutation(n)
    for step in range(STEPS):
        rows = perm[step * M:(step + 1) * M]
        what = f"{name} {'graph' if graph else 'eager'} step {step + 1}"
        replays = _lib.REPLAYS
        before, params = C._ppo_step(model, roll, rows, graph)
        C._assert_replayed(what, _lib.REPLAYS - replays, graph and step > 0)
        dpi, dv = C._check_ppo_heads(what, cfg, net, roll, rows, M, params)
        _check_grads(what, name, cfg, net, params, _x(net, cfg, roll["raw"][rows]), dpi, dv, {}, M)
        C._ppo_adam(what, name, model, before, M)


def _seq_rollout(model, cfg, rng):
    """RNN_NENV environments x RNN_T steps, buffer row t * RNN_NENV + e (the runner's layout), dones "before the step"
    with 20% resets, and non-zero start states."""
    H = model.net.nlstm
    n = RNN_T * RNN_NENV
    dones = (rng.rand(n) < 0.2).astype(np.uint8)
    states0 = (0.5 * rng.randn(RNN_NENV, 2 * H)).astype(np.float32)
    roll = _rollout(model, cfg, rng, n, seq=(dones.reshape(RNN_T, RNN_NENV).astype(np.float64),
                                             states0.astype(np.float64)))
    roll.update(dones=torch.as_tensor(dones).to(DEV), dones_np=dones, states0=torch.as_tensor(states0).to(DEV),
                states0_np=states0)
    return roll


def _envs(perm, step):
    """The environments of minibatch `step`: RNN_E consecutive entries of the permutation, wrapping around."""
    return np.resize(np.roll(perm, -step * RNN_E), RNN_E)


def _seq_step(model, roll, envs, graph):
    """One train_rollout_seq over environments `envs`; returns the pre-step state and parameters and the time-major
    buffer rows of the minibatch (the launch order of one chunk)."""
    rows = np.stack([np.arange(RNN_T) * RNN_NENV + e for e in envs])              # [E, T]
    before, params = C._flat_state(model.net.store), model.net.store.export_tf("params")
    model.train_rollout_seq(C.PPO_LR, C.CLIPRANGE, roll["obs"], roll["acts"], roll["ret"], roll["oldv"],
                            roll["oldnlp"], roll["dones"], roll["states0"], rows, envs, eager=not graph)
    torch.cuda.synchronize()
    return before, params, rows.T.reshape(-1)


def _seq_check(what, name, cfg, net, roll, envs, order, params, dpi, dv, M):
    E = len(envs)
    masks = roll["dones_np"][order].reshape(RNN_T, E).astype(np.float64)
    s0 = roll["states0_np"].astype(np.float64)
    shifted = np.concatenate([np.zeros((1, E)), masks[:-1]])
    below = ("/lstm/", "/c1/", "/c2/", "/c3/", "/fc1/")          # the cell and the tower under it
    mutants = {"start states of rows 0..E-1 (state_idx ignored)": (dict(seq=(masks, s0[:E])), below),
               "reset applied one step late": (dict(seq=(shifted, s0[envs])), below),
               "dWh from h_{t-1} before the mask": (dict(unmasked_dwh=True), ("/lstm/wh",))}
    _check_grads(what, name, cfg, net, params, _x(net, cfg, roll["raw"][order]), dpi, dv, _masks(net, M), M,
                 seq=(masks, s0[envs]), seq_mutants=mutants)


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("name", RNN_PPO)
def test_ppo_recurrent_update_composition_vs_float64(name, graph):
    cfg = N.PPO_RNN_LN_CONFIGS[name]
    M = RNN_E * RNN_T
    model = _ppo_model(name, M, nsteps=RNN_T)
    net = model.net
    rng = np.random.RandomState(11)
    roll = _seq_rollout(model, cfg, rng)
    perm = rng.permutation(RNN_NENV)
    for step in range(STEPS):
        envs = _envs(perm, step)
        what = f"{name} {'graph' if graph else 'eager'} step {step + 1}"
        replays = _lib.REPLAYS
        before, params, order = _seq_step(model, roll, envs, graph)
        C._assert_replayed(what, _lib.REPLAYS - replays, graph and step > 0)
        dpi, dv = C._check_ppo_heads(what, cfg, net, roll, order, M, params)
        _seq_check(what, name, cfg, net, roll, envs, order, params, dpi, dv, M)
        C._ppo_adam(what, name, model, before, M)


def test_ppo_recurrent_chunked_update():
    """(e) for train_rollout_seq: the minibatch's environments in two chunks of RNN_E / 2, graph-captured.  Each
    chunk's rows (head outputs, head gradients, h) are bit-identical to the unchunked run's, and the accumulated gradient
    meets (b) against the mirror seeded with the unchunked run's rows."""
    name = "lstm_box7_gauss3_h128"
    cfg = N.PPO_RNN_LN_CONFIGS[name]
    M, half = RNN_E * RNN_T, RNN_E // 2
    full, chunked = _ppo_model(name, M, nsteps=RNN_T), _ppo_model(name, M, nsteps=RNN_T, chunk=half * RNN_T)
    rng = np.random.RandomState(12)
    roll = _seq_rollout(full, cfg, rng)
    perm = rng.permutation(RNN_NENV)
    for step in range(STEPS):
        envs = _envs(perm, step)
        what = f"{name} chunked step {step + 1}"
        for k in ("params", "m", "v"):
            getattr(full.net.store, k).copy_(getattr(chunked.net.store, k))
        full.net.refresh()
        _, params, order = _seq_step(full, roll, envs, True)
        replays = _lib.REPLAYS
        before, params_c, _ = _seq_step(chunked, roll, envs, True)
        C._assert_replayed(what, _lib.REPLAYS - replays, step > 0)
        assert all(np.array_equal(params[k], params_c[k]) for k in params)
        # the second chunk is environments half.. of the minibatch: rows t * half + e' of its launch order
        sec = torch.as_tensor([t * RNN_E + half + e for t in range(RNN_T) for e in range(half)])
        for a, b in zip(C._ppo_heads(full.net, M), C._ppo_heads(chunked.net, half * RNN_T)):
            assert torch.equal(a[sec], b), "per-row head outputs / gradients depend on the chunking"
        assert torch.equal(full.net.tower_pi.lstm.h[:M][sec], chunked.net.tower_pi.lstm.h[:half * RNN_T])
        dpi, dv = C._check_ppo_heads(what + " (unchunked)", cfg, full.net, roll, order, M, params)
        _seq_check(what, name, cfg, chunked.net, roll, envs, order, params, dpi, dv, M)
        C._ppo_adam(what, name, chunked, before, M)


# ================================================================================================ DQN
# grad_norm_clipping and the importance-weight scale per configuration: with a clip, the first update's clip scales
# some variables and leaves others, and in conv_only_dueling_h256_ln a norm's variable is among the scaled ones
DQN_CLIP = {"mlp_dueling_h64_32_double_ln": 10.0, "mlp_plain_h32_32_ln": None, "conv_only_dueling_h256_ln": 10.0}
DQN_W_SCALE = {"mlp_dueling_h64_32_double_ln": 40.0, "conv_only_dueling_h256_ln": 200.0}


def _dqn_model(name, seed=3):
    from baselines_b200.deepq.build_graph import DQNModel
    from baselines_b200.common import spaces
    cfg = N.DQN_LN_CONFIGS[name]
    oa = cfg["ob"][1]
    ob = spaces.Box(0, 255, oa, np.uint8) if cfg["kind"] != "mlp" else spaces.Box(-5, 5, oa, np.float32)
    model = DQNModel(ob, C.DQN_NA, cfg["kind"], lr=C.DQN_LR, gamma=C.GAMMA, grad_norm_clipping=DQN_CLIP[name],
                     double_q=cfg["double_q"], batch_cap=C.DQN_B, seed=seed, hiddens=cfg["hiddens"],
                     dueling=cfg["dueling"], layer_norm=True)
    rng = np.random.RandomState(seed + 100)
    p = model.q.store.export_tf("params")
    for k in p:
        if "biases" in k or k.endswith("/b:0"):
            p[k] = (p[k] + 0.05 * rng.randn(*p[k].shape)).astype(np.float32)
    L.randomise_norms(p, rng)
    assert sum("LayerNorm" in k for k in p) == 2 * len(cfg["hiddens"]) * (2 if cfg["dueling"] else 1)
    model.q.store.import_tf(p, "params")
    model.q.refresh()
    model.update_target()
    p2 = {k: (v + 0.01 * rng.randn(*v.shape)).astype(np.float32) for k, v in p.items()}
    model.qt.store.import_tf({k.replace("q_func", "target_q_func", 1): v for k, v in p2.items()}, "params")
    model.qt.refresh()
    return model


@pytest.mark.parametrize("replay", [False, True], ids=["gathered", "replay_idx"])
@pytest.mark.parametrize("name", list(N.DQN_LN_CONFIGS))
def test_dqn_layer_norm_update_composition_vs_float64(name, replay):
    cfg = N.DQN_LN_CONFIGS[name]
    B = C.DQN_B
    model = _dqn_model(name)
    q = model.q
    rng = np.random.RandomState(9)
    n = STEPS * B + 41
    b = C._dqn_batch(rng, cfg, n)
    dev = lambda a: torch.as_tensor(a).to(DEV).contiguous()
    store = {k: dev(v) for k, v in b.items()}
    perm = rng.permutation(n)
    mcfg = N.dqn_mirror_cfg(cfg)
    seg_names = [s[0] for s in q.store._specs]
    for step in range(STEPS):
        rows = perm[step * B:(step + 1) * B]
        what = f"{name} {'replay' if replay else 'gathered'} step {step + 1}"
        replays = _lib.REPLAYS
        w = ((rng.rand(B) * 0.9 + 0.1) * DQN_W_SCALE.get(name, 1.0)).astype(np.float32)
        before = C._flat_state(q.store)
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
        C._assert_replayed(what, _lib.REPLAYS - replays, replay and step > 0)
        da, ds = C._check_dqn_heads(what, model, cfg, b, rows, w, B)
        x = C._dqn_x(cfg, b["o_t"][rows])
        masks = C._dqn_masks(q, B)
        ds_d = None if ds is None else ds.to(DEV)
        ref = N.q_ref(params, mcfg, x, da.to(DEV), ds_d, rnd=True, masks=masks, dev=DEV)
        S = N.q_ref(params, mcfg, x, da.to(DEV), ds_d, absolute=True, ref_acts=ref.acts, dev=DEV)
        C._check_masks(what, ref, S, masks)
        got = q.store.export_tf("grads")
        names = list(got)
        _shares(what, ref.grads)
        muts = C._dqn_mutants(cfg, params, x, da.to(DEV), ds_d, masks, mcfg, names)
        muts.update(_norm_mutants(params, ref.grads, B))
        C._assert_grads(what, name, got, ref.grads, S.grads, muts, names, 1.0 / B)
        # (c) per-variable clip_by_norm, then Adam
        g_flat = q.store.grads.detach().double().cpu().numpy()
        off = q.store.segment_offsets()
        clip = DQN_CLIP[name]
        scale = np.ones_like(g_flat)
        facs = []
        for s0, s1 in zip(off[:-1], off[1:]):
            seg = g_flat[s0:s1]
            f = lr.clip_scale(math.fsum(seg * seg), clip) if clip else 1.0
            scale[s0:s1] = f
            facs.append(f)
        print(f"[observed] {what} per-variable clip factors: "
              + ", ".join(f"{nm} {f:.3f}" for nm, f in zip(seg_names, facs)))
        if clip is None:
            assert all(f == 1.0 for f in facs)
        elif step == 0:
            assert min(facs) < 1.0 and max(facs) == 1.0, facs
            assert any(f < 1.0 for nm, f in zip(seg_names, facs) if "/ln" in nm) == (cfg["kind"] == "conv_only"), facs
        C._check_adam(what, q.store, before, g_flat, C._lr_t(C.DQN_LR), model.opt.t, 1e-8, scale, min(facs) < 1.0)
