"""CPU: the float64 network mirror (tests/_net_refs.py), rounding off, equals the CPU oracle (oracle/nets.py) run in
float64 on every network of tests/test_update_composition_gpu.py and tests/test_update_composition_rnn_ln_gpu.py: the
same head outputs, and the same gradient of every TF variable when it is seeded with the oracle's own d(loss)/d(head)
-- from ppo_loss / the DQN Huber loss where the oracle has that network, from a random seed on the head outputs
otherwise.  The layer-normalised networks run the oracle with tests/_layer_norm_refs.py's norms, the recurrent ones
against tests/_lstm_oracle.py (env-major rows there, time-major in the mirror).  This ties the mirror the GPU tests
trust to the restated reference."""
import math

import numpy as np
import pytest
import torch

import _layer_norm_refs as L
import _lstm_oracle as LO
import _net_refs as N
from oracle import nets

RTOL = 1e-12


def _close(got, want, what):
    got, want = torch.as_tensor(got).double(), torch.as_tensor(want).double()
    assert got.shape == want.shape, (what, got.shape, want.shape)
    atol = RTOL * float(want.abs().max()) if want.numel() else 0.0
    err = float((got - want).abs().max()) if want.numel() else 0.0
    assert torch.allclose(got, want, rtol=RTOL, atol=atol), f"{what}: max |mirror - oracle| = {err:.3e}"


def _ppo_case(name, B=7, seed=0):
    cfg = N.PPO_CONFIGS[name] if name in N.PPO_CONFIGS else N.PPO_RNN_LN_CONFIGS[name]
    rng = np.random.RandomState(seed)
    okind = cfg["ob"][0]
    if cfg["kind"] == "cnn":
        obs = rng.randint(0, 256, (B,) + cfg["ob"][1]).astype(np.uint8)
        x = obs
    elif okind == "discrete":
        x = N.encode_obs(rng.randint(0, cfg["ob"][1], B).astype(np.float32), onehot_n=cfg["ob"][1])
    elif okind == "mdisc":
        nv = cfg["ob"][1]
        x = N.encode_obs(np.stack([rng.randint(0, n, B) for n in nv], 1).astype(np.float32), nvec=list(nv))
    else:
        x = (rng.randn(B, *cfg["ob"][1]) * 3).astype(np.float32).astype(np.float64)
    nout = N.ppo_nout(cfg["ac"])
    net_kw = dict(num_layers=cfg.get("num_layers", 2), num_hidden=cfg.get("num_hidden", 64)) \
        if cfg["kind"] == "mlp" else {}
    params = nets.init_policy_params(cfg["kind"], N.in_dim(cfg["ob"]), "box" if cfg["ac"][0] == "gauss" else "discrete",
                                     nout, value_network="copy" if cfg.get("copy") else None, seed=seed, **net_kw)
    # non-zero biases, so that a missing bias term shows
    if cfg.get("layer_norm"):
        params = L.randomise_norms(L.with_policy_norms(params, num_layers=cfg.get("num_layers", 2)), rng)
    params = {k: (v + 0.1 * rng.randn(*v.shape).astype(np.float32)) if k.endswith("/b:0") else v
              for k, v in params.items()}
    return cfg, params, x, nout, rng



def _oracle_policy(tp, cfg, x):
    """oracle/nets.py policy_forward, with the mlp depth of the configuration."""
    scope = "ppo2_model"
    if cfg["kind"] == "cnn":
        lat_fn = lambda pfx: nets.nature_cnn(tp, pfx, x)
    else:
        lat_fn = lambda pfx: nets.mlp(tp, pfx, x, num_layers=cfg.get("num_layers", 2))
    lat = lat_fn(f"{scope}/pi")
    vlat = lat_fn(f"{scope}/vf") if cfg.get("copy") else lat
    pi = lat @ tp[f"{scope}/pi/w:0"] + tp[f"{scope}/pi/b:0"] if f"{scope}/pi/w:0" in tp else lat
    return pi, (vlat @ tp[f"{scope}/vf/w:0"] + tp[f"{scope}/vf/b:0"])[:, 0]


def _check_policy(name, cfg, params, x, tp, pi, v, dpi, dv):
    ref = N.policy_ref(params, N.ppo_mirror_cfg(cfg), x, dpi, dv, identity=N.ppo_identity(cfg))
    _close(ref.pi, pi.detach(), f"{name} pi")
    _close(ref.v, v.detach(), f"{name} v")
    for k, t in tp.items():
        if k.endswith("logstd:0"):
            continue
        _close(ref.grads[k], t.grad, f"{name} d/d {k}")
    if N.ppo_identity(cfg):
        assert "ppo2_model/pi/w:0" not in params
        _close(ref.grads["head_pi/w"], _lat_grad(tp, cfg, x, dpi), f"{name} identity head w")
        _close(ref.grads["head_pi/b"], torch.as_tensor(dpi).sum(0), f"{name} identity head b")


def _lat_grad(tp, cfg, x, dpi):
    """Gradient of the identity head's weight: latent^T dpi."""
    with torch.no_grad():
        lat = nets.mlp(tp, "ppo2_model/pi", torch.as_tensor(x), num_layers=cfg.get("num_layers", 2))
    return lat.t() @ torch.as_tensor(dpi)


@pytest.mark.parametrize("name", list(N.PPO_CONFIGS))
def test_policy_mirror_matches_oracle_forward_and_gradient(name):
    cfg, params, x, nout, rng = _ppo_case(name)
    tp = nets.to_torch(params, torch.float64, requires_grad=True)
    pi, v = _oracle_policy(tp, cfg, torch.as_tensor(x))
    dpi, dv = rng.randn(*pi.shape), rng.randn(*v.shape)
    ((pi * torch.as_tensor(dpi)).sum() + (v * torch.as_tensor(dv)).sum()).backward()
    _check_policy(name, cfg, params, x, tp, pi, v, dpi, dv)


PPO_LOSS_CASES = [n for n, c in N.PPO_CONFIGS.items() if c["ac"][0] in ("cat", "gauss") and c.get("num_layers", 2) == 2]


@pytest.mark.parametrize("name", PPO_LOSS_CASES)
def test_policy_mirror_seeded_by_ppo_loss_matches_oracle_autograd(name, monkeypatch):
    """d(ppo_loss)/d(param) of the oracle == the mirror seeded with the oracle's d(ppo_loss)/d(pi, v)."""
    cfg, params, x, nout, rng = _ppo_case(name, B=9, seed=1)
    B = x.shape[0]
    tp = nets.to_torch(params, torch.float64, requires_grad=True)
    heads = {}
    orig = nets.policy_forward

    def spy(*a, **k):
        pi, ls, vf = orig(*a, **k)
        pi.retain_grad()
        vf.retain_grad()
        heads.update(pi=pi, vf=vf)
        return pi, ls, vf
    monkeypatch.setattr(nets, "policy_forward", spy)
    if cfg["ac"][0] == "cat":
        acts = torch.as_tensor(rng.randint(0, nout, B))
    else:
        acts = torch.as_tensor(rng.randn(B, nout))
    f = lambda a: torch.as_tensor(a, dtype=torch.float64)
    loss, _ = nets.ppo_loss(tp, cfg["kind"], torch.as_tensor(x), acts, f(rng.randn(B)), f(rng.randn(B)),
                            f(rng.randn(B) + math.log(max(nout, 2))), f(rng.randn(B)), 0.2, 0.01, 0.5,
                            value_network="copy" if cfg.get("copy") else None)
    loss.backward()
    pi, vf = heads["pi"], heads["vf"]
    _check_policy(name, cfg, params, x, tp, pi, vf, pi.grad.numpy(), vf.grad.numpy())


def _dqn_case(name, B=7, seed=0):
    cfg = N.DQN_CONFIGS[name] if name in N.DQN_CONFIGS else N.DQN_LN_CONFIGS[name]
    rng = np.random.RandomState(seed)
    nA = 6
    if cfg["kind"] != "mlp":
        x = rng.randint(0, 256, (B,) + cfg["ob"][1]).astype(np.uint8)
    elif cfg["ob"][0] == "discrete":
        x = N.encode_obs(rng.randint(0, cfg["ob"][1], B).astype(np.float32), onehot_n=cfg["ob"][1])
    else:
        x = (rng.randn(B, *cfg["ob"][1]) * 2).astype(np.float32).astype(np.float64)
    params = nets.init_q_params(cfg["kind"], N.in_dim(cfg["ob"]), nA, hiddens=cfg["hiddens"], dueling=cfg["dueling"],
                                seed=seed)
    if cfg.get("layer_norm"):
        params = L.randomise_norms(L.with_q_norms(params, len(cfg["hiddens"])), rng)
    params = {k: (v + 0.1 * rng.randn(*v.shape).astype(np.float32)) if ("/b:0" in k or "biases" in k) else v
              for k, v in params.items()}
    return cfg, params, x, nA, rng


@pytest.mark.parametrize("name", list(N.DQN_CONFIGS) + list(N.DQN_LN_CONFIGS))
def test_q_mirror_seeded_by_td_loss_matches_oracle_autograd(name, monkeypatch):
    """q(s) and d(Huber TD loss)/d(param) of the oracle's DQN step == the mirror's A, S and its gradient seeded with
    d loss / dA = dq - mean(dq), d loss / dS = sum(dq) (dueling) or dq.  The layer-normalised streams run the oracle
    with _layer_norm_refs.q_forward."""
    cfg, params, x, nA, rng = _dqn_case(name)
    if cfg.get("layer_norm"):
        monkeypatch.setattr(nets, "q_forward", L.q_forward)
    B = x.shape[0]
    oracle = nets.DQNOracle(params, cfg["kind"], 0.99, n_hidden=len(cfg["hiddens"]), dueling=cfg["dueling"],
                            double_q=cfg["double_q"], dtype=torch.float64)
    for t in oracle.tp.values():
        t.requires_grad_(True)
    qs = []
    orig = nets.q_forward

    def spy(*a, **k):
        q = orig(*a, **k)
        if q.requires_grad:
            q.retain_grad()
        qs.append(q)
        return q
    monkeypatch.setattr(nets, "q_forward", spy)
    x1 = x[::-1].copy()
    _, loss = oracle.td_and_loss(x, rng.randint(0, nA, B), rng.randn(B), x1, (rng.rand(B) < 0.2).astype(np.float64),
                                 rng.rand(B) + 0.1)
    loss.backward()
    q = qs[0]
    dq = q.grad.numpy()
    if cfg["dueling"]:
        da, ds = dq - dq.mean(1, keepdims=True), dq.sum(1)
    else:
        da, ds = dq, None
    ref = N.q_ref(params, N.dqn_mirror_cfg(cfg), x, da, ds)
    assert list(ref.grads) == list(params)                       # TF names, in creation order
    qm = ref.A if not cfg["dueling"] else ref.S[:, None] + ref.A - ref.A.mean(1, keepdim=True)
    _close(qm, q.detach(), f"{name} q")
    for k, t in oracle.tp.items():
        _close(ref.grads[k], t.grad, f"{name} d/d {k}")


def test_encode_obs_matches_oracle_normalisation():
    """The mirror's float32 encoder (x - mean) * inv_std against the oracle's (x - mean) / std: within fp32 rounding,
    and identical after the +-5 clip."""
    rng = np.random.RandomState(4)
    obs = (rng.randn(50, 11) * 6).astype(np.float32)
    rms = dict(runningsum=rng.randn(11) * 3, runningsumsq=rng.rand(11) * 40 + 10, count=10.0)
    mean = (rms["runningsum"] / rms["count"]).astype(np.float32)
    std = np.sqrt(np.maximum((rms["runningsumsq"] / rms["count"]).astype(np.float32) - mean * mean, np.float32(1e-2)))
    got = N.encode_obs(obs, mean=mean, inv_std=np.float32(1.0) / std)
    want = nets.encode_observation(obs, torch.float32, rms=rms).double().numpy()
    assert np.allclose(got, want, rtol=2 ** -22, atol=0) and (np.abs(want) == 5).any()


@pytest.mark.parametrize("name", ["mlp13_cat15_l3_h20", "mlp11_gauss3_copy_l1_h32"])
def test_policy_mirror_takes_stored_tanh_activations(name):
    """A tanh layer's entry in `masks` replaces its stored activation in the forward: the mirror's own activations
    reproduce its outputs exactly, and a changed activation reaches the heads."""
    cfg, params, x, nout, rng = _ppo_case(name)
    mcfg, ident = N.ppo_mirror_cfg(cfg), N.ppo_identity(cfg)
    z, zv = np.zeros((len(x), nout)), np.zeros(len(x))
    ref = N.policy_ref(params, mcfg, x, z, zv, rnd=True, identity=ident)
    tanh_acts = {k: a for k, a in ref.acts.items() if "mlp_fc" in k}
    same = N.policy_ref(params, mcfg, x, z, zv, rnd=True, masks=tanh_acts, identity=ident)
    assert torch.equal(same.pi, ref.pi) and torch.equal(same.v, ref.v)
    last = [k for k in tanh_acts if k.startswith("ppo2_model/pi/")][-1]
    moved = dict(tanh_acts, **{last: tanh_acts[last] * 0.5})
    other = N.policy_ref(params, mcfg, x, z, zv, rnd=True, masks=moved, identity=ident)
    assert not torch.equal(other.pi, ref.pi)


LN_PPO = [n for n, c in N.PPO_RNN_LN_CONFIGS.items() if c.get("layer_norm")]
RNN_PPO = [n for n, c in N.PPO_RNN_LN_CONFIGS.items() if "nlstm" in c]


@pytest.mark.parametrize("name", LN_PPO)
def test_layer_norm_policy_mirror_matches_oracle(name, monkeypatch):
    """mlp(layer_norm=True): the mirror against oracle/nets.py with _layer_norm_refs.mlp, every norm's gamma and beta
    included, under the reference's names and in its creation order."""
    cfg, params, x, nout, rng = _ppo_case(name)
    assert sum("LayerNorm" in k for k in params) == 4 * (2 if cfg.get("copy") else 1)
    monkeypatch.setattr(nets, "mlp", L.mlp)
    tp = nets.to_torch(params, torch.float64, requires_grad=True)
    pi, v = _oracle_policy(tp, cfg, torch.as_tensor(x))
    dpi, dv = rng.randn(*pi.shape), rng.randn(*v.shape)
    ((pi * torch.as_tensor(dpi)).sum() + (v * torch.as_tensor(dv)).sum()).backward()
    _check_policy(name, cfg, params, x, tp, pi, v, dpi, dv)
    ref = N.policy_ref(params, N.ppo_mirror_cfg(cfg), x, dpi, dv)
    assert list(ref.grads) == [k for k in params if not k.endswith("logstd:0")]


def _recurrent_case(name, T, E, seed=0):
    """Parameters, env-major raw observations / masks (the oracle's rows e*T + t), start states, and the time-major
    order of the mirror's rows."""
    cfg = N.PPO_RNN_LN_CONFIGS[name]
    rng = np.random.RandomState(seed)
    (ok, oa), nout, H = cfg["ob"], N.ppo_nout(cfg["ac"]), cfg["nlstm"]
    onehot = oa if ok == "discrete" else 0
    params = LO.init_recurrent_params(cfg["kind"], oa if ok == "box" else (), "box" if cfg["ac"][0] == "gauss" else
                                      "discrete", nout, nlstm=H, seed=seed, onehot_n=onehot)
    params = {k: (v + 0.1 * rng.randn(*v.shape).astype(np.float32)) if k.endswith("/b:0") else v
              for k, v in params.items()}
    n = T * E
    if cfg["kind"] == "cnn_lstm":
        obs = rng.randint(0, 256, (n,) + oa).astype(np.uint8)
    elif onehot:
        obs = rng.randint(0, onehot, n)
    else:
        obs = (rng.randn(n, *oa) * 2).astype(np.float32)
    masks = (rng.rand(n) < 0.3).astype(np.float64)
    states = rng.randn(E, 2 * H) * 0.5
    tm = np.array([e * T + t for t in range(T) for e in range(E)])
    return cfg, params, obs, masks, states, tm, onehot, rng


def _mirror_rows(cfg, obs, onehot):
    if cfg["kind"] == "cnn_lstm":
        return obs
    return N.encode_obs(obs.astype(np.float32), onehot_n=onehot)


@pytest.mark.parametrize("name", RNN_PPO)
def test_recurrent_policy_mirror_matches_lstm_oracle(name):
    """lstm / cnn_lstm: the mirror over time-major rows with per-row masks and per-environment start states against
    _lstm_oracle.recurrent_forward (a2c/utils.py lstm() through autograd), forward and every TF variable's gradient."""
    T, E = 4, 3
    cfg, params, obs, masks, states, tm, onehot, rng = _recurrent_case(name, T, E)
    tp = nets.to_torch(params, torch.float64, requires_grad=True)
    pi, _, v, _ = LO.recurrent_forward(tp, cfg["kind"], torch.as_tensor(obs), masks, states, E, onehot_n=onehot)
    dpi, dv = rng.randn(*pi.shape), rng.randn(*v.shape)
    ((pi * torch.as_tensor(dpi)).sum() + (v * torch.as_tensor(dv)).sum()).backward()
    seq = (masks.reshape(E, T).T.copy(), states)
    ref = N.policy_ref(params, N.ppo_mirror_cfg(cfg), _mirror_rows(cfg, obs[tm], onehot), dpi[tm], dv[tm], seq=seq)
    _close(ref.pi, pi.detach()[tm], f"{name} pi")
    _close(ref.v, v.detach()[tm], f"{name} v")
    assert list(ref.grads) == [k for k in params if not k.endswith("logstd:0")]
    for k, t in tp.items():
        if not k.endswith("logstd:0"):
            _close(ref.grads[k], t.grad, f"{name} d/d {k}")


@pytest.mark.parametrize("name", ["cnn84_cat6_shared", "mlp376_gauss17_copy_h64"])
def test_sliced_mirror_equals_unsliced(name):
    """policy_ref_sliced over uneven slices (3, 3, 1 rows, ReLU decisions handed in per slice) against one policy_ref
    pass over all rows: the same head outputs, gradients and absolute network S, to float64 rounding; every slice is
    handed to `each` once, in order."""
    cfg, params, x, nout, rng = _ppo_case(name)
    mcfg, ident = N.ppo_mirror_cfg(cfg), N.ppo_identity(cfg)
    dpi, dv = rng.randn(len(x), nout), rng.randn(len(x))
    ref = N.policy_ref(params, mcfg, x, dpi, dv, rnd=True, identity=ident)
    S = N.policy_ref(params, mcfg, x, dpi, dv, absolute=True, ref_acts=ref.acts, identity=ident)
    masks = {k: a for k, a in ref.acts.items() if cfg["kind"] == "cnn"}
    seen = []
    sl = N.policy_ref_sliced(params, mcfg, x, dpi, dv, 3, masks=lambda s, e: {k: m[s:e] for k, m in masks.items()},
                             each=lambda s, e, r, a: seen.append((s, e, len(r.pi), len(a.pi))), identity=ident)
    assert seen == [(0, 3, 3, 3), (3, 6, 3, 3), (6, 7, 1, 1)]
    _close(sl.pi, ref.pi, f"{name} sliced pi")
    _close(sl.v, ref.v, f"{name} sliced v")
    assert list(sl.grads) == list(ref.grads) and list(sl.S) == list(S.grads)
    for k in ref.grads:
        _close(sl.grads[k], ref.grads[k], f"{name} sliced d/d {k}")
        _close(sl.S[k], S.grads[k], f"{name} sliced S of {k}")


@pytest.mark.parametrize("name", ["lstm_box7_gauss3_h128", "mlp11_cat4_shared_ln"])
def test_absolute_mirror_bounds_the_signed_one(name):
    """The absolute network (the error scale S) through a LayerNorm or the LSTM cell: every output and gradient is at
    least as large as the signed run's, element by element."""
    if name in RNN_PPO:
        T, E = 5, 3
        cfg, params, obs, masks, states, tm, onehot, rng = _recurrent_case(name, T, E, seed=3)
        x, kw = _mirror_rows(cfg, obs[tm], onehot), dict(seq=(masks.reshape(E, T).T.copy(), states))
    else:
        cfg, params, x, nout, rng = _ppo_case(name, B=9, seed=3)
        kw = {}
    mcfg = N.ppo_mirror_cfg(cfg)
    n, nout = len(x), N.ppo_nout(cfg["ac"])
    dpi, dv = rng.randn(n, nout), rng.randn(n)
    ref = N.policy_ref(params, mcfg, x, dpi, dv, rnd=True, **kw)
    S = N.policy_ref(params, mcfg, x, dpi, dv, absolute=True, ref_acts=ref.acts, **kw)
    assert (S.pi >= ref.pi.abs() * (1 - 1e-12)).all() and (S.v >= ref.v.abs() * (1 - 1e-12)).all()
    for k, g in ref.grads.items():
        assert (S.grads[k] >= g.abs() * (1 - 1e-9) - 1e-300).all(), k
