"""GPU: the acting passes of every PPO2 and DQN network against the float64 network mirror, at the batch sizes they act
with, eagerly and replayed from a CUDA graph.

Every rollout's actions, values and neglogpacs come from the acting pass, and so does every DQN action.  It does not run
the train forward's launch sequence: PolicyNet.act runs forward(masks=False), so the shift-GEMM convs write no ReLU bit
mask; it runs at B = nenv (or nenv / act_chunks), B = 1 for a single-env run; and it is captured once per rollout slot
and replayed, reading the sampler's stream position (PolicyNet.rng_ctr) and DQN's epsilon and step from device memory.

  1. Model.step / Model.value for every N.PPO_CONFIGS entry at B in BATCHES (and a B > 4096 for mlp):
     a. logits (pi_out) and value against policy_ref(rnd=True) with the ReLU decisions and stored tanh activations of
        the kernels: |got - ref| <= g * S + 2^-23 |ref|, S the mirror's absolute network;
     b. actions equal the float64 sampler at the kernel's logits and the injected noise (Gumbel-max per segment,
        Bernoulli threshold, mu + sigma n), rows at a Gumbel tie excluded; neglogp equals the float64 neglogp of that
        action within NLP_ROUNDINGS fp32 roundings of the sum of its terms' magnitudes;
     c. value() is bit-identical to step()'s value (value() runs the train forward with masks);
     d. a row does not depend on the batch: rows of a smaller acting pass and of the train forward (forward(masks=True)
        gathered through src_idx) are bit-identical to the acting pass's rows.
  2. Graph replay and the sampler stream: replay equals eager bit for bit; rng_ctr advances once per pass and every
     pass's samples are the host Philox4x32-10 stream at that position (_loss_refs.philox_uniforms); chunked acting
     with frame stacking equals an unchunked pass; empirical frequencies of the mcat and bern heads at B = 1 and 7.
  3. Runner.run_device (T = 5, N = 7, host and device env): every slot equals a step on its observations, checked as
     in 1; last_values equal value() at the final observation.
  4. DQN act / q_values for every N.DQN_CONFIGS entry: A, S and q against q_ref(rnd=True) and dueling_q; the greedy
     action is the argmax (lowest index at exact ties); eps = 1 draws exactly the host splitmix64 stream and is uniform;
     eps and the step are read from the device on replay.
  5. The observation encoder's edges: fp16 range (values >= 65520 raise ValueError instead of turning into NaN), the
     precision max(2^-22 |v|, 2^-25), the normalisation clip, one-hot blocks across 8-column groups and out-of-range
     Discrete values.

Tolerances: every g is 3.5x the maximum observed on an H100 80GB HBM3 (700 W power limit); the observed values are
listed next to the constants and each run prints its own [observed] lines.  Every bound is shown to reject the
mutants named next to it.
"""
import numpy as np
import pytest
import torch

import _loss_refs as lr
import _net_refs as N
import _refs as R
from baselines_b200 import _lib, ops
from test_update_composition_gpu import _dqn_masks, _norm_arrays, _ppo_masks, _spaces

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
U32 = 2.0 ** -24
BATCHES = (1, 2, 7, 63, 64, 65, 127, 128, 129, 1000)
BIG_MLP_B = 5000                   # above 4096: more rows than 32 waves of the 128-row GEMM tiles on 132 SMs

# g of the logits / value bound per configuration: 3.5x the maximum observed over every batch size, the runner and the
# encoder-edge tests on an H100 80GB HBM3 (700 W power limit), floor 1e-10.  Observed (pi, v):
_OBSERVED = {
    "cnn84_cat6_shared": (1.46e-09, 9.99e-10),
    "cnn84_cat6_copy": (1.42e-09, 8.52e-10),
    "cnn64_cat6_shared": (2.94e-09, 2.07e-09),
    "mlp376_gauss17_copy_h64": (6.16e-08, 6.70e-08),
    "mlp11_gauss3_copy_h256": (4.58e-08, 1.05e-07),
    "mlp11_gauss3_copy_l1_h32": (3.95e-08, 5.23e-08),
    "mlp13_cat15_l3_h20": (1.10e-07, 6.93e-08),
    "mlp_disc10_cat4": (0.0, 1.17e-08),
    "mlp_mdisc33_mcat33": (0.0, 3.47e-09),
    "mlp5_gauss32_copy_identity": (0.0, 4.37e-08),          # identity head: the logits are the stored latent
    "mlp11_bern5_normalized": (6.52e-09, 6.24e-08),
}
G_PI = {k: 3.5 * max(v[0], 1e-10) for k, v in _OBSERVED.items()}
G_V = {k: 3.5 * max(v[1], 1e-10) for k, v in _OBSERVED.items()}
# g of the hidden mlp layers' pre-activations behind each stored tanh activation, every configuration (PPO2 and DQN)
G_PRE = 3.5 * 7.93e-08                # observed on an H100 80GB HBM3 (700 W power limit): 7.93e-08
# DQN: (A, S) per configuration, same rule; q_values take 2 max(g_A, g_S) on |S| + |A| + mean |A|.  Observed:
_OBSERVED_DQN = {
    "mlp_dueling_h64_32_double": (4.90e-06, 3.06e-06),
    "mlp_plain_h20_max": (3.14e-07, 0.0),
    "mlp_dueling_h20_double": (3.14e-07, 4.95e-08),
    "cnn_dueling_h256": (1.44e-10, 1.35e-10),
    "conv_only_dueling_h256": (7.77e-10, 6.14e-10),
    "mlp_disc7_dueling_h64": (2.67e-09, 2.90e-09),
}
G_A = {k: 3.5 * max(v[0], 1e-10) for k, v in _OBSERVED_DQN.items()}
G_S = {k: 3.5 * max(v[1], 1e-10) for k, v in _OBSERVED_DQN.items()}
# neglogp: |got - ref| <= NLP_ROUNDINGS(n) * 2^-24 * (sum of the magnitudes of its terms), n = logits per row.  The
# kernels evaluate max, n expf, a sum of n terms, logf and one subtraction per segment (cat / mcat), n sigmoid
# cross-entropies of three terms each (bern), or n divisions, squares and sums plus the constant (gauss).  The most
# observed on an H100 is 3.3 roundings.
NLP_ROUNDINGS = lambda n: 4 * n + 16


def _report(what, seen, g):
    print(f"[observed] {what}: g = {seen:.3e} (allowed {g:.3e})")


def _bound(what, got, ref, S, g, mutants):
    """|got - ref| <= g S + 2^-23 |ref|, rejecting every mutant; prints the observed g and each mutant's g."""
    for mn, m in mutants.items():
        print(f"[mutant] {what} {mn}: g = {R.excess(m, ref, S, R.R_F32):.3e}")
    seen = R.assert_within(got, ref, S, g, R.R_F32, mutants, what)
    _report(what, seen, g)
    return seen


# ================================================================================================ PPO2 models
def _act_model(name, B, seed=0):
    """The real Model with nbatch_act = B; biases moved off zero, obs_rms installed for the normalised network."""
    from baselines_b200.common.policies import PolicyBuilder
    from baselines_b200.ppo2.model import Model
    cfg = N.PPO_CONFIGS[name]
    ob, ac = _spaces(cfg)
    kw = dict(num_layers=cfg.get("num_layers", 2), num_hidden=cfg.get("num_hidden", 64)) if cfg["kind"] == "mlp" else {}
    np.random.seed(seed)
    pol = PolicyBuilder(ob, ac, cfg["kind"], value_network="copy" if cfg.get("copy") else None,
                        normalize_observations=cfg.get("normalize", False), **kw)
    model = Model(policy=pol, ob_space=ob, ac_space=ac, nbatch_act=B, nbatch_train=B, nsteps=1, ent_coef=0.01,
                  vf_coef=0.5, max_grad_norm=0.5, comm=False, train_chunk=B)
    net = model.net
    rng = np.random.RandomState(seed + 100)
    p = net.store.export_tf("params")
    for k in p:
        if k.endswith("/b:0") and not k.endswith("logstd:0"):
            p[k] = (p[k] + 0.05 * rng.randn(*p[k].shape)).astype(np.float32)
    if net.pd == "gauss":
        p["ppo2_model/pi/logstd:0"] = (0.2 * rng.randn(1, net.nout)).astype(np.float32)
    model.set_params(p)
    if cfg.get("normalize"):
        d = N.in_dim(cfg["ob"])[0]               # |(x - mean) / std| beyond 5 for a good share of the observations
        net.set_obs_rms(dict(runningsum=rng.randn(d) * 5.0, runningsumsq=rng.rand(d) * 20.0 + 30.0, count=10.0))
    return model


def _act_obs(rng, cfg, B):
    """uint8 frames (cnn), un-rounded float32 at VecNormalize scale (Box, clipped to +-10), integers otherwise."""
    ok, oa = cfg["ob"]
    if cfg["kind"] == "cnn":
        return rng.randint(0, 256, (B,) + oa).astype(np.uint8)
    if ok == "discrete":                             # neighbouring rows differ
        return ((np.arange(B) + rng.randint(oa)) % oa).reshape(B, 1).astype(np.float32)
    if ok == "mdisc":
        c = np.arange(B) + rng.randint(int(np.prod(oa)))
        return np.stack([(c // int(np.prod(oa[i + 1:]))) % k for i, k in enumerate(oa)], 1).astype(np.float32)
    return np.clip(rng.randn(B, *oa) * 3.0, -10.0, 10.0).astype(np.float32)


def _noise(rng, pd, B, nout):
    if pd == "gauss":
        return rng.randn(B, nout).astype(np.float32)
    return (rng.rand(B, nout) * 0.998 + 0.001).astype(np.float32)


def _mirror_x(net, cfg, raw):
    if cfg["kind"] == "cnn":
        return torch.as_tensor(np.asarray(raw)).to(DEV).double()
    ok, oa = cfg["ob"]
    mean, inv_std = _norm_arrays(net)
    return torch.as_tensor(N.encode_obs(np.asarray(raw).reshape(len(raw), -1), onehot_n=oa if ok == "discrete" else 0,
                                        nvec=list(oa) if ok == "mdisc" else None, mean=mean, inv_std=inv_std)).to(DEV)


def _tanh_acts(prefix, tower, B):
    """The kernels' stored tanh activations of an mlp tower, keyed like the mirror's layers."""
    if tower is None or tower.kind != "mlp":
        return {}
    return {f"{prefix}/mlp_fc{i}": tower.hfc[i][:B, :l.N].double() for i, l in enumerate(tower.fcs)}


def _check_tanh(what, ref, S, acts, g=None):
    """Each stored tanh activation the mirror takes from the kernels is fp16(tanh(pre)) of the mirror's pre-activation:
    |s - tanh(pre)| <= half the fp16 spacing at s + 2^-22 |tanh(pre)| (tanhf) + (1 - tanh^2) G_PRE S_pre.  Mutant:
    the layer's output of row i + 1."""
    g = G_PRE if g is None else g
    for k, s_k in acts.items():
        t = torch.tanh(ref.pres[k])
        sp = torch.as_tensor(np.spacing(s_k.abs().cpu().numpy().astype(np.float16)).astype(np.float64)).to(DEV)
        fixed = 0.5 * sp + 2.0 ** -22 * t.abs()
        d = (1 - t * t) * S.pres[k]
        over = ((s_k - t).abs() - fixed).clamp_min(0.0)
        seen = float((over[d > 0] / d[d > 0]).max()) if bool((d > 0).any()) else 0.0
        _report(f"{what} {k.split('/', 1)[1]} stored tanh pre-activation", seen, g)
        assert bool((over <= g * d).all()), (what, k, seen)
        slack = fixed + g * d
        if s_k.shape[0] > 1:
            assert not bool(((torch.roll(s_k, -1, 0) - t).abs() <= slack).all()), (what, k, "row i + 1 accepted")


def _mirror(net, cfg, raw, what):
    """float64 mirror of the last acting pass over `raw` (ReLU decisions and stored tanh activations from the kernels)
    and its absolute network."""
    B = len(raw)
    P = net.store.export_tf("params")
    mcfg, ident = N.ppo_mirror_cfg(cfg), net.pi_identity
    x = _mirror_x(net, cfg, raw)
    masks = _ppo_masks(net, B)
    acts = dict(_tanh_acts("ppo2_model/pi", net.tower_pi, B), **_tanh_acts("ppo2_model/vf", net.tower_vf, B))
    masks.update(acts)
    z = torch.zeros(B, net.nout, dtype=torch.float64, device=DEV)
    zv = torch.zeros(B, dtype=torch.float64, device=DEV)
    ref = N.policy_ref(P, mcfg, x, z, zv, rnd=True, masks=masks, identity=ident, dev=DEV)
    S = N.policy_ref(P, mcfg, x, z, zv, absolute=True, ref_acts=ref.acts, identity=ident, dev=DEV)
    _check_tanh(what, ref, S, acts)
    return ref, S, P


def _sample_ref(pd, pi, noise, nvec, logstd):
    """float64 sampler at logits pi [B, nout] (numpy float64) with the injected noise: (actions, rows to compare)."""
    u = noise.astype(np.float64)
    B = pi.shape[0]
    if pd in ("cat", "mcat"):
        nv = nvec or [pi.shape[1]]
        sc = pi - np.log(-np.log(u))
        acts = np.stack([blk.argmax(1) for blk in np.split(sc, np.cumsum(nv)[:-1], axis=1)], 1)
        ok = lr.gumbel_clear(pi.astype(np.float32), noise, nv)
        return (acts[:, 0] if pd == "cat" else acts), ok
    if pd == "bern":
        p = 1.0 / (1.0 + np.exp(-pi))
        return (u < p).astype(np.float32), np.all(np.abs(u - p) > 1e-6, axis=1)
    return pi + np.exp(logstd.astype(np.float64)) * u, np.ones(B, bool)


def _nlp_ref(pd, pi, acts, nvec, logstd):
    """float64 neglogp of `acts` at logits pi, and the sum of the magnitudes of its terms (the rounding scale)."""
    if pd in ("cat", "mcat"):
        nv = nvec or [pi.shape[1]]
        a = acts.reshape(len(acts), -1)
        nlp, sc = 0.0, 0.0
        for s, blk in enumerate(np.split(pi, np.cumsum(nv)[:-1], axis=1)):
            m = blk.max(1)
            lz = np.log(np.exp(blk - m[:, None]).sum(1))
            la = blk[np.arange(len(blk)), a[:, s]]
            nlp = nlp + m + lz - la
            sc = sc + np.abs(m) + np.abs(lz) + np.abs(la) + 1.0
        return nlp, sc
    if pd == "bern":
        x = acts.astype(np.float64)
        t = np.maximum(pi, 0) - pi * x + np.log1p(np.exp(-np.abs(pi)))
        return t.sum(1), (np.abs(pi) * 2 + 1).sum(1)
    ls = logstd.astype(np.float64)
    t = (acts.astype(np.float64) - pi) / np.exp(ls)
    q = 0.5 * (t * t).sum(1)
    c = 0.5 * np.log(2 * np.pi) * pi.shape[1] + ls.sum()
    return q + c, q + abs(c) + np.abs(ls).sum() + 1.0


def _wrong_action(pd, acts, nvec, nout, logstd):
    """Another action of each row: the neglogp bound must reject the neglogp of this one."""
    if pd == "cat":
        return (acts + 1) % nout
    if pd == "mcat":
        return (acts + 1) % np.asarray(nvec)[None]
    if pd == "bern":
        w = acts.copy()
        w[:, 0] = 1.0 - w[:, 0]
        return w
    return acts + np.exp(logstd)[None].astype(np.float32)


def _check_step(what, name, model, raw, noise, a, v, nlp):
    """1a and 1b for one acting pass (outputs a, v, nlp; the pass must be the last one the model ran)."""
    cfg, net = N.PPO_CONFIGS[name], model.net
    B, nout, pd = len(raw), net.nout, net.pd
    nvec = net.nvec
    pi = net.pi_out[:B, :nout].double()
    ref, S, P = _mirror(net, cfg, raw, what)
    vb = torch.as_tensor(np.asarray(v)).to(DEV).double()
    muts_pi = {"logits read one column off": torch.roll(ref.pi, 1, 1)}
    muts_v = {"value read one column off (the last logit)": ref.pi[:, nout - 1],
              "value head bias left out": ref.v - float(P["ppo2_model/vf/b:0"][0])}
    if B > 1:
        muts_pi["row i's logits taken from row i + 1"] = torch.roll(ref.pi, -1, 0)
        muts_v["row i's value taken from row i + 1"] = torch.roll(ref.v, -1, 0)
    _bound(f"{what} logits", pi, ref.pi, S.pi, G_PI[name], muts_pi)
    _bound(f"{what} value", vb, ref.v, S.v, G_V[name], muts_v)
    # actions: the float64 sampler at the kernel's own logits
    pin = pi.cpu().numpy()
    ls = net.logstd.detach().cpu().numpy() if pd == "gauss" else None
    want, ok = _sample_ref(pd, pin, noise, nvec, ls)
    assert ok.mean() > 0.9 or B < 8, (what, ok.mean())
    a = np.asarray(a)
    if pd == "gauss":
        tol = 8 * U32 * (np.abs(pin) + np.exp(ls)[None] * np.abs(noise))       # expf (2 ulp), product, sum
        assert np.all(np.abs(a - want) <= tol), f"{what} gauss actions"
    else:
        assert np.array_equal(a[ok], want[ok].astype(a.dtype)), f"{what} actions"
    ref_nlp, sc = _nlp_ref(pd, pin, a, nvec, ls)
    k = NLP_ROUNDINGS(nout)
    err = np.abs(np.asarray(nlp, np.float64) - ref_nlp)
    wrong = _nlp_ref(pd, pin, _wrong_action(pd, a, nvec, nout, ls), nvec, ls)[0]
    seen = float((err / (sc * U32)).max())
    print(f"[observed] {what} neglogp: {seen:.2f} fp32 roundings of its scale (allowed {k})")
    assert np.all(err <= k * U32 * sc), (what, seen)
    assert np.any(np.abs(wrong - ref_nlp) > k * U32 * sc), f"{what}: the neglogp bound accepts another action's"


def _ppo_cases():
    out = []
    for name, cfg in N.PPO_CONFIGS.items():
        for B in BATCHES + ((BIG_MLP_B,) if cfg["kind"] == "mlp" else ()):
            out.append(pytest.param(name, B, id=f"{name}-B{B}"))
    return out


@pytest.mark.parametrize("name,B", _ppo_cases())
def test_ppo_step_vs_float64(name, B):
    """1a-1d."""
    cfg = N.PPO_CONFIGS[name]
    model = _act_model(name, B)
    net = model.net
    rng = np.random.RandomState(B)
    raw = _act_obs(rng, cfg, B)
    noise = _noise(rng, net.pd, B, net.nout)
    a, v, _, nlp = model.step(raw, noise=noise)
    pi_step = net.pi_out[:B, :net.nout].clone()
    _check_step(f"{name} B={B}", name, model, raw, noise, a, v, nlp)
    # c. value() runs the train forward (with masks): bit-identical to step()'s value
    assert np.array_equal(model.value(raw), v), "value() differs from step()'s value"
    # d. batch invariance: a smaller acting pass, and the train forward gathered through src_idx
    for k in sorted({1, B // 2 + 1} - {B}):
        a2, v2, _, n2 = model.step(raw[:k], noise=noise[:k])
        assert np.array_equal(v2, v[:k]) and np.array_equal(n2, nlp[:k]) and np.array_equal(a2, a[:k]), (B, k)
        assert torch.equal(net.pi_out[:k, :net.nout], pi_step[:k]), (B, k)
    perm = torch.as_tensor(np.random.RandomState(1).permutation(B)).to(DEV)
    x = net.encode_obs(raw)
    net.forward(x, B, src_idx=perm, masks=True)
    torch.cuda.synchronize()
    assert torch.equal(net.pi_out[:B, :net.nout], pi_step[perm]), "train forward rows differ from the acting pass"
    vt = net.v_out[:B, 0] if net.v_out.dim() == 2 else net.v_out[:B]
    assert torch.equal(vt.cpu(), torch.as_tensor(v)[perm.cpu()]), "train forward values differ from the acting pass"


# ================================================================================================ graph replay
STREAM_CASES = ("cnn84_cat6_shared", "mlp_mdisc33_mcat33", "mlp11_bern5_normalized", "mlp376_gauss17_copy_h64")


def _philox_actions(pd, pi, seed, off, nvec, ls):
    """The kernel's sample at stream position `off` from the host Philox stream (gauss: Box-Muller in float64)."""
    B, n = pi.shape
    u = lr.philox_uniforms(seed, B, n + (n & 1), off)
    if pd == "gauss":
        u1, u2 = u[:, 0::2].astype(np.float64), u[:, 1::2].astype(np.float64)
        r = np.sqrt(-2.0 * np.log(u1))
        z = np.stack([r * np.cos(2 * np.pi * u2), r * np.sin(2 * np.pi * u2)], 2).reshape(B, -1)[:, :n]
        return _sample_ref(pd, pi, z, nvec, ls)
    return _sample_ref(pd, pi, u[:, :n], nvec, ls)


@pytest.mark.parametrize("name", STREAM_CASES)
def test_step_device_replay_equals_eager_and_stream_advances(name):
    """2: three persistent step_device calls (eager, capture + replay, replay) equal three eager passes from the same
    rng_ctr bit for bit; the counter advances by exactly one per pass; each pass samples the host Philox stream at its
    position.  Mutant: the sampler offset not advanced (every pass at the first position)."""
    cfg = N.PPO_CONFIGS[name]
    B = 65
    model = _act_model(name, B)
    net = model.net
    rng = np.random.RandomState(5)
    raw = _act_obs(rng, cfg, B)
    x = net.encode_obs(raw)
    a = torch.zeros(net.action_shape(B), dtype=net.action_dtype, device=DEV)
    v, n = torch.zeros(B, device=DEV), torch.zeros(B, device=DEV)
    ctr0 = int(net.rng_ctr.item())
    seqs = []
    for graph in (True, False):
        net.rng_ctr.fill_(ctr0)
        outs = []
        for k in range(3):
            r0 = _lib.REPLAYS
            if graph:
                model.step_device(x, a, v, n, persistent=True)
            else:
                net.act(x, B, a, v, n, seed=model._rng_seed)
            torch.cuda.synchronize()
            assert _lib.REPLAYS - r0 == (1 if graph and k > 0 else 0), (graph, k)
            assert int(net.rng_ctr.item()) == ctr0 + k + 1, "rng_ctr must advance once per acting pass"
            outs.append((a.clone(), v.clone(), n.clone(), net.pi_out[:B, :net.nout].double().cpu().numpy()))
        seqs.append(outs)
    for (ga, gv, gn, _), (ea, ev, en, _) in zip(*seqs):
        assert torch.equal(ga, ea) and torch.equal(gv, ev) and torch.equal(gn, en), "replay differs from eager"
    ls = net.logstd.detach().cpu().numpy() if net.pd == "gauss" else None
    acts = [o[0].cpu().numpy() for o in seqs[0]]
    assert not np.array_equal(acts[0], acts[1]) and not np.array_equal(acts[1], acts[2]), "replays repeat samples"
    for k, (ak, _, _, pik) in enumerate(seqs[0]):
        want, ok = _philox_actions(net.pd, pik, model._rng_seed, ctr0 + k, net.nvec, ls)
        stale, _ = _philox_actions(net.pd, pik, model._rng_seed, ctr0, net.nvec, ls)
        ak = ak.cpu().numpy()
        if net.pd == "gauss":
            tol = 1e-4 * (1 + np.abs(want))                   # device logf / sinpif / cospif against float64
            assert np.all(np.abs(ak - want) <= tol), (name, k)
            if k:
                assert not np.all(np.abs(stale - want) <= tol), "the stream check cannot see a stale offset"
        else:
            assert ok.mean() > 0.9 and np.array_equal(ak[ok], want[ok].astype(ak.dtype)), (name, k)
            if k:
                assert not np.array_equal(stale[ok], want[ok]), "the stream check cannot see a stale offset"


@pytest.mark.parametrize("name,B", [(n, b) for n in ("mlp_mdisc33_mcat33", "mlp11_bern5_normalized") for b in (1, 7)])
def test_sampler_frequencies_at_small_batches(name, B):
    """2: PASSES replayed acting passes on fixed observations: per row and component, the frequency of every category
    (mcat) or of 1 (bern) is within 5 sigma (+ 1 / PASSES) of the float64 probability at the kernel's logits."""
    PASSES = 4000
    cfg = N.PPO_CONFIGS[name]
    model = _act_model(name, B)
    net = model.net
    raw = _act_obs(np.random.RandomState(11), cfg, B)
    x = net.encode_obs(raw)
    a = torch.zeros(net.action_shape(B), dtype=net.action_dtype, device=DEV)
    v, n = torch.zeros(B, device=DEV), torch.zeros(B, device=DEV)
    hist = torch.zeros((PASSES,) + tuple(a.shape), dtype=a.dtype, device=DEV)
    for k in range(PASSES):
        model.step_device(x, a, v, n, persistent=True)
        hist[k].copy_(a)
    pi = net.pi_out[:B, :net.nout].double().cpu().numpy()
    h = hist.cpu().numpy()
    worst = 0.0
    if net.pd == "mcat":
        off = np.concatenate([[0], np.cumsum(net.nvec)])
        for s, k_ in enumerate(net.nvec):
            l = pi[:, off[s]:off[s + 1]]
            p = np.exp(l - l.max(1, keepdims=True))
            p /= p.sum(1, keepdims=True)
            for c in range(k_):
                f = (h[:, :, s] == c).mean(0)
                z = np.abs(f - p[:, c]) / (np.sqrt(p[:, c] * (1 - p[:, c]) / PASSES) + 1.0 / PASSES)
                worst = max(worst, float(z.max()))
    else:
        p = 1.0 / (1.0 + np.exp(-pi))
        f = h.mean(0)
        worst = float((np.abs(f - p) / (np.sqrt(p * (1 - p) / PASSES) + 1.0 / PASSES)).max())
    print(f"[observed] {name} B={B} sampler frequencies: {worst:.2f} sigma (allowed 5)")
    assert worst <= 5.0, (name, B, worst)


def test_chunked_acting_equals_unchunked(monkeypatch):
    """2: frame-stacked NatureCNN rollout acted in 4 chunks of 7 envs: every chunk's values are bit-identical to an
    unchunked pass over the same stacked observations, its neglogp is the float64 neglogp of the action it returned,
    and the actions lie in range."""
    from baselines_b200.common.vec_env import SyntheticVecEnv, VecFrameStack
    from baselines_b200.ppo2.runner import Runner
    monkeypatch.setenv("B200RL_ACT_CHUNKS", "4")
    Nenv, T = 28, 5
    model = _act_model("cnn84_cat6_shared", Nenv)
    env = VecFrameStack(SyntheticVecEnv(Nenv, (84, 84, 1), np.uint8, n_actions=6, seed=2), 4)
    runner = Runner(env=env, model=model, nsteps=T, gamma=0.99, lam=0.95)
    assert runner.fs and runner.act_chunks == 4
    ro, _ = runner.run_device()
    torch.cuda.synchronize()
    net = model.net
    for t in range(1, T):                               # slots 1.. are acted chunk-wise with the frame upload
        obs = ro.obs[t].clone()
        a, v, n = (torch.zeros_like(x) for x in (ro.actions[t], ro.values[t], ro.neglogpacs[t]))
        net.act(obs, Nenv, a, v, n, seed=model._rng_seed)
        torch.cuda.synchronize()
        assert torch.equal(v, ro.values[t]), f"slot {t}: chunked values differ from an unchunked pass"
        pi = net.pi_out[:Nenv, :6].double().cpu().numpy()
        acts = ro.actions[t].cpu().numpy()
        assert ((acts >= 0) & (acts < 6)).all()
        ref, sc = _nlp_ref("cat", pi, acts, None, None)
        err = np.abs(ro.neglogpacs[t].cpu().numpy() - ref)
        assert np.all(err <= NLP_ROUNDINGS(6) * U32 * sc), (t, float((err / (sc * U32)).max()))


# ================================================================================================ runner
@pytest.mark.parametrize("device_env", [False, True], ids=["host_env", "device_env"])
@pytest.mark.parametrize("name", ["cnn84_cat6_shared", "mlp11_gauss3_copy_h256"])
def test_runner_rollout_vs_float64(name, device_env):
    """3: T = 5, N = 7 with injected noise: every slot's actions / values / neglogpacs are a step on ro.obs[t] (bit for
    bit), checked against the mirror as in 1; last_values equal value() at the final observation and the mirror."""
    from baselines_b200.common.vec_env import DeviceSyntheticVecEnv, SyntheticVecEnv
    from baselines_b200.ppo2.runner import Runner
    cfg = N.PPO_CONFIGS[name]
    T, Nenv = 5, 7
    model = _act_model(name, Nenv)
    net = model.net
    shape = N.in_dim(cfg["ob"])
    dt = np.uint8 if cfg["kind"] == "cnn" else np.float32
    kw = dict(n_actions=6) if net.pd == "cat" else dict(act_dim=net.nout)
    env = (DeviceSyntheticVecEnv if device_env else SyntheticVecEnv)(Nenv, shape, dt, seed=4, **kw)
    runner = Runner(env=env, model=model, nsteps=T, gamma=0.99, lam=0.95)
    noise = _noise(np.random.RandomState(6), net.pd, T * Nenv, net.nout).reshape(T, Nenv, net.nout)
    ro, _ = runner.run_device(noise=noise)
    torch.cuda.synchronize()
    for t in range(T):
        raw = ro.obs[t].cpu().numpy()
        a, v, _, nlp = model.step(raw, noise=noise[t])
        got_a = net.actions_to_numpy(ro.actions[t])
        assert np.array_equal(a, got_a) and np.array_equal(v, ro.values[t].cpu().numpy()) and \
            np.array_equal(nlp, ro.neglogpacs[t].cpu().numpy()), f"slot {t} differs from a step on its observations"
        _check_step(f"{name} runner slot {t}", name, model, raw, noise[t], a, v, nlp)
    last = runner._cur.cpu().numpy()
    lv = model.value(last)
    assert np.array_equal(lv, ro.last_values.cpu().numpy()), "last_values differ from value() at the final observation"
    ref, S, P = _mirror(net, cfg, last, f"{name} runner last_values")
    _bound(f"{name} runner last_values", torch.as_tensor(lv).to(DEV).double(), ref.v, S.v, G_V[name],
           {"value head bias left out": ref.v - float(P["ppo2_model/vf/b:0"][0]),
            "row i's value taken from row i + 1": torch.roll(ref.v, -1, 0)})


# ================================================================================================ DQN
DQN_NA = 6
DQN_BATCHES = (1, 2, 7, 65, 512)


def _dqn_act_model(name, seed=3):
    from baselines_b200.common import spaces
    from baselines_b200.deepq.build_graph import DQNModel
    cfg = N.DQN_CONFIGS[name]
    ok, oa = cfg["ob"]
    if ok == "discrete":
        ob = spaces.Discrete(oa)
    else:
        ob = spaces.Box(0, 255, oa, np.uint8) if cfg["kind"] != "mlp" else spaces.Box(-5, 5, oa, np.float32)
    model = DQNModel(ob, DQN_NA, cfg["kind"], lr=1e-3, gamma=0.99, grad_norm_clipping=10.0, double_q=cfg["double_q"],
                     batch_cap=512, seed=seed, hiddens=cfg["hiddens"], dueling=cfg["dueling"])
    rng = np.random.RandomState(seed + 100)
    p = model.q.store.export_tf("params")
    for k in p:
        if "biases" in k or k.endswith("/b:0"):
            p[k] = (p[k] + 0.05 * rng.randn(*p[k].shape)).astype(np.float32)
    model.q.store.import_tf(p, "params")
    model.q.refresh()
    return model


def _dqn_obs(rng, cfg, B):
    if cfg["kind"] != "mlp":
        return rng.randint(0, 256, (B,) + cfg["ob"][1]).astype(np.uint8)
    if cfg["ob"][0] == "discrete":
        return rng.randint(0, cfg["ob"][1], (B, 1)).astype(np.float32)
    return (rng.randn(B, *cfg["ob"][1]) * 2.0).astype(np.float32)


def name_of(cfg):
    return next(n for n, c in N.DQN_CONFIGS.items() if c is cfg)


def _dqn_mirror(model, cfg, raw):
    B = len(raw)
    q = model.q
    if cfg["kind"] != "mlp":
        x = torch.as_tensor(raw).to(DEV).double()
    else:
        ok, oa = cfg["ob"]
        x = torch.as_tensor(N.encode_obs(raw, onehot_n=oa if ok == "discrete" else 0)).to(DEV)
    mcfg = N.dqn_mirror_cfg(cfg)
    P = q.store.export_tf("params")
    masks = _dqn_masks(q, B)
    acts = _tanh_acts("deepq/q_func", q.trunk, B)
    masks.update(acts)
    sa = torch.zeros(B, DQN_NA, dtype=torch.float64, device=DEV)
    ss = torch.zeros(B, dtype=torch.float64, device=DEV) if cfg["dueling"] else None
    ref = N.q_ref(P, mcfg, x, sa, ss, rnd=True, masks=masks, dev=DEV)
    S = N.q_ref(P, mcfg, x, sa, ss, absolute=True, ref_acts=ref.acts, dev=DEV)
    _check_tanh(f"{name_of(cfg)} B={B}", ref, S, acts)
    return ref, S


@pytest.mark.parametrize("B", DQN_BATCHES)
@pytest.mark.parametrize("name", list(N.DQN_CONFIGS))
def test_dqn_act_and_q_values_vs_float64(name, B):
    """4: the raw head outputs of an acting pass (A, S), q_values and the greedy action against the mirror."""
    cfg = N.DQN_CONFIGS[name]
    model = _dqn_act_model(name)
    q = model.q
    raw = _dqn_obs(np.random.RandomState(B), cfg, B)
    act = model.act_device(torch.as_tensor(raw).to(DEV), B, 0.0).cpu().numpy()
    out = q.out[:B].double()
    ref, S = _dqn_mirror(model, cfg, raw)
    what = f"{name} B={B}"
    mA = {"action scores read one column off": torch.roll(ref.A, 1, 1)}
    if B > 1:
        mA["row i's scores taken from row i + 1"] = torch.roll(ref.A, -1, 0)
    _bound(f"{what} A", out[:, :DQN_NA], ref.A, S.A, G_A[name], mA)
    if cfg["dueling"]:
        mS = {"state score read one column off (the last action score)": ref.A[:, -1]}
        if B > 1:
            mS["row i's state score taken from row i + 1"] = torch.roll(ref.S, -1, 0)
        _bound(f"{what} S", out[:, DQN_NA], ref.S, S.S, G_S[name], mS)
    # the greedy action: the float64 argmax of q formed from the kernel's own head outputs, where the top-2 gap is
    # clear of fp32 rounding
    o = out.cpu().numpy()
    qk = lr.dueling_q(torch.as_tensor(o[:, :DQN_NA]), torch.as_tensor(o[:, DQN_NA]) if cfg["dueling"] else None).numpy()
    top2 = np.sort(qk, 1)[:, -2:]
    clear = (top2[:, 1] - top2[:, 0]) > 1e-5 * (1 + np.abs(qk).max(1))
    assert clear.mean() > 0.9 or B < 8
    assert np.array_equal(act[clear], qk.argmax(1)[clear]), f"{what}: greedy action is not the argmax"
    # q_values: S + A - mean(A) against the mirror's, scale |S| + |A| + mean |A| of the absolute network
    qv = torch.as_tensor(model.q_values(raw)).to(DEV).double()
    qref = lr.dueling_q(ref.A, ref.S)
    if cfg["dueling"]:
        qS = S.S[:, None] + S.A + S.A.mean(1, keepdim=True)
        g = max(G_A[name], G_S[name]) * 2
    else:
        qS, g = S.A, G_A[name]
    mq = {"q read one column off": torch.roll(qref, 1, 1)}
    if B > 1:
        mq["row i's q taken from row i + 1"] = torch.roll(qref, -1, 0)
    _bound(f"{what} q_values", qv, qref, qS, g, mq)


def test_dqn_greedy_takes_lowest_index_at_exact_ties():
    """4: with two identical action-score columns (same weights and bias), rows whose maximum is that pair must take
    the lower index, like tf.argmax."""
    name = "mlp_dueling_h64_32_double"
    cfg = N.DQN_CONFIGS[name]
    model = _dqn_act_model(name)
    q = model.q
    p = q.store.export_tf("params")
    last = f"deepq/q_func/action_value/{N._fc_name(len(cfg['hiddens']))}"
    for lo_, hi_ in ((1, 4),):
        p[f"{last}/weights:0"][:, hi_] = p[f"{last}/weights:0"][:, lo_]
        p[f"{last}/biases:0"][lo_] += 0.3                # the tied pair is the maximum of many rows
        p[f"{last}/biases:0"][hi_] = p[f"{last}/biases:0"][lo_]
    q.store.import_tf(p, "params")
    q.refresh()
    B = 512
    raw = _dqn_obs(np.random.RandomState(3), cfg, B)
    act = model.act_device(torch.as_tensor(raw).to(DEV), B, 0.0).cpu().numpy()
    o = q.out[:B, :DQN_NA].cpu().numpy()
    assert np.array_equal(o[:, 1], o[:, 4])
    tie = o.argmax(1) == 1                               # numpy's argmax takes the first index too
    assert tie.sum() > 20, tie.sum()
    assert np.all(act[tie] == 1), "an exact tie must take the lowest index"


def test_dqn_epsilon_and_step_read_from_device_on_replay(monkeypatch):
    """4: eps = 1 draws exactly the host splitmix64 stream at the step counter and is uniform over nA (chi-square,
    p = 1e-6); the step advances once per act_device call and replays draw new actions; a replay equals an eager run
    at the same step; stochastic=False is greedy after a replay with eps = 1, and update_eps is sticky (build_act).
    Mutants: eps frozen at its captured value (the greedy check sees random actions); the step not advanced."""
    import scipy.stats
    from baselines_b200.deepq.build_graph import build_act
    name = "mlp_dueling_h20_double"
    cfg = N.DQN_CONFIGS[name]
    model = _dqn_act_model(name)
    act = build_act(model)
    B = 512
    raw = _dqn_obs(np.random.RandomState(8), cfg, B)
    greedy = act(raw, stochastic=False)
    draws = []
    for k in range(40):                              # eager, capture + replay, then replays
        step = int(model._step_dev.item())
        r0 = _lib.REPLAYS
        a = act(raw, update_eps=1.0)
        assert _lib.REPLAYS - r0 == 1, "the acting pass must replay from a graph after its first call"
        assert int(model._step_dev.item()) == step + 1, "_step_dev must advance once per act_device call"
        _, want = lr.dqn_act_draws(model._seed, step, B, DQN_NA)
        assert np.array_equal(a, want), f"eps = 1 pass {k}: not the splitmix64 stream at step {step}"
        draws.append(a)
    assert not np.array_equal(draws[-1], draws[-2]), "replays repeat the same draws"
    cnt = np.bincount(np.concatenate(draws), minlength=DQN_NA)
    chi = float(((cnt - cnt.sum() / DQN_NA) ** 2 / (cnt.sum() / DQN_NA)).sum())
    print(f"[observed] eps = 1 chi-square {chi:.2f} over {cnt.sum()} draws (allowed {scipy.stats.chi2.isf(1e-6, 5):.2f})")
    assert chi < scipy.stats.chi2.isf(1e-6, DQN_NA - 1)
    # greedy after replays with eps = 1: eps comes from the device, not from the captured call
    g2 = act(raw, stochastic=False)
    assert np.array_equal(g2, greedy), "stochastic=False is not greedy after a replay with eps = 1"
    assert (greedy != draws[-1]).mean() > 0.5, "the greedy check cannot tell eps = 0 from eps = 1"
    # update_eps is sticky: a call without it keeps eps = 1 ...
    step = int(model._step_dev.item())
    a = act(raw)
    assert np.array_equal(a, lr.dqn_act_draws(model._seed, step, B, DQN_NA)[1]), "eps must stay at its last update"
    # ... until it is updated
    assert np.array_equal(act(raw, update_eps=0.0), greedy)
    # a replay equals an eager run at the same step
    model._step_dev.fill_(step)
    ops.set_scalars(model._eps_dev, 1.0)
    monkeypatch.setenv("B200RL_NO_GRAPHS", "1")
    r0 = _lib.REPLAYS
    eager = model.act_device(torch.as_tensor(raw).to(DEV), B, 1.0).cpu().numpy()
    assert _lib.REPLAYS == r0
    assert np.array_equal(eager, a), "an eager pass differs from the replay at the same step"


# ================================================================================================ encoder edges
F16_MAX_ENC = 65520.0


def _enc(x, in_dim, in_pad, **kw):
    B = x.shape[0]
    out = torch.full((B, 2 * in_pad), float("nan"), dtype=torch.float16, device=DEV)
    flag = torch.zeros(1, dtype=torch.int32, device=DEV)
    raw_dim = x.shape[1]
    ops.obs_encode(torch.as_tensor(x).to(DEV).contiguous(), out, B, raw_dim, in_dim, in_pad, overflow=flag, **kw)
    torch.cuda.synchronize()
    return out, int(flag.item())


EDGE_VALUES = np.array([65504.0, 65519.0, 65519.996, 2.0 ** -3, 2.0 ** -14, 2.0 ** -24, 1e-30, 0.0, 1.0, 3.1415927,
                        1e3 + 1.0 / 3, 2.0 ** -3 * 0.99, 2.0 ** -14 * 1.37, 5e-6, 7e-8], np.float32)


def test_obs_encode_precision_and_range():
    """5: hi + lo is within max(2^-22 |v|, 2^-25) of every value below the fp16 limit, no output is NaN there, the
    flag stays clear, and rows with values at or beyond 65520 set it.  The relative claim alone fails below ~2^-3,
    where lo is fp16-subnormal."""
    vals = np.concatenate([EDGE_VALUES, -EDGE_VALUES])
    rng = np.random.RandomState(0)
    rand = (np.exp(rng.uniform(np.log(1e-9), np.log(6e4), 4000)) * rng.choice([-1, 1], 4000)).astype(np.float32)
    x = np.concatenate([vals, rand, np.zeros((-len(vals) - len(rand)) % 8, np.float32)]).reshape(-1, 8)
    out, flag = _enc(x, 8, 8)
    assert flag == 0, "a value below 65520 set the overflow flag"
    hi, lo = out[:, :8].double().cpu().numpy(), out[:, 8:].double().cpu().numpy()
    assert np.isfinite(hi).all() and np.isfinite(lo).all()
    v = x.astype(np.float64)
    err = np.abs(v - (hi + lo))
    assert np.all(err <= np.maximum(2.0 ** -22 * np.abs(v), 2.0 ** -25)), float((err / np.maximum(
        2.0 ** -22 * np.abs(v), 2.0 ** -25)).max())
    assert np.any(err > 2.0 ** -22 * np.abs(v)), "expected the subnormal lo range to exceed the relative bound"
    assert np.array_equal(hi, v.astype(np.float16).astype(np.float64)), "hi is not fp16(v)"
    for bad in (65520.0, -65520.0, 1e5, -1e5, 3e38, -3e38):
        y = np.zeros((2, 8), np.float32)
        y[1, 3] = bad
        assert _enc(y, 8, 8)[1] == 1, f"{bad} did not set the overflow flag"


def test_obs_encode_clip_both_sides_and_onehot_edges():
    """5: normalisation with inv_std large enough to clip on both sides equals encode_obs exactly; MultiDiscrete
    blocks straddling 8-column groups (nvec 5, 7, 6) with out-of-range and negative values give tf.one_hot's zero
    block; a Discrete value >= n writes only a padding column (or nothing past in_pad), never a real one."""
    rng = np.random.RandomState(1)
    x = (rng.randn(64, 11) * 3).astype(np.float32)
    mean = (rng.randn(11) * 0.5).astype(np.float32)
    inv_std = np.full(11, 40.0, np.float32)
    out, flag = _enc(x, 11, 16, mean=torch.as_tensor(mean).to(DEV), inv_std=torch.as_tensor(inv_std).to(DEV),
                     clip=(-5.0, 5.0))
    want = N.encode_obs(x, mean=mean, inv_std=inv_std)
    hi = out[:, :11].double().cpu().numpy()
    got = hi + out[:, 16:27].double().cpu().numpy()
    assert flag == 0 and (want == 5.0).any() and (want == -5.0).any()
    assert np.array_equal(hi, want.astype(np.float16).astype(np.float64)), "hi is not fp16 of the normalised value"
    assert np.all(np.abs(got - want) <= np.maximum(2.0 ** -22 * np.abs(want), 2.0 ** -25))
    assert np.array_equal(got[np.abs(want) == 5.0], want[np.abs(want) == 5.0]), "a clipped value is not exactly +-5"
    nvec = [5, 7, 6]
    md = np.stack([rng.randint(-2, k + 3, 64) for k in nvec], 1).astype(np.float32)
    out, _ = _enc(md, 18, 24, onehot_n=18, seg_off=ops.segment_table(nvec, DEV))
    ref = np.zeros((64, 18))
    for s, (lo_, k) in enumerate(zip([0, 5, 12], nvec)):
        for b in range(64):
            if 0 <= md[b, s] < k:
                ref[b, lo_ + int(md[b, s])] = 1.0
    o = out.double().cpu().numpy()
    assert np.array_equal(o[:, :18], ref) and not o[:, 18:24].any() and not o[:, 24:].any()
    d = np.array([[0], [9], [10], [12], [15], [16], [-1], [40]], np.float32)
    out, _ = _enc(d, 10, 16, onehot_n=10)
    o = out.double().cpu().numpy()
    assert np.array_equal(o[:, :10], np.eye(10)[[0, 9]].tolist() + [[0] * 10] * 6)
    assert o[2, 10] == 1 and o[3, 12] == 1 and o[4, 15] == 1 and not o[5:].any()   # padding columns only


@pytest.mark.parametrize("name", ["mlp_disc10_cat4", "mlp376_gauss17_copy_h64"])
def test_out_of_range_observations_through_the_model(name):
    """5: through Model.step: a Discrete value >= n acts like tf.one_hot's all-zero row because the padding rows of the
    first layer's forward weights stay zero (asserted directly); Box values up to 65519 give the mirror's result within
    the bound; 1e5 and 3e38 raise ValueError naming the limit instead of acting on NaN, and the model still works."""
    cfg = N.PPO_CONFIGS[name]
    B = 8
    model = _act_model(name, B)
    net = model.net
    l0 = net.tower_pi.fcs[0]
    w = net.w0cat if net.fuse0 else l0.w_fwd
    assert not w[:, l0.K:l0.Kp].any() and not w[:, l0.Kp + l0.K:].any(), "padding columns of the forward weights"
    rng = np.random.RandomState(2)
    noise = _noise(rng, net.pd, B, net.nout)
    if cfg["ob"][0] == "discrete":
        raw = np.array([[0], [3], [9], [10], [12], [15], [-1], [40]], np.float32)
        model.step(raw, noise=noise)
        mirror_raw = np.where((raw >= 0) & (raw < 10), raw, 0)
        pi = net.pi_out[:B, :net.nout].double()
        x = torch.as_tensor(N.encode_obs(mirror_raw, onehot_n=10)).to(DEV)
        x[3:] = 0.0                                                            # tf.one_hot of an out-of-range value
        P = net.store.export_tf("params")
        z, zv = torch.zeros(B, net.nout, device=DEV, dtype=torch.float64), torch.zeros(B, device=DEV, dtype=torch.float64)
        ref = N.policy_ref(P, N.ppo_mirror_cfg(cfg), x, z, zv, rnd=True, masks=_tanh_acts("ppo2_model/pi", net.tower_pi, B),
                           identity=net.pi_identity, dev=DEV)
        S = N.policy_ref(P, N.ppo_mirror_cfg(cfg), x, z, zv, absolute=True, ref_acts=ref.acts,
                         identity=net.pi_identity, dev=DEV)
        _bound(f"{name} out-of-range Discrete logits", pi, ref.pi, S.pi, G_PI[name],
               {"row i's logits taken from row i + 1": torch.roll(ref.pi, -1, 0)})
        return
    raw = np.clip(rng.randn(B, *cfg["ob"][1]) * 3.0, -10, 10).astype(np.float32)
    raw[0, :4] = [65504.0, -65519.0, 65519.0, -65504.0]
    raw[1, 5] = 2.0 ** -24
    raw[2, 7] = 1e-30
    a, v, _, nlp = model.step(raw, noise=noise)
    assert np.isfinite(v).all() and np.isfinite(nlp).all()
    _check_step(f"{name} edge values", name, model, raw, noise, a, v, nlp)
    for bad in (1e5, -1e5, 3e38, 65520.0):
        r2 = raw.copy()
        r2[4, 9] = bad
        with pytest.raises(ValueError, match="65520"):
            model.step(r2, noise=noise)
        with pytest.raises(ValueError, match="65520"):
            model.value(r2)
    a2, v2, _, n2 = model.step(raw, noise=noise)            # the flag was cleared: in-range observations act again
    assert np.array_equal(v2, v) and np.array_equal(n2, nlp)


def test_dqn_out_of_range_observations_raise():
    """5: q_values and build_act raise ValueError naming the limit for an observation value >= 65520."""
    from baselines_b200.deepq.build_graph import build_act
    name = "mlp_plain_h20_max"
    model = _dqn_act_model(name)
    act = build_act(model)
    raw = _dqn_obs(np.random.RandomState(4), N.DQN_CONFIGS[name], 4)
    good = model.q_values(raw)
    assert np.isfinite(good).all()
    raw[2, 1] = 3e38
    with pytest.raises(ValueError, match="65520"):
        model.q_values(raw)
    with pytest.raises(ValueError, match="65520"):
        act(raw, stochastic=False)
    raw[2, 1] = 65519.0
    assert np.isfinite(model.q_values(raw)).all()
