"""GPU: whole PPO2 and DQN updates at the minibatch sizes the benchmark trains with, against the float64 mirror.

test_update_composition_gpu.py checks every parameter's gradient and Adam step at M = 301.  The benchmark trains cfg2
on minibatches of 131 072 images and cfg3 on 262 144 rows, one chunk each, and some behaviour only happens there:
c1's stored activations (hconv[0], [131072, 20*20*32] fp16, 3.36 GB) and its data gradient (dY[0], 3.7 GB) pass byte
2^31; the weight-gradient reductions run over ~10^5 k-blocks; the split-K fc1 / mlp weight gradients, the column sums,
the dL/dlogstd row sum, adv_stats and the float64 loss-statistic atomics accumulate over the whole minibatch.

Each PPO2 configuration builds its model as bench.py's make() does (one chunk per minibatch) from a device rollout of
3 M + 37 rows whose actions, old values and old neglogp sit near the current policy, and runs three train_rollout
calls through src_idx on disjoint slices of a permutation: eager, captured and replayed, replayed (run_epochs' path).
After each one:
  1. every row's stored activations (NatureCNN: c1, c2, c3, fc1; mlp: the tanh layers of both towers) and head
     outputs equal the mirror (rnd=True, the kernels' ReLU decisions) within half a spacing of their format + g S;
     the bound rejects the neighbouring row's values, and a failure names the row and its byte offset in the buffer;
  2. the fp16 head-gradient rows and the five loss statistics equal tests/_loss_refs.py at the kernels' head outputs
     (test_update_composition_gpu._check_ppo_heads), adv_st a two-pass float64 mean and std within the one-pass bound
     of its summation depth (test_update_path_gpu._adv_bound);
  3. every TF variable's gradient equals the mirror within g S + 2^-23 |ref|; each bound rejects "one sample dropped"
     (each head's row with the largest gradient), built as the reference minus the mirror of that row alone, or,
     for the tensors named in WEAK, a block of consecutive rows dropped (see there);
  4. params / m / v equal float64 TF-Adam (the global clip case of each step asserted).
The mirror runs in slices (tests/_net_refs.policy_ref_sliced): a float64 batch of 131 072 images does not fit.  The
composition mistakes of test_update_composition_gpu.py (each a further full mirror pass) are checked there, not here.

cfg4's DQN update runs as bench.py's run_deepq builds it (batch 512 through replay indices, lr 1e-4, grad_norm_clipping
10, hiddens (256,), dueling, double-Q) through test_update_composition_gpu's checks.

Tolerances: every g is 3.5x the maximum observed on an H100 80GB HBM3 (700 W power limit) over two runs of every step,
floor 1e-8; the observed values are listed next to the constants and each run prints its own [observed] lines.
"""
import math
import time
import types

import numpy as np
import pytest
import torch

import _loss_refs as lr
import _net_refs as N
import _refs as R
import test_update_composition_gpu as C
from baselines_b200 import _lib
from test_update_path_gpu import _adv_bound

pytestmark = pytest.mark.gpu

DEV = C.DEV
MIRROR = {"cfg2": "cnn84_cat6_shared", "cfg3": "mlp376_gauss17_copy_h64"}   # the mirror's name of each network
SLICE = {"cfg2": 2048, "cfg3": 32768}          # mirror rows per slice: c1's float64 patches of 2048 images are 1.7 GB
# device memory beside the rollout: the model's workspaces at one 131 072-image chunk (~14 GB), the minibatch's
# gathered images and one slice of the float64 mirror
HEADROOM = {"cfg2": 36 << 30, "cfg3": 8 << 30}
# whether max_grad_norm = 0.5 scales the gradient of steps 1, 2, 3: cfg2's gradient norm is ~12 after the first Adam
# step (clip factors 0.042, 0.034), so both cases are checked there
CLIPPED = {"cfg2": (False, True, True), "cfg3": (False, False, False)}
# |pre| / S within which a kernel ReLU decision may differ from float64: one input activation rounded to the other
# neighbouring fp16 value moves a pre-activation by ~2^-11 of one of its terms, and among the 7e8 decisions of a
# minibatch some lie that close to zero (observed up to 2.86e-6 on c2; test_update_composition_gpu.G_MASK = 1e-6 holds
# at M = 301)
G_MASK = 3.5 * 2.86e-6
DQN_CLIP_CASE = "none"             # which of cfg4's variables grad_norm_clipping = 10 scales in the first update

# g per configuration and tensor: 3.5x the maximum observed on an H100 80GB HBM3 (700 W power limit) over two runs of
# three steps each, floor 1e-8.  Gradients (the same networks at M = 301 / B = 301: test_update_composition_gpu.py's
# cnn84_cat6_shared, mlp376_gauss17_copy_h64 and cnn_dueling_h256 rows):
_OBSERVED = {
    "cfg2": {"pi/c1/w": 2.66e-08, "pi/c1/b": 5.61e-09, "pi/c2/w": 9.86e-08, "pi/c2/b": 3.04e-08, "pi/c3/w": 9.86e-08,
             "pi/c3/b": 7.83e-07, "pi/fc1/w": 1.20e-06, "pi/fc1/b": 9.30e-07, "pi/w": 5.34e-09, "pi/b": 4.59e-09,
             "vf/w": 5.34e-09, "vf/b": 3.60e-10},
    "cfg3": {"pi/mlp_fc0/w": 1.51e-07, "pi/mlp_fc0/b": 7.26e-08, "pi/mlp_fc1/w": 2.04e-07, "pi/mlp_fc1/b": 1.46e-07,
             "vf/mlp_fc0/w": 8.00e-07, "vf/mlp_fc0/b": 3.13e-07, "vf/mlp_fc1/w": 6.38e-07, "vf/mlp_fc1/b": 4.25e-07,
             "pi/w": 3.49e-07, "pi/b": 1.73e-09, "vf/w": 2.71e-07, "vf/b": 6.56e-11},
    "cfg4": {"c1/w": 6.01e-09, "c1/b": 2.43e-09, "c2/w": 3.36e-08, "c2/b": 1.14e-07, "c3/w": 8.12e-09, "c3/b": 3.30e-08,
             "fc1/w": 1.68e-07, "fc1/b": 1.78e-06, "action_value/fully_connected/weights": 3.04e-08,
             "action_value/fully_connected/biases": 1.05e-06, "action_value/fully_connected_1/weights": 6.15e-10,
             "action_value/fully_connected_1/biases": 6.83e-10, "state_value/fully_connected/weights": 3.12e-08,
             "state_value/fully_connected/biases": 0.00e+00, "state_value/fully_connected_1/weights": 3.10e-10,
             "state_value/fully_connected_1/biases": 0.00e+00},
}
# Finding: for these tensors the bound cannot see one dropped sample.  cfg2's pi/c1/w, pi/c1/b, pi/w and vf/w sum
# 131 072 rows whose largest one moves them by 4e-9 to 4e-8 of S, at or below the error observed there (vf/w: a row
# moves it by 3.9e-9 of S, the kernels are off by up to 5.3e-9); cfg4's state_value/fully_connected_1/weights sits at
# the 1e-8 floor (observed 3.1e-10) where one row moves it by 1.4e-8.  For them the mutant drops a block of consecutive
# rows from the row with the largest head gradient on: 64 rows (moving c1 by 1.5e-7 to 3.8e-7 of S); the head weights'
# per-row terms cancel in sign, 64 rows move pi/w by only 1.3e-8 of S, so there 4096 rows.
WEAK = {"cfg2": {"pi/c1/w": 64, "pi/c1/b": 64, "pi/w": 4096, "vf/w": 4096},
        "cfg4": {"state_value/fully_connected_1/weights": 64}}
G = {(c, t): 3.5 * max(v, 1e-8) for c, per in _OBSERVED.items() for t, v in per.items()}
# cfg3's dL/dlogstd: the 1024 fp32 block partials of the Gaussian loss kernel are added in order, so the error grows
# with the minibatch (observed 3.64e-5 of S at M = 262 144; test_update_path_gpu.G_DLOGSTD = 1.3e-6 is fitted at
# B <= 4096).  One row is ~4e-6 of S, below that: the bound rejects the rows of one loss-kernel block (256) dropped.
G_DLOGSTD = 3.5 * 3.64e-05
DLOGSTD_DROP = 256
# stored activations and head outputs, beyond half a spacing of their format
_OBSERVED_FWD = {
    "cfg2": {"pi/c1": 5.97e-08, "pi/c2": 4.22e-06, "pi/c3": 5.97e-07, "pi/fc1": 1.35e-08, "pi": 2.12e-09,
             "vf": 1.86e-09},
    "cfg3": {"pi/mlp_fc0": 1.05e-07, "pi/mlp_fc1": 4.40e-05, "vf/mlp_fc0": 9.20e-08, "vf/mlp_fc1": 5.09e-05,
             "pi": 1.24e-04, "vf": 1.51e-04},
}
G_FWD = {(c, t): 3.5 * max(v, 1e-8) for c, per in _OBSERVED_FWD.items() for t, v in per.items()}


def _bench(key):
    from bench import CFGS
    return CFGS[key]


def _bytes(n, shape, dtype):
    return n * math.prod(shape) * torch.empty((), dtype=dtype).element_size()


def _release(*objs):
    """Free the device memory held by the models and buffers of a test, also where a failure's traceback still refers
    to them: every tensor reachable through the project's objects loses its storage, captured graphs are dropped."""
    seen = set()

    def walk(o):
        if id(o) in seen:
            return
        seen.add(id(o))
        if isinstance(o, torch.Tensor):
            if o.is_cuda:
                o.untyped_storage().resize_(0)
        elif isinstance(o, (list, tuple)):
            for v in o:
                walk(v)
        elif isinstance(o, dict):
            for v in o.values():
                walk(v)
        elif type(o).__module__.startswith("baselines_b200") and hasattr(o, "__dict__"):
            if hasattr(o, "graphs") and hasattr(o.graphs, "clear"):
                o.graphs.clear()
            for v in vars(o).values():
                walk(v)
    torch.cuda.synchronize()
    for o in objs:
        walk(o)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


@pytest.fixture
def held():
    """A list the test puts its models and device buffers in; released when the test ends, pass or fail."""
    objs = []
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    yield objs
    print(f"[cost] wall {time.time() - t0:.1f} s, peak device memory {torch.cuda.max_memory_allocated() / 1e9:.1f} GB")
    _release(*objs)
    objs.clear()


def _need(nbytes):
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip(f"needs {nbytes} bytes ({nbytes / 1e9:.1f} GB) of free device memory; {free / 1e9:.1f} GB free")


# ================================================================================================ PPO2
def _bench_model(key):
    """bench.py make(): build_policy with the configuration's network and value_network, Model with its coefficients,
    nbatch_train and train_chunk; then biases off zero and a non-zero logstd (test_update_composition_gpu)."""
    from baselines_b200.common.policies import build_policy
    from baselines_b200.ppo2.model import Model
    cfg, mc = _bench(key), N.PPO_CONFIGS[MIRROR[key]]
    ob, ac = C._spaces(mc)
    assert (cfg["network"], tuple(cfg["ob_shape"]), cfg["value_network"] == "copy") == \
        (mc["kind"], mc["ob"][1], bool(mc.get("copy"))), (key, MIRROR[key])
    assert (cfg["n_actions"] or cfg["act_dim"]) == mc["ac"][1]
    M = cfg["nenvs"] * cfg["nsteps"] // cfg["nminibatches"]
    np.random.seed(0)
    env = types.SimpleNamespace(observation_space=ob, action_space=ac)
    model = Model(policy=build_policy(env, cfg["network"], value_network=cfg["value_network"]), ob_space=ob,
                  ac_space=ac, nbatch_act=cfg["nenvs"], nbatch_train=M, nsteps=cfg["nsteps"],
                  ent_coef=cfg["ent_coef"], vf_coef=cfg["vf_coef"], max_grad_norm=cfg["max_grad_norm"], comm=False,
                  train_chunk=cfg["train_chunk"])
    assert model.chunk == M, (key, model.chunk, M)           # the benchmark's single-chunk launch sequence
    C._move_off_zero(model, 0)
    assert model.net.obs_rms is None and model.net.pi_identity == N.ppo_identity(mc)
    return model, cfg, mc, M


def _rollout(model, mc, n, seed):
    """A flat device rollout of n rows: uint8 images or float32 rows (N(0, 9)); actions, values and neglogp from the
    policy's own acting pass, old values and old neglogp moved off them so that both clip branches occur."""
    net = model.net
    g = torch.Generator(device=DEV).manual_seed(seed)
    shape = mc["ob"][1]
    if mc["kind"] == "cnn":
        obs = torch.empty((n,) + shape, dtype=torch.uint8, device=DEV).random_(0, 256, generator=g)
    else:
        obs = torch.randn((n,) + shape, device=DEV, generator=g) * 3.0
    acts = torch.empty(net.action_shape(n), dtype=net.action_dtype, device=DEV)
    v, nlp = torch.empty(n, device=DEV), torch.empty(n, device=DEV)
    for s in range(0, n, net.cap):
        e = min(s + net.cap, n)
        model.step_device(obs[s:e], acts[s:e], v[s:e], nlp[s:e])
    oldnlp = nlp + 0.15 * torch.randn(n, device=DEV, generator=g)
    oldv = v + 0.3 * torch.randn(n, device=DEV, generator=g)
    ret = oldv + torch.randn(n, device=DEV, generator=g)
    torch.cuda.synchronize()
    host = lambda t: t.cpu().numpy()
    return dict(obs=obs, acts=acts, ret=ret, oldv=oldv, oldnlp=oldnlp, acts_np=host(acts),
                np=dict(ret=host(ret), oldv=host(oldv), oldnlp=host(oldnlp)))


def _stored_layers(net, mc, B, start):
    """(mirror name, the kernels' stored fp16 activations of rows start .. start+B, bytes per row of their buffer)."""
    out = []
    towers = [("pi", net.tower_pi)] + ([("vf", net.tower_vf)] if net.tower_vf is not None else [])
    for nm, t in towers:
        if t.kind == "cnn":
            for i, c in enumerate(t.convs):
                out.append((f"ppo2_model/{nm}/{c.name.split('/')[-1]}", N.kernel_act(t, i, B, start),
                            c.OH * c.OW * c.nf * 2))
            out.append((f"ppo2_model/{nm}/fc1", t.hfc[0][start:start + B, :t.fcs[0].N], t.ld_hfc[0] * 2))
        else:
            for i, l in enumerate(t.fcs):
                out.append((f"ppo2_model/{nm}/mlp_fc{i}", t.hfc[i][start:start + B, :l.N], t.ld_hfc[i] * 2))
    return out


def _check_rows(what, key, layer, got, want, S, start, row_bytes, r, tiny, fwd_seen):
    """got (rows start ..) within g S + r |want| + tiny of want: r, tiny half a spacing of got's format.  A failure
    names the worst row and its byte offset in the kernels' buffer; the bound must reject the neighbouring row's
    values.  Records the observed g and the mutant's in fwd_seen."""
    B = got.shape[0]
    got, want, S = (t.double().reshape(B, -1) for t in (got, want, S))
    short = C._short(layer)
    g = G_FWD[(key, short)]
    if not R.within(got, want, S, g, r, tiny):
        e = ((got - want).abs() - g * S - r * want.abs() - tiny).amax(1)
        row = int(e.argmax())
        raise AssertionError(f"{what} {short}: row {start + row} (byte {(start + row) * row_bytes} of its buffer) is "
                             f"off by {float(e[row]):.3e} beyond g = {g:.1e}: got {got[row][:4].tolist()} ..., "
                             f"want {want[row][:4].tolist()} ...")
    seen = R.assert_within(got, want, S, g, r, {"the neighbouring row's values": torch.roll(want, 1, 0)},
                           f"{what} {short} rows {start}..", tiny)
    mut = R.excess(torch.roll(want, 1, 0), want, S, r)
    o, m = fwd_seen.get(short, (0.0, math.inf))
    fwd_seen[short] = (max(o, seen), min(m, mut))


def _check_forward_slice(what, key, net, mc, s, e, ref, S, fwd_seen, mask_seen, masks):
    """Per-row checks of one mirror slice: the kernels' ReLU decisions (G_MASK), stored activations, head outputs."""
    for k, (w, nd) in C._check_masks(what, ref, S, masks, report=False, g_mask=G_MASK).items():
        o, n_ = mask_seen.get(k, (0.0, 0))
        mask_seen[k] = (max(o, w), n_ + nd)
    for layer, got, row_bytes in _stored_layers(net, mc, e - s, s):
        pre = ref.pres[layer]
        want = pre * masks[layer] if layer in masks else torch.tanh(pre)
        _check_rows(what, key, layer, got, want, S.pres[layer], s, row_bytes, R.R_F16, 2.0 ** -25, fwd_seen)
    nout = net.nout
    _check_rows(what, key, "pi", net.pi_out[s:e, :nout], ref.pi, S.pi, s, net.ld_pi * 4, C.U32, 1e-30, fwd_seen)
    _check_rows(what, key, "vf", net.v_out[s:e, 0], ref.v, S.v, s, net.ld_v * 4, C.U32, 1e-30, fwd_seen)


def _rows_dropped(params, mcfg, x, dpi, dv, masks_of, ident, ref_grads, k=1):
    """The reference with rows left out, as the reference minus the mirror of those rows alone (the gradient is a sum
    of per-row terms).  k = 1: each head's row of largest gradient loses that head's seed (the row's data gradients
    are rounded as a whole, so the row runs with and without it); k > 1: the k rows from the row with the largest
    policy gradient on lose their whole loss."""
    ip, iv = int(dpi.abs().sum(1).argmax()), int(dv.abs().argmax())
    out = {n: g.clone() for n, g in ref_grads.items()}
    run = lambda s, e, sp, sv: N.policy_ref(params, mcfg, x[s:e], sp, sv, rnd=True, masks=masks_of(s, e),
                                            identity=ident, dev=DEV).grads
    if k > 1:
        s = min(ip, len(dv) - k)
        full = run(s, s + k, dpi[s:s + k], dv[s:s + k])
        for n in out:
            out[n] -= full[n]
        return out
    for r in sorted({ip, iv}):
        sp, sv = dpi[r:r + 1], dv[r:r + 1]
        full = run(r, r + 1, sp, sv)
        part = run(r, r + 1, sp * (r != ip), sv * (r != iv))
        for n in out:
            out[n] -= full[n] - part[n]
    return out


def _check_adv(what, net, roll, rows, M):
    R_, V = roll["np"]["ret"][rows], roll["np"]["oldv"][rows]
    d = R_.astype(np.float64) - V
    mean, std = lr.adv_moments(R_, V)
    bound, k = _adv_bound(d, M)
    i = int(np.abs(d).argmax())
    x = np.delete(d, i)
    m = x.sum() / M
    t = lambda a: torch.as_tensor(np.asarray(a, np.float64))
    seen = R.assert_within(t(net.adv_st.cpu().numpy()), t([mean, std]), t(bound), 1.0, 0.0,
                           {"row with the largest |R - V| dropped": t([m, math.sqrt((x * x).sum() / M - m * m)])},
                           f"{what} adv_st")
    print(f"[observed] {what} adv_st M={M} k={k}: {seen:.3e} of the one-pass bound")


@pytest.mark.parametrize("key", list(MIRROR))
def test_ppo_update_at_bench_minibatch_vs_float64(key, held):
    mc = N.PPO_CONFIGS[MIRROR[key]]
    cfg = _bench(key)
    M = cfg["nenvs"] * cfg["nsteps"] // cfg["nminibatches"]
    n = C.STEPS * M + 37
    _need(_bytes(n, mc["ob"][1], torch.uint8 if mc["kind"] == "cnn" else torch.float32) + HEADROOM[key])
    model, cfg, mc, M = _bench_model(key)
    held.append(model)
    net = model.net
    mcfg, ident = N.ppo_mirror_cfg(mc), net.pi_identity
    roll = _rollout(model, mc, n, 11)
    held.append(roll)
    perm = np.random.RandomState(12).permutation(n)
    for step in range(C.STEPS):
        rows = perm[step * M:(step + 1) * M]
        what = f"{key} step {step + 1}"
        replays = _lib.REPLAYS
        before, params = C._ppo_step(model, roll, rows, True, lr_=cfg["lr"], cliprange=cfg["cliprange"])
        C._assert_replayed(what, _lib.REPLAYS - replays, step > 0)
        # 2. heads, loss statistics, advantage moments
        dpi, dv = C._check_ppo_heads(what, mc, net, roll, rows, M, params, clip=cfg["cliprange"],
                                     ent=cfg["ent_coef"], vfc=cfg["vf_coef"], stats=model._stats_out.cpu().numpy(),
                                     g_dlogstd=G_DLOGSTD, dlogstd_drop=DLOGSTD_DROP)
        _check_adv(what, net, roll, rows, M)
        # 1. and 3. the mirror, slice by slice
        ridx = torch.as_tensor(rows).to(DEV)
        x = roll["obs"].index_select(0, ridx)
        if mc["kind"] != "cnn":
            x = x.double()                           # a Box without normalisation: the encoder's float32 rows
        held.append(x)
        masks_of = lambda s, e: C._ppo_masks(net, e - s, s)
        fwd_seen, mask_seen = {}, {}
        sl = N.policy_ref_sliced(params, mcfg, x, dpi.to(DEV), dv.to(DEV), SLICE[key], masks=masks_of,
                                 each=lambda s, e, ref, S: _check_forward_slice(what, key, net, mc, s, e, ref, S,
                                                                                fwd_seen, mask_seen, masks_of(s, e)),
                                 identity=ident, dev=DEV)
        for k, (w, nd) in mask_seen.items():
            C._report(f"{what} {C._short(k)} ReLU decisions ({nd} differ) |pre|/S", w, G_MASK)
        for short, (o, m) in fwd_seen.items():
            print(f"[mutant] {what} forward {short} the neighbouring row's values: g = {m:.3e}")
            C._report(f"{what} forward {short}", o, G_FWD[(key, short)])
        got = net.store.export_tf("grads")
        names = [k for k in got if not k.endswith("logstd:0")]
        args = (params, mcfg, x, dpi.to(DEV), dv.to(DEV), masks_of, ident, sl.grads)
        weak = WEAK.get(key, {})
        muts = {"one sample dropped": (_rows_dropped(*args), {k for k in names if C._short(k) not in weak})}
        for blk in sorted(set(weak.values())):
            muts[f"{blk} consecutive rows dropped"] = (_rows_dropped(*args, k=blk),
                                                       {k for k in names if weak.get(C._short(k)) == blk})
        C._assert_grads(what, key, got, sl.grads, sl.S, muts, names, 1.0 / M, G)
        del x, sl, muts
        held.pop()
        # 4. Adam
        C._ppo_adam(what, key, model, before, M, lr_=cfg["lr"], clipped=CLIPPED[key][step])


# ================================================================================================ DQN
def test_dqn_update_at_bench_batch_vs_float64(held):
    """cfg4 as run_deepq builds it: batch 512 through replay indices, three steps, test_update_composition_gpu's
    checks (head gradients, every variable's gradient with its mutants, per-variable clip, Adam)."""
    cfg = _bench("cfg4")
    name = "cnn_dueling_h256"
    mc = N.DQN_CONFIGS[name]
    assert (cfg["network"], tuple(cfg["ob_shape"]), cfg["n_actions"], mc["hiddens"], mc["dueling"], mc["double_q"]) \
        == ("cnn", mc["ob"][1], C.DQN_NA, (256,), True, True)
    C._dqn_update_run(name, True, B=cfg["batch"], lr_=cfg["lr"], clip=10.0, case=DQN_CLIP_CASE, g_table=G,
                      table_key="cfg4", block=(64, set(WEAK["cfg4"])))
