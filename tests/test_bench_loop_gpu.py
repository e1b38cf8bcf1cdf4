"""GPU: the PPO2 update loop as bench.py times it -- runner.run_device() then run_epochs(..., shuffle="device"), update
after update on one Model and one Runner -- and the device minibatch shuffle behind it.

  1. ops.shuffle_indices equals the host restatement _shuffle_ref.shuffle_ref element for element at cfg2's and cfg3's
     rollout shapes and at n = 1, 2, 7, 4^10, 4^10 + 1, 4^12 + 1 (half_bits 1 .. 13; at 4^12 + 1 the domain is almost
     4x the range, so cycle walking runs longest), for keys with bits 31 and 63 set as well as the keys run_epochs draws.
  2. The minibatches the kernel gives at cfg2 and cfg3 (two epochs keyed as run_epochs keys them) look like those of a
     uniform random permutation, each family at p = 1e-6 after a Bonferroni correction over its members
     (_shuffle_ref.minibatch_pvalues): samples per timestep and per environment in every minibatch, the overlap of every
     pair of minibatches of the two epochs, and the low bits of (i, pi(i)).
  3. bench's update loop at reduced sizes (cfg2's NatureCNN and cfg3's mlp / gauss17 / value_network='copy' with a
     train chunk that splits every minibatch), 3 updates with graphs:
     a. every epoch's key is run_epochs_keys of the numpy state before the update, keys are pairwise distinct, and the
        shuffle buffer of every epoch equals shuffle_ref for its key;
     b. a second model from the same initial state trained with run_epochs(perms=the recorded buffers as env-major
        indices), also from graphs, gives bit-identical rollouts, parameters and Adam moments after every update (the
        weight-gradient reductions run in a fixed order); the loss statistics, float64 atomic sums, agree to 1e-12;
        the same perms run eagerly agrees by test_round2_gpu's graph-versus-eager criterion;
     c. rollout k continues rollout k - 1: observation, reward and done rows are the env's pool and table entries at
        the env's running step, dones[0] is the previous rollout's last dones, actions and neglogp are the host Philox
        stream at the position of the acting pass (the counter runs on across rollouts), values and last_values are
        the forward at the stored observations, advs / returns are oracle.gae.gae_reference_order bit for bit;
     d. the host SyntheticVecEnv with the same seed (bench's `e2e` arm) gives bit-identical rollouts and parameters
        over 2 updates.
  4. A recurrent policy under shuffle="device" shuffles environments on the host (np.random.shuffle) and is
     bit-identical to perms drawn from the same numpy state.
"""
import numpy as np
import pytest
import torch

import _shuffle_ref as S
from bench import CFGS
from test_act_path_gpu import NLP_ROUNDINGS, U32, _nlp_ref, _philox_actions

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
RUN_KEYS = S.run_epochs_keys(np.random.RandomState(0).get_state(), 2)
KEYS = [0x1234567890ABCDEF, (1 << 63) | (1 << 31) | 0x5A5A, (1 << 63) | 0x1234567890ABCDEF, (1 << 64) - 1, 0, 1] + RUN_KEYS
BIG = 1 << 22                      # above this many samples only four keys (the host restatement takes seconds each)
P_FAMILY = 1e-6


def _kernel(n, key, T=0, N=0):
    from baselines_b200 import ops
    out = torch.full((n,), -1, dtype=torch.int64, device=DEV)
    ops.shuffle_indices(out, n, key, T, N)
    return out.cpu().numpy()


# ================================================================================================ 1. kernel = host
SHAPES = [(CFGS["cfg2"]["nsteps"] * CFGS["cfg2"]["nenvs"], CFGS["cfg2"]["nsteps"], CFGS["cfg2"]["nenvs"]),
          (CFGS["cfg3"]["nsteps"] * CFGS["cfg3"]["nenvs"], CFGS["cfg3"]["nsteps"], CFGS["cfg3"]["nenvs"])] + \
         [(n, 0, 0) for n in (1, 2, 7, 4 ** 10, 4 ** 10 + 1, 4 ** 12 + 1)]


@pytest.mark.parametrize("n,T,N", SHAPES, ids=[f"n{n}-T{T}-N{N}" for n, T, N in SHAPES])
def test_shuffle_kernel_equals_host_restatement(n, T, N):
    keys = KEYS if n <= BIG else [KEYS[0], KEYS[1], KEYS[3], RUN_KEYS[0]]
    for key in keys:
        got = _kernel(n, key, T, N)
        want = S.shuffle_ref(n, key, T, N)
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, f"key {key:#x}: {bad.size} of {n} differ, first at {bad[:4]}: {got[bad[:4]]} vs {want[bad[:4]]}"


# ================================================================================================ 2. statistics
@pytest.mark.parametrize("cfg", ["cfg2", "cfg3"])
def test_device_minibatches_look_like_a_uniform_shuffle(cfg):
    c = CFGS[cfg]
    T, N = c["nsteps"], c["nenvs"]
    m = T * N // c["nminibatches"]
    epochs = [_kernel(T * N, k, T, N) for k in RUN_KEYS]
    p, most = S.minibatch_pvalues(epochs, T, N, m)
    for fam, v in p.items():
        print(f"[observed] {cfg} {fam}: {len(v)} tests, smallest p {v.min():.3e} (allowed {P_FAMILY / len(v):.3e})")
    print(f"[observed] {cfg}: largest overlap of two minibatches of different epochs {most} of {m}")
    assert most < m, "an epoch-2 minibatch repeats an epoch-1 minibatch as a set"
    for fam, v in p.items():
        assert v.min() > P_FAMILY / len(v), (cfg, fam, float(v.min()))


# ================================================================================================ 3. the update loop
LOOPS = {
    "cfg2": dict(N=64, T=32, nminibatches=4, noptepochs=CFGS["cfg2"]["noptepochs"], train_chunk=None),
    "cfg3": dict(N=256, T=32, nminibatches=4, noptepochs=CFGS["cfg3"]["noptepochs"], train_chunk=768),
}
ROLLOUT_FIELDS = ("obs", "actions", "values", "neglogpacs", "rewards", "dones", "advs", "returns", "last_values",
                  "last_dones")


def _make(cfg, L, env_kind):
    """bench.py run_ppo2.make() at the reduced sizes L, on a device or host synthetic env with bench's seed."""
    from baselines_b200.common.policies import build_policy
    from baselines_b200.common.vec_env import DeviceSyntheticVecEnv, SyntheticVecEnv
    from baselines_b200.ppo2.model import Model
    from baselines_b200.ppo2.runner import Runner
    N, T = L["N"], L["T"]
    env_kw = dict(n_actions=cfg["n_actions"] or 6, act_dim=cfg["act_dim"])
    ob_dtype = np.dtype(cfg["ob_dtype"])
    np.random.seed(0)
    if env_kind == "device":
        env = DeviceSyntheticVecEnv(N, cfg["ob_shape"], ob_dtype, seed=0, device=DEV, **env_kw)
    else:
        env = SyntheticVecEnv(N, cfg["ob_shape"], ob_dtype, seed=0, **env_kw)
    policy = build_policy(env, cfg["network"], value_network=cfg["value_network"])
    model = Model(policy=policy, ob_space=env.observation_space, ac_space=env.action_space, nbatch_act=N,
                  nbatch_train=N * T // L["nminibatches"], nsteps=T, ent_coef=cfg["ent_coef"], vf_coef=cfg["vf_coef"],
                  max_grad_norm=cfg["max_grad_norm"], comm=False, train_chunk=L["train_chunk"])
    return model, Runner(env=env, model=model, nsteps=T, gamma=cfg["gamma"], lam=cfg["lam"])


def _tables(cfg, N):
    """The synthetic process's observation pool, reward and done tables (seed 0), on the host."""
    from baselines_b200.common.vec_env import SyntheticVecEnv
    h = SyntheticVecEnv(N, cfg["ob_shape"], np.dtype(cfg["ob_dtype"]), n_actions=cfg["n_actions"] or 6,
                        act_dim=cfg["act_dim"], seed=0)
    return [p.numpy() for p in h.pool], h.rews, h.dones


def _check_rollout(what, cfg, model, runner, tables, k, ctr0, prev_last_dones):
    """3c for rollout k (0-based) of a runner whose env started at step 0; returns copies of the rollout arrays."""
    from oracle.gae import gae_reference_order
    ro, net = runner.rollout, model.net
    T, N = ro.T, ro.N
    g0 = k * T                                          # env steps taken before this rollout
    torch.cuda.synchronize()
    pool, rews, dones = tables
    g = g0 + np.arange(T)
    obs = ro.obs.cpu().numpy()
    for t in range(T):
        assert np.array_equal(obs[t].reshape(pool[0].shape), pool[(g0 + t) % len(pool)]), f"{what}: obs row {t}"
    assert np.array_equal(runner._cur.cpu().numpy().reshape(pool[0].shape), pool[(g0 + T) % len(pool)]), \
        f"{what}: bootstrap observation"
    assert np.array_equal(ro.rewards.cpu().numpy(), rews[(g + 1) % 64]), f"{what}: rewards"
    want_d = dones[g % 64].copy()
    if g0 == 0:
        want_d[0] = False                               # nothing is done before the first step
    got_d = ro.dones.cpu().numpy().astype(bool)
    last_d = ro.last_dones.cpu().numpy().astype(bool)
    assert np.array_equal(got_d, want_d), f"{what}: dones"
    assert np.array_equal(got_d[0], np.zeros(N, bool) if prev_last_dones is None else prev_last_dones), \
        f"{what}: dones[0] is not the previous rollout's last dones"
    assert np.array_equal(last_d, dones[(g0 + T) % 64]), f"{what}: last_dones"
    assert int(net.rng_ctr.item()) == ctr0 + g0 + T, f"{what}: the sampler counter did not run on across rollouts"
    # acting passes: the forward at the stored observations, sampled at the Philox stream position of that pass
    ls = net.logstd.detach().cpu().numpy() if net.pd == "gauss" else None
    acts = net.actions_to_numpy(ro.actions)
    nlps = ro.neglogpacs.cpu().numpy()
    for t in range(T + 1):
        x = net.encode_obs(ro.obs[t] if t < T else runner._cur)
        net.forward(x, N, masks=False)
        v = net.v_out[:N, 0] if net.v_out.dim() == 2 else net.v_out[:N]
        if t == T:
            assert torch.equal(v, ro.last_values), f"{what}: last_values differ from the forward at the final obs"
            break
        assert torch.equal(v, ro.values[t]), f"{what}: values of step {t} differ from the forward at its obs"
        pi = net.pi_out[:N, :net.nout].double().cpu().numpy()
        pos = ctr0 + g0 + t
        want, ok = _philox_actions(net.pd, pi, model._rng_seed, pos, net.nvec, ls)
        stale, _ = _philox_actions(net.pd, pi, model._rng_seed, ctr0 + t, net.nvec, ls)
        a = acts[t]
        if net.pd == "gauss":
            tol = 1e-4 * (1 + np.abs(want))               # device logf / sinpif / cospif against float64
            assert np.all(np.abs(a - want) <= tol), f"{what}: step {t} actions are not the stream at {pos}"
            if pos != ctr0 + t:
                assert not np.all(np.abs(stale - want) <= tol), "the stream check cannot see a reset counter"
        else:
            assert ok.mean() > 0.9 and np.array_equal(a[ok], want[ok].astype(a.dtype)), \
                f"{what}: step {t} actions are not the stream at {pos}"
            if pos != ctr0 + t:
                assert not np.array_equal(stale[ok], want[ok]), "the stream check cannot see a reset counter"
        ref, sc = _nlp_ref(net.pd, pi, a, net.nvec, ls)
        assert np.all(np.abs(nlps[t].astype(np.float64) - ref) <= NLP_ROUNDINGS(net.nout) * U32 * sc), \
            f"{what}: step {t} neglogp"
    adv, ret = gae_reference_order(ro.rewards.cpu().numpy(), ro.values.cpu().numpy(), got_d,
                                   ro.last_values.cpu().numpy(), last_d, cfg["gamma"], cfg["lam"])
    assert np.array_equal(ro.advs.cpu().numpy(), adv) and np.array_equal(ro.returns.cpu().numpy(), ret), \
        f"{what}: advs / returns differ from gae_reference_order"
    out = {f: getattr(ro, f).clone() for f in ROLLOUT_FIELDS}
    out["cur"] = runner._cur.clone()
    return out, last_d


def _run(what, cfgname, env_kind, updates, monkeypatch, perms=None):
    """bench's update() `updates` times: run_device, then run_epochs with shuffle="device" (or the given perms); every
    rollout is checked (3c).  Returns per update: the numpy state before it, the recorded (key, buffer) per epoch, the
    rollout, the loss statistics, parameters and Adam moments after it; and the replay count."""
    from baselines_b200 import _lib
    from baselines_b200.ppo2 import ppo2
    cfg, L = CFGS[cfgname], LOOPS[cfgname]
    N, T = L["N"], L["T"]
    nbatch = N * T
    model, runner = _make(cfg, L, env_kind)
    tables = _tables(cfg, N)
    calls = []
    real = ppo2.ops_shuffle

    def recording_shuffle(out, n, key, T_, N_):
        real(out, n, key, T_, N_)
        calls.append((key, out.data_ptr(), out.clone()))
    monkeypatch.setattr(ppo2, "ops_shuffle", recording_shuffle)
    ctr0 = int(model.net.rng_ctr.item())
    r0 = _lib.REPLAYS
    res, prev = [], None
    for u in range(updates):
        state = np.random.get_state()
        c0 = len(calls)
        ro, _ = runner.run_device()
        roll, prev = _check_rollout(f"{what} rollout {u + 1}", cfg, model, runner, tables, u, ctr0, prev)
        st = ppo2.run_epochs(model, ro, cfg["lr"], cfg["cliprange"], nbatch, nbatch // L["nminibatches"],
                             L["noptepochs"], DEV, perms=None if perms is None else perms[u], shuffle="device")
        stats = torch.stack(st).cpu().numpy()
        store = model.net.store
        res.append(dict(state=state, calls=calls[c0:], roll=roll, stats=stats, params=model.get_params(),
                        m=store.m.clone(), v=store.v.clone(), t=model.opt.t))
    torch.cuda.synchronize()
    monkeypatch.setattr(ppo2, "ops_shuffle", real)
    return res, _lib.REPLAYS - r0


def _same_rollout(a, b):
    return all(torch.equal(a[f], b[f]) for f in a)


def _same_update(a, b):
    """Bit-identical parameters and Adam moments; the float64 atomic loss sums to 1e-12 (relative above 1)."""
    same_p = all(np.array_equal(a["params"][k], b["params"][k]) for k in a["params"])
    stats_ok = np.all(np.abs(a["stats"] - b["stats"]) <= 1e-12 * np.maximum(np.abs(b["stats"]), 1.0))
    return same_p and torch.equal(a["m"], b["m"]) and torch.equal(a["v"], b["v"]) and stats_ok and a["t"] == b["t"]


@pytest.mark.parametrize("cfgname", ["cfg2", "cfg3"])
def test_bench_update_loop(cfgname, monkeypatch):
    L = LOOPS[cfgname]
    N, T, nep = L["N"], L["T"], L["noptepochs"]
    nbatch = N * T
    updates = 3
    monkeypatch.delenv("B200RL_NO_GRAPHS", raising=False)
    dev_run, replays = _run(f"{cfgname} device shuffle", cfgname, "device", updates, monkeypatch)
    assert replays >= 2 * (T + 1 + L["nminibatches"] * nep), "updates 2 and 3 must replay from graphs"
    # a. keys and buffers
    all_keys = []
    for u, r in enumerate(dev_run):
        keys = [k for k, _, _ in r["calls"]]
        assert keys == S.run_epochs_keys(r["state"], nep), f"update {u + 1}: keys are not run_epochs' draws"
        assert len({p for _, p, _ in r["calls"]}) == 1, "every epoch shuffles into the rollout's one buffer"
        for key, _, buf in r["calls"]:
            assert np.array_equal(buf.cpu().numpy(), S.shuffle_ref(nbatch, key, T, N)), f"update {u + 1} key {key:#x}"
        all_keys += keys
    assert len(set(all_keys)) == len(all_keys) == updates * nep, "epoch keys repeat"
    # b. the same sequence with the recorded permutations injected (graphs), then eagerly
    perms = [[S.flat_of_offsets(buf.cpu().numpy(), T, N) for _, _, buf in r["calls"]] for r in dev_run]
    perm_run, _ = _run(f"{cfgname} perms", cfgname, "device", updates, monkeypatch, perms=perms)
    for u, (a, b) in enumerate(zip(dev_run, perm_run)):
        assert not b["calls"], "run_epochs(perms=...) must not shuffle on the device"
        assert _same_rollout(a["roll"], b["roll"]), f"update {u + 1}: rollouts differ"
        assert _same_update(a, b), f"update {u + 1}: the device-shuffle update differs from its injected permutation"
    monkeypatch.setenv("B200RL_NO_GRAPHS", "1")
    eager_run, eager_replays = _run(f"{cfgname} perms eager", cfgname, "device", updates, monkeypatch, perms=perms)
    monkeypatch.delenv("B200RL_NO_GRAPHS")
    assert eager_replays == 0
    assert _same_rollout(eager_run[0]["roll"], perm_run[0]["roll"]), "rollout 1 starts from identical parameters"
    pe, pg = eager_run[-1]["params"], perm_run[-1]["params"]
    n = sum(v.size for v in pe.values())
    diff = max(float(np.abs(pe[k] - pg[k]).max()) for k in pe)
    mdiff = sum(float(np.abs(pe[k] - pg[k]).sum()) for k in pe) / n
    print(f"[observed] {cfgname}: graphs-vs-eager params max {diff:.2e} mean {mdiff:.2e} "
          f"(graph-vs-graph spread 0: the two graph runs are bit-identical)")
    # test_round2_gpu's criterion with the measured run-to-run spread, here 0
    assert mdiff <= 2e-6 and diff <= 1e-3, (mdiff, diff)
    assert np.allclose(eager_run[-1]["stats"], perm_run[-1]["stats"], rtol=5e-3, atol=5e-3)
    assert eager_run[-1]["t"] == perm_run[-1]["t"] == updates * L["nminibatches"] * nep
    # d. the host env with the same seed
    host_run, _ = _run(f"{cfgname} host env", cfgname, "host", 2, monkeypatch)
    for u, (a, h) in enumerate(zip(dev_run, host_run)):
        assert [k for k, _, _ in h["calls"]] == [k for k, _, _ in a["calls"]]
        assert _same_rollout(a["roll"], h["roll"]), f"update {u + 1}: host-env rollout differs from the device env's"
        assert _same_update(a, h), f"update {u + 1}: host-env update differs from the device env's"


# ================================================================================================ 4. recurrent
def test_recurrent_device_shuffle_takes_the_host_path(monkeypatch):
    from baselines_b200.common.policies import build_policy
    from baselines_b200.common.vec_env import DeviceSyntheticVecEnv
    from baselines_b200.ppo2 import ppo2
    from baselines_b200.ppo2.model import Model
    from baselines_b200.ppo2.runner import Runner
    N, T, nmb, nep = 16, 8, 4, 3
    monkeypatch.delenv("B200RL_NO_GRAPHS", raising=False)

    def no_device_shuffle(*a):
        raise AssertionError("a recurrent policy must not shuffle on the device")
    monkeypatch.setattr(ppo2, "ops_shuffle", no_device_shuffle)
    runs = []
    for use_perms in (False, True):
        np.random.seed(0)
        env = DeviceSyntheticVecEnv(N, (11,), np.float32, act_dim=3, seed=0, device=DEV)
        model = Model(policy=build_policy(env, "lstm", nlstm=64), ob_space=env.observation_space,
                      ac_space=env.action_space, nbatch_act=N, nbatch_train=N * T // nmb, nsteps=T, ent_coef=0.0,
                      vf_coef=0.5, max_grad_norm=0.5, comm=False)
        assert model.recurrent
        runner = Runner(env=env, model=model, nsteps=T, gamma=0.99, lam=0.95)
        out = []
        for u in range(2):
            state = np.random.get_state()
            perms = None
            if use_perms:                                    # np.random.shuffle(envinds) replayed from that state
                rs = np.random.RandomState()
                rs.set_state(runs[0][u]["state"])
                envinds, perms = np.arange(N), []
                for _ in range(nep):
                    rs.shuffle(envinds)
                    perms.append(envinds.copy())
            ro, _ = runner.run_device()
            st = ppo2.run_epochs(model, ro, 3e-4, 0.2, N * T, N * T // nmb, nep, DEV, perms=perms, shuffle="device")
            out.append(dict(state=state, stats=torch.stack(st).cpu().numpy(), params=model.get_params(),
                            m=model.net.store.m.clone(), v=model.net.store.v.clone(), t=model.opt.t,
                            roll={f: getattr(ro, f).clone() for f in ROLLOUT_FIELDS}))
        runs.append(out)
    s0, s1 = runs[0][0]["state"], runs[0][1]["state"]
    assert s0[2] != s1[2] or not np.array_equal(s0[1], s1[1]), "the host shuffle did not draw from the numpy stream"
    for u, (a, b) in enumerate(zip(*runs)):
        assert _same_rollout(a["roll"], b["roll"]), f"update {u + 1}: recurrent rollouts differ"
        assert _same_update(a, b), f"update {u + 1}: recurrent update differs from perms of the same numpy state"
