"""DQN parameter-space noise on the GPU (deepq/build_graph.py:202-314): the perturbation and KL / scale-adaptation kernels,
and the act function built on them (one shared trunk, perturbed and adaptive stream copies)."""
import numpy as np
import pytest
import torch

import _layer_norm_refs as L

pytestmark = pytest.mark.gpu


def _jobs(rows):
    return torch.tensor(rows, dtype=torch.int64, device="cuda")


def test_param_perturb_injected_noise_is_exact_and_copies_stay_copies():
    from baselines_b200 import ops
    rng = np.random.RandomState(0)
    src = torch.from_numpy(rng.randn(5000).astype(np.float32)).cuda()
    jobs = [(10, 0, 1000, 1), (2000, 1000, 7, 0), (3000, 1008, 1537, 1)]      # 1007 is a gap no job writes
    dst = torch.full((2600,), 9.0, dtype=torch.float32, device="cuda")
    n = torch.from_numpy(rng.randn(2600).astype(np.float32)).cuda()
    scale = torch.tensor([0.37], dtype=torch.float32, device="cuda")
    ctr = torch.zeros(1, dtype=torch.int64, device="cuda")
    ops.param_perturb(src, dst, _jobs(jobs), 3, 1537, scale, 1, ctr, normals=n)
    got, s, nn_ = dst.cpu().numpy(), src.cpu().numpy(), n.cpu().numpy()
    want = np.full(2600, 9.0, np.float32)
    want[0:1000] = s[10:1010] + np.float32(0.37) * nn_[0:1000]                 # float32 multiply, then float32 add
    want[1000:1007] = s[2000:2007]
    want[1008:2545] = s[3000:4537] + np.float32(0.37) * nn_[1008:2545]
    assert np.array_equal(got, want)


def test_param_perturb_philox_stream_replays_on_the_host():
    from baselines_b200 import ops
    N, seed = 40000, 987654321
    src = torch.zeros(N, dtype=torch.float32, device="cuda")
    scale = torch.ones(1, dtype=torch.float32, device="cuda")
    outs = []
    for off in (0, 3):
        dst = torch.empty(N, dtype=torch.float32, device="cuda")
        ctr = torch.full((1,), off, dtype=torch.int64, device="cuda")
        ops.param_perturb(src, dst, _jobs([(0, 0, N, 1)]), 1, N, scale, seed, ctr)
        outs.append(dst.cpu().numpy())
        ref = L.philox_normals(seed, off, np.arange(N))
        assert np.allclose(outs[-1], ref, atol=2e-5, rtol=1e-5), float(np.abs(outs[-1] - ref).max())
        assert abs(outs[-1].mean()) < 0.02 and abs(outs[-1].std() - 1.0) < 0.02
    assert not np.array_equal(outs[0], outs[1])


@pytest.mark.parametrize("B", [1, 32, 300, 1000])
@pytest.mark.parametrize("dueling", [True, False])
def test_adapt_kernel_mean_kl_and_both_scale_updates(B, dueling):
    from baselines_b200 import ops
    rng = np.random.RandomState(B)
    nA, ld = 6, 16
    a, b = rng.randn(B, ld).astype(np.float32), rng.randn(B, ld).astype(np.float32)
    b[:, :nA + 1] = a[:, :nA + 1] + 0.3 * b[:, :nA + 1]

    def q(o):
        o = o.astype(np.float64)
        return o[:, nA:nA + 1] + o[:, :nA] - o[:, :nA].mean(1, keepdims=True) if dueling else o[:, :nA]
    ref = L.mean_kl(q(a), q(b))
    for thr, up in ((ref * 2, True), (ref / 2, False)):
        scale = torch.tensor([0.02], dtype=torch.float32, device="cuda")
        t = torch.tensor([thr], dtype=torch.float32, device="cuda")
        kl = torch.zeros(1, dtype=torch.float32, device="cuda")
        ops.dqn_param_noise_adapt(torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda(), ld, nA, dueling, B, scale, t, kl)
        assert abs(kl.item() - ref) <= 2e-5 * abs(ref) + 1e-7, (kl.item(), ref)
        want = np.float32(0.02) * np.float32(1.01) if up else np.float32(0.02) / np.float32(1.01)
        assert np.float32(scale.item()) == np.float32(want)
    # the bound tells KL(p || q) from KL(q || p)
    assert abs(L.mean_kl(q(b), q(a)) - ref) > 2e-5 * abs(ref) + 1e-7


# --------------------------------------------------------------------------------------------------- the act function
def _model(seed=3, B=32, **kw):
    from baselines_b200.common import spaces
    from baselines_b200.deepq.build_graph import DQNModel
    kw = dict(dict(hiddens=(64,), dueling=True, layer_norm=True), **kw)
    np.random.seed(seed)                       # the model draws the seed of its random streams from numpy's global state
    return DQNModel(spaces.Box(-5, 5, (8,), np.float32), 5, "mlp", lr=1e-3, gamma=0.99, grad_norm_clipping=10,
                    batch_cap=B, seed=seed, param_noise=True, **kw)


def _q_float64(model, copy_=None, obs=None):
    """Q values in float64 from the model's float32 variables, the stream fully_connected ones taken from copy_."""
    from oracle import nets
    tp = dict(model.q.store.export_tf("params"))
    if copy_ is not None:
        for k, v in copy_.export_tf().items():
            tp[k.replace(copy_.scope, "deepq/q_func", 1)] = v
    tp = nets.to_torch(tp, torch.float64)
    with torch.no_grad():
        return L.q_forward(tp, "mlp", torch.as_tensor(obs), "deepq/q_func", len(model.q.hiddens), model.q.dueling).numpy()


def test_reset_perturbs_the_fully_connected_variables_only_and_they_stay_until_the_next_reset():
    from baselines_b200.deepq.build_graph import build_act
    model = _model()
    pn, act = model.pn, build_act(model)
    rng = np.random.RandomState(0)
    obs = rng.randn(16, 8).astype(np.float32)
    qv = model.q.store.export_tf("params")
    fc = {k for k in qv if "fully_connected" in k}
    assert {k.replace("perturbed_q_func", "q_func") for k in pn.perturbed.export_tf()} == fc
    assert fc and all("mlp_fc" not in k and "LayerNorm" not in k for k in fc)      # trunk and norms are q_func's own
    before, adaptive0 = pn.perturbed.export_tf(), pn.adaptive.params.clone()
    for k, v in before.items():                                                    # until the first reset: q_func
        assert np.array_equal(v, qv[k.replace("perturbed_q_func", "q_func")])
    pn.normals = torch.from_numpy(rng.randn(pn.perturbed.numel).astype(np.float32)).cuda()
    n = pn.normals.cpu().numpy()
    act(obs, reset=True, update_param_noise_threshold=0.05)
    after = pn.perturbed.export_tf()
    for k, (o, sh) in pn.perturbed.tf_names.items():
        want = qv[k.replace("perturbed_q_func", "q_func")] + np.float32(0.01) * n[o:o + int(np.prod(sh))].reshape(sh)
        assert np.array_equal(after[k], want), k
    assert torch.equal(pn.adaptive.params, adaptive0)                              # no scale update: untouched
    # greedy actions are the argmax of the PERTURBED scores
    a = act(obs, stochastic=False, update_param_noise_threshold=0.05)
    qp = _q_float64(model, pn.perturbed, obs)
    top2 = np.sort(qp, 1)[:, -2:]
    clear = top2[:, 1] - top2[:, 0] > 1e-2
    assert clear.sum() >= 8 and np.array_equal(a[clear], qp.argmax(1)[clear])
    out = pn.perturbed.out[:16].cpu().numpy()
    assert np.array_equal(a, (out[:, 5:6] + out[:, :5] - out[:, :5].mean(1, keepdims=True)).argmax(1))
    # calls without reset, scale updates and a change of q_func leave the perturbed copy alone
    pn.normals = None
    for _ in range(3):
        act(obs, update_param_noise_threshold=0.05, update_param_noise_scale=True)
    model.q.store.params.mul_(1.5)
    model.q.refresh()
    act(obs, update_param_noise_threshold=0.05)
    assert all(np.array_equal(v, after[k]) for k, v in pn.perturbed.export_tf().items())
    assert not torch.equal(pn.adaptive.params, adaptive0)


def test_mean_kl_against_float64_and_reset_uses_the_scale_before_the_update():
    from baselines_b200.deepq.build_graph import build_act
    model = _model()
    pn, act = model.pn, build_act(model)
    rng = np.random.RandomState(1)
    obs = rng.randn(32, 8).astype(np.float32)
    pn.scale.fill_(0.2)                                              # a perturbation large enough for a KL well above fp16
    pn.normals = torch.from_numpy(rng.randn(pn.perturbed.numel).astype(np.float32)).cuda()
    n = pn.normals.cpu().numpy()
    act(obs, reset=True, update_param_noise_threshold=1e9, update_param_noise_scale=True)
    ref = L.mean_kl(_q_float64(model, None, obs), _q_float64(model, pn.adaptive, obs))
    got = pn.mean_kl.item()
    assert ref > 1e-3 and abs(got - ref) <= 0.05 * ref + 1e-4, (got, ref)          # fp16 operands on both sides
    assert np.float32(pn.scale.item()) == np.float32(np.float32(0.2) * np.float32(1.01))
    qv = model.q.store.export_tf("params")
    for k, (o, sh) in pn.perturbed.tf_names.items():                  # perturbed with 0.2, not 0.2 * 1.01
        want = qv[k.replace("perturbed_q_func", "q_func")] + np.float32(0.2) * n[o:o + int(np.prod(sh))].reshape(sh)
        assert np.array_equal(pn.perturbed.export_tf()[k], want), k


def _drive(model, calls, obs):
    from baselines_b200.deepq.build_graph import build_act
    act, pn, sm = build_act(model), model.pn, L.ParamNoiseState()
    trace = []
    for kw in calls:
        a = act(obs, **kw)
        sm.call(pn.mean_kl.item(), **kw)
        assert np.float32(pn.scale.item()) == sm.scale and np.float32(pn.threshold.item()) == sm.threshold
        assert np.float32(model._eps_dev.item()) == sm.eps
        trace.append((a.copy(), pn.scale.item(), pn.mean_kl.item()))
    return trace


def _calls(n, seed):
    rng = np.random.RandomState(seed)
    calls = []
    for i in range(n):
        kw = dict(reset=bool(rng.rand() < 0.15), update_param_noise_scale=bool(rng.rand() < 0.7))
        if rng.rand() < 0.8:
            kw["update_param_noise_threshold"] = float(rng.choice([-1.0, 1e-4, 5e-3, 0.05]))
        if rng.rand() < 0.3:
            kw["update_eps"] = float(rng.choice([-1.0, 0.0, 0.1]))
        calls.append(kw)
    return calls


def test_two_hundred_mixed_calls_follow_the_float32_state_machine_replayed_or_eager(monkeypatch):
    """Scale, threshold and eps after every one of 200 calls with mixed flags equal the float32 state machine fed with
    the measured mean_kl; and the sequences replayed from captured graphs give the same actions, scales and mean_kl as
    the eager ones."""
    obs = np.random.RandomState(2).randn(4, 8).astype(np.float32)
    calls = _calls(200, 5)
    traces = []
    for no_graphs in ("0", "1"):
        monkeypatch.setenv("B200RL_NO_GRAPHS", no_graphs)
        model = _model(seed=7)
        traces.append(_drive(model, calls, obs))
        if no_graphs == "0":
            assert {k[0] for k in model.graphs.graphs} == {"act_pn"} and len(model.graphs.graphs) >= 3
    scales = {t[1] for t in traces[0]}
    assert len(scales) > 20                                          # the scale moved both ways
    for (a0, s0, k0), (a1, s1, k1) in zip(*traces):
        assert np.array_equal(a0, a1) and s0 == s1 and k0 == k1


def test_save_act_load_act_continues_with_the_saved_perturbation(tmp_path):
    from baselines_b200 import deepq
    from baselines_b200.common import spaces
    from baselines_b200.deepq.build_graph import DQNModel, build_act
    params = dict(ob_space=spaces.Box(-5, 5, (8,), np.float32), num_actions=5, network="mlp", lr=1e-3, gamma=0.99,
                  grad_norm_clipping=10, batch_cap=32, seed=3, param_noise=True, hiddens=(64,), layer_norm=True)
    model = DQNModel(**params)
    aw = deepq.ActWrapper(build_act(model), params, model)
    obs = np.random.RandomState(3).randn(32, 8).astype(np.float32)
    model.pn.scale.fill_(0.3)
    for i in range(3):
        aw(obs, reset=(i == 0), update_param_noise_threshold=0.01, update_param_noise_scale=True)
    want = aw(obs, stochastic=False, update_param_noise_threshold=0.01)
    plain = _q_float64(model, None, obs).argmax(1)
    assert not np.array_equal(want, plain)                            # the perturbation matters at this scale
    path = str(tmp_path / "act.pkl")
    aw.save_act(path)
    import joblib
    aw.save(str(tmp_path / "vars"))
    keys = set(joblib.load(str(tmp_path / "vars")))
    for k in ("deepq/param_noise_scale:0", "deepq/param_noise_threshold:0",
              "deepq/perturbed_q_func/action_value/fully_connected/weights:0",
              "deepq/perturbed_q_func/state_value/fully_connected_1/biases:0",
              "deepq/adaptive_q_func/action_value/fully_connected_1/weights:0",
              "deepq/q_func/action_value/LayerNorm/gamma:0"):
        assert k in keys, k
    again = deepq.load_act(path)
    assert np.float32(again.model.pn.scale.item()) == np.float32(model.pn.scale.item())
    assert np.float32(again.model.pn.threshold.item()) == np.float32(0.01)
    assert np.array_equal(again(obs, stochastic=False, update_param_noise_threshold=0.01), want)
    # a file without the noise keys loads as before: the noise state stays what it was
    d = {k: v for k, v in joblib.load(str(tmp_path / "vars")).items() if "param_noise" not in k and "perturbed" not in k
         and "adaptive" not in k}
    joblib.dump(d, str(tmp_path / "old"))
    again.model.pn.scale.fill_(0.125)
    again.load(str(tmp_path / "old"))
    assert again.model.pn.scale.item() == 0.125


def test_deepq_learn_with_param_noise_and_layer_norm_solves_identity_env():
    """deepq.learn(param_noise=True, layer_norm=True) on the contextual-bandit identity env of test_deepq_gpu, at that
    test's threshold: 0.9 mean reward over 200 greedy steps of q_func, the network that was trained.  The perturbed
    network only changes at an episode's start, so exploration is one draw per episode: with that test's 50-step
    episodes and 4000 steps (80 draws) the one run made reached 0.58; the budget here is 6000 steps of 5-step episodes
    (1200 draws), set from one run."""
    from baselines_b200 import deepq
    from baselines_b200.common import spaces

    class Env:
        def __init__(self, n=5, ep_len=50):
            self.n, self.ep_len = n, ep_len
            self.observation_space = spaces.Box(0, 1, (n,), np.float32)
            self.action_space = spaces.Discrete(n)
            self.rng = np.random.RandomState(0)

        def _ob(self):
            o = np.zeros(self.n, np.float32)
            o[self.s] = 1
            return o

        def reset(self):
            self.s, self.t = self.rng.randint(self.n), 0
            return self._ob()

        def step(self, a):
            r = 1.0 if int(a) == self.s else 0.0
            self.s, self.t = self.rng.randint(self.n), self.t + 1
            return self._ob(), r, self.t >= self.ep_len, {}

    env = Env(ep_len=5)
    act = deepq.learn(env, "mlp", seed=0, lr=1e-3, total_timesteps=6000, buffer_size=2000, exploration_fraction=0.3,
                      exploration_final_eps=0.02, train_freq=1, batch_size=32, print_freq=None, checkpoint_freq=None,
                      learning_starts=200, gamma=0.0, target_network_update_freq=200, prioritized_replay=True,
                      hiddens=(64,), dueling=True, layer_norm=True, param_noise=True)
    pn = act.model.pn
    assert pn.ctr.item() > 6000 and pn.scale.item() != np.float32(0.01)       # it perturbed and adapted throughout
    ob, tot = env.reset(), 0.0
    for _ in range(200):
        ob, r, d, _ = env.step(int(act.model.q_values(ob[None]).argmax(1)[0]))
        tot += r
        if d:
            ob = env.reset()
    assert tot / 200 > 0.9, tot / 200
