"""Recurrent PPO2 policies (lstm, cnn_lstm) on the LSTM sequence kernels (csrc/lstm.cu).

Error bounds.  The kernels take Wh as fp16 and keep c, h, the gates and dc in fp32; the float64 references below use the
same fp16-rounded weights, so what remains is fp32 rounding: a dot product of H (forward) or 4H (backward) terms of
size <= |h| |w| <= 1 has error <= n * 2^-24 * sum |terms| (~1e-5 at n = 512), and the cell adds a few ulps per step.
That bounds one step a priori.  Over T steps the error is fed back through Wh; 2e-4 absolute on h, c and the state (1e-3
scaled on dz) is a margin over that per-step bound times the sequence length seen here, not a worst case proven for
every input: it is ~10x the largest error measured on an H100 and far below the size of a wrong formula (each
one-mistake reference below misses by more than 10x the bound).  fp16 outputs add half an fp16 spacing (2^-11
relative)."""
import numpy as np
import pytest
import torch

from _lstm_oracle import lstm_steps as ref_forward, lstm_steps_backward as ref_backward

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _masks(kind, T, B, rng):
    if kind == "zeros":
        return np.zeros((T, B))
    if kind == "ones":
        return np.ones((T, B))
    return (rng.random((T, B)) < 0.2).astype(np.float64)


def _case(H, B, T, mkind, seed=0):
    rng = np.random.default_rng(seed + 7 * B + T + H)
    wh = (rng.standard_normal((H, 4 * H)) / np.sqrt(H)).astype(np.float16).astype(np.float64)
    xg = rng.standard_normal((T * B, 4 * H)).astype(np.float32)
    s0 = rng.standard_normal((B, 2 * H)).astype(np.float32) * 0.5
    masks = _masks(mkind, T, B, rng)
    dh = rng.standard_normal((T * B, H)).astype(np.float16)
    return wh, xg, s0, masks, dh


def _run_kernels(H, B, T, wh, xg, s0, masks, dh):
    from baselines_b200 import ops
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dt)
    xg_d, wh_d, whT_d = t(xg, torch.float32), t(wh, torch.float16), t(wh.T, torch.float16)
    m_d, s_d = t(masks.reshape(-1), torch.uint8), t(s0, torch.float32)
    h = torch.zeros(T * B, H, dtype=torch.float16, device=DEV)
    hp = torch.zeros_like(h)
    c = torch.zeros(T * B, H, dtype=torch.float32, device=DEV)
    gates = torch.zeros(T * B, 4 * H, dtype=torch.float32, device=DEV)
    s_out = torch.zeros(B, 2 * H, dtype=torch.float32, device=DEV)
    ops.lstm_seq_fwd(xg_d, 4 * H, wh_d, m_d, s_d, h, H, T, B, H, state_out=s_out, hprev_out=hp, gates_out=gates,
                     c_out=c)
    dz = torch.zeros(T * B, 4 * H, dtype=torch.float16, device=DEV)
    ops.lstm_seq_bwd(t(dh, torch.float16), H, gates, c, m_d, s_d, whT_d, dz, 4 * H, T, B, H)
    g = lambda a: a.double().cpu().numpy()
    return g(h), g(hp), g(c), g(gates), g(s_out), g(dz)


@pytest.mark.parametrize("H", [64, 128])
@pytest.mark.parametrize("B", [1, 63, 64, 65, 1000])
@pytest.mark.parametrize("T", [1, 5, 128])
@pytest.mark.parametrize("mkind", ["zeros", "ones", "random"])
def test_sequence_kernels_against_float64(H, B, T, mkind):
    wh, xg, s0, masks, dh = _case(H, B, T, mkind)
    h, hp, c, gates, s_out, dz = _run_kernels(H, B, T, wh, xg, s0, masks, dh)
    rh, rc, rg, rhp, rs = ref_forward(xg.astype(np.float64), wh, masks, s0.astype(np.float64), T, B, H)
    tol16 = 2e-4 + 2.0 ** -11                        # fp16 outputs: + half an ulp (2^-11 relative)
    assert (np.abs(h - rh) <= 2e-4 + 2.0 ** -11 * np.abs(rh)).all()
    assert (np.abs(hp - rhp) <= 2e-4 + 2.0 ** -11 * np.abs(rhp)).all()      # the start state's h is not bounded by 1
    assert np.abs(c - rc).max() <= 2e-4 * max(1.0, np.abs(rc).max())
    assert np.abs(gates - rg).max() <= 2e-4
    assert np.abs(s_out - rs).max() <= 2e-4 * max(1.0, np.abs(rc).max())
    rdz = ref_backward(dh.astype(np.float64), rg, rc, masks, s0.astype(np.float64), wh, T, B, H)
    scale = max(1.0, np.abs(rdz).max())
    err_dz = np.abs(dz - rdz).max()
    bound = 1e-3 * scale + 2.0 ** -11 * np.abs(rdz).max()
    assert err_dz <= bound, (err_dz, bound)
    # each bound rejects a reference with one plausible mistake
    if T > 1 and mkind == "random" and B >= 63:
        for mistake in ("mask_after", "swap_fi"):
            wrong = ref_forward(xg.astype(np.float64), wh, masks, s0.astype(np.float64), T, B, H, mistake=mistake)
            assert np.abs(h - wrong[0]).max() > 10 * tol16, mistake
        wrong_dz = ref_backward(dh.astype(np.float64), rg, rc, masks, s0.astype(np.float64), wh, T, B, H,
                                mistake="no_carry")
        assert np.abs(dz - wrong_dz).max() > 10 * bound


def _assert_float64_bounds(H, B, T, wh, xg, s0, masks, dh, h, hp, c, gates, s_out, dz):
    """The bounds of test_sequence_kernels_against_float64 (s_out None: not written)."""
    rh, rc, rg, rhp, rs = ref_forward(xg.astype(np.float64), wh, masks, s0.astype(np.float64), T, B, H)
    assert (np.abs(h - rh) <= 2e-4 + 2.0 ** -11 * np.abs(rh)).all()
    assert (np.abs(hp - rhp) <= 2e-4 + 2.0 ** -11 * np.abs(rhp)).all()
    assert np.abs(c - rc).max() <= 2e-4 * max(1.0, np.abs(rc).max())
    assert np.abs(gates - rg).max() <= 2e-4
    if s_out is not None:
        assert np.abs(s_out - rs).max() <= 2e-4 * max(1.0, np.abs(rc).max())
    rdz = ref_backward(dh.astype(np.float64), rg, rc, masks, s0.astype(np.float64), wh, T, B, H)
    assert np.abs(dz - rdz).max() <= 1e-3 * max(1.0, np.abs(rdz).max()) + 2.0 ** -11 * np.abs(rdz).max()


@pytest.mark.parametrize("H", [64, 128])
@pytest.mark.parametrize("B,T", [(37, 5), (9, 1)])
def test_sequence_kernels_in_the_operand_forms_training_uses(H, B, T):
    """The forms nn.LSTM.forward / backward call the kernels in: gates_out is xg (ldxg = 4H), masks gathered through
    mask_idx and start states through state_idx from a larger permuted rollout, and row pitches ldh, lddh > H and
    lddz > 4H.  Every output is bit-identical to the contiguous call on the equivalent dense operands, meets the float64
    bounds, and leaves the padding columns as they were."""
    from baselines_b200 import ops
    wh, xg, _, _, dh = _case(H, B, T, "random", seed=11)
    rng = np.random.default_rng(H + B)
    n_roll, n_env = 3 * T * B + 5, 2 * B + 3                 # the rollout the minibatch's rows and states come from
    masks_roll = (rng.random(n_roll) < 0.25).astype(np.uint8)
    states_roll = (rng.standard_normal((n_env, 2 * H)) * 0.5).astype(np.float32)
    mask_idx = rng.permutation(n_roll)[:T * B]
    state_idx = rng.permutation(n_env)[:B]
    masks = masks_roll[mask_idx].reshape(T, B).astype(np.float64)
    s0 = states_roll[state_idx]
    dense = _run_kernels(H, B, T, wh, xg, s0, masks, dh)

    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dt)
    ldh, lddh, lddz = H + 8, H + 16, 4 * H + 8
    xg_d = t(xg, torch.float32)                              # receives the gates in place
    h = torch.full((T * B, ldh), -7.0, dtype=torch.float16, device=DEV)
    hp = torch.zeros(T * B, H, dtype=torch.float16, device=DEV)
    c = torch.zeros(T * B, H, dtype=torch.float32, device=DEV)
    s_out = torch.zeros(B, 2 * H, dtype=torch.float32, device=DEV)
    m_d, mi_d = t(masks_roll, torch.uint8), t(mask_idx, torch.int64)
    s_d, si_d = t(states_roll, torch.float32), t(state_idx, torch.int64)
    ops.lstm_seq_fwd(xg_d, 4 * H, t(wh, torch.float16), m_d, s_d, h, ldh, T, B, H, mask_idx=mi_d, state_idx=si_d,
                     state_out=s_out, hprev_out=hp, gates_out=xg_d, c_out=c)
    dh_d = torch.full((T * B, lddh), 3.0, dtype=torch.float16, device=DEV)
    dh_d[:, :H] = t(dh, torch.float16)
    dz = torch.full((T * B, lddz), 5.0, dtype=torch.float16, device=DEV)
    ops.lstm_seq_bwd(dh_d, lddh, xg_d, c, m_d, s_d, t(wh.T, torch.float16), dz, lddz, T, B, H, mask_idx=mi_d,
                     state_idx=si_d)
    torch.cuda.synchronize()
    assert torch.all(h[:, H:] == -7.0) and torch.all(dh_d[:, H:] == 3.0) and torch.all(dz[:, 4 * H:] == 5.0)
    assert torch.equal(s_d, t(states_roll, torch.float32))   # the rollout's states are only read
    g = lambda a: a.double().cpu().numpy()
    got = (g(h[:, :H]), g(hp), g(c), g(xg_d), g(s_out), g(dz[:, :4 * H]))
    for name, a, b in zip(("h", "hprev", "c", "gates", "state_out", "dz"), got, dense):
        assert np.array_equal(a, b), name
    _assert_float64_bounds(H, B, T, wh, xg, s0, masks, dh, *got)
    # the gather matters: the rollout's first rows and states are another input
    plain = _run_kernels(H, B, T, wh, xg, states_roll[:B], masks_roll[:T * B].reshape(T, B).astype(np.float64), dh)
    assert not np.array_equal(plain[0], got[0])

    if T == 1:
        # acting: the state advances in place (state_out is state_in, no state_idx)
        st = t(s0, torch.float32)
        h1 = torch.zeros(B, H, dtype=torch.float16, device=DEV)
        mk = t(masks.reshape(-1), torch.uint8)
        ops.lstm_seq_fwd(t(xg, torch.float32), 4 * H, t(wh, torch.float16), mk, st, h1, H, 1, B, H, state_out=st)
        torch.cuda.synchronize()
        assert torch.equal(h1.double().cpu(), torch.from_numpy(dense[0])) and np.array_equal(g(st), dense[4])


@pytest.mark.parametrize("H", [64, 128])
def test_lstm_layer_gradients_against_float64(H):
    """LSTM layer: dWh = hprev^T dz, dWx = x^T dz, db = colsum(dz), dx = dz Wx^T on the GEMM, against float64."""
    from baselines_b200 import nn
    rng = np.random.default_rng(H)
    T, B, nin = 16, 65, 48
    store = nn.ParamStore(torch.device(DEV))
    lstm = nn.LSTM(store, "pi", "ppo2_model/pi", nin, H, lambda shape, scale: nn.ortho_init(shape, scale, np.random))
    store.finalize()
    lstm.materialize(T * B)
    store.views["pi/lstm/wx/b"].copy_(torch.from_numpy(rng.standard_normal(4 * H).astype(np.float32) * 0.1))
    lstm.refresh()
    x = rng.standard_normal((T * B, nin)).astype(np.float16)
    masks = (rng.random((T, B)) < 0.2).astype(np.float64)
    s0 = (rng.standard_normal((B, 2 * H)) * 0.5).astype(np.float32)
    x_d = torch.from_numpy(x).to(DEV)
    m_d = torch.from_numpy(masks.reshape(-1).astype(np.uint8)).to(DEV)
    s_d = torch.from_numpy(s0).to(DEV)
    seq = nn.Seq(T, B, m_d, None, s_d, None, None)
    h, _ = lstm.forward(x_d, nin, seq)
    dh = rng.standard_normal((T * B, H)).astype(np.float16)
    lstm.dh.copy_(torch.from_numpy(dh))
    dx = torch.zeros(T * B, nin, dtype=torch.float16, device=DEV)
    store.grads.zero_()
    lstm.backward(1.0, dx=dx, ldo=nin)
    torch.cuda.synchronize()
    wx = store.views["pi/lstm/wx/w"].cpu().numpy().astype(np.float16).astype(np.float64)
    wh = store.views["pi/lstm/wh"].cpu().numpy().astype(np.float16).astype(np.float64)
    b = store.views["pi/lstm/wx/b"].cpu().numpy().astype(np.float64)
    xg = x.astype(np.float64) @ wx + b
    rh, rc, rg, rhp, _ = ref_forward(xg, wh, masks, s0.astype(np.float64), T, B, H)
    assert np.abs(h.double().cpu().numpy() - rh).max() <= 2e-4 + 2.0 ** -11
    rdz = ref_backward(dh.astype(np.float64), rg, rc, masks, s0.astype(np.float64), wh, T, B, H)
    # the GEMMs read dz and hprev as fp16: the references use the same roundings of the float64 values
    rdz16 = rdz.astype(np.float16).astype(np.float64)
    rhp16 = rhp.astype(np.float16).astype(np.float64)
    g = lambda n: store.gviews[n].cpu().numpy().astype(np.float64)
    for got, want in ((g("pi/lstm/wh"), rhp16.T @ rdz16), (g("pi/lstm/wx/w"), x.astype(np.float64).T @ rdz16),
                      (g("pi/lstm/wx/b"), rdz16.sum(0)), (dx.double().cpu().numpy(), rdz16 @ wx.T)):
        # fp16 roundings of dz / hprev differ by one ulp between kernel and reference: 2^-10 relative per term
        bound = 2.0 ** -9 * np.abs(want).max() + 2e-3 * np.sqrt(T * B) * 2.0 ** -10 * max(1.0, np.abs(rdz).max())
        assert np.abs(got - want).max() <= bound, (np.abs(got - want).max(), bound)


# ------------------------------------------------------------------------------------------- whole-model tests
def _model(network, ob_space, ac_space, nenv, nsteps, nminibatches=1, seed=0, train_chunk=None, **kw):
    from baselines_b200.common.policies import build_policy
    from baselines_b200.ppo2.model import Model

    class E:
        pass
    env = E()
    env.observation_space, env.action_space, env.num_envs = ob_space, ac_space, nenv
    np.random.seed(seed)
    policy = build_policy(env, network, **kw)
    return Model(policy=policy, ob_space=ob_space, ac_space=ac_space, nbatch_act=nenv,
                 nbatch_train=nenv * nsteps // nminibatches, nsteps=nsteps, ent_coef=0.01, vf_coef=0.5,
                 max_grad_norm=0.5, comm=False, train_chunk=train_chunk)


def _spaces(kind):
    from baselines_b200.common import spaces
    if kind == "box":
        return spaces.Box(-5, 5, (7,), np.float32), spaces.Discrete(4)
    if kind == "discrete":
        return spaces.Discrete(5), spaces.Discrete(3)
    return spaces.Box(0, 255, (84, 84, 4), np.uint8), spaces.Discrete(6)


def _obs(kind, T, N, rng):
    if kind == "box":
        return rng.standard_normal((T, N, 7)).astype(np.float32)
    if kind == "discrete":
        return rng.integers(0, 5, (T, N)).astype(np.int64)
    return rng.integers(0, 256, (T, N, 84, 84, 4)).astype(np.uint8)


@pytest.mark.parametrize("kind,network,nlstm", [("box", "lstm", 128), ("discrete", "lstm", 64),
                                                ("atari", "cnn_lstm", 128)])
def test_acting_equals_training_bitwise(kind, network, nlstm):
    """T chained T = 1 acting passes give the same h, state and values bit for bit as one train-forward sequence, and
    the result of a row does not depend on how many rows run with it."""
    from baselines_b200 import nn
    rng = np.random.default_rng(1)
    T, N = 6, 5
    ob, ac = _spaces(kind)
    model = _model(network, ob, ac, N, T, nlstm=nlstm)
    net = model.net
    H = net.nlstm
    obs = _obs(kind, T, N, rng)
    dones = (rng.random((T, N)) < 0.3).astype(np.uint8)
    s0 = (rng.standard_normal((N, 2 * H)) * 0.3).astype(np.float32)
    st = torch.from_numpy(s0).to(DEV)
    mk = torch.zeros(N, dtype=torch.uint8, device=DEV)
    a = torch.zeros(net.action_shape(N), dtype=net.action_dtype, device=DEV)
    v = torch.zeros(N, device=DEV)
    nlp = torch.zeros(N, device=DEV)
    acts_h, acts_v = [], []
    for t in range(T):
        x = net.encode_obs(obs[t])
        mk.copy_(torch.from_numpy(dones[t]))
        model.step_device(x, a, v, nlp, state=st, mask=mk)
        acts_h.append(net.tower_pi.lstm.h[:N].clone())
        acts_v.append(v.clone())
    xs = net.encode_obs(obs.reshape((T * N,) + obs.shape[2:]))
    d_all = torch.from_numpy(dones.reshape(-1)).to(DEV)
    s0_d = torch.from_numpy(s0).to(DEV)
    s_out = torch.zeros_like(s0_d)
    net.forward(xs, T * N, seq=nn.Seq(T, N, d_all, None, s0_d, None, s_out))
    h_seq = net.tower_pi.lstm.h[:T * N].view(T, N, H).clone()
    v_seq = net.v_out[:T * N, 0].view(T, N)
    for t in range(T):
        assert torch.equal(h_seq[t], acts_h[t]), t
        assert torch.equal(v_seq[t], acts_v[t]), t
    assert torch.equal(s_out, st)
    # one environment alone gives the same bits as inside the batch
    s1 = torch.from_numpy(s0[2:3].copy()).to(DEV)
    net.forward(net.encode_obs(obs[:, 2]), T, seq=nn.Seq(T, 1, torch.from_numpy(dones[:, 2].copy()).to(DEV), None, s1,
                                                         None, None))
    assert torch.equal(net.tower_pi.lstm.h[:T], h_seq[:, 2])


def _vec_env(kind, N, seed):
    from baselines_b200.common.vec_env import DummyVecEnv
    from baselines_b200 import envs
    from baselines_b200.common import spaces

    class Rand(envs.Env):
        def __init__(self, i):
            self.observation_space, self.action_space = _spaces(kind)
            self.rng = np.random.default_rng(seed * 100 + i)
            self.t = 0

        def _ob(self):
            return _obs(kind, 1, 1, self.rng)[0, 0]

        def reset(self):
            self.t = 0
            return self._ob()

        def step(self, a):
            self.t += 1
            done = self.rng.random() < 0.15
            return self._ob(), float(self.rng.standard_normal()), done, {}
    return DummyVecEnv([lambda i=i: Rand(i) for i in range(N)])


@pytest.mark.parametrize("kind,network", [("box", "lstm"), ("discrete", "lstm"), ("atari", "cnn_lstm")])
def test_update_first_minibatch_and_determinism(kind, network):
    """The first minibatch of the first epoch sees exactly the acting pass (approxkl == clipfrac == 0); two runs of a
    whole update are bit-identical; the runner returns the rollout-start states and carries them across rollouts."""
    from baselines_b200.ppo2.runner import Runner
    from baselines_b200.ppo2.ppo2 import run_epochs
    T, N = 8, 4
    params = []
    for run in range(2):
        ob, ac = _spaces(kind)
        model = _model(network, ob, ac, N, T, nminibatches=2, nlstm=64 if kind == "discrete" else 128)
        runner = Runner(env=_vec_env(kind, N, 3), model=model, nsteps=T, gamma=0.99, lam=0.95)
        out = runner.run()
        assert out[6].shape == (N, 2 * model.net.nlstm) and not out[6].any()     # zero initial state
        np.random.seed(5)
        ro = runner.rollout
        stats = run_epochs(model, ro, 3e-4, 0.2, N * T, N * T // 2, 2, DEV)
        st0 = stats[0].cpu().numpy()
        assert st0[3] == 0.0 and st0[4] == 0.0, st0                 # approxkl, clipfrac
        out2 = runner.run()
        assert np.array_equal(out2[6], runner.rollout.states0.cpu().numpy())
        assert out2[6].any()                                         # the state carried over from the first rollout
        params.append(model.get_params())
    for k in params[0]:
        assert np.array_equal(params[0][k], params[1][k]), k


def test_graph_replay_matches_eager(monkeypatch):
    """The graph-replayed acting and train sequences compute what the eager ones do."""
    from baselines_b200.ppo2.runner import Runner
    from baselines_b200.ppo2.ppo2 import run_epochs
    res = []
    for no_graphs in ("1", "0"):
        monkeypatch.setenv("B200RL_NO_GRAPHS", no_graphs)
        ob, ac = _spaces("box")
        model = _model("lstm", ob, ac, 4, 8, nminibatches=2)
        runner = Runner(env=_vec_env("box", 4, 3), model=model, nsteps=8, gamma=0.99, lam=0.95)
        for _ in range(3):
            runner.run_device()
            np.random.seed(2)
            run_epochs(model, runner.rollout, 3e-4, 0.2, 32, 16, 2, DEV)
        res.append((model.get_params(), runner.rollout.values.cpu().numpy()))
    for k in res[0][0]:
        assert np.array_equal(res[0][0][k], res[1][0][k]), k
    assert np.array_equal(res[0][1], res[1][1])


def test_checkpoint_round_trip(tmp_path):
    from baselines_b200.common import spaces
    ob, ac = _spaces("atari")
    m1 = _model("cnn_lstm", ob, ac, 2, 4, nlstm=64)
    p = m1.get_params()
    for k, shape in (("wx", (512, 256)), ("wh", (64, 256)), ("b", (256,))):
        assert p[f"ppo2_model/pi/lstm/{k}:0"].shape == shape
    path = str(tmp_path / "ck")
    m1.save(path)
    m2 = _model("cnn_lstm", ob, ac, 2, 4, nlstm=64, seed=1)
    m2.load(path)
    p2 = m2.get_params()
    for k in p:
        assert np.array_equal(p[k], p2[k]), k
    obs = np.random.default_rng(0).integers(0, 256, (2, 84, 84, 4)).astype(np.uint8)
    s = np.random.default_rng(1).standard_normal((2, 128)).astype(np.float32)
    v1, v2 = m1.value(obs, S=s, M=[False, True]), m2.value(obs, S=s, M=[False, True])
    assert np.array_equal(v1, v2)


def test_fixed_sequence_learns():
    """The reference's test_fixed_sequence for ppo2 + lstm: a memory task only a recurrent policy can solve."""
    from baselines_b200.common.vec_env import DummyVecEnv
    from baselines_b200.envs import FixedSequenceEnv
    from baselines_b200.ppo2 import ppo2

    def env_fn():
        e = FixedSequenceEnv(n_actions=10, episode_len=5)
        e.seed(0)
        return e
    env = DummyVecEnv([env_fn])
    model = ppo2.learn(network="lstm", env=env, total_timesteps=50000, seed=0, nsteps=10, ent_coef=0.0,
                       nminibatches=1)
    env = DummyVecEnv([env_fn])
    total, done = 0.0, True
    for _ in range(10000):                        # common/tests/util.py simple_test
        if done:
            obs = env.reset()
            state = model.initial_state
        a, _, state, _ = model.step(obs, S=state, M=[False])
        obs, rew, done, _ = env.step(a)
        total += float(rew[0])
    assert total / 10000 > 0.7, total / 10000


def test_cli_trains_and_saves(tmp_path):
    import subprocess
    import sys
    import os
    out = str(tmp_path / "model")
    env = dict(os.environ)
    r = subprocess.run([sys.executable, "-m", "baselines_b200.run", "--alg=ppo2", "--env=CartPole-v0", "--network=lstm",
                        "--num_timesteps=2048", "--nsteps=128", "--nminibatches=1", "--nlstm=64",
                        f"--save_path={out}"], capture_output=True, text=True, env=env,
                       cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))), timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    import joblib
    d = joblib.load(out)
    assert d["ppo2_model/pi/lstm/wh:0"].shape == (64, 256)
