"""GPU: the HER kernels (csrc/her.cu) against exact numpy restatements, whole train steps against the float64 mirror of
tests/_her_refs.py, graph replay against eager, the host reward path, seeded determinism, checkpoints, learning and the
command line."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import _her_refs as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", autouse=True)
def _lib():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from baselines_b200 import build_ext
    build_ext.build()


def _split(x0, in_pad, n):
    x = x0.cpu().numpy()
    return x[:, :n], x[:, in_pad:in_pad + n]


def _value(x0, in_pad, n):
    hi, lo = _split(x0, in_pad, n)
    return (hi.astype(np.float32) + lo.astype(np.float32)).astype(np.float32)


def _agent(dimo=5, dimg=3, dimu=4, T=10, layers=2, hidden=64, batch_size=256, buffer_episodes=12, rbs=2,
           relative_goals=False, max_u=1.0, action_l2=1.0, clip_return=True, replay_strategy='future',
           reward=('sparse', 0.0625), seed=0, norm_clip=5):
    from baselines_b200.her.ddpg import DDPG
    from baselines_b200.her.experiment.config import simple_goal_subtract
    from baselines_b200.her.her_sampler import make_sample_her_transitions

    def reward_fun(ag_2, g, info):
        d = np.linalg.norm(ag_2 - g, axis=-1)
        return -(d > reward[1]).astype(np.float32) if reward[0] == 'sparse' else -d
    sampler = make_sample_her_transitions(replay_strategy, 4, reward_fun)
    sampler.device_reward = reward
    gamma = 1. - 1. / (T + 1)
    return DDPG(input_dims={'o': dimo, 'g': dimg, 'u': dimu, 'info_is_success': 1}, buffer_size=buffer_episodes * (T + 1),
                hidden=hidden, layers=layers, network_class='baselines.her.actor_critic:ActorCritic', polyak=0.95,
                batch_size=batch_size, Q_lr=1e-3, pi_lr=1e-3, norm_eps=0.01, norm_clip=norm_clip, max_u=max_u,
                action_l2=action_l2, clip_obs=200., scope='ddpg', T=T + 1, rollout_batch_size=rbs,
                subtract_goals=simple_goal_subtract, relative_goals=relative_goals, clip_pos_returns=True,
                clip_return=(1. / (1. - gamma)) if clip_return else np.inf, bc_loss=0, q_filter=0, num_demo=0,
                demo_batch_size=0, prm_loss_weight=0, aux_loss_weight=0, sample_transitions=sampler, gamma=gamma,
                seed=seed)


def _episodes(agent, rng, n, dtype=np.float32, scale=1.0):
    T, d = agent.T - 1, agent.input_dims
    ep = {'o': rng.randn(n, T + 1, d['o']) * 3 * scale, 'ag': rng.randn(n, T + 1, d['g']) * scale,
          'g': rng.randn(n, T, d['g']) * scale, 'u': rng.uniform(-1, 1, (n, T, d['u'])) * np.asarray(agent.max_u),
          'info_is_success': rng.randint(0, 2, (n, T, 1))}
    return {k: v.astype(dtype) for k, v in ep.items()}


def _host_ring(agent):
    b = agent.buffer.buffers
    return tuple(b[k].cpu().numpy() for k in ('o', 'ag', 'g', 'u'))


def _stats(agent):
    return ((agent.o_stats.mean.cpu().numpy(), agent.o_stats.std.cpu().numpy()),
            (agent.g_stats.mean.cpu().numpy(), agent.g_stats.std.cpu().numpy()))


# ---------------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("relative", [False, True])
@pytest.mark.parametrize("rtype", ["sparse", "dense"])
def test_cache_uploaded_sample_relabels_rewards_and_encodes_bit_for_bit(relative, rtype):
    from baselines_b200 import ops
    rng = np.random.RandomState(1)
    thr = 0.0625
    agent = _agent(relative_goals=relative, reward=(rtype, thr), max_u=[1.0, 0.5, 2.0, 1.5], buffer_episodes=8)
    # the constructor's 0 * target + 1 * main leaves the targets equal to the main networks, bit for bit
    for t, m in ((agent.target_pi, agent.main_pi), (agent.target_Q, agent.main_Q)):
        assert torch.equal(t.store.params.view(torch.int32), m.store.params.view(torch.int32))
    np.random.seed(3)
    for _ in range(7):                            # 14 episodes into 8 slots: the ring fills, then random replacement
        agent.store_episode(_episodes(agent, rng, 2))
    assert agent.buffer.current_size == agent.buffer.size
    # goals at exactly the threshold distance from ag_2 (dyadic values: the differences are exact)
    b = agent.buffer.buffers
    b['g'][0, 3] = torch.tensor([0.25, 0.5, -0.75], dtype=torch.float64)
    b['ag'][0, 4] = torch.tensor([0.25 + thr, 0.5, -0.75], dtype=torch.float64)
    ring = _host_ring(agent)
    T = agent.T - 1
    B = agent.cap
    sel = agent.buffer.draw(B)
    sel[:4] = [[0, 3, -1], [0, 3, 4], [1, T - 1, T], [2, 0, T]]   # at the threshold, relabelled, future_t = T
    S = agent.graphs.upload("sel", sel, agent.cap, (3,), torch.int64, agent.device)
    pi, Q, tpi, tQ = agent.main_pi, agent.main_Q, agent.target_pi, agent.target_Q
    st = _stats(agent)
    ops.her_sample(agent.buffer.ring, S, B, relative, 200., agent.o_stats.mean, agent.o_stats.std, agent.g_stats.mean, agent.g_stats.std, 5.0,
                   agent.max_u_dev, {'sparse': 1, 'dense': 2}[rtype], thr, agent.r, pi.x0, tpi.x0, pi.in_pad, Q.x0,
                   tQ.x0, Q.in_pad)
    torch.cuda.synchronize()
    ref = R.sample(ring, sel, relative, 200., st, 5.0, np.asarray([1.0, 0.5, 2.0, 1.5], np.float32),
                   reward=(rtype, thr))
    assert np.array_equal(agent.r[:B].cpu().numpy().view(np.uint32), ref['r'].view(np.uint32))
    if rtype == 'sparse':
        assert ref['r'][0] == 0.0                 # exactly at the threshold: not "> threshold"
    dimo, dimg = agent.dimo, agent.dimg
    want = {
        'pi': np.concatenate([ref['o'], ref['g']], 1), 'tpi': np.concatenate([ref['o_2'], ref['g_2']], 1),
        'Q': np.concatenate([ref['o'], ref['g'], ref['u_in']], 1), 'tQ': np.concatenate([ref['o_2'], ref['g_2']], 1)}
    for name, net, rows, n in (('pi', pi, B, dimo + dimg), ('tpi', tpi, B, dimo + dimg), ('Q', Q, B, Q.nin),
                               ('tQ', tQ, B, dimo + dimg)):
        hi, lo = _split(net.x0[:rows], net.in_pad, n)
        whi, wlo = R.halves(want[name])
        assert np.array_equal(hi.view(np.uint16), whi.view(np.uint16)), name
        assert np.array_equal(lo.view(np.uint16), wlo.view(np.uint16)), name
    hi, lo = _split(Q.x0[B:2 * B], Q.in_pad, dimo + dimg)
    assert np.array_equal(hi.view(np.uint16), R.halves(want['pi'])[0].view(np.uint16))
    # the tempting relabelling mistakes give other goals
    for bad in ('ag_t', 'ag_t1'):
        wrong = R.sample(ring, sel, relative, 200., st, 5.0, np.ones(4, np.float32), reward=(rtype, thr),
                         relabel_at=bad)
        assert not np.array_equal(wrong['g'], ref['g'])


def test_normaliser_bit_for_bit_over_several_stores():
    rng = np.random.RandomState(2)
    for relative, dtype in ((False, np.float32), (True, np.float32), (False, np.float64)):
        agent = _agent(relative_goals=relative)
        state = [(agent.o_stats.state.cpu().numpy(), agent.o_stats.mean.cpu().numpy(), agent.o_stats.std.cpu().numpy()),
                 (agent.g_stats.state.cpu().numpy(), agent.g_stats.mean.cpu().numpy(), agent.g_stats.std.cpu().numpy())]
        for k in range(4):
            ep = _episodes(agent, rng, 2, dtype)
            ep['o'][:, :, 0] = 0.0                # a zero column: its variance is 0 and its std the eps floor
            np.random.seed(10 + k)
            agent.store_episode(ep)
            np.random.seed(10 + k)
            n, T = ep['u'].shape[:2]
            e, t, f = agent.sample_transitions.draw(n, T, n * T)
            sel = np.stack([e, t, f], 1)
            prev = state
            state = R.norm_update([state[0][0], state[1][0]], None, None, ep, sel, relative, 200., 0.01)
            for (st, m, sd), nz in ((state[0], agent.o_stats), (state[1], agent.g_stats)):
                assert np.array_equal(nz.state.cpu().numpy().view(np.uint32), st.view(np.uint32))
                assert np.array_equal(nz.mean.cpu().numpy().view(np.uint32), m.view(np.uint32))
                assert np.array_equal(nz.std.cpu().numpy().view(np.uint32), sd.view(np.uint32))
        assert agent.o_stats.std[0].item() == np.float32(0.01)
        # count starting at 0 instead of 1 gives other statistics
        bad = R.norm_update([prev[0][0], prev[1][0]], None, None, ep, sel, relative, 200., 0.01, count0=0.0)
        assert not np.array_equal(bad[0][1], state[0][1])


# -------------------------------------------------------------------------------------------------- whole steps
BASE = dict(layers=2, hidden=64, clip_return=True, action_l2=1.0, max_u=1.0, replay_strategy='future')
CASES = {
    "l1_h256": dict(layers=1, hidden=256),
    "l3_h256_clip_inf": dict(layers=3, hidden=256, clip_return=False),
    "l2_maxu_vec_l2_0": dict(max_u=[2.0, 0.5, 1.5, 1.0], action_l2=0.0),
    "l2_maxu_scalar_none": dict(max_u=2.0, replay_strategy='none'),
    "l2_maxu_vec_l2_1": dict(max_u=[2.0, 0.5, 1.5, 1.0], action_l2=1.0),
}
# 3 x 256 ReLU towers read fp16 activations and weights: about 1.4e-2 of the layer scale was seen at B = 256
TOL = {1: 3e-2, 256: 3e-2, 1024: 3e-2}


def _bound(dev, ref, scale):
    return float(np.max(np.abs(np.asarray(dev, np.float64) - ref))) / (scale + 1e-12)


def _layer_scales(rg):
    layer = lambda k: k.rsplit("/", 1)[0]
    top = {}
    for k, r in rg.items():
        top[layer(k)] = max(top.get(layer(k), 0.0), float(np.max(np.abs(r))))
    return {k: top[layer(k)] for k in rg}


def _worst(dev, rg, sc=None):
    sc = sc or _layer_scales(rg)
    return max(_bound(dev[k], r, sc[k]) for k, r in rg.items())


def _pi_scales(P, inp, rc, masks):
    """Per pi variable: its layer's largest entry of the -mean(Q_pi) part of the gradient plus that of the action_l2
    part.  The two parts can cancel (one sample at B = 1): against the scale of their sum the fp16 rounding of each
    would look arbitrarily large, against the parts' scales it does not."""
    q_part = R.train_step(P, inp, dict(rc, action_l2=0.0), pi_masks=masks)["pi_grads"]
    full = R.train_step(P, inp, rc, pi_masks=masks)["pi_grads"]
    l2_part = {k: full[k] - q_part[k] for k in full}
    a, b = _layer_scales(q_part), _layer_scales(l2_part)
    return {k: a[k] + b[k] for k in full}


def _prepared(case, B):
    cfg = dict(BASE, **CASES[case])
    agent = _agent(layers=cfg['layers'], hidden=cfg['hidden'], batch_size=B, clip_return=cfg['clip_return'],
                   action_l2=cfg['action_l2'], max_u=cfg['max_u'], replay_strategy=cfg['replay_strategy'],
                   buffer_episodes=40)
    rng = np.random.RandomState(4)
    np.random.seed(5)
    for _ in range(6):
        agent.store_episode(_episodes(agent, rng, 2))
    for _ in range(2):
        agent.train_device()
        agent.update_target_net()
    # a target critic that answers about +3: y = r + gamma Q' is then positive where r = 0, so the upper clip at 0 acts
    agent.target_Q.head.b.fill_(3.0)
    agent.target_Q.refresh()
    return cfg, agent


@pytest.mark.parametrize("B", [1, 256, 1024])
@pytest.mark.parametrize("case", sorted(CASES))
def test_train_step_against_float64(case, B):
    cfg, agent = _prepared(case, B)
    P = {}
    for net in (agent.main_pi, agent.main_Q, agent.target_pi, agent.target_Q):
        P.update(net.tf_variables())
    m_prev = {n: (net.store.export_tf("m"), net.store.export_tf("v")) for n, net in
              (("pi", agent.main_pi), ("Q", agent.main_Q))}
    sel = agent.sample_batch()
    inp = R.sample(_host_ring(agent), sel, False, 200., _stats(agent), 5.0,
                   np.broadcast_to(np.asarray(cfg['max_u'], np.float32), (agent.dimu,)), reward=('sparse', 0.0625))
    rc = dict(scope='ddpg', layers=cfg['layers'], max_u=np.broadcast_to(np.asarray(cfg['max_u'], np.float64),
                                                                        (agent.dimu,)),
              gamma=agent.gamma, clip_return=agent.clip_return, clip_pos_returns=True, action_l2=cfg['action_l2'],
              dimu=agent.dimu)
    agent.stage_batch(sel)
    loss, q_pi = agent.train_device(stage=False)
    # the actor's hidden ReLU decisions: where a float64 pre-activation is within fp16 resolution of zero the device's
    # is as right as the mirror's, and at B = 1 one such unit decides a whole column of its layer's gradient
    masks = [h[:B, :agent.hidden].cpu().numpy() > 0 for h in agent.main_pi.h]
    n_amb, agree = R.ambiguous_units(P, 'ddpg/main/pi', np.concatenate([inp['o'], inp['g']], 1), cfg['layers'], masks)
    assert agree and n_amb <= max(2, B * cfg["hidden"] * cfg["layers"] // 20), (n_amb, agree)
    ref = R.train_step(P, inp, rc, pi_masks=masks)
    tol = TOL[B]
    grads = {}
    pi_sc = _pi_scales(P, inp, rc, masks)
    for net, rg, sc in ((agent.main_Q, ref["Q_grads"], None), (agent.main_pi, ref["pi_grads"], pi_sc)):
        dg = net.store.export_tf("grads")
        grads.update(dg)
        print(case, B, net.scope, "worst", _worst(dg, rg, sc), flush=True)
        assert _worst(dg, rg, sc) < tol, (case, B, _worst(dg, rg, sc))
    assert abs(loss.item() - ref["loss"]) <= tol * (abs(ref["loss"]) + 1e-3)
    y = agent.y[:B].cpu().numpy()
    np.testing.assert_allclose(y, ref["y"], rtol=1e-4, atol=1e-4)
    assert (y <= 0).all()
    np.testing.assert_allclose(q_pi.cpu().numpy(), ref["q_pi"], rtol=tol, atol=tol * (np.abs(ref["q_pi"]).max() + 1e-3))
    # each bound rejects the tempting mistakes that apply to this configuration
    mistakes = ['no_upper_clip']
    if cfg['action_l2'] > 0:
        mistakes.append('l2_over_B')
    if np.any(np.asarray(cfg['max_u']) != 1.0):
        mistakes.append('u_not_scaled')
    for bad in mistakes:
        wrong = R.train_step(P, inp, rc, variant=bad, pi_masks=masks)
        if bad == 'no_upper_clip':
            if np.array_equal(wrong['y'], ref['y']):
                continue
            assert not np.allclose(y, wrong['y'], rtol=1e-4, atol=1e-4), bad
            continue
        w = max(_worst(agent.main_Q.store.export_tf("grads"), wrong["Q_grads"]),
                _worst(agent.main_pi.store.export_tf("grads"), wrong["pi_grads"], pi_sc))
        print(case, B, bad, "rejected by", w, flush=True)
        assert w > tol, (bad, w)
    # Adam on each network from the device's own gradients
    for name, net in (("pi", agent.main_pi), ("Q", agent.main_Q)):
        mm, vv = net.store.export_tf("m"), net.store.export_tf("v")
        for k in mm:
            g = grads[k].astype(np.float64)
            m0, v0 = m_prev[name][0][k], m_prev[name][1][k]
            np.testing.assert_allclose(mm[k], 0.9 * m0 + 0.1 * g, rtol=1e-5, atol=1e-9 + 1e-6 * np.abs(g).max())
            np.testing.assert_allclose(vv[k], 0.999 * v0 + 0.001 * g * g, rtol=1e-4, atol=1e-12 + 1e-6 * (g * g).max())
    # Polyak, bit for bit with polyak * target + (1 - polyak) * main in float32
    before = {**agent.target_pi.tf_variables(), **agent.target_Q.tf_variables()}
    main = {**agent.main_pi.tf_variables(), **agent.main_Q.tf_variables()}
    agent.update_target_net()
    after = {**agent.target_pi.tf_variables(), **agent.target_Q.tf_variables()}
    for k, v in after.items():
        want = np.float32(0.95) * before[k] + np.float32(1. - 0.95) * main[k.replace('/target/', '/main/')]
        assert np.array_equal(v.view(np.uint32), want.astype(np.float32).view(np.uint32)), k


def _train_run(graphs_on, monkeypatch, host_reward=False):
    monkeypatch.setenv("B200RL_NO_GRAPHS", "0" if graphs_on else "1")
    agent = _agent(batch_size=256, buffer_episodes=40)
    if host_reward:
        agent.sample_transitions.device_reward = None
    rng = np.random.RandomState(6)
    np.random.seed(7)
    for _ in range(3):
        agent.store_episode(_episodes(agent, rng, 2))
        for _ in range(3):
            agent.train_device()
        agent.update_target_net()
    return agent.get_variables(), np.random.get_state()[1].copy()


def test_graph_replay_equals_eager_and_host_reward_equals_device_rule(monkeypatch):
    eager, s0 = _train_run(False, monkeypatch)
    graph, s1 = _train_run(True, monkeypatch)
    host, s2 = _train_run(True, monkeypatch, host_reward=True)
    assert np.array_equal(s0, s1) and np.array_equal(s0, s2)
    for k in eager:
        assert np.array_equal(eager[k], graph[k]), k
        assert np.array_equal(eager[k], host[k]), k


# ------------------------------------------------------------------------------------------ learn, save, command line
def _learn(tmp, seed=0, epochs=1, **kw):
    from baselines_b200 import logger
    from baselines_b200.common.cmd_util import make_vec_env
    from baselines_b200.her.her import learn
    logger.configure(str(tmp), format_strs=["csv"])
    env = make_vec_env('PointReach-v0', 'robotics', 2, seed, flatten_dict_observations=False)
    n_cycles = kw.pop('n_cycles', 5)
    params = dict(n_cycles=n_cycles, n_batches=kw.pop('n_batches', 10), n_test_rollouts=kw.pop('n_test_rollouts', 2),
                  buffer_size=kw.pop('buffer_size', 100000))
    params.update(kw.pop('override', {}))
    return learn(network='mlp', env=env, total_timesteps=epochs * n_cycles * 50 * 2, seed=seed,
                 override_params=params, **kw)


def test_seeded_learn_is_deterministic_and_checkpoints_round_trip(tmp_path):
    a = _learn(tmp_path / "a", seed=3, save_path=str(tmp_path / "pols"))
    b = _learn(tmp_path / "b", seed=3)
    va, vb = a.get_variables(), b.get_variables()
    names = list(va)
    assert names[:10] == [f'ddpg/{s}/{n}:0' for s in ('o_stats', 'g_stats') for n in ('sum', 'sumsq', 'count', 'mean',
                                                                                         'std')]
    order = [k.split('/')[1] + '/' + k.split('/')[2] for k in names[10:]]
    assert order == sorted(order, key=['main/pi', 'main/Q', 'target/pi', 'target/Q'].index)
    assert va['ddpg/main/pi/_0/kernel:0'].shape == (4 + 2, 256) and va['ddpg/main/Q/_3/kernel:0'].shape == (256, 1)
    for k in va:
        assert np.array_equal(va[k], vb[k]), k
    assert os.path.exists(tmp_path / "pols" / "policy_best.pkl") and os.path.exists(tmp_path / "pols" / "policy_0.pkl")
    keys = open(tmp_path / "a" / "progress.csv").readline().strip().split(",")
    for k in ('epoch', 'test/success_rate', 'test/mean_Q', 'test/episode', 'train/success_rate', 'train/episode',
              'stats_o/mean', 'stats_o/std', 'stats_g/mean', 'stats_g/std'):
        assert k in keys
    assert os.path.exists(tmp_path / "a" / "params.json")
    a.save(str(tmp_path / "ck"))
    c = _learn(tmp_path / "c", seed=4, epochs=0, load_path=str(tmp_path / "ck"))
    vc = c.get_variables()
    assert list(vc) == names
    for k in va:
        assert np.array_equal(va[k], vc[k]), k


def test_her_learns_point_reach(tmp_path):
    policy = _learn(tmp_path, seed=0, epochs=8, n_cycles=10, n_batches=40, n_test_rollouts=10)
    from baselines_b200 import logger  # noqa: F401
    import csv
    rows = list(csv.DictReader(open(tmp_path / "progress.csv")))
    rates = [float(r['test/success_rate']) for r in rows]
    print("test/success_rate per epoch:", rates, flush=True)
    _learn(tmp_path / "none", seed=0, epochs=8, n_cycles=10, n_batches=40, n_test_rollouts=10, replay_strategy='none')
    none = [float(r['test/success_rate']) for r in csv.DictReader(open(tmp_path / "none" / "progress.csv"))]
    print("replay_strategy='none':", none)
    assert max(none[-2:]) < max(rates[-2:])
    assert max(rates[-2:]) >= SUCCESS_THRESHOLD, rates


# On an H100 80GB HBM3 at a 700 W power limit this seeded run gave test/success_rate 0.30, 0.30, 0.40, 0.65, 0.25,
# 0.20, 0.45, 0.60 over its 8 epochs, and replay_strategy='none' 0.00, 0.05, 0.05, 0.00, 0.00, 0.05, 0.10, 0.20
SUCCESS_THRESHOLD = 0.4


def test_command_line_trains_and_saves(tmp_path):
    env = dict(os.environ, PYTHONPATH=ROOT)
    out = subprocess.run([sys.executable, "-m", "baselines_b200.run", "--alg=her", "--env=PointReach-v0",
                          "--num_timesteps=1000", "--n_cycles=2", "--n_batches=2", "--n_test_rollouts=1",
                          f"--save_path={tmp_path / 'ck'}", f"--log_path={tmp_path / 'log'}"],
                         cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    import joblib
    d = joblib.load(tmp_path / "ck")
    assert 'ddpg/main/pi/_0/kernel:0' in d and 'ddpg/o_stats/count:0' in d
