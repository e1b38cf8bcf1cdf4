"""CPU: HER's host side -- the sampler's numpy stream, the rollout worker, the float64 mirror of tests/_her_refs.py
against numpy loops and central differences, the normaliser restatement, the refusals, dispatch, the goal environment
and dict observations through the vec envs."""
import numpy as np
import pytest

import _her_refs as R


def test_dispatch():
    from baselines_b200.her.her import learn
    from baselines_b200.run import get_learn_function
    assert get_learn_function('her') is learn


def test_refusals():
    from baselines_b200.her.experiment import config
    from baselines_b200.her.her import learn
    from baselines_b200.her.her_sampler import make_sample_her_transitions
    with pytest.raises(NotImplementedError):
        learn(network='mlp', env=None, total_timesteps=1, demo_file='demo.npz')
    with pytest.raises(NotImplementedError):
        learn(network='mlp', env=None, total_timesteps=1, replay_strategy='final')
    with pytest.raises(NotImplementedError):
        make_sample_her_transitions('episode', 4, None)
    params = config.prepare_params(dict(config.DEFAULT_PARAMS, env_name='PointReach-v0', replay_strategy='future',
                                        network_class='my.module:Net'))
    with pytest.raises(NotImplementedError):
        config.configure_ddpg(dims=config.configure_dims(params), params=params)


def _reference_draws(rollout_batch_size, T, batch_size, future_p):
    """her_sampler.py:27-37 in the reference's order."""
    episode_idxs = np.random.randint(0, rollout_batch_size, batch_size)
    t_samples = np.random.randint(T, size=batch_size)
    her_indexes = np.where(np.random.uniform(size=batch_size) < future_p)
    future_offset = np.random.uniform(size=batch_size) * (T - t_samples)
    future_offset = future_offset.astype(int)
    future_t = (t_samples + 1 + future_offset)[her_indexes]
    return episode_idxs, t_samples, her_indexes[0], future_t


@pytest.mark.parametrize("strategy", ["future", "none"])
def test_sampler_draws_and_stream(strategy):
    from baselines_b200.her.her_sampler import make_sample_her_transitions

    def reward_fun(ag_2, g, info):
        return -(np.linalg.norm(ag_2 - g, axis=-1) > 0.05).astype(np.float32)
    s = make_sample_her_transitions(strategy, 4, reward_fun)
    rng = np.random.RandomState(0)
    E, T, B = 7, 9, 300
    batch = {'o': rng.randn(E, T + 1, 3), 'ag': rng.randn(E, T + 1, 2), 'g': rng.randn(E, T, 2),
             'u': rng.randn(E, T, 2), 'info_is_success': rng.randn(E, T, 1)}
    batch['o_2'], batch['ag_2'] = batch['o'][:, 1:], batch['ag'][:, 1:]
    np.random.seed(5)
    ep, t, her, ft = _reference_draws(E, T, B, 1 - 1 / 5 if strategy == 'future' else 0)
    after = np.random.uniform()
    np.random.seed(5)
    tr = s(batch, B)
    assert np.random.uniform() == after
    g = batch['g'][ep, t].copy()
    g[her] = batch['ag'][ep[her], ft]
    assert np.array_equal(tr['g'], g) and np.array_equal(tr['o'], batch['o'][ep, t])
    assert np.array_equal(tr['r'], reward_fun(batch['ag'][ep, t + 1], g, None))
    np.random.seed(5)
    e2, t2, f2 = s.draw(E, T, B)
    assert np.array_equal(e2, ep) and np.array_equal(t2, t)
    assert np.array_equal(np.nonzero(f2 >= 0)[0], her) and np.array_equal(f2[her], ft)
    assert np.random.uniform() == after
    if strategy == 'future':
        assert (ft <= T).all() and (ft > t[her]).all() and (ft == T).any()


def test_rollout_worker_episode_and_stream():
    """RolloutWorker over the goal env with a fixed linear policy: the episode dict's shapes and values, the success
    history and the numpy draws of get_actions' host half (ddpg.py:145-153)."""
    from baselines_b200 import logger
    from baselines_b200.common.vec_env import DummyVecEnv
    from baselines_b200 import envs
    from baselines_b200.her.ddpg import postprocess_actions
    from baselines_b200.her.rollout import RolloutWorker

    class Policy:
        def get_actions(self, o, ag, g, noise_eps=0., random_eps=0., use_target_net=False, compute_Q=False):
            u = np.tanh((g - ag) * 10).astype(np.float32)
            u = postprocess_actions(u, noise_eps, random_eps, 1.0, 2)
            return [u, np.zeros((len(o), 1), np.float32)] if compute_Q else u

    def make(i):
        def f():
            e = envs.make('PointReach-v0')
            e.seed(i)
            return e
        return f
    venv = DummyVecEnv([make(0), make(1)])
    dims = {'o': 4, 'g': 2, 'u': 2, 'info_is_success': 1}
    w = RolloutWorker(venv, Policy(), dims, logger, T=50, rollout_batch_size=2, noise_eps=0.2, random_eps=0.3)
    np.random.seed(0)
    ep = w.generate_rollouts()
    assert ep['o'].shape == (2, 50, 4) and ep['ag'].shape == (2, 50, 2)
    assert ep['u'].shape == (2, 49, 2) and ep['g'].shape == (2, 49, 2) and ep['info_is_success'].shape == (2, 49, 1)
    assert ep['o'].dtype == np.float32
    # the next observation continues from the action taken
    np.testing.assert_allclose(ep['ag'][:, 1], np.clip(np.clip(ep['u'][:, 0], -1, 1) * 0.1, -1, 1), atol=1e-7)
    # 50 get_actions calls (the last one's step ends the episode), each one randn, binomial and uniform draw
    np.random.seed(0)
    for _ in range(50):
        np.random.randn(2, 2)
        np.random.binomial(1, 0.3, 2)
        np.random.uniform(low=-1.0, high=1.0, size=(2, 2))
    state_ref = np.random.get_state()
    np.random.seed(0)
    w2 = RolloutWorker(DummyVecEnv([make(0), make(1)]), Policy(), dims, logger, T=50, rollout_batch_size=2,
                       noise_eps=0.2, random_eps=0.3)
    w2.generate_rollouts()
    state = np.random.get_state()
    assert np.array_equal(state[1], state_ref[1]) and state[2] == state_ref[2]
    logs = dict(w.logs('train'))
    assert set(logs) == {'train/success_rate', 'train/episode'} and logs['train/episode'] == 2


def test_postprocess_actions_matches_reference_order():
    from baselines_b200.her.ddpg import postprocess_actions
    u = np.random.RandomState(1).uniform(-1, 1, (5, 3)).astype(np.float32)
    np.random.seed(3)
    got = postprocess_actions(u.copy(), 0.2, 0.3, 1.5, 3)
    np.random.seed(3)
    v = u.copy()
    v += 0.2 * 1.5 * np.random.randn(*v.shape)
    v = np.clip(v, -1.5, 1.5)
    v += np.random.binomial(1, 0.3, v.shape[0]).reshape(-1, 1) * (np.random.uniform(-1.5, 1.5, (5, 3)) - v)
    assert np.array_equal(got, v)


# ---------------------------------------------------------------------------------------------- the float64 mirror
def _params(rng, dimo, dimg, dimu, L, H):
    P = {}
    for scope in ('ddpg/main', 'ddpg/target'):
        for net, nin, nout in (('pi', dimo + dimg, dimu), ('Q', dimo + dimg + dimu, 1)):
            k = nin
            for i, n in enumerate([H] * L + [nout]):
                P[f'{scope}/{net}/_{i}/kernel:0'] = rng.randn(k, n) * 0.5
                P[f'{scope}/{net}/_{i}/bias:0'] = rng.randn(n) * 0.1
                k = n
    return P


def _losses(P, inp, cfg):
    """Q_loss and pi_loss by plain loops over the samples, for central differences."""
    mu = np.asarray(cfg['max_u'], np.float64)
    L, B = cfg['layers'], len(inp['r'])

    def net(scope, x):
        h = x
        for i in range(L + 1):
            h = h @ P[f'{scope}/_{i}/kernel:0'] + P[f'{scope}/_{i}/bias:0']
            if i < L:
                h = np.maximum(h, 0)
        return h
    ql, pl = 0.0, 0.0
    for b in range(B):
        og2 = np.concatenate([inp['o_2'][b], inp['g_2'][b]])
        pit = mu * np.tanh(net('ddpg/target/pi', og2))
        qt = net('ddpg/target/Q', np.concatenate([og2, pit / mu]))[0]
        y = min(max(inp['r'][b] + cfg['gamma'] * qt, -cfg['clip_return']), 0.0)
        og = np.concatenate([inp['o'][b], inp['g'][b]])
        q = net('ddpg/main/Q', np.concatenate([og, inp['u_in'][b]]))[0]
        ql += (y - q) ** 2 / B
        pi = mu * np.tanh(net('ddpg/main/pi', og))
        pl += -net('ddpg/main/Q', np.concatenate([og, pi / mu]))[0] / B
        pl += cfg['action_l2'] * np.sum((pi / mu) ** 2) / (B * cfg['dimu'])
    return ql, pl


def test_mirror_against_loops_and_central_differences():
    rng = np.random.RandomState(0)
    dimo, dimg, dimu, L, H, B = 3, 2, 2, 2, 5, 6
    P = _params(rng, dimo, dimg, dimu, L, H)
    inp = dict(o=rng.randn(B, dimo), g=rng.randn(B, dimg), o_2=rng.randn(B, dimo), g_2=rng.randn(B, dimg),
               u_in=rng.uniform(-1, 1, (B, dimu)), r=-rng.randint(0, 2, B).astype(np.float64))
    cfg = dict(scope='ddpg', layers=L, max_u=np.array([1.5, 0.5]), gamma=0.98, clip_return=50., clip_pos_returns=True,
               action_l2=1.0, dimu=dimu)
    ref = R.train_step(P, inp, cfg)
    ql, pl = _losses(P, inp, cfg)
    assert abs(ref['loss'] - ql) < 1e-12 and abs(ref['pi_loss'] - pl) < 1e-12
    eps = 1e-6
    for grads, which in ((ref['Q_grads'], 0), (ref['pi_grads'], 1)):
        for k, gk in grads.items():
            flat = P[k].reshape(-1)
            num = np.zeros_like(flat)
            for i in range(flat.size):
                old = flat[i]
                flat[i] = old + eps
                up = _losses(P, inp, cfg)[which]
                flat[i] = old - eps
                dn = _losses(P, inp, cfg)[which]
                flat[i] = old
                num[i] = (up - dn) / (2 * eps)
            np.testing.assert_allclose(gk.reshape(-1), num, rtol=1e-5, atol=1e-7, err_msg=k)
    # the tempting mistakes are visible to the mirror
    for bad in ('l2_over_B', 'u_not_scaled'):
        w = R.train_step(P, inp, cfg, variant=bad)
        assert not np.allclose(w['pi_grads']['ddpg/main/pi/_0/kernel:0'], ref['pi_grads']['ddpg/main/pi/_0/kernel:0']) \
            or not np.allclose(w['Q_grads']['ddpg/main/Q/_0/kernel:0'], ref['Q_grads']['ddpg/main/Q/_0/kernel:0'])


def test_normaliser_restatement_against_direct_evaluation():
    """tests/_her_refs.norm_update against normalizer.py:64-118 evaluated directly, in float32 and float64 batches."""
    rng = np.random.RandomState(1)
    E, T, dimo, dimg = 3, 6, 4, 2
    for dtype in (np.float32, np.float64):
        ep = {'o': rng.randn(E, T + 1, dimo).astype(dtype), 'ag': rng.randn(E, T + 1, dimg).astype(dtype),
              'g': rng.randn(E, T, dimg).astype(dtype)}
        sel = np.stack([rng.randint(0, E, 18), rng.randint(0, T, 18), np.where(rng.rand(18) < 0.5, T, -1)], 1)
        st = [np.concatenate([np.zeros(2 * d, np.float32), np.ones(1, np.float32)]) for d in (dimo, dimg)]
        got = R.norm_update(st, None, None, ep, sel, True, 200., 0.01)
        o = ep['o'][sel[:, 0], sel[:, 1]]
        g = ep['g'][sel[:, 0], sel[:, 1]].copy()
        m = sel[:, 2] >= 0
        g[m] = ep['ag'][sel[m, 0], sel[m, 2]]
        g = g - ep['ag'][sel[:, 0], sel[:, 1]]
        for v, (s_, mean, std), D in ((o, got[0], dimo), (g, got[1], dimg)):
            col = np.zeros(D, dtype)
            sq = np.zeros(D, dtype)
            for row in v:
                col = (col + row).astype(dtype)
                sq = (sq + row * row).astype(dtype)
            ls, lq = np.float32(0) + col.astype(np.float32), sq.astype(np.float32)
            cnt = np.float32(1) + np.float32(len(v))
            want_mean = (ls / cnt).astype(np.float32)
            var = (lq / cnt - want_mean * want_mean).astype(np.float32)
            want_std = np.sqrt(np.maximum(np.float32(1e-4), var)).astype(np.float32)
            assert np.array_equal(mean, want_mean) and s_[-1] == cnt
            np.testing.assert_allclose(std, want_std, rtol=1e-6)


# ---------------------------------------------------------------------------------------------- host plumbing
def test_goal_env_and_dict_observations():
    from baselines_b200 import envs
    from baselines_b200.common.cmd_util import make_vec_env
    from baselines_b200.her.experiment import config
    e = envs.make('PointReach-v0')
    assert e._max_episode_steps == 50 and e.unwrapped.reward_type == 'sparse'
    ob = e.reset()
    assert set(ob) == {'observation', 'achieved_goal', 'desired_goal'}
    # the rule of compute_reward, including distances exactly at the threshold
    a = np.array([[0.0, 0.0], [0.1, 0.0], [0.1000001, 0.0]])
    assert list(e.compute_reward(a, np.zeros((3, 2)), {})) == [0.0, 0.0, -1.0]
    assert config.device_reward_rule(e, 2) == ('sparse', 0.1)
    assert config.device_reward_rule(envs.make('PointReachDense-v0'), 2) == ('dense', 0.1)

    class Other:
        reward_type, distance_threshold = 'sparse', 0.1

        def compute_reward(self, achieved_goal, desired_goal, info):
            return -(np.linalg.norm(achieved_goal - desired_goal, axis=-1) >= 0.1).astype(np.float32)
    assert config.device_reward_rule(Other(), 2) is None        # differs exactly at the threshold
    v = make_vec_env('PointReach-v0', 'robotics', 1, 0, flatten_dict_observations=False)
    o = v.reset()
    assert o['observation'].shape == (1, 4) and o['desired_goal'].shape == (1, 2)
    o2, r, d, info = v.step(np.zeros((1, 2), np.float32))
    assert o2['achieved_goal'].shape == (1, 2) and 'is_success' in info[0]
    f = make_vec_env('PointReach-v0', 'robotics', 1, 0)
    assert f.reset().shape == (1, 8)
