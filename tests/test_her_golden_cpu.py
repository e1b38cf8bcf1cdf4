"""CPU: HER's sampler, episode storage slots and rollout worker against fixtures produced by executing the reference's
her_sampler.py, replay_buffer.py, rollout.py and ddpg.py get_actions (tools/gen_her_golden.py)."""
import os

import numpy as np
import pytest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _fx(name):
    return np.load(os.path.join(GOLDEN, f"her_{name}.npz"))


def reward_fun(ag_2, g, info):
    return -(np.linalg.norm(ag_2 - g, axis=-1) > 0.1).astype(np.float32)


def policy_pi(o, g):
    """The fixture's fixed network: pi = tanh(W [o | g])."""
    W = np.linspace(-1.5, 1.5, (o.shape[1] + g.shape[1]) * 2).reshape(-1, 2)
    return np.tanh(np.concatenate([o, g], 1) @ W).astype(np.float32)


@pytest.mark.parametrize("strategy", ["future", "none"])
def test_sampler_matches_executed_reference(strategy):
    from baselines_b200.her.her_sampler import make_sample_her_transitions
    fx = _fx("sampler")
    batch = {k[6:]: fx[k] for k in fx.files if k.startswith("batch_")}
    batch['o_2'], batch['ag_2'] = batch['o'][:, 1:, :], batch['ag'][:, 1:, :]
    s = make_sample_her_transitions(strategy, 4, reward_fun)
    np.random.seed(11)
    tr = s(batch, 200)
    for k in ('o', 'o_2', 'ag', 'ag_2', 'g', 'u', 'r'):
        assert np.array_equal(tr[k], fx[f"{strategy}_{k}"]), k
    assert np.array_equal(np.random.uniform(size=4), fx[f"{strategy}_after"])
    # the integers the device receives select the same transitions and goals
    np.random.seed(11)
    ep, t, ft = s.draw(6, 9, 200)
    assert np.array_equal(batch['o'][ep, t], fx[f"{strategy}_o"])
    g = batch['g'][ep, t].copy()
    g[ft >= 0] = batch['ag'][ep[ft >= 0], ft[ft >= 0]]
    assert np.array_equal(g, fx[f"{strategy}_g"])
    assert np.array_equal(np.random.uniform(size=4), fx[f"{strategy}_after"])


def test_storage_slots_match_executed_reference():
    """Consecutive slots, the overflow that fills the ring, then full-ring replacement with repeated slots."""
    from baselines_b200.her.replay_buffer import storage_idx
    fx = _fx("storage")
    np.random.seed(21)
    cur = 0
    for k in range(8):
        idx, cur = storage_idx(cur, 5, 3)
        assert np.array_equal(idx, fx[f"slots{k}"]) and cur == fx[f"size{k}"], k
    assert np.array_equal(np.random.uniform(size=4), fx["after"])


def test_rollout_worker_matches_executed_reference():
    from baselines_b200 import envs, logger
    from baselines_b200.common.vec_env import DummyVecEnv
    from baselines_b200.her.ddpg import postprocess_actions
    from baselines_b200.her.rollout import RolloutWorker
    fx = _fx("rollout")

    class Policy:
        def get_actions(self, o, ag, g, noise_eps=0., random_eps=0., use_target_net=False, compute_Q=False):
            o, g = np.clip(o, -200., 200.), np.clip(g, -200., 200.)
            pi = policy_pi(o.reshape(-1, 4), g.reshape(-1, 2))
            u = postprocess_actions(pi.copy(), noise_eps, random_eps, 1.0, 2)
            return [u, pi.sum(axis=1, keepdims=True)] if compute_Q else u

    def make(i):
        def f():
            e = envs.make('PointReach-v0')
            e.seed(i)
            return e
        return f
    dims = {'o': 4, 'g': 2, 'u': 2, 'info_is_success': 1}
    np.random.seed(31)
    w = RolloutWorker(DummyVecEnv([make(0), make(1)]), Policy(), dims, logger, T=50, rollout_batch_size=2,
                      noise_eps=0.2, random_eps=0.3)
    ev = RolloutWorker(DummyVecEnv([make(2), make(3)]), Policy(), dims, logger, T=50, rollout_batch_size=2,
                       exploit=True, compute_Q=True)
    for k in range(2):
        ep = w.generate_rollouts()
        for key, v in ep.items():
            assert v.dtype == fx[f"train{k}_{key}"].dtype and np.array_equal(v, fx[f"train{k}_{key}"]), (k, key)
    ep = ev.generate_rollouts()
    for key, v in ep.items():
        assert np.array_equal(v, fx[f"eval_{key}"]), key
    assert np.array_equal(np.array(w.success_history), fx["train_success"])
    assert np.array_equal(np.array(ev.success_history), fx["eval_success"])
    assert np.array_equal(np.array(ev.Q_history), fx["eval_Q"])
    assert np.array_equal(np.random.uniform(size=4), fx["after"])
