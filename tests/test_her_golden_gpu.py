"""GPU: HER's device episode ring and a learn-shaped sequence of train steps against fixtures produced by executing the
reference's replay_buffer.py and ddpg.py store_episode / sample_batch (tools/gen_her_golden.py), and the normaliser of
one-column observations and goals, which numpy sums pairwise."""
import os

import numpy as np
import pytest
import torch

import _her_refs as R

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module", autouse=True)
def _lib():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from baselines_b200 import build_ext
    build_ext.build()


def _fx(name):
    return np.load(os.path.join(GOLDEN, f"her_{name}.npz"))


def reward_fun(ag_2, g, info):
    return -(np.linalg.norm(ag_2 - g, axis=-1) > 0.1).astype(np.float32)


def _episode(fx, prefix):
    return {k[len(prefix):]: fx[k] for k in fx.files if k.startswith(prefix)}


def test_device_ring_matches_executed_reference_storage():
    """Wrap, overflow and full-ring replacement, a repeated slot keeping the last of its episodes."""
    from baselines_b200.her.replay_buffer import ReplayBuffer
    fx = _fx("storage")
    T = 4
    shapes = {'o': (T + 1, 3), 'ag': (T + 1, 2), 'g': (T, 2), 'u': (T, 2), 'info_is_success': (T, 1)}
    buf = ReplayBuffer(shapes, 5 * (T + 1), T + 1, None)
    np.random.seed(21)
    for k in range(8):
        buf.store_episode(_episode(fx, f"ep{k}_"))
        assert buf.current_size == fx[f"size{k}"]
    for key in shapes:
        assert np.array_equal(buf.buffers[key].cpu().numpy(), fx[f"buf_{key}"]), key
    assert np.array_equal(np.random.uniform(size=4), fx["after"])


def test_learn_shaped_sequence_matches_reference_stream_and_rewards():
    """store_episode (storage slots and the normaliser's sample) and three train steps per cycle over six cycles, the
    ring full after four: numpy's global stream after each cycle equals the reference's, and the rewards of each
    cycle's first batch, relabelled and recomputed on the device, equal the reference's."""
    from baselines_b200.her.ddpg import DDPG
    from baselines_b200.her.experiment.config import simple_goal_subtract
    from baselines_b200.her.her_sampler import make_sample_her_transitions
    fx = _fx("stream")
    T, B = 6, 32
    sampler = make_sample_her_transitions('future', 4, reward_fun)
    sampler.device_reward = ('sparse', 0.1)
    gamma = 1. - 1. / (T + 1)
    agent = DDPG(input_dims={'o': 3, 'g': 2, 'u': 2, 'info_is_success': 1}, buffer_size=8 * (T + 1), hidden=64,
                 layers=2, network_class='baselines.her.actor_critic:ActorCritic', polyak=0.95, batch_size=B,
                 Q_lr=1e-3, pi_lr=1e-3, norm_eps=0.01, norm_clip=5, max_u=1.0, action_l2=1.0, clip_obs=200.,
                 scope='ddpg', T=T + 1, rollout_batch_size=2, subtract_goals=simple_goal_subtract, relative_goals=False,
                 clip_pos_returns=True, clip_return=1. / (1. - gamma), bc_loss=0, q_filter=0, num_demo=0,
                 demo_batch_size=0, prm_loss_weight=0, aux_loss_weight=0, sample_transitions=sampler, gamma=gamma,
                 seed=0)
    np.random.seed(41)
    for c in range(6):
        agent.store_episode(_episode(fx, f"ep{c}_"))
        for k in range(3):
            agent.train_device()
            if k == 0:
                r = agent.r[:B].cpu().numpy()
                assert np.array_equal(r.view(np.uint32), fx[f"batch{c}_r"].astype(np.float32).view(np.uint32)), c
        st = np.random.get_state()
        assert np.array_equal(st[1], fx[f"state{c}"]) and st[2] == fx[f"pos{c}"], c
    assert agent.buffer.current_size == agent.buffer.size


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_normaliser_one_column_bit_for_bit(dtype):
    """dimo = dimg = 1: numpy's v.sum(axis=0) of an [N, 1] batch is a pairwise sum (N = 140: its recursive case)."""
    from test_her_gpu import _agent, _episodes
    rng = np.random.RandomState(3)
    agent = _agent(dimo=1, dimg=1, dimu=2, T=70, relative_goals=True, buffer_episodes=8)
    state = [agent.o_stats.state.cpu().numpy(), agent.g_stats.state.cpu().numpy()]
    for k in range(3):
        ep = _episodes(agent, rng, 2, dtype, scale=7.0)
        np.random.seed(50 + k)
        agent.store_episode(ep)
        np.random.seed(50 + k)
        n, T = ep['u'].shape[:2]
        e, t, f = agent.sample_transitions.draw(n, T, n * T)
        out = R.norm_update(state, None, None, ep, np.stack([e, t, f], 1), True, 200., 0.01)
        state = [out[0][0], out[1][0]]
        for (st, m, sd), nz in ((out[0], agent.o_stats), (out[1], agent.g_stats)):
            assert np.array_equal(nz.state.cpu().numpy().view(np.uint32), st.view(np.uint32))
            assert np.array_equal(nz.mean.cpu().numpy().view(np.uint32), m.view(np.uint32))
            assert np.array_equal(nz.std.cpu().numpy().view(np.uint32), sd.view(np.uint32))
