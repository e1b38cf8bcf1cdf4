"""GPU parity of the DQN learner against the CPU oracle (oracle/nets.py DQNOracle restates
deepq/build_graph.py:380-444; PARITY UNPINNED at the TF boundary) and of the device replay buffer against
the oracle PER arithmetic (pinned bit-exactly to the executed reference by tests/test_oracle_golden.py)."""
import random

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _space(shape, dtype):
    from baselines_b200.common import spaces
    return spaces.Box(0, 255, shape, dtype) if dtype == np.uint8 else spaces.Box(-5, 5, shape, dtype)


@pytest.mark.parametrize("network,ob_shape,dtype,dueling", [("cnn", (84, 84, 4), np.uint8, True),
                                                            ("conv_only", (84, 84, 4), np.uint8, True),
                                                            ("mlp", (8,), np.float32, True),
                                                            ("mlp", (8,), np.float32, False)])
def test_dqn_train_step_matches_oracle(network, ob_shape, dtype, dueling):
    from baselines_b200.deepq.build_graph import DQNModel
    from oracle import nets
    nA, seed = 6, 3
    B = 256 if dtype == np.uint8 else 64
    model = DQNModel(_space(ob_shape, dtype), nA, network, lr=1e-4, gamma=0.99, grad_norm_clipping=10, batch_cap=B,
                     seed=seed, hiddens=(256,), dueling=dueling)
    qp = nets.init_q_params(network, ob_shape, nA, hiddens=(256,), dueling=dueling, seed=seed)
    mp = model.q.store.export_tf("params")
    assert set(mp) == set(qp)
    for k in qp:
        assert np.array_equal(mp[k], qp[k]), k
    oracle = nets.DQNOracle(qp, network, 0.99, n_hidden=1, dueling=dueling, grad_norm_clipping=10.0)
    rng = np.random.RandomState(0)

    def obs():
        if dtype == np.uint8:
            return rng.randint(0, 256, (B,) + ob_shape).astype(np.uint8)
        return (rng.randn(B, *ob_shape) * 2.0).astype(np.float32)      # un-rounded float32 (no fp16 pre-rounding)

    dev = model.device
    for it in range(3):
        # Adam's first steps move every weight by ~lr regardless of |g| (m/sqrt(v) = +-1), so sign flips of
        # near-zero gradients make two correct implementations drift apart; re-synchronise the state so that
        # every iteration compares ONE step from identical parameters / Adam slots / target network.
        model.q.store.import_tf({k: v.numpy() for k, v in oracle.tp.items()}, "params")
        model.q.store.import_tf({k: v.numpy() for k, v in oracle.m.items()}, "m")
        model.q.store.import_tf({k: v.numpy() for k, v in oracle.v.items()}, "v")
        model.qt.store.import_tf({k: v.numpy() for k, v in oracle.tt.items()}, "params")
        model.opt.t = oracle.t
        model.q.refresh()
        model.qt.refresh()
        o_t, o_1 = obs(), obs()
        act = rng.randint(0, nA, B).astype(np.int64)
        rew = rng.randn(B).astype(np.float32)
        done = (rng.rand(B) < 0.1).astype(np.float32)
        w = (rng.rand(B) * 0.9 + 0.1).astype(np.float32)
        # double-Q picks argmax_a q_online(s'): where the top-2 gap is inside the fp16 error the two paths may
        # legitimately pick different actions, so mark those transitions terminal (target = reward only)
        qn = np.sort(oracle.q_values(o_1), axis=1)
        done[(qn[:, -1] - qn[:, -2]) < 3e-2] = 1.0
        f = lambda z: torch.as_tensor(z).to(dev)
        td = model.train_device(f(o_t), f(o_1), f(act), f(rew), f(done), f(w), None, B).cpu().numpy()
        td_o = oracle.train(1e-4, o_t, act, rew, o_1, done, w)
        assert np.allclose(td, td_o, atol=5e-3 * max(1.0, np.abs(td_o).max())), (it, np.abs(td - td_o).max())
        g = model.q.store.export_tf("grads")
        num = sum(float(((g[k] - oracle.last_grads[k]) ** 2).sum()) for k in g)
        den = sum(float((oracle.last_grads[k] ** 2).sum()) for k in g)
        per = {k.split("q_func/")[-1]: round(float((((g[k] - oracle.last_grads[k]) ** 2).sum() /
                                                    max((oracle.last_grads[k] ** 2).sum(), 1e-30)) ** 0.5), 4) for k in g}
        print(f"[{network}] it={it} grad rel err total={(num / den) ** 0.5:.4f} per-var={per}")
        # ~1e-2 observed; after update_target the TD errors shrink and cancellation raises the RELATIVE error
        assert (num / den) ** 0.5 < 5e-2, (it, (num / den) ** 0.5, per)
        p, po = model.q.store.export_tf("params"), {k: v.numpy() for k, v in oracle.tp.items()}
        err = max(float(np.abs(p[k] - po[k]).max()) for k in p)
        # the reference's tolerance.  One Adam step moves each element by at most ~lr whatever the gradient, so this
        # bounds the step and cannot detect a gradient error (see test_update_composition_gpu.py)
        assert err < 3e-3, (it, err)
        if it == 1:
            model.update_target()
            oracle.update_target()
    qv = model.q_values(o_t[:8])
    assert np.allclose(qv, oracle.q_values(o_t[:8]), atol=2e-2)


def test_prioritized_replay_buffer_matches_oracle():
    from baselines_b200.deepq.replay_buffer import PrioritizedReplayBuffer
    from oracle.segment_tree import PrioritizedSampler
    size, alpha, batch = 300, 0.6, 32
    buf = PrioritizedReplayBuffer(size, alpha)
    per = PrioritizedSampler(size, alpha)
    rng = np.random.RandomState(1)
    for i in range(350):                                   # wraps the ring
        o = rng.randint(0, 256, (4, 4, 1)).astype(np.uint8)
        buf.add(o, i % 3, float(i), o, float(i % 7 == 0))
        per.add()
    assert len(buf) == 300
    for r in range(5):
        random.seed(100 + r)
        u = [random.random() for _ in range(batch)]
        random.seed(100 + r)
        out = buf.sample(batch, beta=0.5)
        idx_o = per.sample_idx(u)
        assert list(out[6]) == idx_o                       # same python-RNG stream -> same indices
        assert np.allclose(out[5], per.weights(idx_o, 0.5), rtol=1e-12)
        assert out[0].shape == (batch, 4, 4, 1) and out[2].dtype == np.float64
        pr = np.abs(rng.randn(batch)) + 1e-6
        buf.update_priorities(out[6], pr)
        per.update_priorities(idx_o, pr)
        assert buf._max_priority == per.max_priority
    assert np.array_equal(buf._it_sum.cpu().numpy(), per.sum_tree.value)
    assert np.array_equal(buf._it_min.cpu().numpy(), per.min_tree.value)
    # device priority path: (|td| + eps) ** alpha, running max
    idx, w32, w64 = buf.sample_device(batch, 0.4)
    td = torch.randn(batch, device=buf.device)
    buf.update_priorities_device(idx, td, 1e-6)
    assert buf._max_priority >= float(np.abs(td.cpu().numpy()).max())


def test_deepq_learn_solves_identity_env():
    """deepq on a contextual-bandit identity env (common/tests/test_identity.py shape): must learn a == s."""
    from baselines_b200.common import spaces
    from baselines_b200 import deepq

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

    env = Env()
    act = deepq.learn(env, "mlp", seed=0, lr=1e-3, total_timesteps=4000, buffer_size=2000, exploration_fraction=0.3,
                      exploration_final_eps=0.02, train_freq=1, batch_size=32, print_freq=None, checkpoint_freq=None,
                      learning_starts=200, gamma=0.0, target_network_update_freq=200, prioritized_replay=True,
                      hiddens=(64,), dueling=True)
    ob, tot = env.reset(), 0.0
    for _ in range(200):
        a = act(ob[None], stochastic=False)[0]
        ob, r, d, _ = env.step(a)
        tot += r
        if d:
            ob = env.reset()
    assert tot / 200 > 0.9, tot / 200
    a, _, _, _ = act.step(ob)
    assert a.shape == (1,)
