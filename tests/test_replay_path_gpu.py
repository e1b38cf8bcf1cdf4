"""GPU: the prioritized replay path of deepq.learn, bit for bit against tests/_replay_refs.py.

Kernels at their edges (tree_set chunking and duplicates, every tree_range_sum range, per_sample strata and boundaries,
per_priorities dtypes and invalid priorities, the correctly rounded pow), then PrioritizedReplayBuffer driven with the
learner's own call pattern, and deepq.learn itself recorded and replayed through the reference.  Nothing here has a
tolerance: indices, float64 and float32 weights, the max priority and both trees are compared exactly.
"""
import random

import numpy as np
import pytest
import torch

from _replay_refs import ReferenceReplay, build_trees, cr_pow, leaf_values, reference_priorities, running_max
from oracle.segment_tree import SumTree

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from baselines_b200 import ops as o
    return o


def dev(a):
    return torch.as_tensor(np.ascontiguousarray(a)).cuda()


def _empty_trees(cap):
    return (torch.zeros(2 * cap, dtype=torch.float64, device="cuda"),
            torch.full((2 * cap,), float("inf"), dtype=torch.float64, device="cuda"))


def _upload_trees(s_np, m_np):
    return dev(s_np.copy()), dev(m_np.copy())


# ------------------------------------------------------------------------------------------ pow
def _sweep_values(n, seed=0):
    rng = np.random.RandomState(seed)
    x = np.exp2(rng.uniform(-24.0, 20.0, n)).astype(np.float32)
    p2 = np.array([2.0 ** k for k in range(-149, 128)], np.float32)
    sub = (rng.randint(1, 1 << 23, 4096).astype(np.uint32)).view(np.float32)       # float32 subnormals
    extra = np.concatenate([p2, np.nextafter(p2, np.float32(np.inf)), np.nextafter(p2, np.float32(0)), sub,
                            np.array([0.0, np.finfo(np.float32).max], np.float32)])
    return np.concatenate([x, extra])


# Correctly rounded pow on the device against the correctly rounded host value, over 2^21 log-uniform float32
# priorities in [2^-24, 2^20] plus 0, subnormals, every power of two and its float32 neighbours, at every exponent the
# replay uses.  Measured on an NVIDIA H100 80GB HBM3 (700 W limit): 0 device mismatches at every exponent, while the
# host's glibc 2.39 float.__pow__ differs from the correctly rounded value on 1718 / 1757 / 1748 / 0 / 1769 / 1752 /
# 1796 of the 2 102 081 values (the counts are printed for each run).
@pytest.mark.parametrize("y", [0.5, 0.6, 0.7, 1.0, -0.4, -0.7, -1.0])
def test_device_pow_is_correctly_rounded(ops, y):
    x = _sweep_values(1 << 21).astype(np.float64)
    out = torch.empty(len(x), dtype=torch.float64, device="cuda")
    ops.per_pow(dev(x), y, out)
    want = cr_pow(x, y)
    got = out.cpu().numpy()
    bad = np.flatnonzero(got != want)
    host = np.array([v ** y if v > 0 else w for v, w in zip(x.tolist(), want.tolist())])
    print(f"pow sweep y={y}: n={len(x)} device!=correctly-rounded {len(bad)}, host float.__pow__ "
          f"!=correctly-rounded {int((host != want).sum())}")
    assert len(bad) == 0, [(x[i].hex(), got[i].hex(), want[i].hex()) for i in bad[:5]]


# ------------------------------------------------------------------------------------------ tree_set
def _tree_set_case(ops, cap, idx, vals, rng):
    """Pre-fill every leaf, then one tree_set of (idx, vals); expected = sequential writes, the last one winning."""
    init = np.exp2(rng.uniform(-10, 10, cap))
    s, m = _empty_trees(cap)
    ops.tree_set(s, m, cap, dev(np.arange(cap, dtype=np.int64)), dev(init))
    ops.tree_set(s, m, cap, dev(idx), dev(vals))
    leaves = init.copy()
    for i, v in zip(idx.tolist(), vals.tolist()):
        leaves[i] = v
    ws, wm = build_trees(cap, leaves)
    assert np.array_equal(s.cpu().numpy(), ws) and np.array_equal(m.cpu().numpy(), wm)


@pytest.mark.parametrize("cap", [1, 2, 4096, 1 << 20])
@pytest.mark.parametrize("n", [1, 1023, 1024, 1025, 2049])
def test_tree_set_chunks_and_duplicates(ops, cap, n):
    rng = np.random.RandomState(cap + n)
    idx = rng.randint(0, cap, n).astype(np.int64)
    if n > 900 and cap > 1:
        idx[5] = idx[900]                               # duplicate inside one 1024-chunk
        if n > 1030:
            idx[1000] = idx[1030] = min(3, cap - 1)     # duplicate across the chunk boundary: the later chunk wins
    vals = np.exp2(rng.uniform(-20, 20, n))
    _tree_set_case(ops, cap, idx, vals, rng)
    _tree_set_case(ops, cap, np.full(n, cap // 2, np.int64), vals, rng)          # all indices equal


# ------------------------------------------------------------------------------------------ tree_range_sum
def test_tree_range_sum_every_range_small_and_random_at_2pow20(ops):
    rng = np.random.RandomState(3)
    for cap in (1, 2, 4, 8, 16, 32, 64):
        leaves = np.exp2(rng.uniform(-30, 30, cap)) * rng.rand(cap)
        s_np, _ = build_trees(cap, leaves)
        ref = SumTree(cap)
        ref.value = s_np
        s, _ = _upload_trees(*build_trees(cap, leaves))
        ranges = [(a, e) for a in range(cap) for e in range(-cap + 1, cap + 1)
                  if (e + cap if e < 0 else e) - 1 >= a]
        out = torch.empty(len(ranges), dtype=torch.float64, device="cuda")
        for k, (a, e) in enumerate(ranges):
            ops.tree_range_sum(s, cap, a, e, out[k:k + 1])
        got = out.cpu().numpy()
        want = np.array([ref.reduce(a, e) for a, e in ranges])
        assert np.array_equal(got, want), cap
    cap = 1 << 20
    leaves = np.exp2(rng.uniform(-20, 20, cap))
    s_np, _ = build_trees(cap, leaves)
    ref = SumTree(cap)
    ref.value = s_np
    s = dev(s_np)
    lo = rng.randint(0, cap, 10000)
    hi = rng.randint(0, cap, 10000)
    ranges = [(int(min(a, b)), int(max(a, b)) + 1) for a, b in zip(lo, hi)]
    out = torch.empty(len(ranges), dtype=torch.float64, device="cuda")
    for k, (a, e) in enumerate(ranges):
        ops.tree_range_sum(s, cap, a, e, out[k:k + 1])
    assert np.array_equal(out.cpu().numpy(), np.array([ref.reduce(a, e) for a, e in ranges]))


# ------------------------------------------------------------------------------------------ per_sample
def _ref_with_leaves(cap, n_stored, leaves, alpha=0.6):
    ref = ReferenceReplay(cap, alpha)
    ref.leaves[:n_stored] = leaves
    ref.stored[:n_stored] = True
    ref.n = n_stored
    ref._dirty = True
    return ref


def _check_sample(ops, ref, uniforms, beta):
    cap = ref.sum_tree.capacity
    s, m = _upload_trees(*ref.trees())
    B = len(uniforms)
    idx = torch.empty(B, dtype=torch.int64, device="cuda")
    w64 = torch.empty(B, dtype=torch.float64, device="cuda")
    w32 = torch.empty(B, dtype=torch.float32, device="cuda")
    bad = torch.zeros(1, dtype=torch.int32, device="cuda")
    ops.per_sample(s, m, cap, ref.n, dev(np.asarray(uniforms, np.float64)), beta, idx, w64, w32, bad)
    want = np.asarray(ref.sample_idx(uniforms), np.int64)
    want_w = ref.weights(want, beta)
    got = idx.cpu().numpy()
    assert np.array_equal(got, want)
    assert got.max() < ref.n
    assert np.array_equal(w64.cpu().numpy(), want_w)
    assert np.array_equal(w32.cpu().numpy(), want_w.astype(np.float32))
    assert np.array_equal(w32.cpu().numpy(), w64.cpu().numpy().astype(np.float32))
    assert int(bad[0]) == 0
    return got


@pytest.mark.parametrize("n_stored,cap", [(2, 2), (3, 4), (100, 128), (1023, 1024), (1024, 1024)])
@pytest.mark.parametrize("batch", [1, 255, 256, 257, 512])
def test_per_sample_strata_weights_and_unstored_tail(ops, n_stored, cap, batch):
    rng = np.random.RandomState(n_stored * 1000 + batch)
    pri = np.exp(rng.uniform(np.log(1e-6), np.log(1e6), n_stored)).astype(np.float32)   # 1e-6 .. 1e6
    ref = _ref_with_leaves(cap, n_stored, leaf_values(pri, 0.6))
    u = rng.rand(batch)
    u[0] = 0.0
    u[-1] = np.nextafter(1.0, 0.0)
    got = _check_sample(ops, ref, u, 0.4 + 0.6 * rng.rand())
    assert got.max() < n_stored                          # the zero tail past n_stored is never sampled


def test_per_sample_mass_on_a_left_subtree_sum_goes_right(ops):
    """Power-of-two priorities make every prefix sum exact; a mass equal to one must take the right branch (the
    reference's strict `left > mass`), landing on the leaf that starts there."""
    leaves = np.array([1.0, 2.0, 4.0, 1.0, 4.0, 2.0, 2.0, 8.0])     # the first 7 sum to p_total = 16
    ref = _ref_with_leaves(8, 8, leaves)
    prefix = np.concatenate([[0.0], np.cumsum(leaves[:7])])
    for j in range(7):
        got = _check_sample(ops, ref, [prefix[j] / 16.0], 0.5)
        assert got[0] == j
    # batch 4: every = 4, masses u*4 + 4i; u = 0 puts them on 0, 4, 8, 12, of which 0, 8 and 12 are the prefix sums
    # where leaves 0, 4 and 5 start
    got = _check_sample(ops, ref, [0.0] * 4, 0.5)
    assert list(got) == [0, 2, 4, 5]


# ------------------------------------------------------------------------------------------ per_priorities
TD_EDGES = np.array([0.0, -0.0, 1e-45, -1e-45, 2.0 ** -130, 1.17e-38, 0.5, -0.75, 1.0, -1e-6, 3.0e38,
                     -np.finfo(np.float32).max, 123.456, -1e3], np.float32)


@pytest.mark.parametrize("eps", [0.0, 1e-6])
@pytest.mark.parametrize("maxp0", [0.25, 1.0, 1e39])
def test_per_priorities_float32_priorities_and_running_max(ops, eps, maxp0):
    td = TD_EDGES if eps > 0 else TD_EDGES[np.abs(TD_EDGES) > 0]
    td = np.concatenate([td, np.random.RandomState(5).randn(300).astype(np.float32)])
    powered = torch.empty(len(td), dtype=torch.float64, device="cuda")
    maxp = torch.full((1,), maxp0, dtype=torch.float64, device="cuda")
    bad = torch.zeros(1, dtype=torch.int32, device="cuda")
    ops.per_priorities(dev(td), eps, 0.6, powered, maxp, bad)
    p = reference_priorities(td, eps)
    assert np.array_equal(powered.cpu().numpy(), leaf_values(p, 0.6))
    assert float(maxp[0]) == running_max(maxp0, p)
    assert maxp0 == 1e39 or float(maxp[0]) == float(np.float32(float(maxp[0])))     # a float32 value
    assert int(bad[0]) == 0


@pytest.mark.parametrize("td0,eps", [(np.nan, 1e-6), (0.0, 0.0), (-0.0, 0.0)])
def test_per_priorities_flags_priorities_that_are_not_positive(ops, td0, eps):
    td = np.array([0.5, td0, 2.0], np.float32)
    powered = torch.empty(3, dtype=torch.float64, device="cuda")
    maxp = torch.ones(1, dtype=torch.float64, device="cuda")
    bad = torch.zeros(1, dtype=torch.int32, device="cuda")
    ops.per_priorities(dev(td), eps, 0.6, powered, maxp, bad)
    assert int(bad[0]) == 1
    assert float(maxp[0]) == float(np.float32(2.0 + np.float32(eps)))


def _filled_buffer(size, alpha=0.6, n=None):
    from baselines_b200.deepq.replay_buffer import PrioritizedReplayBuffer
    buf = PrioritizedReplayBuffer(size, alpha)
    o = np.zeros(2, np.float32)
    for i in range(size if n is None else n):
        buf.add(o, i % 3, float(i), o, 0.0)
    return buf


@pytest.mark.parametrize("case", ["nan", "zero"])
def test_invalid_priority_raises_and_sampling_stays_in_range(ops, case):
    size, B = 100, 32                                   # capacity 128: the right-most leaf is not stored
    buf = _filled_buffer(size)
    random.seed(0)
    idx, _, _ = buf.sample_device(B, 0.4)
    td = torch.randn(B, device="cuda")
    if case == "nan":
        td[7] = float("nan")
        buf.update_priorities_device(idx, td, 1e-6)
    else:
        td[7] = 0.0
        buf.update_priorities_device(idx, td, 0.0)
    torch.cuda.synchronize()                            # deepq.learn: the next act
    with pytest.raises(AssertionError, match="priority > 0"):
        buf.sample_device(B, 0.4)
    with pytest.raises(AssertionError, match="priority > 0"):
        buf.update_priorities_device(idx, td, 1e-6)
    # the poisoned tree itself: sampling returns stored indices and raises the flag
    u = dev(np.linspace(0.0, np.nextafter(1.0, 0.0), B))
    idx2 = torch.empty(B, dtype=torch.int64, device="cuda")
    w64 = torch.empty(B, dtype=torch.float64, device="cuda")
    bad = torch.zeros(1, dtype=torch.int32, device="cuda")
    ops.per_sample(buf._it_sum, buf._it_min, buf._cap, len(buf), u, 0.4, idx2, w64, None, bad)
    got = idx2.cpu().numpy()
    assert got.min() >= 0 and got.max() < size
    assert int(bad[0]) == 1


# ------------------------------------------------------------------------------------------ the learner's pattern
def _td(rng, B, t):
    """Seeded float32 TD errors spread over ~8 decades, so that a few transitions dominate the sum and sampled batches
    repeat indices; now and then one large error lifts the max priority."""
    td = rng.standard_normal(B) * np.exp(rng.uniform(-9.0, 9.0, B))
    if t % 7 == 0:
        td[0] = 50.0 + t
    return td.astype(np.float32)


def _run_learner_pattern(buf, ref, steps, learning_starts, B, rng, check_every, t0=0, total=None):
    from baselines_b200.common.schedules import LinearSchedule
    beta_schedule = LinearSchedule(total or steps, initial_p=0.4, final_p=1.0)
    o = np.zeros(2, np.float32)
    pending, dup_seen = 0, False
    for t in range(t0, steps):
        buf.add(o, t % 3, float(t), o, 0.0)
        pending += 1
        if t > learning_starts:
            beta = beta_schedule.value(t)
            u = [random.random() for _ in range(B)]
            idx, w32, w64 = buf.sample_device(B, beta=beta, uniforms=u)
            td = _td(rng, B, t)
            buf.update_priorities_device(idx, dev(td), 1e-6)
            want_idx, want_w64, want_w32, want_maxp = ref.step(pending, u, beta, td, 1e-6)
            pending = 0
            got = idx.cpu().numpy()
            assert np.array_equal(got, want_idx), t
            assert np.array_equal(w64.cpu().numpy(), want_w64), t
            assert np.array_equal(w32.cpu().numpy(), want_w32), t
            assert buf._max_priority == want_maxp, t
            dup_seen |= len(set(got.tolist())) < B
            if t % check_every == 0 or t == steps - 1:
                s, m = ref.trees()
                assert np.array_equal(buf._it_sum.cpu().numpy(), s), t
                assert np.array_equal(buf._it_min.cpu().numpy(), m), t
    return dup_seen


@pytest.mark.parametrize("size,steps,learning_starts", [(100, 400, 50), (300, 700, 120), (50000, 50600, 50100)])
def test_prioritized_buffer_along_the_learner_pattern(size, steps, learning_starts):
    """One add per step (staged STAGE = 64 at a time), then from learning_starts sample_device at the schedule's beta
    and update_priorities_device with seeded float32 TD errors; the ring wraps (for 50 000 inside a staged block) and
    transitions keep entering after the max priority has left 1."""
    buf = _filled_buffer(size, n=0)
    ref = ReferenceReplay(size, 0.6)
    random.seed(size)
    rng = np.random.RandomState(size)
    dup = _run_learner_pattern(buf, ref, steps, learning_starts, 32, rng, check_every=50)
    assert dup and buf._max_priority > 1.0


def test_prioritized_buffer_cfg4_size(ops):
    """cfg-4: 10^6 transitions in a 2^20 tree, filled with add_batch, then 50 learner steps at batch 512."""
    from baselines_b200.deepq.replay_buffer import PrioritizedReplayBuffer
    from baselines_b200.common.schedules import LinearSchedule
    size, B = 10 ** 6, 512
    buf = PrioritizedReplayBuffer(size, 0.6)
    ref = ReferenceReplay(size, 0.6)
    k = 1 << 18
    for s in range(0, size, k):
        n = min(k, size - s)
        o = torch.zeros(n, 1, dtype=torch.uint8, device="cuda")
        buf.add_batch(o, torch.zeros(n, dtype=torch.int64, device="cuda"), torch.zeros(n, device="cuda"), o,
                      torch.zeros(n, device="cuda"))
        ref.add(n)
    random.seed(4)
    rng = np.random.RandomState(4)
    sched = LinearSchedule(100, initial_p=0.4, final_p=1.0)
    dup = False
    for t in range(50):
        if t == 25:                                     # more transitions after updates: max_priority ** alpha != 1
            o = torch.zeros(1000, 1, dtype=torch.uint8, device="cuda")
            z = torch.zeros(1000, device="cuda")
            buf.add_batch(o, z.long(), z, o, z)
            ref.add(1000)
        u = [random.random() for _ in range(B)]
        idx, w32, w64 = buf.sample_device(B, beta=sched.value(t), uniforms=u)
        td = _td(rng, B, t)
        buf.update_priorities_device(idx, dev(td), 1e-6)
        want_idx, want_w64, want_w32, want_maxp = ref.step(0, u, sched.value(t), td, 1e-6)
        got = idx.cpu().numpy()
        assert np.array_equal(got, want_idx), t
        assert np.array_equal(w64.cpu().numpy(), want_w64), t
        assert np.array_equal(w32.cpu().numpy(), want_w32), t
        assert buf._max_priority == want_maxp, t
        dup |= len(set(got.tolist())) < B
    s, m = ref.trees()
    assert np.array_equal(buf._it_sum.cpu().numpy(), s)
    assert np.array_equal(buf._it_min.cpu().numpy(), m)
    assert dup and buf._max_priority > 1.0


def test_uniform_buffer_add_and_add_batch_interleaved():
    """ReplayBuffer's stored arrays after single adds (staged) and add_batch calls that cross a stage and the wrap."""
    from baselines_b200.deepq.replay_buffer import ReplayBuffer
    size = 100
    buf = ReplayBuffer(size)
    want = {k: np.zeros(size, dt) for k, dt in (("obs", np.float32), ("act", np.int64), ("rew", np.float32),
                                                 ("done", np.float32))}
    nxt, rng = 0, np.random.RandomState(6)
    for r in range(12):
        k = int(rng.randint(1, 90))
        if r % 2:
            ob = rng.randn(k, 1).astype(np.float32)
            act, rew, done = rng.randint(0, 5, k), rng.randn(k).astype(np.float32), (rng.rand(k) < .3).astype(np.float32)
            buf.add_batch(ob, act, rew, ob + 1, done)
        for i in range(k):
            if not r % 2:
                ob1 = rng.randn(1).astype(np.float32)
                a1, r1, d1 = int(rng.randint(0, 5)), float(np.float32(rng.randn())), float(rng.rand() < .3)
                buf.add(ob1, a1, r1, ob1 + 1, d1)
            j = (nxt + i) % size
            if r % 2:
                want["obs"][j], want["act"][j], want["rew"][j], want["done"][j] = ob[i, 0], act[i], rew[i], done[i]
            else:
                want["obs"][j], want["act"][j], want["rew"][j], want["done"][j] = ob1[0], a1, r1, d1
        nxt = (nxt + k) % size
        buf._flush()
        n = len(buf)
        assert np.array_equal(buf._obs_t[:n, 0].cpu().numpy(), want["obs"][:n])
        assert np.array_equal(buf._obs_tp1[:n, 0].cpu().numpy(), want["obs"][:n] + 1)
        assert np.array_equal(buf._actions[:n].cpu().numpy(), want["act"][:n])
        assert np.array_equal(buf._rewards[:n].cpu().numpy(), want["rew"][:n])
        assert np.array_equal(buf._dones[:n].cpu().numpy(), want["done"][:n])
    assert nxt != 0 and len(buf) == size


# ------------------------------------------------------------------------------------------ deepq.learn itself
@pytest.mark.parametrize("train_freq", [1, 4])
def test_deepq_learn_prioritized_replay_recorded_and_replayed(monkeypatch, train_freq):
    from baselines_b200.common import spaces
    from baselines_b200.common.schedules import LinearSchedule
    from baselines_b200.deepq import deepq
    from baselines_b200.deepq.replay_buffer import PrioritizedReplayBuffer

    log = []

    class Recording(PrioritizedReplayBuffer):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            log.append(("init", self))

        def add(self, *a, **k):
            log.append(("add",))
            return super().add(*a, **k)

        def sample_device(self, batch_size, beta, uniforms=None):
            u = [random.random() for _ in range(batch_size)]            # as the base class draws them
            idx, w32, w64 = super().sample_device(batch_size, beta, uniforms=u)
            log.append(("sample", beta, u, idx.clone(), w32.clone(), w64.clone()))
            return idx, w32, w64

        def update_priorities_device(self, idx, td_errors, eps):
            log.append(("update", idx.clone(), td_errors.clone(), eps))  # td_errors is a view of a persistent buffer
            return super().update_priorities_device(idx, td_errors, eps)

    class Env:
        def __init__(self, n=4):
            self.n = n
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
            r = float(int(a) == self.s) + self.rng.randn()
            self.s, self.t = self.rng.randint(self.n), self.t + 1
            return self._ob(), r, self.t >= 20, {}

    monkeypatch.setattr(deepq, "PrioritizedReplayBuffer", Recording)
    T, size, ls, B, alpha, eps = 600, 200, 50, 32, 0.6, 1e-6
    deepq.learn(Env(), "mlp", seed=0, lr=1e-3, total_timesteps=T, buffer_size=size, train_freq=train_freq,
                batch_size=B, print_freq=None, checkpoint_freq=None, learning_starts=ls, gamma=0.9,
                target_network_update_freq=100, prioritized_replay=True, prioritized_replay_alpha=alpha,
                prioritized_replay_eps=eps, hiddens=(16,))
    buf = log[0][1]
    ref = ReferenceReplay(size, alpha)
    sched = LinearSchedule(T, initial_p=0.4, final_p=1.0)
    trained = [t for t in range(T) if t > ls and t % train_freq == 0]
    betas, pending, last_idx, n_up = [], 0, None, 0
    for rec in log[1:]:
        if rec[0] == "add":
            pending += 1
        elif rec[0] == "sample":
            _, beta, u, idx, w32, w64 = rec
            betas.append(beta)
            ref.add(pending)
            pending = 0
            want = np.asarray(ref.sample_idx(u), np.int64)
            assert np.array_equal(idx.cpu().numpy(), want)
            ww = ref.weights(want, beta)
            assert np.array_equal(w64.cpu().numpy(), ww) and np.array_equal(w32.cpu().numpy(), ww.astype(np.float32))
            last_idx = want
        else:
            _, idx, td, e = rec
            assert e == eps and np.array_equal(idx.cpu().numpy(), last_idx)    # td[b] goes back to idx[b]
            ref.update_priorities(last_idx, reference_priorities(td.cpu().numpy(), e))
            n_up += 1
    ref.add(pending)
    buf._flush()
    assert betas == [sched.value(t) for t in trained]                   # the schedule's t and the train gating
    assert n_up == len(trained)
    s, m = ref.trees()
    assert np.array_equal(buf._it_sum.cpu().numpy(), s) and np.array_equal(buf._it_min.cpu().numpy(), m)
    assert buf._max_priority == ref.max_priority and ref.max_priority > 1.0
