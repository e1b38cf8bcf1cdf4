"""CPU: the prioritized-replay reference semantics of tests/_replay_refs.py (priority dtype, leaf rule, running max,
vectorised tree build, the step driver) against the sequential oracle and against decimal arithmetic."""
import decimal

import numpy as np

from _replay_refs import (ReferenceReplay, build_trees, cr_pow, leaf_values, reference_priorities,
                                running_max)
from oracle.segment_tree import MinTree, PrioritizedSampler, SumTree


def _decimal_pow(x, y):
    with decimal.localcontext() as ctx:
        ctx.prec = 60
        return float(decimal.Decimal(float(x)) ** decimal.Decimal(float(y)))


def test_float32_td_plus_python_eps_stays_float32():
    td = np.array([-3.5, 0.0, -0.0, 1e-30, 2.0 ** -140, 0.1, 3e38], np.float32)
    assert (np.abs(td) + 1e-6).dtype == np.float32                  # deepq.py:302 under NumPy 1.x and 2.x alike
    p = reference_priorities(td, 1e-6)
    assert p.dtype == np.float32
    want = [np.float32(np.float64(abs(float(t))) + np.float64(np.float32(1e-6))) for t in td]
    assert np.array_equal(p, np.array(want, np.float32))
    assert p[0] == np.float32(3.500001) and p[1] == p[2] == np.float32(1e-6)
    assert float(p[5]) != abs(0.1) + 1e-6                             # float32, not the float64 sum
    assert np.array_equal(reference_priorities(td, 0.0), np.abs(td))
    assert np.isnan(reference_priorities(np.array([np.nan], np.float32), 1e-6)[0])


def test_leaf_is_float64_pow_of_the_float32_priority():
    p = reference_priorities(np.array([0.3, 7.25, 1e-5], np.float32), 1e-6)
    leaves = leaf_values(p, 0.6)
    assert leaves.dtype == np.float64
    for pi, li in zip(p, leaves):
        assert li == _decimal_pow(float(pi), 0.6)
        # NumPy 2 evaluates np.float32 ** float in float32; NumPy 1.x (the reference's) in float64
        assert li != float(np.float32(float(pi) ** 0.6)) or li == float(np.float32(li))


def test_cr_pow_matches_decimal():
    rng = np.random.RandomState(0)
    x32 = np.exp2(rng.uniform(-24, 20, 3000)).astype(np.float32)
    special = np.array([2.0 ** k for k in range(-149, 128, 7)], np.float32)
    x = np.concatenate([x32, special, np.nextafter(special, np.float32(np.inf)),
                        np.nextafter(special, np.float32(0))]).astype(np.float64)
    x = np.concatenate([x, rng.uniform(1e-3, 1e6, 500)])             # double arguments, like p * n in the weights
    for y in (0.5, 0.6, 0.7, -0.4, -0.7, -1.0, -0.43):
        got = cr_pow(x, y)
        want = np.array([_decimal_pow(v, y) for v in x.tolist()])
        assert np.array_equal(got, want), (y, int((got != want).sum()))
    assert cr_pow(4.0, 0.5) == 2.0 and cr_pow(3.0, 1.0) == 3.0 and cr_pow(0.0, 0.6) == 0.0
    assert cr_pow(5.0, 0.0) == 1.0 and cr_pow(0.0, -0.4) == float("inf")


def test_vectorised_tree_build_equals_sequential_set():
    rng = np.random.RandomState(1)
    for cap in (1, 2, 8, 64, 1024):
        s, m = SumTree(cap), MinTree(cap)
        leaves = np.zeros(cap)
        written = np.zeros(cap, bool)
        for _ in range(3 * cap):
            i = int(rng.randint(cap))
            v = float(np.abs(rng.randn()) ** 0.6) * 10.0 ** rng.randint(-6, 7)
            s.set(i, v)
            m.set(i, v)
            leaves[i] = v
            written[i] = True
        bs, bm = build_trees(cap, leaves, np.where(written, leaves, np.inf))
        assert np.array_equal(bs, s.value) and np.array_equal(bm, m.value), cap


def test_duplicate_index_last_write_wins_and_max_counts_every_entry():
    ref = ReferenceReplay(8, 0.6)
    ref.add(8)
    td = np.array([100.0, 0.5, 2.0, 0.25], np.float32)
    ref.update_priorities([3, 3, 5, 5], reference_priorities(td, 1e-6))
    p = reference_priorities(td, 1e-6)
    assert ref.leaves[3] == cr_pow(float(p[1]), 0.6)                  # the later entry for index 3
    assert ref.leaves[5] == cr_pow(float(p[3]), 0.6)
    assert ref.max_priority == float(p[0])                            # max over all four, not over the survivors
    assert running_max(1.0, p) == float(p[0]) and running_max(200.0, p) == 200.0
    # the next add enters with max_priority ** alpha of that float32 value
    ref.add(1)
    assert ref.leaves[0] == cr_pow(float(np.float32(100.000001)), 0.6)


def test_driver_equals_sequential_oracle_with_the_same_leaf_rule():
    """ReferenceReplay (rebuilt trees, float32 priorities) against PrioritizedSampler's own sequential sets fed the
    same leaf values, over adds that wrap the ring, duplicate indices and priority updates between adds."""
    size, alpha, batch = 100, 0.6, 32
    rng = np.random.RandomState(2)
    ref = ReferenceReplay(size, alpha)
    seq = PrioritizedSampler(size, alpha)
    for step in range(40):
        k = int(rng.randint(2, 9))                                   # the p_total quirk needs n >= 2
        ref.add(k)
        for _ in range(k):
            i = seq.next_idx
            seq.add()
            v = cr_pow(seq.max_priority, alpha)
            seq.sum_tree.set(i, v)
            seq.min_tree.set(i, v)
        u = rng.rand(batch)
        beta = 0.4 + 0.01 * step
        td = (rng.randn(batch) * 10.0 ** rng.randint(-3, 3)).astype(np.float32)
        idx, w64, w32, maxp = ref.step(0, u, beta, td, 1e-6)
        want_idx = seq.sample_idx(u)
        assert list(idx) == want_idx
        total = seq.sum_tree.sum()
        max_w = cr_pow(seq.min_tree.min() / total * seq.n, -beta)
        want_w = np.array([cr_pow(seq.sum_tree.get(i) / total * seq.n, -beta) / max_w for i in want_idx])
        assert np.array_equal(w64, want_w) and np.array_equal(w32, want_w.astype(np.float32))
        pr = reference_priorities(td, 1e-6)
        for i, p in zip(want_idx, pr):
            v = cr_pow(float(p), alpha)
            seq.sum_tree.set(i, v)
            seq.min_tree.set(i, v)
            seq.max_priority = max(seq.max_priority, float(p))
        assert maxp == seq.max_priority
        s, m = ref.trees()
        assert np.array_equal(s, seq.sum_tree.value) and np.array_equal(m, seq.min_tree.value)
    assert seq.max_priority != 1.0 and len(set(ref.leaves[:size].tolist())) > 50
