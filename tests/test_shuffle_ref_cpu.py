"""CPU: the host restatement of the device minibatch shuffle (_shuffle_ref) and the key / buffer plumbing of
ppo2.run_epochs(shuffle="device").

  1. shuffle_ref is a bijection of [0, n) for n at and around every power of four up to 4^10 (half_bits 1 .. 11, the
     domain up to almost 4x the range) and at a prime; with (T, N) it is the plain permutation composed with the sf01
     map, so every output is a buffer offset t*N + e; different keys give different permutations, and so do keys that
     differ only in bit 63.
  2. The vectorised numpy network equals a scalar restatement in python integers masked to 32 bits.
  3. run_epochs(shuffle="device") with a recording stand-in for the kernel and the model: one shuffle per epoch into
     the rollout's one shuffle buffer, keyed as run_epochs_keys says; the minibatches are consecutive slices of that
     epoch's buffer.
  4. The minibatch statistics the GPU test applies to the kernel accept the 6-round network at the cfg2 shape and
     reject a 2-round one.
"""
import numpy as np
import pytest
import torch

import _shuffle_ref as S

SIZES = sorted({1, 2, 3, 4, 5, 15, 16, 17, 63, 64, 65, 100003} |
               {4 ** k + d for k in range(1, 11) for d in (-1, 1)})


def _split(n):
    """(T, N) with T * N == n, T the largest divisor <= sqrt(n)."""
    T = max(d for d in range(1, int(n ** 0.5) + 1) if n % d == 0)
    return T, n // T


@pytest.mark.parametrize("n", SIZES)
def test_shuffle_ref_is_a_bijection_with_and_without_the_buffer_map(n):
    key = 0x9E3779B97F4A7C15 ^ n
    p = S.shuffle_ref(n, key)
    assert p.dtype == np.int64 and p.shape == (n,)
    assert np.array_equal(np.sort(p), np.arange(n))
    T, N = _split(n)
    q = S.shuffle_ref(n, key, T, N)
    assert np.array_equal(np.sort(q), np.arange(n))
    t, e = q // N, q % N                               # every output is t*N + e with t < T, e < N
    assert np.all((t >= 0) & (t < T) & (e >= 0) & (e < N))
    assert np.array_equal(q, (p % T) * N + p // T), "the (T, N) output is not the sf01 map of the plain permutation"
    assert np.array_equal(S.flat_of_offsets(q, T, N), p)


@pytest.mark.parametrize("n", [n for n in SIZES if n >= 64])
def test_different_keys_give_different_permutations(n):
    keys = [0, 1, 0x1234567890ABCDEF, 0x1234567890ABCDEF ^ (1 << 63), 1 << 32, (1 << 64) - 1]
    perms = [S.shuffle_ref(n, k) for k in keys]
    for a in range(len(keys)):
        for b in range(a):
            assert not np.array_equal(perms[a], perms[b]), (hex(keys[a]), hex(keys[b]))


def test_half_bits_as_the_host_function_derives_it():
    assert [S.half_bits(n) for n in (1, 2, 4, 5, 16, 17)] == [1, 1, 1, 2, 2, 3]
    assert S.half_bits(4 ** 10) == 10 and S.half_bits(4 ** 10 + 1) == 11 and S.half_bits(4 ** 12 + 1) == 13
    assert S.half_bits(128 * 4096) == 10 and S.half_bits(512 * 16384) == 12


def _scalar_shuffle(n, key):
    """shuffle_indices_kernel for one lane at a time in python integers."""
    M = 0xFFFFFFFF
    hb = S.half_bits(n)
    mask = (1 << hb) - 1
    rk = [(((key >> (8 * r)) & M) * 0x9E3779B1 + ((key >> 32) & M) + 0x7F4A7C15 * (r + 1)) & M for r in range(6)]

    def f(x, k):
        x = (x ^ k) & M
        x = (x * 0x9E3779B1) & M
        x ^= x >> 15
        x = (x * 0x85EBCA77) & M
        x ^= x >> 13
        return x

    out = []
    for i in range(n):
        x = i
        while True:
            l, r = (x >> hb) & mask, x & mask
            for k in rk:
                l, r = r, l ^ (f(r, k) & mask)
            x = (l << hb) | r
            if x < n:
                break
        out.append(x)
    return np.array(out, np.int64)


@pytest.mark.parametrize("n,key", [(1, 5), (7, 0xFFFFFFFFFFFFFFFF), (65, 0x8000000080000000), (1000, 0x1234567890ABCDEF),
                                   (4 ** 6 + 1, 0x7FFFFFFE7FFFFFFE)])
def test_vectorised_network_equals_a_scalar_restatement(n, key):
    assert np.array_equal(S.shuffle_ref(n, key), _scalar_shuffle(n, key))


# ------------------------------------------------------------------------------------------ run_epochs plumbing
class _Rollout:
    def __init__(self, T, N):
        self.T, self.N = T, N
        self.buf = torch.full((T * N,), -1, dtype=torch.int64)

    def flat(self, name):
        return torch.zeros(self.T * self.N)

    def shuffle_buffer(self):
        return self.buf


class _Model:
    recurrent = False

    def __init__(self):
        self.minibatches = []

    def train_rollout(self, lr, clip, obs, actions, returns, values, neglogp, mb):
        self.minibatches.append(mb.clone())
        return torch.zeros(5, dtype=torch.float64)


@pytest.mark.parametrize("noptepochs", [1, 4])
def test_run_epochs_device_shuffle_keys_buffer_and_minibatches(monkeypatch, noptepochs):
    """3.  Mutants caught here: one key per update instead of per epoch, the two draws swapped, epoch 0's buffer reused
    for every epoch, a minibatch taken from the wrong slice."""
    from baselines_b200.ppo2 import ppo2
    T, N, nmb = 8, 12, 4
    n, m = T * N, T * N // nmb
    calls = []

    def fake_shuffle(out, n_, key, T_, N_):
        assert (n_, T_, N_) == (n, T, N)
        out.copy_(torch.from_numpy(S.shuffle_ref(n_, key, T_, N_)))
        calls.append((key, out))

    monkeypatch.setattr(ppo2, "ops_shuffle", fake_shuffle)
    np.random.seed(123)
    state = np.random.get_state()
    ro, model = _Rollout(T, N), _Model()
    stats = ppo2.run_epochs(model, ro, 1e-3, 0.2, n, m, noptepochs, "cpu", shuffle="device")
    assert len(stats) == noptepochs * nmb
    keys = S.run_epochs_keys(state, noptepochs)
    assert [k for k, _ in calls] == keys
    assert all(out is ro.buf for _, out in calls), "every epoch shuffles into the rollout's one shuffle buffer"
    assert len(set(keys)) == noptepochs and all(k >> 32 for k in keys)
    for ep, key in enumerate(keys):
        want = S.shuffle_ref(n, key, T, N)
        for b in range(nmb):
            got = model.minibatches[ep * nmb + b].numpy()
            assert np.array_equal(got, want[b * m:(b + 1) * m]), (ep, b)
    # the numpy stream moved by exactly two draws per epoch
    rs = np.random.RandomState()
    rs.set_state(state)
    rs.randint(0, 2 ** 31 - 1, size=2 * noptepochs)
    assert np.random.randint(0, 2 ** 31) == rs.randint(0, 2 ** 31)


def test_run_epochs_keys_replays_the_draws_in_order():
    np.random.seed(7)
    st = np.random.get_state()
    a, b, c, d = (int(np.random.randint(0, 2 ** 31 - 1)) for _ in range(4))
    assert S.run_epochs_keys(st, 2) == [a | (b << 32), c | (d << 32)]


# ------------------------------------------------------------------------------------------ statistical power
def test_minibatch_statistics_accept_six_rounds_and_reject_two():
    """4: at cfg2's shape (n = 524 288, T = 128, N = 4096, 4 minibatches of 131 072), two epoch keys drawn as run_epochs
    draws them.  Each family is tested at p = 1e-6 after a Bonferroni correction over its members."""
    T, N, m = 128, 4096, 131072
    keys = S.run_epochs_keys(np.random.RandomState(0).get_state(), 2)
    for rounds, accept in ((6, True), (2, False)):
        p, most = S.minibatch_pvalues([S.shuffle_ref(T * N, k, T, N, rounds=rounds) for k in keys], T, N, m)
        worst = {f: float(v.min() * len(v)) for f, v in p.items()}
        print(f"[observed] {rounds} rounds: Bonferroni-scaled smallest p per family {worst}; largest overlap {most}")
        assert most < m
        assert all(w > 1e-6 for w in worst.values()) == accept, (rounds, worst)
