"""Host restatement of the device minibatch shuffle (csrc/optim.cu shuffle_indices_kernel, b200rl_shuffle_indices) and
of the epoch keys ppo2.run_epochs draws for it.

shuffle_ref(n, key, T, N) returns what the kernel writes for sample i: a 6-round Feistel network over 2 * half_bits
bits (the smallest power of four >= n, at least 4), in wrapping uint32 arithmetic, re-encrypted until the value lands
in [0, n) (cycle walking), then the env-major flat index j = e*T + t mapped to its buffer offset t*N + e.
"""
import numpy as np

ROUNDS = 6
_M32 = 0xFFFFFFFF


def half_bits(n):
    """b200rl_shuffle_indices: the Feistel halves are half_bits wide, 4^half_bits >= n, half_bits >= 1."""
    hb = 1
    while (1 << (2 * hb)) < n:
        hb += 1
    return hb


def round_keys(key, rounds=ROUNDS):
    """rk[r] = uint32(key >> 8r) * 0x9E3779B1 + uint32(key >> 32) + 0x7F4A7C15 * (r + 1), all mod 2^32."""
    key &= (1 << 64) - 1
    return [(((key >> (8 * r)) & _M32) * 0x9E3779B1 + (key >> 32) + 0x7F4A7C15 * (r + 1)) & _M32
            for r in range(rounds)]


def feistel_round(x, k):
    """The kernel's round function on a uint32 array (numpy array arithmetic wraps mod 2^32)."""
    x = x ^ np.uint32(k)
    x = x * np.uint32(0x9E3779B1)
    x ^= x >> np.uint32(15)
    x = x * np.uint32(0x85EBCA77)
    x ^= x >> np.uint32(13)
    return x


def encrypt(x, rk, hb):
    """One pass of the network over uint64 values x < 4^hb."""
    mask = np.uint32((1 << hb) - 1)
    l = ((x >> np.uint64(hb)).astype(np.uint32)) & mask
    r = x.astype(np.uint32) & mask
    for k in rk:
        l, r = r, l ^ (feistel_round(r, k) & mask)
    return (l.astype(np.uint64) << np.uint64(hb)) | r.astype(np.uint64)


def shuffle_ref(n, key, T=0, N=0, rounds=ROUNDS):
    """int64[n]: out[i] of shuffle_indices_kernel for this key; with T > 0 (T * N == n) the buffer offset of the
    env-major flat index, (j % T) * N + j // T.  rounds: only for showing what a weaker network looks like."""
    assert n > 0 and (T == 0 or T * N == n)
    hb, rk = half_bits(n), round_keys(key, rounds)
    x = np.arange(n, dtype=np.uint64)
    todo = np.arange(n)
    while todo.size:                                    # cycle walking: only the lanes still >= n are re-encrypted
        y = encrypt(x[todo], rk, hb)
        x[todo] = y
        todo = todo[y >= np.uint64(n)]
    j = x.astype(np.int64)
    return (j % T) * N + j // T if T > 0 else j


def flat_of_offsets(o, T, N):
    """Inverse of the sf01 map: buffer offset t*N + e -> env-major flat index e*T + t."""
    o = np.asarray(o, dtype=np.int64)
    return (o % N) * T + o // N


def run_epochs_keys(seed_state, noptepochs):
    """The keys ppo2.run_epochs(shuffle="device") passes to shuffle_indices, one per epoch, when the global numpy
    stream is at seed_state (np.random.get_state()): two randint(0, 2^31 - 1) draws per epoch, the first the low word,
    the second the high word."""
    rs = np.random.RandomState()
    rs.set_state(seed_state)
    keys = []
    for _ in range(noptepochs):
        lo = int(rs.randint(0, 2 ** 31 - 1))
        hi = int(rs.randint(0, 2 ** 31 - 1))
        keys.append(lo | (hi << 32))
    return keys


# ------------------------------------------------------------------------------------------ minibatch statistics
def _chi2_sf(x, df):
    import scipy.stats
    return scipy.stats.chi2.sf(x, df)


def minibatch_pvalues(epochs, T, N, m):
    """Upper-tail p-values of what a uniform random permutation gives the minibatches of `epochs` (buffer-offset arrays
    of n = T * N samples, one per epoch, cut into minibatches of m), per family:
      timestep  per epoch and minibatch: Pearson chi-square of the counts per timestep; each count is
                Hypergeometric(n, N, m), so X^2 (n - 1) / (n - m) is chi-square with T - 1 degrees of freedom;
      env       the same over the N environments (T samples each), N - 1 degrees of freedom;
      overlap   per pair (minibatch a of epoch 0, minibatch b of epoch 1): the shared samples, Hypergeometric(n, m, m),
                two-sided;
      lowbits   per epoch: chi-square independence of (i mod 2^k, pi(i) mod 2^k) and of (i mod 2^k, floor(pi(i) 2^k / n))
                for k = 3, 4, pi(i) the env-major flat index of sample i, (2^k - 1)^2 degrees of freedom.
    Also returns the largest overlap (m means epoch 1 repeats one of epoch 0's minibatches as a set)."""
    import scipy.stats
    n = T * N
    K = n // m
    fpc = (n - 1) / (n - m)                             # finite-population factor of sampling without replacement
    mb = np.arange(n) // m
    out = {"timestep": [], "env": [], "overlap": None, "lowbits": []}
    for o in epochs:
        for fam, cls, C in (("timestep", o // N, T), ("env", o % N, N)):
            c = np.bincount(mb * C + cls, minlength=K * C).reshape(K, C).astype(np.float64)
            x2 = ((c - m / C) ** 2).sum(1) / (m / C) * fpc
            out[fam].extend(_chi2_sf(x2, C - 1))
        i = np.arange(n)
        j = flat_of_offsets(o, T, N)
        for k in (3, 4):
            b = 1 << k
            for col in (j % b, (j * b) // n):
                c = np.bincount((i % b) * b + col, minlength=b * b).reshape(b, b).astype(np.float64)
                e = np.outer(c.sum(1), c.sum(0)) / n
                out["lowbits"].append(_chi2_sf(((c - e) ** 2 / e).sum(), (b - 1) ** 2))
    lab = []
    for o in epochs[:2]:
        lab_e = np.empty(n, np.int64)
        lab_e[o] = mb
        lab.append(lab_e)
    ov = np.bincount(lab[0] * K + lab[1], minlength=K * K)
    h = scipy.stats.hypergeom(n, m, m)
    out["overlap"] = np.minimum(1.0, 2 * np.minimum(h.sf(ov - 1), h.cdf(ov)))
    out = {k: np.asarray(v, np.float64) for k, v in out.items()}
    return out, int(ov.max())
