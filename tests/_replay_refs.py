"""Reference semantics of the prioritized replay path that deepq.learn runs, in the reference's dtypes.

The reference (deepq/deepq.py:302, deepq/replay_buffer.py:100-191) computes
* new priorities ``np.abs(td_errors) + prioritized_replay_eps`` on the float32 TD errors of its graph: a float32 array
  plus a python float stays float32, so each priority is fl32(|td| + fl32(eps));
* leaves ``priority ** alpha``: under NumPy 1.x (which TF1 pins) an np.float32 scalar to a python float power is a
  float64 pow of the float32 value; NumPy 2 would evaluate it in float32, so the rule is written out here instead of
  being taken from executing the reference with the installed NumPy;
* ``_max_priority = max(_max_priority, priority)`` over every entry, duplicates included, keeping the float32 value;
  new transitions enter with ``_max_priority ** alpha``;
* weights ``(p * n) ** -beta / (p_min * n) ** -beta`` in float64.

Every pow is the correctly rounded one (``cr_pow``).  The host libm is not an exact target: glibc >= 2.28 documents its
pow to 0.52 ulp, and on glibc 2.39 ``float.__pow__`` differs from the correctly rounded result for about 1 in 1500
float32 priorities.  Holding both host and device to the correctly rounded value makes the leaves independent of the
libm that happens to evaluate them.

The trees reuse ``oracle/segment_tree.py``; ``build_trees`` is a vectorised bottom-up build of the same node values.
"""
import decimal

import numpy as np

from oracle.segment_tree import MinTree, PrioritizedSampler, SumTree


def cr_pow(x, y):
    """Correctly rounded x ** y for float64 x > 0 (array or scalar) and a float y.  An x87 long-double powl (about
    2^-63 relative) decides every value whose rounding it settles with a 2x margin; the rest (~0.2%) go to decimal at
    60 digits."""
    scalar = np.ndim(x) == 0
    x = np.atleast_1d(np.asarray(x, dtype=np.float64))
    out = np.empty_like(x)
    pos = (x > 0) & np.isfinite(x)
    with np.errstate(all="ignore"):
        out[~pos] = np.power(x[~pos], y)                                 # 0, inf, NaN: IEEE special values
    xp = x[pos]
    r = np.power(xp.astype(np.longdouble), np.longdouble(y))
    lo = (r * (1 - np.longdouble(2.0 ** -62))).astype(np.float64)
    hi = (r * (1 + np.longdouble(2.0 ** -62))).astype(np.float64)
    res = lo.copy()
    amb = np.flatnonzero(lo != hi)
    if len(amb):
        with decimal.localcontext() as ctx:
            ctx.prec = 60
            dy = decimal.Decimal(float(y))
            res[amb] = [float(decimal.Decimal(v) ** dy) for v in xp[amb].tolist()]
    out[pos] = res
    if y == 1.0:
        out[pos] = xp
    if y == 0.0:
        out[:] = 1.0
    return float(out[0]) if scalar else out


def reference_priorities(td32, eps):
    """deepq.py:302 on float32 TD errors: fl32(|td| + fl32(eps)), as float32."""
    td32 = np.asarray(td32)
    assert td32.dtype == np.float32
    return (np.abs(td32) + np.float32(eps)).astype(np.float32)


def leaf_values(priorities, alpha):
    """replay_buffer.py:188-189 with NumPy 1.x scalar promotion: float(p) ** alpha in float64 (correctly rounded)."""
    return cr_pow(np.asarray(priorities, dtype=np.float32).astype(np.float64), float(alpha))


def running_max(maxp, priorities):
    """replay_buffer.py:191, in update order, over every entry (duplicates included)."""
    for p in np.asarray(priorities).tolist():
        maxp = max(maxp, float(p))
    return maxp


def build_trees(capacity, leaves_sum, leaves_min=None):
    """Sum and min node arrays from their leaves, bottom-up: node = op(left, right), which is what a sequence of
    SumTree.set / MinTree.set leaves behind for the same final leaves."""
    s = np.zeros(2 * capacity, np.float64)
    m = np.full(2 * capacity, np.inf, np.float64)
    s[capacity:] = leaves_sum
    m[capacity:] = leaves_sum if leaves_min is None else leaves_min
    lo = capacity
    while lo > 1:
        hi, lo = lo, lo // 2
        s[lo:hi] = s[2 * lo:2 * hi:2] + s[2 * lo + 1:2 * hi:2]
        m[lo:hi] = np.minimum(m[2 * lo:2 * hi:2], m[2 * lo + 1:2 * hi:2])
    return s, m


class ReferenceReplay(PrioritizedSampler):
    """PrioritizedSampler driven one recorded learner step at a time, with the float32 priority rule above.  The leaves
    are kept as one array and the trees are rebuilt from it (``build_trees``) whenever they are read."""

    def __init__(self, size, alpha):
        super().__init__(size, alpha)
        cap = self.sum_tree.capacity
        self.leaves = np.zeros(cap, np.float64)
        self.stored = np.zeros(cap, bool)
        self._dirty = False

    def _sync(self):
        if self._dirty:
            cap = self.sum_tree.capacity
            self.sum_tree.value, self.min_tree.value = build_trees(cap, self.leaves,
                                                                   np.where(self.stored, self.leaves, np.inf))
            self._dirty = False

    def trees(self):
        self._sync()
        return self.sum_tree.value, self.min_tree.value

    def add(self, k=1):
        """k transitions at the ring position, each entering with max_priority ** alpha (replay_buffer.py:100-105)."""
        idx = (self.next_idx + np.arange(k)) % self.maxsize
        self.next_idx = int((self.next_idx + k) % self.maxsize)
        self.n = min(self.n + k, self.maxsize)
        self.leaves[idx] = cr_pow(self.max_priority, self.alpha)
        self.stored[idx] = True
        self._dirty = True
        return idx

    def sample_idx(self, uniforms):
        self._sync()
        return super().sample_idx(uniforms)

    def weights(self, idxes, beta):
        self._sync()
        total = self.sum_tree.sum()
        p_min = self.min_tree.min() / total
        max_w = cr_pow(p_min * self.n, -beta)
        p = np.array([self.sum_tree.get(int(i)) for i in idxes]) / total
        return cr_pow(p * self.n, -beta) / max_w

    def update_priorities(self, idxes, priorities):
        """replay_buffer.py:169-191 for float32 priorities: leaves in update order (the last write to an index wins)."""
        idxes = np.asarray(idxes, dtype=np.int64)
        priorities = np.asarray(priorities, dtype=np.float32)
        assert len(idxes) == len(priorities)
        assert np.all(priorities > 0), "assert priority > 0"
        assert np.all((idxes >= 0) & (idxes < self.n))
        vals = leaf_values(priorities, self.alpha)
        _, first_rev = np.unique(idxes[::-1], return_index=True)        # the last write to each index
        last = len(idxes) - 1 - first_rev
        self.leaves[idxes[last]] = vals[last]
        self._dirty = True
        self.max_priority = running_max(self.max_priority, priorities)

    def step(self, adds, uniforms, beta, td32=None, eps=None):
        """One learner step: `adds` transitions, a sample with these uniforms at this beta, then (when td32 is given)
        update_priorities(idx, reference_priorities(td32, eps)).  Returns (idx, w64, w32, max_priority)."""
        if adds:
            self.add(adds)
        idx = np.asarray(self.sample_idx(uniforms), dtype=np.int64)
        w64 = self.weights(idx, beta)
        if td32 is not None:
            self.update_priorities(idx, reference_priorities(td32, eps))
        return idx, w64, w64.astype(np.float32), self.max_priority


__all__ = ["cr_pow", "reference_priorities", "leaf_values", "running_max", "build_trees", "ReferenceReplay",
           "SumTree", "MinTree"]
