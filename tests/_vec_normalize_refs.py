"""Order-explicit numpy restatement of VecNormalize (common/vec_env.py) and RunningMeanStd (running_mean_std.py): every
add in the order numpy performs it, so that the device kernels have a reference to match bit for bit.

* batch moments along axis 0 (np.mean / np.var in the dtype of x): with D >= 2 columns each column is summed
  sequentially in row order; with D == 1 (and for the 1-D discounted return) numpy's pairwise sum is used;
* the Chan combination of running_mean_std.py, left to right (float64, but bv * n in the batch's dtype);
* the step order of VecNormalize.step_wait.
"""
import numpy as np


def pairwise_sum(a):
    """np.add.reduce of a 1-D array in a's dtype: the reduction starts from +0 and adds numpy's pairwise sum
    (loops_utils.h pairwise_sum) of the whole array."""
    a = np.asarray(a)
    return a.dtype.type(a.dtype.type(0.0) + _pairwise(a))


def _pairwise(a):
    n = a.shape[0]
    dt = a.dtype.type
    if n < 8:
        res = dt(0.0)
        for i in range(n):
            res = dt(res + a[i])
        return res
    if n <= 128:
        r = a[:8].copy()
        m = n - n % 8
        for i in range(8, m, 8):
            r = r + a[i:i + 8]
        res = dt(dt(dt(r[0] + r[1]) + dt(r[2] + r[3])) + dt(dt(r[4] + r[5]) + dt(r[6] + r[7])))
        for i in range(m, n):
            res = dt(res + a[i])
        return res
    n2 = n // 2
    n2 -= n2 % 8
    return dt(_pairwise(a[:n2]) + _pairwise(a[n2:]))


def column_sum(x2):
    """Sequential sum over rows of an [N, D] array from +0, column by column (numpy's axis-0 reduction, D >= 2)."""
    s = np.zeros(x2.shape[1], x2.dtype)
    for i in range(x2.shape[0]):
        s += x2[i]
    return s


def batch_moments(x):
    """(mean, var) of x along axis 0, in x's dtype, shaped like x[0]."""
    x = np.asarray(x)
    N = x.shape[0]
    x2 = x.reshape(N, -1)
    dt = x.dtype.type
    if x2.shape[1] == 1:
        m = dt(pairwise_sum(x2[:, 0]) / dt(N))
        d = (x2[:, 0] - m)
        v = dt(pairwise_sum(d * d) / dt(N))
        return np.full(x.shape[1:], m, x.dtype), np.full(x.shape[1:], v, x.dtype)
    m = (column_sum(x2) / dt(N)).astype(x.dtype)
    d = x2 - m
    v = (column_sum(d * d) / dt(N)).astype(x.dtype)
    return m.reshape(x.shape[1:]), v.reshape(x.shape[1:])


def combine(mean, var, count, bm, bv, n):
    """running_mean_std.py:22-34 left to right, in float64 except bv * n: numpy keeps that product in the batch's
    dtype (a Python int does not widen a float32 array), so for float32 observations it is a float32 multiply."""
    bm, bv = np.asarray(bm), np.asarray(bv)
    delta = bm - mean
    tot = count + n
    new_mean = mean + delta * n / tot
    m2 = var * count + bv * n + delta * delta * count * n / tot
    return new_mean, m2 / tot, tot


class RefVecNormalize:
    """VecNormalize over raw (obs, rews, news) batches; obs/rews come back as the float32 the Runner stores."""

    def __init__(self, ob_shape, num_envs, ob=True, ret=True, clipob=10., cliprew=10., gamma=0.99, epsilon=1e-8):
        self.ob = ((np.zeros(ob_shape), np.ones(ob_shape), 1e-4) if ob else None)
        self.rt = ((np.zeros(()), np.ones(()), 1e-4) if ret else None)
        self.clipob, self.cliprew, self.gamma, self.epsilon = clipob, cliprew, gamma, epsilon
        self.ret = np.zeros(num_envs)

    def obfilt(self, x):
        if self.ob is None:
            return np.asarray(x).astype(np.float32)
        bm, bv = batch_moments(x)
        self.ob = combine(*self.ob, bm, bv, x.shape[0])
        mean, var, _ = self.ob
        y = (x.astype(np.float64) - mean) / np.sqrt(var + self.epsilon)
        return np.clip(y, -self.clipob, self.clipob).astype(np.float32)

    def reset(self, x):
        self.ret = np.zeros_like(self.ret)
        return self.obfilt(x)

    def step(self, x, rews, news):
        self.ret = self.ret * self.gamma + rews
        y = self.obfilt(x)
        r = np.asarray(rews)
        if self.rt is not None:
            bm, bv = batch_moments(self.ret)
            self.rt = combine(*self.rt, bm, bv, self.ret.shape[0])
            r = np.clip(r / np.sqrt(self.rt[1] + self.epsilon), -self.cliprew, self.cliprew)
        self.ret[np.asarray(news, dtype=np.bool_)] = 0.
        return y, r.astype(np.float32)
