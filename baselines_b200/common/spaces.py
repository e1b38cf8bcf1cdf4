"""Minimal gym.spaces stand-ins (gym is an external dependency of the reference and is absent here).

Only what the learner boundary needs (SURVEY.md 8b): `.shape`, `.dtype`, `.n`, `.nvec`, `.sample()`.  Real
gym spaces are accepted everywhere too: the code duck-types on these attributes (is_discrete / is_multi_discrete /
is_multi_binary / is_box tell the four apart).
"""
import numpy as np


class Box:
    def __init__(self, low, high, shape=None, dtype=np.float32):
        self.dtype = np.dtype(dtype)
        if shape is None:
            low, high = np.asarray(low), np.asarray(high)
            shape = low.shape
        self.shape = tuple(shape)
        self.low = np.broadcast_to(np.asarray(low, dtype=self.dtype), self.shape).copy()
        self.high = np.broadcast_to(np.asarray(high, dtype=self.dtype), self.shape).copy()

    def seed(self, seed=None):
        self._rng = np.random.RandomState(seed)

    def sample(self):
        rng = getattr(self, "_rng", None) or np.random
        if self.dtype.kind in "iu":
            return rng.randint(self.low.astype(np.int64), self.high.astype(np.int64) + 1).astype(self.dtype)
        return rng.uniform(self.low, self.high).astype(self.dtype)

    def contains(self, x):
        x = np.asarray(x)
        return x.shape == self.shape and bool(np.all(x >= self.low) and np.all(x <= self.high))

    def __repr__(self):
        return f"Box{self.shape}"


class Discrete:
    def __init__(self, n):
        self.n = int(n)
        self.shape = ()
        self.dtype = np.dtype(np.int64)

    def seed(self, seed=None):
        self._rng = np.random.RandomState(seed)

    def sample(self):
        return int((getattr(self, "_rng", None) or np.random).randint(self.n))

    def contains(self, x):
        return 0 <= int(x) < self.n

    def __repr__(self):
        return f"Discrete({self.n})"


class MultiDiscrete:
    """gym.spaces.MultiDiscrete: a vector of independent Discrete(nvec[i]) components, int64."""

    def __init__(self, nvec):
        nv = np.asarray(nvec, dtype=np.int64)
        if nv.ndim != 1 or nv.size == 0 or np.any(nv < 1):
            raise ValueError(f"MultiDiscrete needs a non-empty 1-d nvec of entries >= 1, got {nvec!r}")
        self.nvec = nv
        self.shape = nv.shape
        self.dtype = np.dtype(np.int64)

    def seed(self, seed=None):
        self._rng = np.random.RandomState(seed)

    def sample(self):
        rng = getattr(self, "_rng", None) or np.random
        return (rng.random_sample(self.nvec.shape) * self.nvec).astype(self.dtype)

    def contains(self, x):
        x = np.asarray(x)
        return x.shape == self.shape and x.dtype.kind in "iu" and bool(np.all((x >= 0) & (x < self.nvec)))

    def __repr__(self):
        return f"MultiDiscrete({self.nvec.tolist()})"


class MultiBinary:
    """gym.spaces.MultiBinary: n independent bits, int8."""

    def __init__(self, n):
        self.n = int(n)
        if self.n < 1:
            raise ValueError(f"MultiBinary needs n >= 1, got {n!r}")
        self.shape = (self.n,)
        self.dtype = np.dtype(np.int8)

    def seed(self, seed=None):
        self._rng = np.random.RandomState(seed)

    def sample(self):
        return (getattr(self, "_rng", None) or np.random).randint(2, size=self.n).astype(self.dtype)

    def contains(self, x):
        x = np.asarray(x)
        return x.shape == self.shape and bool(np.all((x == 0) | (x == 1)))

    def __repr__(self):
        return f"MultiBinary({self.n})"


class Dict:
    """gym.spaces.Dict: a mapping of named spaces (goal environments: observation / achieved_goal / desired_goal)."""

    def __init__(self, spaces):
        from collections import OrderedDict
        items = spaces.items() if isinstance(spaces, dict) else spaces
        self.spaces = OrderedDict(sorted(items) if isinstance(spaces, dict) and
                                  not isinstance(spaces, OrderedDict) else items)
        self.shape, self.dtype = None, None

    def seed(self, seed=None):
        for s in self.spaces.values():
            s.seed(seed)

    def sample(self):
        from collections import OrderedDict
        return OrderedDict((k, s.sample()) for k, s in self.spaces.items())

    def contains(self, x):
        return isinstance(x, dict) and x.keys() == self.spaces.keys() and \
            all(s.contains(x[k]) for k, s in self.spaces.items())

    def __getitem__(self, key):
        return self.spaces[key]

    def __repr__(self):
        return "Dict(" + ", ".join(f"{k}:{s}" for k, s in self.spaces.items()) + ")"


def is_discrete(space):
    """Discrete: `.n` and a scalar shape (gym's MultiBinary also has `.n`, with shape (n,))."""
    return hasattr(space, "n") and not hasattr(space, "nvec") and tuple(getattr(space, "shape", ())) == ()


def is_multi_discrete(space):
    return hasattr(space, "nvec")


def is_multi_binary(space):
    return hasattr(space, "n") and not hasattr(space, "nvec") and tuple(getattr(space, "shape", ())) == (int(space.n),)


def is_box(space):
    return hasattr(space, "low") and hasattr(space, "high")


def is_dict(space):
    return hasattr(space, "spaces") and isinstance(space.spaces, dict)
