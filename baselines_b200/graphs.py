"""CUDA-graph replay of fixed launch sequences.

One PPO2 minibatch is ~120 C-ABI calls, one acting pass 7, one deepq train step ~90; each call costs tens of
microseconds of host time (argument marshalling through ctypes), which exceeds the kernels' own duration for the
small networks (cfg-3 mlp, cfg-4 batch 512) and for the 4096-sample acting passes.  A sequence whose pointers and
shapes do not change is therefore captured once with torch.cuda.graph and replayed; everything that does change
between replays (Adam step size, clip range, sampler stream position, minibatch indices) lives in device memory
(ops.set_scalars / ops.counter_add / fixed index buffers), so a replay computes exactly what the eager sequence would.

B200RL_NO_GRAPHS=1 disables replay (every call runs eagerly) -- used by tests to check both paths agree.
"""
import gc
import os

import torch

from . import _lib


def enabled():
    return os.environ.get("B200RL_NO_GRAPHS", "0") != "1"


class GraphCache:
    """key -> captured graph.  The first call with a key runs eagerly (it also performs one-time work such as
    cudaFuncSetAttribute inside the library); the second call captures and replays; later calls replay."""

    def __init__(self, max_graphs=1024):
        self.graphs = {}          # key -> (graph, number of library kernels launches captured in it)
        self.seen = set()
        self.max_graphs = max_graphs
        self.homes = {}

    def home(self, name, rows, trailing, dtype, device):
        """The fixed buffer `name` with at least `rows` rows of shape `trailing`: captured graphs read it, each call
        refills it.  Its leading dimension may grow; its trailing shape and dtype are fixed.  A request that does not
        fit allocates it anew at exactly that size; replacing an earlier buffer drops every graph and the seen set,
        since a graph captured over the old buffer would otherwise replay reading freed memory."""
        buf = self.homes.get(name)
        if buf is None or buf.shape[0] < rows or buf.shape[1:] != tuple(trailing) or buf.dtype != dtype:
            if buf is not None:
                self.clear()
            buf = self.homes[name] = torch.zeros((rows,) + tuple(trailing), dtype=dtype, device=device)
        return buf

    def run(self, key, fn, allow_fallback=False):
        if not enabled() or _lib._prof is not None:            # per-call profiling needs the eager sequence
            fn()
            return
        ent = self.graphs.get(key)
        if ent is None:
            if key not in self.seen or len(self.graphs) >= self.max_graphs:
                if len(self.seen) < 65536:
                    self.seen.add(key)
                fn()
                return
            g = torch.cuda.CUDAGraph()
            before = _lib.LAUNCHES
            # torch.cuda.graph collects garbage before the capture begins; a collection DURING the capture could free a
            # pinned host buffer of a dead object, whose release makes a CUDA call that invalidates the capture
            gc_on = gc.isenabled()
            gc.disable()
            try:
                with torch.cuda.graph(g):
                    fn()
            except Exception as ex:                              # noqa: BLE001 -- e.g. a collective that cannot be captured
                if not allow_fallback:
                    raise
                import warnings
                warnings.warn(f"CUDA-graph capture of {key[0]!r} failed ({ex!r}); this sequence stays eager")
                torch.cuda.synchronize()
                self.seen.discard(key)
                self.max_graphs = 0                              # stop capturing in this cache
                _lib.LAUNCHES = before
                fn()
                return
            finally:
                if gc_on:
                    gc.enable()
            ent = self.graphs[key] = (g, _lib.LAUNCHES - before)
            _lib.LAUNCHES = before                               # nothing ran during capture
        ent[0].replay()
        _lib.LAUNCHES += ent[1]                                  # kernels executed by the replay
        _lib.REPLAYS += 1

    def clear(self):
        self.graphs.clear()
        self.seen.clear()
