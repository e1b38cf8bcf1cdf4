"""Generate tests/golden/ddpg_*.npz by EXECUTING the reference's pure-numpy DDPG modules: baselines/ddpg/memory.py
(Memory / RingBuffer sampling across a wrap of a small ring) and baselines/ddpg/noise.py (Ornstein-Uhlenbeck and normal
action noise, AdaptiveParamNoiseSpec.adapt).  Both are loaded by file path (baselines/ddpg/__init__.py is empty, but the
package's siblings import TensorFlow).

    python tools/gen_ddpg_golden.py /path/to/openai/baselines

The fixtures are committed; the tests never read the reference.
"""
import importlib.util
import os
import sys

import numpy as np

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def _load(ref, name):
    spec = importlib.util.spec_from_file_location(f"_ref_ddpg_{name}", os.path.join(ref, "baselines", "ddpg", f"{name}.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main(ref):
    memory, noise = _load(ref, "memory"), _load(ref, "noise")
    # memory: a ring of 10 rows, 27 appends (it wraps twice), samples of 16 from a seeded stream
    rng = np.random.RandomState(0)
    obs0, acts = rng.randn(27, 3).astype(np.float32), rng.uniform(-1, 1, (27, 2)).astype(np.float32)
    rews, terms, obs1 = rng.randn(27).astype(np.float32), (rng.rand(27) < 0.3).astype(np.float32), \
        rng.randn(27, 3).astype(np.float32)
    m = memory.Memory(limit=10, action_shape=(2,), observation_shape=(3,))
    out = {"obs0": obs0, "actions": acts, "rewards": rews, "terminals1": terms, "obs1": obs1}
    k = 0
    for n in (12, 27):                                  # after 12 appends the ring has wrapped once, after 27 twice
        while k < n:
            m.append(obs0[k], acts[k], rews[k], obs1[k], terms[k])
            k += 1
        np.random.seed(n)
        b = m.sample(batch_size=16)
        out.update({f"n{n}_start": m.observations0.start, f"n{n}_length": m.observations0.length})
        out.update({f"n{n}_{key}": v for key, v in b.items()})
    np.savez(os.path.join(OUT, "ddpg_memory.npz"), **out)
    # noise: 50 draws of each from seeded streams, with a reset after 20 for OU
    np.random.seed(1)
    ou = noise.OrnsteinUhlenbeckActionNoise(mu=np.zeros(3), sigma=0.2 * np.ones(3))
    ou_seq = [ou() for _ in range(20)]
    ou.reset()
    ou_seq += [ou() for _ in range(30)]
    np.random.seed(2)
    nn = noise.NormalActionNoise(mu=np.zeros(3), sigma=0.1 * np.ones(3))
    normal_seq = [nn() for _ in range(50)]
    spec = noise.AdaptiveParamNoiseSpec(initial_stddev=0.2, desired_action_stddev=0.2)
    dists = np.random.RandomState(3).uniform(0, 0.4, 200)
    trace = []
    for d in dists:
        spec.adapt(d)
        trace.append(spec.current_stddev)
    np.savez(os.path.join(OUT, "ddpg_noise.npz"), ou=np.array(ou_seq), normal=np.array(normal_seq), dists=dists,
             adapt=np.array(trace))


if __name__ == "__main__":
    if len(sys.argv) != 2:
        raise SystemExit("usage: python tools/gen_ddpg_golden.py /path/to/openai/baselines")
    main(sys.argv[1])
