"""Generate tests/golden/her_*.npz by EXECUTING the reference's HER modules: baselines/her/her_sampler.py (the
`future` and `none` samplers), replay_buffer.py (episode storage through wrap, overflow and full-ring replacement),
rollout.py (RolloutWorker) driven by ddpg.py's own get_actions, and ddpg.py's store_episode / sample_batch for a
learn-shaped sequence of numpy draws.  TensorFlow, mpi4py and the reference's logger / tf_util / mpi_adam are replaced
by import stubs: the code executed here is numpy only; the network is a fixed numpy function standing in for sess.run.

    python tools/gen_her_golden.py /path/to/openai/baselines

The fixtures are committed; the tests never read the reference.
"""
import importlib
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, ROOT)


def _stub(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


def _load_reference(ref):
    """baselines.her.* from the reference tree; everything it imports besides numpy is a stub."""
    class _Anything:
        def __init__(self, *a, **k):
            pass

        def __getattr__(self, name):
            return _Anything()

        def __call__(self, *a, **k):
            return _Anything()
    def _tf_attr(name):
        if name.startswith('__'):
            raise AttributeError(name)
        return _Anything()
    tf = _stub("tensorflow")
    tf.__getattr__ = _tf_attr
    contrib = _stub("tensorflow.contrib")
    staging = _stub("tensorflow.contrib.staging", StagingArea=_Anything)
    tf.contrib, contrib.staging = contrib, staging
    _stub("mpi4py", MPI=_Anything())
    quiet = lambda *a, **k: None
    baselines = _stub("baselines")
    baselines.__path__ = []
    logger = _stub("baselines.logger", info=quiet, warn=quiet, debug=quiet, log=quiet, record_tabular=quiet,
                   dump_tabular=quiet, get_dir=lambda: None)
    common = _stub("baselines.common")
    common.__path__ = []
    common.tf_util = _stub("baselines.common.tf_util", get_session=_Anything, numel=_Anything)
    common.mpi_adam = _stub("baselines.common.mpi_adam", MpiAdam=_Anything)
    her = _stub("baselines.her")
    her.__path__ = [os.path.join(ref, "baselines", "her")]
    baselines.logger, baselines.common, baselines.her = logger, common, her
    return {name: importlib.import_module(f"baselines.her.{name}")
            for name in ("her_sampler", "replay_buffer", "rollout", "ddpg")}


def reward_fun(ag_2, g, info):
    """gym robotics' sparse goal reward with threshold 0.1 (PointReach-v0's)."""
    return -(np.linalg.norm(ag_2 - g, axis=-1) > 0.1).astype(np.float32)


def episodes(rng, n, T, dimo=3, dimg=2, dimu=2):
    """A batch of n float32 episodes of T transitions, as RolloutWorker returns them."""
    return {'o': rng.randn(n, T + 1, dimo).astype(np.float32), 'ag': rng.randn(n, T + 1, dimg).astype(np.float32),
            'g': rng.randn(n, T, dimg).astype(np.float32), 'u': rng.uniform(-1, 1, (n, T, dimu)).astype(np.float32),
            'info_is_success': rng.randint(0, 2, (n, T, 1)).astype(np.float32)}


def policy_pi(o, g):
    """The fixed numpy network of the rollout fixture: pi = tanh(W [o | g]), Q = sum(pi)."""
    W = np.linspace(-1.5, 1.5, (o.shape[1] + g.shape[1]) * 2).reshape(-1, 2)
    return np.tanh(np.concatenate([o, g], 1) @ W).astype(np.float32)


def gen_sampler(mods):
    out = {}
    rng = np.random.RandomState(0)
    E, T, B = 6, 9, 200
    batch = episodes(rng, E, T)
    batch = {k: v.astype(np.float64) for k, v in batch.items()}
    out.update({f"batch_{k}": v for k, v in batch.items()})
    for strategy in ("future", "none"):
        sample = mods["her_sampler"].make_sample_her_transitions(strategy, 4, reward_fun)
        b = dict(batch)
        b['o_2'], b['ag_2'] = b['o'][:, 1:, :], b['ag'][:, 1:, :]
        np.random.seed(11)
        tr = sample(b, B)
        for k in ('o', 'o_2', 'ag', 'ag_2', 'g', 'u', 'r'):
            out[f"{strategy}_{k}"] = tr[k]
        out[f"{strategy}_after"] = np.random.uniform(size=4)
    np.savez(os.path.join(OUT, "her_sampler.npz"), **out)


def gen_storage(mods):
    """Episodes of batch 3 into a ring of 5: consecutive, then an overflow (one consecutive slot, two drawn), then
    full-ring replacement with repeated slots."""
    rng = np.random.RandomState(1)
    T, size, n_stores = 4, 5, 8
    shapes = {'o': (T + 1, 3), 'ag': (T + 1, 2), 'g': (T, 2), 'u': (T, 2), 'info_is_success': (T, 1)}
    buf = mods["replay_buffer"].ReplayBuffer(shapes, size * (T + 1), T + 1, None)
    slots, out = [], {}
    rec = buf._get_storage_idx
    buf._get_storage_idx = lambda inc=None: slots.append(np.atleast_1d(rec(inc)).copy()) or slots[-1]
    np.random.seed(21)
    repeated = False
    for k in range(n_stores):
        ep = episodes(rng, 3, T)
        buf.store_episode(ep)
        repeated |= len(set(slots[-1].tolist())) < 3
        for key, v in ep.items():
            out[f"ep{k}_{key}"] = v
        out[f"slots{k}"] = slots[-1]
        out[f"size{k}"] = np.int64(buf.current_size)
    assert repeated, "the fixture must store into a repeated slot"
    for key in shapes:
        out[f"buf_{key}"] = buf.buffers[key]
    out["after"] = np.random.uniform(size=4)
    np.savez(os.path.join(OUT, "her_storage.npz"), **out)


def _ref_agent(mods, dimo, dimg, dimu, T, batch_size=0, buffer=None, sample_transitions=None):
    """A reference her/ddpg.py DDPG whose host methods run as written; the TF pieces are a numpy function."""
    DDPG = mods["ddpg"].DDPG
    agent = DDPG.__new__(DDPG)

    class Net:
        pi_tf, Q_pi_tf, o_tf, g_tf, u_tf = "pi", "Q_pi", "o", "g", "u"

    class Sess:
        def run(self, vals, feed_dict):
            pi = policy_pi(feed_dict["o"], feed_dict["g"])
            return [pi if v == "pi" else pi.sum(axis=1, keepdims=True) for v in vals]

    class Stats:
        def update(self, v):
            pass

        def recompute_stats(self):
            pass
    agent.__dict__.update(dimo=dimo, dimg=dimg, dimu=dimu, max_u=1.0, relative_goals=False, clip_obs=200.,
                          subtract_goals=lambda a, b: a - b, main=Net(), target=Net(), sess=Sess(), bc_loss=0,
                          batch_size=batch_size, buffer=buffer, sample_transitions=sample_transitions,
                          o_stats=Stats(), g_stats=Stats(), T=T,
                          stage_shapes={k: None for k in ('ag', 'g', 'info_is_success', 'o', 'u', 'o_2', 'g_2', 'r')})
    return agent


def gen_rollout(mods):
    from baselines_b200 import envs
    from baselines_b200.common.vec_env import DummyVecEnv

    def make(i):
        def f():
            e = envs.make('PointReach-v0')
            e.seed(i)
            return e
        return f
    dims = {'o': 4, 'g': 2, 'u': 2, 'info_is_success': 1}
    agent = _ref_agent(mods, 4, 2, 2, 50)
    np.random.seed(31)
    w = mods["rollout"].RolloutWorker(DummyVecEnv([make(0), make(1)]), agent, dims, None, T=50, rollout_batch_size=2,
                                      noise_eps=0.2, random_eps=0.3)
    ev = mods["rollout"].RolloutWorker(DummyVecEnv([make(2), make(3)]), agent, dims, None, T=50, rollout_batch_size=2,
                                       exploit=True, compute_Q=True)
    out = {}
    for k in range(2):
        ep = w.generate_rollouts()
        for key, v in ep.items():
            out[f"train{k}_{key}"] = v
    ep = ev.generate_rollouts()
    for key, v in ep.items():
        out[f"eval_{key}"] = v
    out["train_success"] = np.array(w.success_history)
    out["eval_success"] = np.array(ev.success_history)
    out["eval_Q"] = np.array(ev.Q_history)
    out["after"] = np.random.uniform(size=4)
    np.savez(os.path.join(OUT, "her_rollout.npz"), **out)


def gen_stream(mods):
    """learn's per-cycle draws: store_episode (storage slots and the normaliser's sample over the new episodes), then
    n_batches sample_batch calls, over 6 cycles into a ring that fills after 4."""
    rng = np.random.RandomState(2)
    T, rbs, size, n_batches, B = 6, 2, 8, 3, 32
    sample = mods["her_sampler"].make_sample_her_transitions('future', 4, reward_fun)
    shapes = {'o': (T + 1, 3), 'ag': (T + 1, 2), 'g': (T, 2), 'u': (T, 2), 'info_is_success': (T, 1)}
    buf = mods["replay_buffer"].ReplayBuffer(shapes, size * (T + 1), T + 1, sample)
    agent = _ref_agent(mods, 3, 2, 2, T + 1, batch_size=B, buffer=buf, sample_transitions=sample)
    out = {}
    np.random.seed(41)
    for c in range(6):
        ep = episodes(rng, rbs, T)
        for key, v in ep.items():
            out[f"ep{c}_{key}"] = v
        agent.store_episode(ep)
        for k in range(n_batches):
            batch = agent.sample_batch()
            if k == 0:
                out[f"batch{c}_g"] = batch[1]      # stage_shapes order: ag, g, ...
                out[f"batch{c}_r"] = batch[-1]
        out[f"state{c}"] = np.random.get_state()[1].copy()
        out[f"pos{c}"] = np.int64(np.random.get_state()[2])
    np.savez(os.path.join(OUT, "her_stream.npz"), **out)


def main(ref):
    import baselines_b200.envs  # noqa: F401 -- the package (and torch) before the stubs
    import baselines_b200.common.vec_env  # noqa: F401
    mods = _load_reference(ref)
    gen_sampler(mods)
    gen_storage(mods)
    gen_rollout(mods)
    gen_stream(mods)
    print("wrote tests/golden/her_{sampler,storage,rollout,stream}.npz")


if __name__ == "__main__":
    main(sys.argv[1])
