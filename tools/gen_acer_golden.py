"""Generate tests/golden/acer_*.npz by EXECUTING the reference's numpy-only ACER host code: baselines/acer/buffer.py
(Buffer put / get through a ring wrap, `_stack_obs`) and baselines/acer/runner.py (Runner.run over the reference's own
common/runners.py and common/vec_env/vec_frame_stack.py).  gym.spaces is replaced by this package's spaces module and
VecEnv / VecEnvWrapper by minimal stand-ins with the reference's step protocol; the model and the environment are
scripted from arrays stored in the fixtures, so the tests can replay them.

    python tools/gen_acer_golden.py /path/to/openai/baselines

The fixtures are committed; the tests never read the reference.
"""
import importlib.util
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, ROOT)

from baselines_b200.common import spaces  # noqa: E402


def _stub(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    m.__path__ = []
    sys.modules[name] = m
    return m


class VecEnv:
    def __init__(self, num_envs, observation_space, action_space):
        self.num_envs, self.observation_space, self.action_space = num_envs, observation_space, action_space

    def step(self, actions):
        self.step_async(actions)
        return self.step_wait()


class VecEnvWrapper(VecEnv):
    def __init__(self, venv, observation_space=None, action_space=None):
        self.venv = venv
        super().__init__(venv.num_envs, observation_space or venv.observation_space,
                         action_space or venv.action_space)

    def step_async(self, actions):
        self.venv.step_async(actions)


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


def load_reference(ref):
    _stub("gym", spaces=spaces)
    sys.modules["gym.spaces"] = spaces
    for p in ("baselines", "baselines.common", "baselines.common.vec_env", "baselines.acer"):
        _stub(p)
    _stub("baselines.common.vec_env.vec_env", VecEnv=VecEnv, VecEnvWrapper=VecEnvWrapper)
    b = os.path.join(ref, "baselines")
    fs = _load("baselines.common.vec_env.vec_frame_stack", os.path.join(b, "common", "vec_env", "vec_frame_stack.py"))
    _load("baselines.common.runners", os.path.join(b, "common", "runners.py"))
    buf = _load("baselines.acer.buffer", os.path.join(b, "acer", "buffer.py"))
    run = _load("baselines.acer.runner", os.path.join(b, "acer", "runner.py"))
    return fs, buf, run


class ScriptedEnv(VecEnv):
    """Frames, rewards and dones from arrays: reset() returns frames[0], step k returns frames[k + 1]."""

    def __init__(self, frames, rewards, dones, nA):
        n = frames.shape[1]
        lo, hi = (0, 255) if frames.dtype == np.uint8 else (-10.0, 10.0)
        super().__init__(n, spaces.Box(lo, hi, frames.shape[2:], frames.dtype), spaces.Discrete(nA))
        self.frames, self.rewards, self.dones, self.k = frames, rewards, dones, 0

    def reset(self):
        return self.frames[0].copy()

    def step_async(self, actions):
        self.actions = actions

    def step_wait(self):
        k = self.k
        self.k += 1
        return self.frames[k + 1].copy(), self.rewards[k].copy(), self.dones[k].copy(), [{} for _ in range(self.num_envs)]


class ScriptedModel:
    """_step returns actions[k] and mus[k] on call k, whatever the observation."""

    def __init__(self, actions, mus):
        self.actions, self.mus, self.k, self.initial_state = actions, mus, 0, None

    def _step(self, obs, S=None, M=None):
        k = self.k
        self.k += 1
        return self.actions[k].copy(), self.mus[k].copy(), None


def frames_of(rng, shape, dtype):
    if dtype == np.uint8:
        return rng.randint(0, 256, shape).astype(np.uint8)
    return (rng.randn(*shape) * 3).astype(np.float32)


class _Env:
    def __init__(self, ob_shape, dtype, nA, nenv, nstack):
        self.observation_space = spaces.Box(0, 255, ob_shape, dtype)
        self.action_space = spaces.Discrete(nA)
        self.num_envs, self.nstack = nenv, nstack


# (name, nenv, nsteps, frame, nc, nstack, dtype)
CASES = [("u8_s4", 3, 5, (4, 3), 1, 4, np.uint8), ("f32_s1", 2, 6, (), 4, 1, np.float32),
         ("f32_s4c2", 2, 4, (3,), 2, 4, np.float32), ("u8_s1", 2, 3, (2, 2), 3, 1, np.uint8)]


def segments(rng, n, nenv, nsteps, frame, nc, nstack, dtype, nA):
    out = []
    for _ in range(n):
        d = rng.rand(nenv, nsteps) < 0.3
        d[0, 0] = d[-1, -1] = True
        m = np.concatenate([rng.rand(nenv, 1) < 0.3, d], axis=1)
        out.append((frames_of(rng, (nenv, nsteps + nstack) + frame + (nc,), dtype),
                    rng.randint(0, nA, (nenv, nsteps)).astype(np.int64), rng.randn(nenv, nsteps).astype(np.float32),
                    rng.dirichlet(np.ones(nA), (nenv, nsteps)).astype(np.float32), d, m))
    return out


def gen_buffer(buf):
    """Buffer put / get before and after the ring wraps (num_in_buffer < size, then = size), a learn-shaped sequence
    of has_atleast / poisson / get, and _stack_obs on each segment; the numpy stream after each phase."""
    out = {}
    for name, nenv, nsteps, frame, nc, nstack, dtype in CASES:
        rng = np.random.RandomState(len(name) + nenv)
        nA = 5
        env = _Env(frame + (nc * nstack,), dtype, nA, nenv, nstack)
        segs = segments(rng, 9, nenv, nsteps, frame, nc, nstack, dtype, nA)
        for i, s in enumerate(segs):
            for k, a in zip(("enc", "act", "rew", "mus", "dones", "masks"), s):
                out[f"{name}/seg{i}/{k}"] = a
            out[f"{name}/seg{i}/stacked"] = buf._stack_obs(s[0], s[4], nsteps)
        b = buf.Buffer(env, nsteps, size=nsteps * 5)             # 5 slots
        np.random.seed(11)
        gets = []
        for i, s in enumerate(segs):
            b.put(*s)
            if i in (2, 7):                                        # 3 slots of 5 filled; after the wrap
                gets.append((i, b.get()))
        for j, (i, g) in enumerate(gets):
            for k, a in zip(("obs", "act", "rew", "mus", "dones", "masks"), g):
                out[f"{name}/get{j}/{k}"] = a
            out[f"{name}/get{j}/after_put"] = np.int64(i)
        out[f"{name}/stream_after_get"] = np.random.rand(4)
        # learn-shaped: one put per on-policy call, then poisson(replay_ratio) gets once has_atleast(replay_start)
        b = buf.Buffer(env, nsteps, size=nsteps * 5)
        np.random.seed(12)
        calls = []
        for i, s in enumerate(segs):
            b.put(*s)
            if b.has_atleast(2 * nsteps):
                n = np.random.poisson(4)
                for _ in range(n):
                    calls.append((i, b.get()[1]))
        out[f"{name}/learn/after_put"] = np.array([c[0] for c in calls], np.int64)
        out[f"{name}/learn/actions"] = np.array([c[1] for c in calls])
        out[f"{name}/stream_after_learn"] = np.random.rand(4)
    np.savez(os.path.join(OUT, "acer_buffer.npz"), **out)


def gen_runner(fs, run):
    """Two Runner.run() calls of the reference over its own VecFrameStack."""
    out = {}
    for name, nenv, nsteps, frame, nc, nstack, dtype in CASES:
        rng = np.random.RandomState(100 + len(name))
        nA = 5
        K = 2 * nsteps
        frames = frames_of(rng, (K + 1, nenv) + frame + (nc,), dtype)
        rewards = rng.randn(K, nenv).astype(np.float32)
        dones = rng.rand(K, nenv) < 0.25
        dones[0, 0] = dones[nsteps - 1, -1] = dones[nsteps, 0] = True
        actions = rng.randint(0, nA, (K, nenv)).astype(np.int64)
        mus = rng.dirichlet(np.ones(nA), (K, nenv)).astype(np.float32)
        for k, a in (("frames", frames), ("rewards", rewards), ("dones", dones), ("actions", actions), ("mus", mus)):
            out[f"{name}/script/{k}"] = a
        env = fs.VecFrameStack(ScriptedEnv(frames, rewards, dones, nA), nstack)
        r = run.Runner(env=env, model=ScriptedModel(actions, mus), nsteps=nsteps)
        for c in range(2):
            res = r.run()
            for k, a in zip(("enc", "obs", "act", "rew", "mus", "dones", "masks"), res):
                out[f"{name}/run{c}/{k}"] = a
    np.savez(os.path.join(OUT, "acer_runner.npz"), **out)


def main(ref):
    fs, buf, run = load_reference(ref)
    gen_buffer(buf)
    gen_runner(fs, run)
    print("wrote tests/golden/acer_{buffer,runner}.npz")


if __name__ == "__main__":
    main(sys.argv[1])
