"""ACER host logic against the reference's own outputs (tests/golden/acer_*.npz, tools/gen_acer_golden.py): the
stacking rule of _stack_obs, and Runner.run -- the segment it stores, and the stacked observations it trains from."""
import numpy as np
import pytest

import _acer_golden as G
import _acer_refs as AR
from baselines_b200.acer.runner import Runner
from baselines_b200.common.vec_env import VecFrameStack


@pytest.mark.parametrize("case", G.CASES, ids=[c[0] for c in G.CASES])
def test_stack_rule_is_the_references(case):
    name, nenv, nsteps = case[:3]
    g = G.load("buffer")
    for i in range(9):
        enc, _, _, _, dones, _ = G.segment(g, name, i)
        want = g[f"{name}/seg{i}/stacked"]
        got = AR.stack_obs(enc, dones, nsteps)
        assert got.dtype == want.dtype and got.tobytes() == want.tobytes()


@pytest.mark.parametrize("case", G.CASES, ids=[c[0] for c in G.CASES])
def test_runner_segments_are_the_references(case):
    """Two Runner.run() calls over this package's VecFrameStack: the stored frames, actions, rewards, mus, dones
    (shifted by one) and masks (with the initial dones) equal the reference runner's, and the stacked observations
    the on-policy call trains from -- the runner's own stacks, or the re-stacked frames -- equal its mb_obs."""
    name, nenv, nsteps, frame, nc, nstack, dtype = case
    g = G.load("runner")
    s = lambda k: g[f"{name}/script/{k}"]
    env = VecFrameStack(G.ScriptedEnv(s("frames"), s("rewards"), s("dones"), G.NA), nstack)
    r = Runner(env, G.ScriptedModel(s("actions"), s("mus"), "cpu"), nsteps)
    for c in range(2):
        rew, dones = r.run()
        w = lambda k: g[f"{name}/run{c}/{k}"]
        seg = r.seg
        assert seg.enc_obs[0].numpy().tobytes() == w("enc").tobytes()
        assert np.array_equal(seg.actions[0].numpy(), w("act"))
        assert seg.rewards[0].numpy().tobytes() == w("rew").tobytes() and rew.tobytes() == w("rew").tobytes()
        assert seg.mus[0].numpy().tobytes() == w("mus").tobytes()
        assert np.array_equal(seg.dones[0].numpy().astype(bool), w("dones")) and np.array_equal(dones, w("dones"))
        assert np.array_equal(seg.masks[0].numpy().astype(bool), w("masks"))
        if r.mb_obs is not None:
            assert r.mb_obs.numpy().tobytes() == w("obs").tobytes()
        else:
            assert AR.stack_obs(w("enc"), w("dones"), nsteps).tobytes() == w("obs").tobytes()
        assert (r.mb_obs is not None) == (nc > 1 and nstack > 1)
