"""ACER's device replay against the reference's own outputs (tests/golden/acer_*.npz): Buffer put / get before and
after the ring wraps, the slots a learn-shaped sequence draws and numpy's stream after it, acer_stack_obs on every
segment, and the on-policy batch re-stacked from the device segment of a Runner."""
import numpy as np
import pytest
import torch

import _acer_golden as G
from baselines_b200 import ops
from baselines_b200.acer.buffer import Buffer
from baselines_b200.acer.runner import Runner
from baselines_b200.common.vec_env import VecFrameStack

pytestmark = pytest.mark.gpu
IDS = [c[0] for c in G.CASES]


def _same(got, want):
    got = got.cpu().numpy() if torch.is_tensor(got) else got
    if want.dtype == bool:
        got = got.astype(bool)
    assert got.shape == want.shape and got.dtype == want.dtype and got.tobytes() == want.tobytes()


@pytest.mark.parametrize("case", G.CASES, ids=IDS)
def test_buffer_put_get_through_the_wrap(case):
    name, nenv, nsteps, frame, nc, nstack, dtype = case
    g = G.load("buffer")
    b = Buffer(G.BufferEnv(frame, nc, nstack, dtype, nenv), nsteps, size=nsteps * 5)
    assert b.size == 5
    np.random.seed(11)
    j = 0
    for i in range(9):
        b.put(*G.segment(g, name, i))
        if i in (2, 7):
            assert int(g[f"{name}/get{j}/after_put"]) == i
            assert b.num_in_buffer == min(5, i + 1) and b.can_sample()
            for got, k in zip(b.get(), ("obs", "act", "rew", "mus", "dones", "masks")):
                _same(got, g[f"{name}/get{j}/{k}"])
            j += 1
    assert np.array_equal(np.random.rand(4), g[f"{name}/stream_after_get"])


@pytest.mark.parametrize("case", G.CASES, ids=IDS)
def test_learn_shaped_draws_and_stream(case):
    name, nenv, nsteps, frame, nc, nstack, dtype = case
    g = G.load("buffer")
    b = Buffer(G.BufferEnv(frame, nc, nstack, dtype, nenv), nsteps, size=nsteps * 5)
    np.random.seed(12)
    calls = []
    for i in range(9):
        b.put(*G.segment(g, name, i))
        if b.has_atleast(2 * nsteps):
            for _ in range(np.random.poisson(4)):
                calls.append((i, b.get()[1].cpu().numpy()))
    assert np.array_equal([c[0] for c in calls], g[f"{name}/learn/after_put"])
    assert np.array_equal(np.array([c[1] for c in calls]), g[f"{name}/learn/actions"])
    assert np.array_equal(np.random.rand(4), g[f"{name}/stream_after_learn"])


@pytest.mark.parametrize("case", G.CASES, ids=IDS)
def test_stack_kernel_on_every_segment(case):
    name, nenv, nsteps, frame, nc, nstack, dtype = case
    g = G.load("buffer")
    for i in range(9):
        enc, _, _, _, dones, _ = G.segment(g, name, i)
        want = g[f"{name}/seg{i}/stacked"]
        ring = torch.from_numpy(enc[None]).cuda()
        d = torch.from_numpy(dones[None].astype(np.uint8)).cuda()
        out = torch.zeros((nenv * (nsteps + 1),) + want.shape[2:], dtype=ring.dtype, device="cuda")
        ops.acer_stack_obs(ring, None, nenv, nsteps, nstack, d, out)
        assert out.cpu().numpy().tobytes() == want.tobytes()


@pytest.mark.parametrize("case", G.CASES, ids=IDS)
def test_runner_on_policy_batch_on_the_device(case):
    name, nenv, nsteps, frame, nc, nstack, dtype = case
    g = G.load("runner")
    s = lambda k: g[f"{name}/script/{k}"]
    env = VecFrameStack(G.ScriptedEnv(s("frames"), s("rewards"), s("dones"), G.NA), nstack)
    r = Runner(env, G.ScriptedModel(s("actions"), s("mus"), "cuda"), nsteps)
    for c in range(2):
        r.run()
        want = g[f"{name}/run{c}/obs"]
        if r.mb_obs is not None:
            got = r.mb_obs
        else:
            got = torch.zeros((nenv * (nsteps + 1),) + want.shape[2:], dtype=r.seg.enc_obs.dtype, device="cuda")
            ops.acer_stack_obs(r.seg.enc_obs, None, nenv, nsteps, nstack, r.seg.dones, got)
        assert got.cpu().numpy().tobytes() == want.tobytes()
