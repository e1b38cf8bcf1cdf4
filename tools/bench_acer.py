"""Time ACER's device calls on the GPU and print one JSON line: the on-policy and replay train calls (re-stacking
included), the acting call, Buffer.put, and the re-stack kernel's bytes over its time against a measured
device-to-device copy bandwidth.  Shapes: the Atari cnn (84x84x4 uint8, 6 actions) at nenv 16 / 64 / 256 and the
CartPole mlp (4 floats, 2 actions, value_network='copy'), nsteps 20.

    python tools/bench_acer.py [--iters 50] [--nenvs 16,64,256]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from baselines_b200 import ops  # noqa: E402
from baselines_b200.acer import acer as A  # noqa: E402
from baselines_b200.acer.buffer import Buffer  # noqa: E402
from baselines_b200.common import spaces  # noqa: E402
from baselines_b200.common.policies import build_policy  # noqa: E402


class _Env:
    def __init__(self, ob, nA, n, nstack):
        self.observation_space, self.action_space, self.num_envs, self.nstack = ob, spaces.Discrete(nA), n, nstack


def _time(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1000.0 / iters        # microseconds per call


def case(kind, nenv, nsteps, iters):
    np.random.seed(0)
    if kind == "cnn":
        ob, nA, nstack, kw = spaces.Box(0, 255, (84, 84, 4), np.uint8), 6, 4, {}
    else:
        ob, nA, nstack, kw = spaces.Box(-1, 1, (4,), np.float32), 2, 1, dict(value_network="copy")
    env = _Env(ob, nA, nenv, nstack)
    model = A.Model(policy=build_policy(env, kind, estimate_q=True, **kw), ob_space=ob, ac_space=env.action_space,
                    nenvs=nenv, nsteps=nsteps, ent_coef=0.01, q_coef=0.5, gamma=0.99, max_grad_norm=10, lr=7e-4,
                    rprop_alpha=0.99, rprop_epsilon=1e-5, total_timesteps=int(1e7), lrschedule='constant', c=10.0,
                    trust_region=True, alpha=0.99, delta=1)
    buf = Buffer(env, nsteps, size=nsteps * 50, device=model.device)
    seg = buf.ring
    if kind == "cnn":
        seg.enc_obs.copy_(torch.randint(0, 256, seg.enc_obs.shape, dtype=torch.uint8))
    else:
        seg.enc_obs.normal_()
    seg.actions.random_(0, nA)
    seg.rewards.normal_()
    seg.mus.fill_(1.0 / nA)
    seg.dones.copy_((torch.rand(seg.dones.shape) < 0.02).to(torch.uint8))
    buf.num_in_buffer = buf.size
    one = [a[0] for a in seg.arrays()]
    r = dict(kind=kind, nenv=nenv, nsteps=nsteps)
    r["train_on_policy_us"] = _time(lambda: model.train_device(seg, None, 0, with_stats=False), iters)
    r["train_replay_us"] = _time(lambda: model.train_device(seg, buf.sample_slots(), 0, with_stats=False), iters)
    r["train_replay_with_stats_us"] = _time(lambda: model.train_device(seg, buf.sample_slots(), 0), iters)
    obs = (np.random.randint(0, 256, (nenv,) + ob.shape).astype(np.uint8) if kind == "cnn"
           else np.random.randn(nenv, *ob.shape).astype(np.float32))
    a = torch.zeros(nenv, dtype=torch.int64, device="cuda")
    mu = torch.zeros(nenv, nA, device="cuda")
    r["act_us"] = _time(lambda: model.step_device(obs, a, mu), iters)
    r["put_us"] = _time(lambda: buf.put(*one), iters)
    out = model.obs_buf
    idx = buf.sample_slots()
    r["stack_us"] = _time(lambda: ops.acer_stack_obs(seg.enc_obs, idx, nenv, nsteps, nstack, seg.dones, out), iters)
    # bytes the re-stack must move: the stacked rows written and the segments' frames read once
    nbytes = out.numel() * out.element_size() + nenv * (nsteps + nstack) * seg.enc_obs[0, 0, 0].numel() * \
        seg.enc_obs.element_size()
    r["stack_GBps"] = nbytes / (r["stack_us"] * 1e3)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--nenvs", default="16,64,256")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_acer needs a GPU"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    x = torch.empty(1 << 28, dtype=torch.uint8, device="cuda")
    y = torch.empty_like(x)
    copy_us = _time(lambda: y.copy_(x), 20)
    res = dict(gpu=q[0] if q else torch.cuda.get_device_name(), d2d_copy_GBps=2 * x.numel() / (copy_us * 1e3),
               cases=[case("cnn", int(n), 20, args.iters) for n in args.nenvs.split(",")] +
               [case("mlp", 1, 20, args.iters)])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
