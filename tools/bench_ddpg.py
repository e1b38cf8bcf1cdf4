"""DDPG timings on one GPU: the train iteration (train + update_target_net, graph replay) at B = 64, 256 and 1024 for a
HalfCheetah shape (obs 17, act 6) and a Humanoid shape (obs 376, act 17), mlp 64x64 with layer norm; the acting call
at nenvs 1 and 16; adapt_param_noise; and, for comparison, the same train iteration at B = 64 as torch-CPU float32
autograd (tests/_ddpg_refs.py's mirror in float32).  CUDA events around each window, median of 20 windows after
warm-up.  Prints one JSON line with the card's name and power limit.

    python tools/bench_ddpg.py [--windows 20] [--iters 50]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl = [s.strip() for s in out.split(",")]
        return name, pl
    except Exception:                                   # noqa: BLE001
        return torch.cuda.get_device_name(0), "unknown"


def _agent(ob, nA, B, param_noise=True):
    from baselines_b200.ddpg.ddpg_learner import DDPG
    from baselines_b200.ddpg.memory import Memory
    from baselines_b200.ddpg.models import Actor, Critic
    from baselines_b200.ddpg.noise import AdaptiveParamNoiseSpec
    np.random.seed(0)
    kw = dict(num_layers=2, num_hidden=64, layer_norm=True)
    mem = Memory(100000, (nA,), (ob,))
    agent = DDPG(Actor(nA, **kw), Critic(**kw), mem, (ob,), (nA,), gamma=0.99, tau=0.01, batch_size=B,
                 critic_l2_reg=1e-2, param_noise=AdaptiveParamNoiseSpec(0.2, 0.2) if param_noise else None, seed=0)
    agent.initialize()
    rng = np.random.RandomState(1)
    for _ in range(20):
        o = rng.randn(100, ob).astype(np.float32)
        agent.store_transition(o, rng.uniform(-1, 1, (100, nA)), rng.randn(100), o, np.zeros(100))
    return agent


def _time(fn, windows, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(windows):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1) * 1000.0 / iters)
    return float(np.median(ms))


def _cpu_oracle_us(ob, nA, B, reps=20):
    import _ddpg_refs as R
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    rng = np.random.RandomState(0)
    P = {}
    for sc in ("actor", "critic", "target_actor", "target_critic"):
        nin = ob + (nA if "critic" in sc else 0)
        for i in range(2):
            P[f"{sc}/mlp_fc{i}/w:0"], P[f"{sc}/mlp_fc{i}/b:0"] = rng.randn(nin, 64) * 0.1, np.zeros(64)
            P[f"{sc}/{R.ln_scope(i)}/beta:0"], P[f"{sc}/{R.ln_scope(i)}/gamma:0"] = np.zeros(64), np.ones(64)
            nin = 64
        h = "dense" if "actor" in sc else "output"
        P[f"{sc}/{h}/kernel:0"] = rng.randn(64, nA if "actor" in sc else 1) * 3e-3
        P[f"{sc}/{h}/bias:0"] = np.zeros(nA if "actor" in sc else 1)
    batch = dict(obs0=rng.randn(B, ob), obs1=rng.randn(B, ob), actions=rng.uniform(-1, 1, (B, nA)),
                 rewards=rng.randn(B), terminals1=np.zeros(B))
    cfg = dict(num_layers=2, layer_norm=True, gamma=0.99, normalize_returns=False, popart=False, critic_l2_reg=1e-2)
    old = R._t
    R._t = lambda a: torch.tensor(np.asarray(a, np.float32), dtype=torch.float32)   # the fp32 arm
    try:
        R.train_step(P, batch, cfg)
        t0 = time.perf_counter()
        for _ in range(reps):
            R.train_step(P, batch, cfg)
        return (time.perf_counter() - t0) * 1e6 / reps
    finally:
        R._t = old


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=20)
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ddpg needs a CUDA device")
    from baselines_b200 import build_ext
    build_ext.build()
    name, pl = _card()
    res = {"card": name, "power_limit": pl, "train_iter_us": {}, "act_us": {}, "adapt_us": {}}
    for shape, (ob, nA) in (("halfcheetah", (17, 6)), ("humanoid", (376, 17))):
        for B in (64, 256, 1024):
            ag = _agent(ob, nA, B)
            idxs = ag.memory.sample_indices(B)

            def it():
                ag.train_device(idxs)
                ag.update_target_net()
            res["train_iter_us"][f"{shape}_B{B}"] = round(_time(it, a.windows, a.iters), 1)
            if B == 64:
                res["adapt_us"][shape] = round(_time(lambda: ag.adapt_param_noise_device(idxs), a.windows, a.iters), 1)
                for n in (1, 16):
                    obs = np.random.RandomState(n).randn(n, ob).astype(np.float32)
                    res["act_us"][f"{shape}_n{n}"] = round(_time(lambda: ag.step(obs), a.windows, 10), 1)
        res.setdefault("cpu_fp32_train_us", {})[f"{shape}_B64"] = round(_cpu_oracle_us(ob, nA, 64), 1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
