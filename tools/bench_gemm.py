#!/usr/bin/env python
"""Stand-alone timing of every plain wgmma GEMM launch (b200rl_gemm_f16, csrc/gemm_wgmma.cu) of the benchmark's PPO2
workloads: one cfg-2 NatureCNN training minibatch (B = 131072: fc1 forward, data and weight gradient, the head GEMMs)
and one acting pass (B = 4096), and one cfg-3 mlp training minibatch (B = 262144).

Each launch is timed where the model issues it, on the model's own buffers: CUDA events around the launch, median of
10 after 3 warm-ups, with an L2 flush (write of a 512 MB buffer) before each timed launch, as in
tools/bench_conv_shift.py.  Flops and bytes are the algorithmic ones ops.gemm reports; the output gives each launch's
share of the HBM and of the tensor roofline (H100 SXM data sheet: 3350 GB/s, 989 dense fp16 TFLOP/s -- a card with a
lower power limit or clock reaches less), and the card's name, power limit and SM clock.

    python tools/bench_gemm.py                                 # the library in this tree; prints one JSON object
    python tools/bench_gemm.py --compare A.so B.so --rounds 5  # two builds of libb200rl.so, alternating per launch

--compare times every launch on both libraries in turn (A, B, A, B, ...; --rounds of each), in one process on the
same inputs.  The model itself runs on the library of this tree; both builds must export the same C-ABI.
A weight-gradient launch accumulates into its gradient, so the replays change the model's gradients: the tool
measures time only.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

os.environ["B200RL_NO_GRAPHS"] = "1"            # eager launches: each one is intercepted and timed where it runs
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_GBS, TENSOR_TFLOPS = 3350.0, 989.0
NAME = "b200rl_gemm_f16"


def _load(path):
    from baselines_b200 import _lib
    lib = C.CDLL(os.path.abspath(path))
    lib.b200rl_last_error.restype = C.c_char_p
    fn = getattr(lib, NAME)
    fn.argtypes = _lib.SIGNATURES[NAME]
    fn.restype = C.c_int
    return lib


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else None
    except (OSError, subprocess.SubprocessError):
        return None


def _sm_clock():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return float(q[0]) if q else None
    except (OSError, subprocess.SubprocessError, ValueError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--compare", nargs=2, metavar=("LIB_A", "LIB_B"), default=None)
    ap.add_argument("--rounds", type=int, default=3, help="--compare: timed rounds per library, alternating")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--configs", default="cfg2,cfg3")
    args = ap.parse_args()

    import torch
    import __graft_entry__
    __graft_entry__.build()
    from baselines_b200 import _lib
    from baselines_b200.common import spaces
    from baselines_b200.common.policies import build_policy
    from baselines_b200.ppo2.model import Model
    assert torch.cuda.is_available(), "bench_gemm times GPU kernels: it needs a GPU"

    libs = [(p, _load(p)) for p in args.compare] if args.compare else [("tree", _lib.load())]
    flush = torch.empty(128 << 20, dtype=torch.float32, device="cuda")
    phase = {"tag": ""}
    results, clocks = [], []
    orig_call = _lib.call

    def time_on(lib, call_args):
        fn = getattr(lib, NAME)
        for _ in range(args.warmup):
            fn(*call_args)
        ts = []
        for _ in range(args.iters):
            flush.fill_(1.0)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            rc = fn(*call_args)
            e1.record()
            torch.cuda.synchronize()
            if rc != 0:
                raise RuntimeError(f"{NAME} failed (rc={rc}): {lib.b200rl_last_error().decode()}")
            ts.append(e0.elapsed_time(e1))
        return float(np.median(ts))

    def call(name, *call_args, label=None, flops=0, nbytes=0):
        if name != NAME:
            return orig_call(name, *call_args, label=label, flops=flops, nbytes=nbytes)
        torch.cuda.synchronize()
        ms = {p: [] for p, _ in libs}
        for _ in range(args.rounds if args.compare else 1):
            for p, lib in libs:
                ms[p].append(time_on(lib, call_args))
        clk = _sm_clock()
        if clk:
            clocks.append(clk)
        M, N, K = call_args[5], call_args[6], call_args[7]
        r = {"launch": (label or name) + phase["tag"], "M": M, "N": N, "K": K, "flops": flops, "bytes": nbytes}
        for p, v in ms.items():
            t = float(np.median(v))
            key = "" if not args.compare else ("A." if p == args.compare[0] else "B.")
            r[key + "ms"] = t
            if args.compare:
                r[key + "ms_rounds"] = v
            r[key + "tflops"] = flops / (t / 1e3) / 1e12
            r[key + "gbs"] = nbytes / (t / 1e3) / 1e9
            r[key + "frac_tensor"] = r[key + "tflops"] / TENSOR_TFLOPS
            r[key + "frac_hbm"] = r[key + "gbs"] / HBM_GBS
        if args.compare:
            r["B_over_A"] = r["B.ms"] / r["A.ms"]
        results.append(r)

    def run(tag, model, train_args, act_obs):
        model.train(*train_args)                       # warm every shape once
        if act_obs is not None:
            model.step(act_obs)
        torch.cuda.synchronize()
        _lib.call = call
        try:
            phase["tag"] = f"@{tag}.train"
            model.train(*train_args)
            if act_obs is not None:
                phase["tag"] = f"@{tag}.act"
                model.step(act_obs)
        finally:
            _lib.call = orig_call

    cfgs = args.configs.split(",")
    if "cfg2" in cfgs:
        class E2:
            observation_space = spaces.Box(0, 255, (84, 84, 4), np.uint8)
            action_space = spaces.Discrete(6)
            num_envs = 4096
        n_train, n_act = 131072, 4096
        np.random.seed(0)
        model = Model(policy=build_policy(E2, "cnn"), ob_space=E2.observation_space, ac_space=E2.action_space,
                      nbatch_act=n_act, nbatch_train=n_train, nsteps=n_train // n_act, ent_coef=0.01, vf_coef=0.5,
                      max_grad_norm=0.5, comm=False)
        rng = np.random.RandomState(0)
        obs = rng.randint(0, 256, (n_train, 84, 84, 4), dtype=np.uint8)
        values = rng.randn(n_train).astype(np.float32)
        run("cfg2", model, (2.5e-4, 0.1, obs, (values + rng.randn(n_train)).astype(np.float32), None,
                            rng.randint(0, 6, n_train), values, np.full(n_train, np.log(6), np.float32)), obs[:n_act])
        del model, obs
    if "cfg3" in cfgs:
        class E3:
            observation_space = spaces.Box(-np.inf, np.inf, (376,), np.float32)
            action_space = spaces.Box(-1.0, 1.0, (17,), np.float32)
            num_envs = 16384
        n_train = 262144
        np.random.seed(0)
        model = Model(policy=build_policy(E3, "mlp", value_network="copy"), ob_space=E3.observation_space,
                      ac_space=E3.action_space, nbatch_act=E3.num_envs, nbatch_train=n_train, nsteps=512,
                      ent_coef=0.0, vf_coef=0.5, max_grad_norm=0.5, comm=False, train_chunk=262144)
        rng = np.random.RandomState(0)
        obs = rng.randn(n_train, 376).astype(np.float32)
        values = rng.randn(n_train).astype(np.float32)
        run("cfg3", model, (3e-4, 0.2, obs, (values + rng.randn(n_train)).astype(np.float32), None,
                            rng.randn(n_train, 17).astype(np.float32), values,
                            np.full(n_train, 17 * 0.5 * np.log(2 * np.pi * np.e), np.float32)), None)
    out = {"device": torch.cuda.get_device_name(), "card": _card(),
           "sm_clock_mhz_median": float(np.median(clocks)) if clocks else None,
           "how": "CUDA events per launch, median of %d after %d warm-ups, 512 MB L2 flush before each"
                  % (args.iters, args.warmup),
           "peaks": {"hbm_gbs": HBM_GBS, "tensor_tflops": TENSOR_TFLOPS, "src": "H100 SXM data sheet"},
           "launches": results}
    if args.compare:
        out["libs"] = {"A": args.compare[0], "B": args.compare[1]}
        out["rounds"] = args.rounds
    print(json.dumps(out))


if __name__ == "__main__":
    main()
