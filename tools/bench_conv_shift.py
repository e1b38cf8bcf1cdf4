#!/usr/bin/env python
"""Stand-alone timing of every shift-GEMM convolution launch (csrc/conv_shift.cu) of the cfg-2 workload: one PPO2
NatureCNN training minibatch (B = 131072: forward of c1 from uint8, c2, c3; data gradient of c3, c2; weight gradient
of c3, c2, c1) and one acting pass (B = 4096: the three forwards).

Each launch is timed where the model issues it, on the model's own buffers: CUDA events around the launch, median of
10 after 3 warm-ups, with an L2 flush (write of a 512 MB buffer) before each timed launch, as in tools/microbench.py.
Flops and bytes are the algorithmic ones ops.conv_shift_* report; the output gives each launch's share of the HBM
and of the tensor roofline (H100 SXM data sheet: 3350 GB/s, 989 dense fp16 TFLOP/s -- a card with a lower power
limit or clock reaches less).

    python tools/bench_conv_shift.py                       # the library in this tree; prints one JSON object
    python tools/bench_conv_shift.py --compare A.so B.so   # two builds of libb200rl.so, alternating per launch

--compare times every launch on both libraries in turn (A, B, A, B, ...; --rounds of each), in one process on the
same inputs.  The model itself runs on the library of this tree; both builds must export the same C-ABI.
A weight-gradient launch accumulates into its gradient, so the replays change the model's gradients: the tool
measures time only.
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

os.environ["B200RL_NO_GRAPHS"] = "1"            # eager launches: each one is intercepted and timed where it runs
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_GBS, TENSOR_TFLOPS = 3350.0, 989.0


def _load(path):
    from baselines_b200 import _lib
    lib = C.CDLL(os.path.abspath(path))
    lib.b200rl_last_error.restype = C.c_char_p
    for name in ("b200rl_conv_shift_fwd", "b200rl_conv_shift_wgrad"):
        fn = getattr(lib, name)
        fn.argtypes = _lib.SIGNATURES[name]
        fn.restype = C.c_int
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--compare", nargs=2, metavar=("LIB_A", "LIB_B"), default=None)
    ap.add_argument("--rounds", type=int, default=3, help="--compare: timed rounds per library, alternating")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import torch
    import __graft_entry__
    __graft_entry__.build()
    from baselines_b200 import _lib
    from baselines_b200.common import spaces
    from baselines_b200.common.policies import build_policy
    from baselines_b200.ppo2.model import Model
    assert torch.cuda.is_available(), "bench_conv_shift times GPU kernels: it needs a GPU"

    libs = [(p, _load(p)) for p in args.compare] if args.compare else [("tree", _lib.load())]
    flush = torch.empty(128 << 20, dtype=torch.float32, device="cuda")
    phase = {"tag": ""}
    results = []
    orig_call = _lib.call

    def time_on(lib, name, call_args):
        fn = getattr(lib, name)
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
                raise RuntimeError(f"{name} failed (rc={rc}): {lib.b200rl_last_error().decode()}")
            ts.append(e0.elapsed_time(e1))
        return float(np.median(ts))

    def call(name, *call_args, label=None, flops=0, nbytes=0):
        if not name.startswith("b200rl_conv_shift"):
            return orig_call(name, *call_args, label=label, flops=flops, nbytes=nbytes)
        torch.cuda.synchronize()
        ms = {p: [] for p, _ in libs}
        for _ in range(args.rounds if args.compare else 1):
            for p, lib in libs:
                ms[p].append(time_on(lib, name, call_args))
        r = {"launch": (label or name) + phase["tag"], "flops": flops, "bytes": nbytes}
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

    class E:
        observation_space = spaces.Box(0, 255, (84, 84, 4), np.uint8)
        action_space = spaces.Discrete(6)
        num_envs = 4096

    n_train, n_act = 131072, 4096
    np.random.seed(0)
    model = Model(policy=build_policy(E, "cnn"), ob_space=E.observation_space, ac_space=E.action_space,
                  nbatch_act=n_act, nbatch_train=n_train, nsteps=n_train // n_act, ent_coef=0.01, vf_coef=0.5,
                  max_grad_norm=0.5, comm=False)
    rng = np.random.RandomState(0)
    obs = rng.randint(0, 256, (n_train, 84, 84, 4), dtype=np.uint8)
    actions = rng.randint(0, 6, n_train)
    values = rng.randn(n_train).astype(np.float32)
    returns = (values + rng.randn(n_train)).astype(np.float32)
    nlp = np.full(n_train, np.log(6), np.float32)
    model.train(2.5e-4, 0.1, obs, returns, None, actions, values, nlp)      # warm every shape once
    model.step(obs[:n_act])
    torch.cuda.synchronize()
    _lib.call = call
    try:
        phase["tag"] = "@train"
        model.train(2.5e-4, 0.1, obs, returns, None, actions, values, nlp)
        phase["tag"] = "@act"
        model.step(obs[:n_act])
    finally:
        _lib.call = orig_call
    out = {"device": torch.cuda.get_device_name(), "how": "CUDA events per launch, median of %d after %d warm-ups, "
           "512 MB L2 flush before each" % (args.iters, args.warmup), "peaks": {"hbm_gbs": HBM_GBS,
           "tensor_tflops": TENSOR_TFLOPS, "src": "H100 SXM data sheet"}, "launches": results}
    if args.compare:
        out["libs"] = {"A": args.compare[0], "B": args.compare[1]}
        out["rounds"] = args.rounds
    print(json.dumps(out))


if __name__ == "__main__":
    main()
