"""Stand-alone timing of VecNormalize on the device (csrc/vec_normalize.cu).

* Kernels at 16384 x 376 (the MuJoCo Humanoid shape of cfg-3) in float32 and float64 and at 256 x 376: the moments,
  the combine, the normalisation and the reward step.  CUDA events around each launch, 3 warm-ups, the median of 20,
  a 512 MB write between iterations so inputs come from HBM.
* The column moments against their chain bound 2 * N * L / clock: each column is 2 * N dependent adds.  L (cycles per
  add) is measured in the same run by a one-thread dependent-add chain (b200rl_vecnorm_add_latency); the clock is the
  card's maximum SM clock, so the ratio is conservative if the card runs slower.
* The normalisation against the H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s (bytes: x in, float32 out).
* ms per env step of a cfg-3-shaped rollout (16384 envs, 376 float32 observations, Box(17), mlp with
  value_network='copy', 8 steps; the median of 3 rollouts after 2 warm-ups) through VecNormalize(SyntheticVecEnv) on the host path (the
  wrapper hidden under a forwarding wrapper) and on the device path, and through VecNormalize(DeviceSyntheticVecEnv).

Prints one JSON object, with the GPU name and power limit read in the same run.

    python tools/bench_vec_normalize.py
"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench_action_heads import HBM_BYTES_PER_S, _gpu, _time  # noqa: E402
from baselines_b200 import ops  # noqa: E402


def _max_sm_clock_hz():
    try:
        out = subprocess.run(["nvidia-smi", f"--id={torch.cuda.current_device()}", "--query-gpu=clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        return float(out.strip().splitlines()[0]) * 1e6
    except (OSError, subprocess.SubprocessError, ValueError, IndexError):
        return None


def add_latency(f64):
    out = torch.zeros(2, dtype=torch.float64, device="cuda")
    for _ in range(2):
        ops.vecnorm_add_latency(f64, 1 << 20, out)
    torch.cuda.synchronize()
    return float(out[0])


def kernels(N, D, dtype, flush, rng, lat, clock):
    tdt = torch.float32 if dtype == np.float32 else torch.float64
    x = torch.from_numpy((1e4 + rng.randn(N, D)).astype(dtype)).cuda()
    rew = torch.from_numpy(rng.randn(N).astype(dtype)).cuda()
    news = torch.from_numpy((rng.rand(N) < 0.01).astype(np.uint8)).cuda()
    ws = torch.zeros(2 * D, dtype=torch.float64, device="cuda")
    rms = torch.cat([torch.zeros(D), torch.ones(2 * D), torch.tensor([1e-4])]).double().cuda()
    rrms = torch.tensor([0.0, 1.0, 1.0, 1e-4], dtype=torch.float64, device="cuda")
    ret = torch.zeros(N, dtype=torch.float64, device="cuda")
    out, rout = torch.zeros(N, D, device="cuda"), torch.zeros(N, device="cuda")
    esize = x.element_size()
    res = {"N": N, "D": D, "dtype": str(tdt).replace("torch.", "")}
    for name, fn in (("moments", lambda: ops.vecnorm_moments(x, ws)),
                     ("combine", lambda: ops.vecnorm_combine(rms, ws, N, 1e-8, tdt == torch.float32)),
                     ("normalize", lambda: ops.vecnorm_normalize(x, rms, 10.0, out)),
                     ("rewards", lambda: ops.vecnorm_rewards(rew, news, ret, rrms, 0.99, 1e-8, 10.0, rout))):
        med, best = _time(fn, flush)
        res[name + "_us"] = round(med, 2)
        if name == "moments" and clock:
            bound_us = 2.0 * N * lat * 1e6 / clock
            res["moments_chain_bound_us"] = round(bound_us, 2)
            res["moments_over_chain_bound"] = round(med / bound_us, 3)
        if name == "normalize":
            nbytes = N * D * (esize + 4.0)
            res["normalize_bytes"] = int(nbytes)
            res["normalize_share_of_3.35TB/s"] = round(nbytes / (med * 1e-6) / HBM_BYTES_PER_S, 3)
    return res


def rollout_ms_per_step(kind, N=16384, T=8):
    from baselines_b200.common.policies import build_policy
    from baselines_b200.common.vec_env import (DeviceSyntheticVecEnv, SyntheticVecEnv, VecEnvWrapper,
                                               VecNormalize)
    from baselines_b200.ppo2.model import Model
    from baselines_b200.ppo2.runner import Runner

    class Fwd(VecEnvWrapper):
        def reset(self):
            return self.venv.reset()

        def step_wait(self):
            return self.venv.step_wait()
    if kind == "device_env":
        env = VecNormalize(DeviceSyntheticVecEnv(N, ob_shape=(376,), ob_dtype=np.float32, act_dim=17))
    else:
        env = VecNormalize(SyntheticVecEnv(N, ob_shape=(376,), ob_dtype=np.float32, act_dim=17))
        if kind == "host":
            env = Fwd(env)
    np.random.seed(0)
    policy = build_policy(env, "mlp", value_network="copy")
    model = Model(policy=policy, ob_space=env.observation_space, ac_space=env.action_space, nbatch_act=N,
                  nbatch_train=N * T // 4, nsteps=T, ent_coef=0.0, vf_coef=0.5, max_grad_norm=0.5, comm=False)
    runner = Runner(env=env, model=model, nsteps=T, gamma=0.99, lam=0.95)
    assert runner.vn == (kind != "host")
    ts = []
    for k in range(5):                                   # 2 warm-up rollouts, the median of 3
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        runner.run_device()
        torch.cuda.synchronize()
        if k >= 2:
            ts.append((time.perf_counter() - t0) * 1e3 / T)
    return round(float(np.median(ts)), 3)


def main():
    assert torch.cuda.is_available(), "bench_vec_normalize needs a GPU"
    rng = np.random.RandomState(0)
    flush = torch.empty(128 << 20, device="cuda")
    clock = _max_sm_clock_hz()
    lat = {"float32": add_latency(False), "float64": add_latency(True)}
    res = {"gpu": _gpu(), "max_sm_clock_mhz": None if clock is None else clock / 1e6,
           "add_latency_cycles": {k: round(v, 2) for k, v in lat.items()}, "kernels": []}
    for N, D, dt in ((16384, 376, np.float32), (16384, 376, np.float64), (256, 376, np.float32)):
        res["kernels"].append(kernels(N, D, dt, flush, rng, lat["float32" if dt == np.float32 else "float64"],
                                      clock))
    res["rollout_ms_per_step"] = {k: rollout_ms_per_step(k) for k in ("host", "device", "device_env")}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
