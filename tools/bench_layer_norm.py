"""Stand-alone timing of layer normalisation: the ln_fwd / ln_bwd kernels at 262144 x 64 (a cfg-3 minibatch chunk),
131072 x 64 and 512 x 256 (a deepq stream at batch 512), and what `layer_norm=True` adds to a cfg-3-shaped PPO2 `mlp`
update (376 observations, Box(17) actions, value_network='copy', 65536 samples) and to a deepq train step at B = 512;
and a deepq act call at B = 1 with epsilon-greedy exploration and with parameter-space noise.

Kernels: CUDA events around each launch, 3 warm-ups, the median of 20 iterations, and a 512 MB write between
iterations so the inputs come from HBM (L2 is 50 MB).  Bytes are what each kernel must move (forward: fp32 z in, fp16 y
out; backward: fp32 z and fp16 du in, fp16 dz out), compared with the H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s.
Whole updates: CUDA events around one call with its launch sequence replayed from a captured graph, median of 20,
with and without layer_norm alternating.  Prints one JSON object, with the GPU name and power limit read in the same
run.

    python tools/bench_layer_norm.py
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench_action_heads import HBM_BYTES_PER_S, _gpu, _time  # noqa: E402
from baselines_b200 import nn, ops  # noqa: E402


def kernels(rows, N, flush, rng):
    z = torch.from_numpy(rng.randn(rows, N).astype(np.float32)).cuda()
    du = torch.from_numpy((rng.randn(rows, N) * 0.1).astype(np.float16)).cuda()
    gamma, beta = torch.ones(N, device="cuda"), torch.zeros(N, device="cuda")
    y, dz = torch.empty_like(du), torch.empty_like(du)
    dg, db = torch.zeros(N, device="cuda"), torch.zeros(N, device="cuda")
    out = {"rows": rows, "N": N}
    for name, fn, nbytes in (
            ("ln_fwd", lambda: ops.ln_fwd(z, N, gamma, beta, y, N, rows, N, ops.ACT_TANH, nn.LN_EPS), rows * N * 6.0),
            ("ln_bwd", lambda: ops.ln_bwd(du, N, z, N, gamma, dz, N, dg, db, rows, N, 1.0 / rows, nn.LN_EPS),
             rows * N * 8.0)):
        med, best = _time(fn, flush)
        out[name] = {"us": round(med, 2), "us_min": round(best, 2), "bytes": int(nbytes),
                     "share_of_3.35TB/s": nbytes / (med * 1e-6) / HBM_BYTES_PER_S}
    return out


def _time_pair(fns, iters=20, warmup=4):
    """Median ms of each callable, the callables alternating."""
    for _ in range(warmup):
        for fn in fns:
            fn()
    ts = [[] for _ in fns]
    for _ in range(iters):
        for i, fn in enumerate(fns):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ts[i].append(e0.elapsed_time(e1))
    return [round(float(np.median(t)), 4) for t in ts]


def ppo2_update(rng, M=65536):
    from baselines_b200.common import spaces
    from baselines_b200.common.policies import build_policy
    from baselines_b200.ppo2.model import Model

    class E:
        observation_space = spaces.Box(-10, 10, (376,), np.float32)
        action_space = spaces.Box(-1, 1, (17,), np.float32)
        num_envs = M // 16
    dev = torch.device("cuda")
    obs = torch.from_numpy(rng.randn(M, 376).astype(np.float32)).to(dev)
    act = torch.from_numpy(rng.randn(M, 17).astype(np.float32)).to(dev)
    val = torch.from_numpy(rng.randn(M).astype(np.float32)).to(dev)
    ret = val + 0.7 * torch.from_numpy(rng.randn(M).astype(np.float32)).to(dev)
    nlp = torch.full((M,), 24.0, device=dev)
    idx = torch.from_numpy(rng.permutation(M)).to(dev)
    fns = []
    for ln in (False, True):
        np.random.seed(0)
        m = Model(policy=build_policy(E, "mlp", value_network="copy", layer_norm=ln), ob_space=E.observation_space,
                  ac_space=E.action_space, nbatch_act=M // 16, nbatch_train=M, nsteps=16, ent_coef=0.0, vf_coef=0.5,
                  max_grad_norm=0.5, comm=False)
        fns.append(lambda m=m: m.train_rollout(3e-4, 0.2, obs, act, ret, val, nlp, idx))
    plain, normed = _time_pair(fns)
    return {"samples": M, "ms_plain": plain, "ms_layer_norm": normed,
            "what": "Model.train_rollout: one shuffled minibatch of device-resident rollout arrays (graph replay)"}


def dqn_step(rng, B=512):
    from baselines_b200.common import spaces
    from baselines_b200.deepq.build_graph import DQNModel
    dev = torch.device("cuda")
    n = 4096
    obs = torch.from_numpy(rng.randn(n, 8).astype(np.float32)).to(dev)
    act = torch.from_numpy(rng.randint(0, 6, n)).to(dev)
    rew = torch.from_numpy(rng.randn(n).astype(np.float32)).to(dev)
    done = torch.zeros(n, device=dev)
    idx = torch.from_numpy(rng.randint(0, n, B)).to(dev)
    w = torch.ones(B, device=dev)
    fns = []
    for ln in (False, True):
        m = DQNModel(spaces.Box(-5, 5, (8,), np.float32), 6, "mlp", lr=1e-4, gamma=0.99, grad_norm_clipping=10,
                     batch_cap=B, seed=0, hiddens=(256,), dueling=True, layer_norm=ln)
        fns.append(lambda m=m: m.train_device(obs, obs, act, rew, done, w, idx, B))
    plain, normed = _time_pair(fns)
    return {"B": B, "ms_plain": plain, "ms_layer_norm": normed,
            "what": "DQNModel.train_device through the resident-replay path (graph replay)"}


def dqn_act(rng):
    """One act call at B = 1 (observation already on the device): epsilon-greedy, and parameter-space noise with the
    scale update every call as deepq.learn makes it (trunk once, three stream passes, one perturbation, the KL)."""
    from baselines_b200.common import spaces
    from baselines_b200.deepq.build_graph import DQNModel
    ob = torch.from_numpy(rng.randn(1, 8).astype(np.float32)).cuda()
    fns = []
    for pn in (False, True):
        m = DQNModel(spaces.Box(-5, 5, (8,), np.float32), 6, "mlp", lr=1e-4, batch_cap=32, seed=0, hiddens=(256,),
                     dueling=True, layer_norm=True, param_noise=pn)
        fns.append((lambda m=m: m.act_device_param_noise(ob, 1, 0.0, False, True)) if pn else
                   (lambda m=m: m.act_device(ob, 1, 0.1)))
    plain, noisy = _time_pair(fns)
    return {"B": 1, "ms_eps_greedy": plain, "ms_param_noise": noisy, "what": "act_device / act_device_param_noise "
            "(update_param_noise_scale=True, no reset), graph replay, layer_norm=True in both"}


def main():
    if not torch.cuda.is_available():
        raise SystemExit("bench_layer_norm.py times CUDA kernels and needs a GPU")
    rng = np.random.RandomState(0)
    flush = torch.empty(128 * 1024 * 1024, dtype=torch.float32, device="cuda")     # 512 MB > 50 MB L2
    res = [kernels(rows, N, flush, rng) for rows, N in ((262144, 64), (131072, 64), (512, 256))]
    del flush
    print(json.dumps({"gpu": _gpu(), "timing": "kernels: CUDA events, 3 warm-ups, median of 20, 512 MB L2 flush between "
                      "iterations; updates: CUDA events, 4 warm-ups, median of 20, variants alternating",
                      "peak_hbm_bytes_per_s": HBM_BYTES_PER_S, "kernels": res, "ppo2_mlp_update": ppo2_update(rng),
                      "deepq_train_step": dqn_step(rng), "deepq_act_call": dqn_act(rng)}))


if __name__ == "__main__":
    main()
