"""Speed of the LSTM sequence kernels (csrc/lstm.cu) and of a cnn_lstm PPO2 update.  Prints one JSON line.

  lstm_seq_fwd / lstm_seq_bwd alone, H = 128: a train minibatch (1024 envs x 128 steps) and an acting pass
  (4096 envs x 1 step); a cnn_lstm PPO2 update over a 1024 envs x 128 steps rollout, 4 minibatches x 4 epochs.
Times are CUDA events around repeated launches after a warm-up; bytes and FLOPs are algorithmic (what the math must
read, write and compute once), so GB/s and TFLOP/s are lower bounds of what the hardware did.  The card's name and
power limit are read in the same run."""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _time(fn, reps, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def kernels(T, B, H=128, reps=20):
    from baselines_b200 import ops
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(0)
    rows = T * B
    xg = torch.randn(rows, 4 * H, device=dev, generator=g)
    wh = (torch.randn(H, 4 * H, device=dev, generator=g) / H ** 0.5).half()
    whT = wh.t().contiguous()
    masks = (torch.rand(rows, device=dev, generator=g) < 0.01).to(torch.uint8)
    s0 = torch.zeros(B, 2 * H, device=dev)
    h = torch.empty(rows, H, dtype=torch.float16, device=dev)
    hp, dh = torch.empty_like(h), torch.randn(rows, H, device=dev, generator=g).half()
    c = torch.empty(rows, H, device=dev)
    gates = torch.empty(rows, 4 * H, device=dev)
    dz = torch.empty(rows, 4 * H, dtype=torch.float16, device=dev)
    train = T > 1
    fwd = lambda: ops.lstm_seq_fwd(xg, 4 * H, wh, masks, s0, h, H, T, B, H, state_out=None if train else s0,
                                   hprev_out=hp if train else None, gates_out=gates if train else None,
                                   c_out=c if train else None)
    fwd()
    bwd = lambda: ops.lstm_seq_bwd(dh, H, gates, c, masks, s0, whT, dz, 4 * H, T, B, H)
    flops = 8.0 * rows * H * H
    out = {}
    for name, fn, nbytes in (("fwd", fwd, rows * (16 * H + 2 * H + (22 * H if train else 0))),
                             ("bwd", bwd, rows * (2 * H + 16 * H + 8 * H + 8 * H))):
        if name == "bwd" and not train:
            continue
        ms = _time(fn, reps)
        out[name] = dict(ms=round(ms, 4), gflops=round(flops / ms / 1e6, 1), gbs=round(nbytes / ms / 1e6, 1))
    return out


def cnn_lstm_update(N=1024, T=128, nminibatches=4, noptepochs=4, reps=3):
    from baselines_b200.common import spaces
    from baselines_b200.common.policies import build_policy
    from baselines_b200.ppo2.model import Model
    from baselines_b200.ppo2.ppo2 import run_epochs
    from baselines_b200.ppo2.runner import Rollout

    class E:
        pass
    env = E()
    env.observation_space, env.action_space, env.num_envs = spaces.Box(0, 255, (84, 84, 4), np.uint8), spaces.Discrete(6), N
    np.random.seed(0)
    policy = build_policy(env, "cnn_lstm")
    model = Model(policy=policy, ob_space=env.observation_space, ac_space=env.action_space, nbatch_act=N,
                  nbatch_train=N * T // nminibatches, nsteps=T, ent_coef=0.01, vf_coef=0.5, max_grad_norm=0.5,
                  comm=False)
    dev = model.device
    ro = Rollout(T, N, (84, 84, 4), torch.uint8, True, 0, dev, state_dim=2 * model.net.nlstm)
    g = torch.Generator(device=dev).manual_seed(1)
    ro.obs.copy_(torch.randint(0, 256, ro.obs.shape, device=dev, generator=g, dtype=torch.uint8))
    ro.actions.copy_(torch.randint(0, 6, ro.actions.shape, device=dev, generator=g))
    ro.returns.normal_(generator=g)
    ro.values.normal_(generator=g)
    ro.neglogpacs.uniform_(1.0, 2.5, generator=g)
    ro.dones.copy_((torch.rand(T, N, device=dev, generator=g) < 0.01).to(torch.uint8))
    ms = _time(lambda: run_epochs(model, ro, 2.5e-4, 0.1, N * T, N * T // nminibatches, noptepochs, dev), reps, 1)
    return dict(ms=round(ms, 1), frames_per_s=round(N * T / ms * 1e3))


def card():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                             str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl


def main():
    from baselines_b200 import build_ext
    build_ext.build()
    name, pl = card()
    res = {"card": name, "power_limit": pl, "H": 128,
           "train_1024x128": kernels(128, 1024), "act_4096x1": kernels(1, 4096),
           "cnn_lstm_update_1024x128_4mb_4ep": cnn_lstm_update()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
