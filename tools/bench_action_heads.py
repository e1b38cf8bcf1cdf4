"""Stand-alone timing of the PPO2 action-head kernels: act (sample + neglogp) and loss (PPO loss + logit gradient) for
Discrete(6), MultiDiscrete (3,)*8 and (7, 5, 3, 2), and MultiBinary(16), at B = 4096 (one acting pass) and B = 131072
(one train chunk), in the fused [pi | vf] head layout the policy uses.

CUDA events around each launch, 3 warm-ups, the median of 20 iterations, and a 512 MB write between iterations so the
inputs come from HBM (L2 is 50 MB).  Bytes are what each kernel must move, computed from the shapes; bytes/s is
compared with the H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s.  Prints one JSON object, with the GPU name and
power limit read in the same run.

    python tools/bench_action_heads.py
"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from baselines_b200 import ops  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
HEADS = [("Discrete(6)", "cat", [6]), ("MultiDiscrete((3,)*8)", "mcat", [3] * 8),
         ("MultiDiscrete((7,5,3,2))", "mcat", [7, 5, 3, 2]), ("MultiBinary(16)", "bern", 16)]


def _pad(n, m):
    return (n + m - 1) // m * m


def _time(fn, flush, iters=20, warmup=3):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        flush.fill_(1.0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts)) * 1e3, float(np.min(ts)) * 1e3


def _gpu():
    info = {"name": torch.cuda.get_device_name(), "power_limit": "not read"}
    try:
        out = subprocess.run(["nvidia-smi", f"--id={torch.cuda.current_device()}", "--query-gpu=name,power.limit",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        if out:
            info["name"], info["power_limit"] = [s.strip() for s in out.split(",", 1)]
    except (OSError, subprocess.SubprocessError):
        pass
    return info


def case(label, pd, arg, B, flush, rng):
    nout = sum(arg) if pd != "bern" else arg
    k = 1 if pd == "cat" else (len(arg) if pd == "mcat" else arg)
    seg = ops.segment_table(arg, "cuda") if pd == "mcat" else None
    ld, ld_g = _pad(nout + 1, 16), _pad(nout + 1, 64)
    head = torch.from_numpy(rng.randn(B, ld).astype(np.float32)).cuda()
    grad = torch.zeros(B, ld_g, dtype=torch.float16, device="cuda")
    adt = torch.float32 if pd == "bern" else torch.int64
    a = torch.zeros((B,) if pd == "cat" else (B, k), dtype=adt, device="cuda")
    val, nlp = torch.zeros(B, device="cuda"), torch.zeros(B, device="cuda")
    ctr = torch.zeros(1, dtype=torch.int64, device="cuda")
    if pd == "bern":
        step = lambda: ops.bern_step(head, ld, nout, head[:, nout:], ld, a, val, nlp, B, seed=1, offset_dev=ctr)
    else:
        step = lambda: ops.cat_step(head, ld, nout, head[:, nout:], ld, a, val, nlp, B, seed=1, offset_dev=ctr,
                                    seg_off=seg)
    step()
    ret = torch.from_numpy(rng.randn(B).astype(np.float32)).cuda()
    oldv = torch.from_numpy(rng.randn(B).astype(np.float32)).cuda()
    oldnlp = (nlp + 0.05 * torch.from_numpy(rng.randn(B).astype(np.float32)).cuda()).contiguous()
    adv_st = torch.tensor([0.0, 1.0], dtype=torch.float64, device="cuda")
    stats = torch.zeros(5, dtype=torch.float64, device="cuda")
    common = (a, None, ret, oldv, oldnlp, adv_st, 0.2, 0.01, 0.5, grad, ld_g, grad[:, nout:], ld_g, stats, B)
    if pd == "bern":
        loss = lambda: ops.bern_loss(head, ld, nout, head[:, nout:], ld, *common)
    else:
        loss = lambda: ops.cat_loss(head, ld, nout, head[:, nout:], ld, *common, seg_off=seg)
    abytes = a.element_size() * k
    # act: read the logits and the value, write actions, value and neglogp
    step_bytes = B * (4.0 * nout + 4 + abytes + 8)
    # loss: read logits, value, actions, return, old value, old neglogp; write the fp16 gradient row (whole 16-byte
    # groups) and dv
    loss_bytes = B * (4.0 * nout + 4 + abytes + 12 + 2.0 * _pad(nout, 8) + 2)
    out = {}
    for name, fn, nbytes in (("step", step, step_bytes), ("loss", loss, loss_bytes)):
        med, best = _time(fn, flush)
        out[name] = {"us": round(med, 2), "us_min": round(best, 2), "bytes": int(nbytes),
                     "bytes_per_s": nbytes / (med * 1e-6), "share_of_3.35TB/s": nbytes / (med * 1e-6) / HBM_BYTES_PER_S}
    return {"head": label, "B": B, "nout": nout, **out}


def main():
    if not torch.cuda.is_available():
        raise SystemExit("bench_action_heads.py times CUDA kernels and needs a GPU")
    rng = np.random.RandomState(0)
    flush = torch.empty(128 * 1024 * 1024, dtype=torch.float32, device="cuda")     # 512 MB > 50 MB L2
    res = [case(label, pd, arg, B, flush, rng) for label, pd, arg in HEADS for B in (4096, 131072)]
    print(json.dumps({"gpu": _gpu(), "timing": "CUDA events, 3 warm-ups, median of 20, 512 MB L2 flush between "
                      "iterations", "peak_hbm_bytes_per_s": HBM_BYTES_PER_S, "cases": res}))


if __name__ == "__main__":
    main()
