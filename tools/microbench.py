#!/usr/bin/env python
"""Stand-alone timings of the two north-star kernels (GAE scan, NatureCNN fc1 GEMM) with CUDA events on the
launching stream, >=3 warm-ups, and an L2 flush (write of a 512 MB buffer) between timed iterations.

    python tools/microbench.py            # prints one JSON object
Used by bench.py (extra `targets` key); `tools/microbench.py --only gae|fc1` runs one case."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from baselines_b200 import ops  # noqa: E402


def _time(fn, iters=10, warmup=3, flush=None):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        if flush is not None:
            flush.fill_(1.0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts)), float(np.min(ts))


def gae_case(T, N, variant, flush):
    g = torch.Generator(device="cuda").manual_seed(0)
    rew = torch.randn(T, N, device="cuda", generator=g)
    val = torch.randn(T, N, device="cuda", generator=g)
    done = (torch.rand(T, N, device="cuda", generator=g) < 0.01).to(torch.uint8)
    lv = torch.randn(N, device="cuda", generator=g)
    ld = torch.zeros(N, dtype=torch.uint8, device="cuda")
    adv, ret = torch.empty_like(rew), torch.empty_like(rew)
    med, best = _time(lambda: ops.gae_scan(rew, val, done, lv, ld, adv, ret, 0.99, 0.95, variant), flush=flush)
    nbytes = 17.0 * T * N + 5.0 * N
    return {"T": T, "N": N, "variant": variant, "ms": med, "ms_best": best, "bytes": nbytes,
            "gbs": nbytes / (med * 1e-3) / 1e9}


def fc1_case(M, kind, flush, K=3136, N=512):
    A = (torch.randn(M, K, device="cuda") * 0.1).half()
    W = (torch.randn(N, K, device="cuda") * 0.1).half()
    if kind == "fwd":
        C = torch.empty(M, N, dtype=torch.float16, device="cuda")
        bias = torch.zeros(N, device="cuda")
        fn = lambda: ops.gemm(A, W, C, M=M, N=N, K=K, lda=K, ldb=K, ldc=N, bias=bias, mode=ops.MODE_F16_ACT,
                              act=ops.ACT_RELU)
    elif kind == "dgrad":
        dz = (torch.randn(M, N, device="cuda") * 0.1).half()
        Wb = (torch.randn(K, N, device="cuda") * 0.1).half()
        out = torch.empty(M, K, dtype=torch.float16, device="cuda")
        fn = lambda: ops.gemm(dz, Wb, out, M=M, N=K, K=N, lda=N, ldb=N, ldc=K, saved=A, ld_saved=K,
                              mode=ops.MODE_F16_DACT, act=ops.ACT_RELU)
    else:
        dz = (torch.randn(M, N, device="cuda") * 0.1).half()
        gw = torch.zeros(K, N, device="cuda")
        tiles = -(-K // 128) * -(-N // 128)
        split = max(1, min((M // 64) // 2, -(-296 // tiles)))
        fn = lambda: ops.gemm(A, dz, gw, M=K, N=N, K=M, lda=K, ldb=N, ldc=N, mn_major=True,
                              mode=ops.MODE_F32_ATOMIC, alpha=1.0, split_k=split)
    med, best = _time(fn, flush=flush)
    flops = 2.0 * M * N * K
    return {"M": M, "K": K, "N": N, "kind": kind, "ms": med, "ms_best": best, "flops": flops,
            "tflops": flops / (med * 1e-3) / 1e12}


def gae_cpu_case(T, N):
    """The reference's numpy GAE loop (ppo2/runner.py:53-65, restated in oracle/gae.py) on the host, same sizes."""
    import time
    from oracle.gae import gae_reference_order
    rng = np.random.RandomState(0)
    rew, val = rng.randn(T, N).astype(np.float32), rng.randn(T, N).astype(np.float32)
    done = rng.rand(T, N) < 0.01
    lv, ld = rng.randn(N).astype(np.float32), np.zeros(N, dtype=np.bool_)
    gae_reference_order(rew[:8], val[:8], done[:8], lv, ld, 0.99, 0.95)
    t0 = time.perf_counter()
    gae_reference_order(rew, val, done, lv, ld, 0.99, 0.95)
    ms = (time.perf_counter() - t0) * 1e3
    return {"T": T, "N": N, "ms": ms, "gbs": (17.0 * T * N + 5.0 * N) / (ms * 1e-3) / 1e9, "kind": "port (numpy, 1 thread)"}


def per_case(flush, cap=1 << 20, batch=512, alpha=0.6, beta=0.4):
    """cfg-4: prioritized replay at capacity 2^20 -- stratified sample of 512 + importance weights, and the
    2 x 512 priority writes of one train step (replay_buffer.py:107-115,157-165,169-191); the CPU leg is the
    oracle port of the same arithmetic (oracle/segment_tree.py), trees filled level by level (same node values)."""
    import random
    import time
    from oracle.segment_tree import PrioritizedSampler
    rng = np.random.RandomState(0)
    pr = np.abs(rng.randn(cap)) + 1e-6
    vals = pr ** alpha
    dev = "cuda"
    it_sum = torch.zeros(2 * cap, dtype=torch.float64, device=dev)
    it_min = torch.full((2 * cap,), float("inf"), dtype=torch.float64, device=dev)
    ops.tree_set(it_sum, it_min, cap, torch.arange(cap, device=dev), torch.from_numpy(vals).to(dev))
    random.seed(0)
    u_host = np.array([random.random() for _ in range(batch)])
    u = torch.from_numpy(u_host).to(dev)
    idx = torch.empty(batch, dtype=torch.int64, device=dev)
    w64 = torch.empty(batch, dtype=torch.float64, device=dev)
    w32 = torch.empty(batch, dtype=torch.float32, device=dev)
    ms_s, _ = _time(lambda: ops.per_sample(it_sum, it_min, cap, cap, u, beta, idx, w64, w32), flush=flush)
    newv = torch.from_numpy((np.abs(rng.randn(batch)) + 1e-6) ** alpha).to(dev)
    torch.cuda.synchronize()
    upd_idx = idx.clone()
    ms_u, _ = _time(lambda: ops.tree_set(it_sum, it_min, cap, upd_idx, newv), flush=flush)
    # CPU port on the same tree
    ps = PrioritizedSampler(cap, alpha)
    ps.n = cap
    for tree, red in ((ps.sum_tree, np.add), (ps.min_tree, np.minimum)):
        tree.value[cap:] = vals
        lvl = cap
        while lvl > 1:
            half = lvl // 2
            tree.value[half:lvl] = red(tree.value[lvl:2 * lvl:2], tree.value[lvl + 1:2 * lvl:2])
            lvl = half
    t0 = time.perf_counter()
    ci = ps.sample_idx(list(u_host))
    cw = ps.weights(ci, beta)
    t1 = time.perf_counter()
    ps.update_priorities(ci, list(np.abs(rng.randn(batch)) + 1e-6))
    t2 = time.perf_counter()
    idx_same = bool(np.array_equal(np.array(ci), idx.cpu().numpy()))     # integer work: must be identical
    w_err = float(np.max(np.abs(w64.cpu().numpy() - cw) / cw))           # pow() of libm vs CUDA: a few ulps
    return {"capacity": cap, "batch": batch, "gpu_sample_us": ms_s * 1e3, "gpu_update_us": ms_u * 1e3,
            "cpu_sample_ms": (t1 - t0) * 1e3, "cpu_update_ms": (t2 - t1) * 1e3, "cpu_kind": "port (python, 1 thread)",
            "indices_equal_port": idx_same, "weights_max_rel_err_vs_port": w_err}


def replay_gather_case(flush, batch=512, pool=32768):
    """cfg-4: the observation gather of one replay sample (replay_buffer.py:33-43 `_encode_sample`: obs_t and
    obs_tp1 of 512 random transitions) as it runs on the device: index gather + uint8 -> fp16 cast in one pass per
    array.  Algorithmic bytes = 2 arrays x 512 x 28224 x (1 B read + 2 B written) = 86.7 MB (SURVEY 8d: 28.9 MB of
    uint8 reads).  The pool (2 x 0.92 GB) is larger than L2."""
    n_el = 84 * 84 * 4
    g = torch.Generator(device="cuda").manual_seed(0)
    obs_t = torch.randint(0, 256, (pool, n_el), dtype=torch.uint8, device="cuda", generator=g)
    obs_1 = torch.randint(0, 256, (pool, n_el), dtype=torch.uint8, device="cuda", generator=g)
    idx = torch.randint(0, pool, (batch,), device="cuda", generator=g)
    out_t = torch.empty(batch, n_el, dtype=torch.float16, device="cuda")
    out_1 = torch.empty(batch, n_el, dtype=torch.float16, device="cuda")

    def fn():
        ops.im2col(obs_t, out_t, batch, 1, 1, n_el, 1, 1, False, src_idx=idx, tag="replay_gather")
        ops.im2col(obs_1, out_1, batch, 1, 1, n_el, 1, 1, False, src_idx=idx, tag="replay_gather")
    ms, best = _time(fn, flush=flush)
    ok = bool(torch.equal(out_t, obs_t[idx].half()) and torch.equal(out_1, obs_1[idx].half()))
    nbytes = 2.0 * batch * n_el * 3
    return {"batch": batch, "pool": pool, "ms": ms, "ms_best": best, "bytes": nbytes, "gbs": nbytes / (ms * 1e-3) / 1e9,
            "matches_torch_index": ok}


def dqn_case(flush, batch=512):
    """cfg-4: one deepq train step (build_graph.py:388-430) at batch 512: conv_only + dueling, double-Q -> three
    forwards, one backward, per-variable clip, Adam; observations gathered from a device-resident buffer."""
    from baselines_b200.common import spaces
    from baselines_b200.deepq.build_graph import DQNModel
    m = DQNModel(spaces.Box(0, 255, (84, 84, 4), np.uint8), 6, "conv_only", lr=1e-4, gamma=0.99, grad_norm_clipping=10,
                 batch_cap=batch, seed=0, hiddens=(256,), dueling=True)
    dev = m.device
    g = torch.Generator(device="cuda").manual_seed(0)
    o_t = torch.randint(0, 256, (batch, 84, 84, 4), dtype=torch.uint8, device=dev, generator=g)
    o_1 = torch.randint(0, 256, (batch, 84, 84, 4), dtype=torch.uint8, device=dev, generator=g)
    act = torch.randint(0, 6, (batch,), device=dev, generator=g)
    rew = torch.randn(batch, device=dev, generator=g)
    done = (torch.rand(batch, device=dev, generator=g) < 0.05).float()
    w = torch.rand(batch, device=dev, generator=g) * 0.9 + 0.1
    ms, best = _time(lambda: m.train_device(o_t, o_1, act, rew, done, w, None, batch), flush=flush)
    return {"batch": batch, "ms": ms, "ms_best": best, "transitions_per_s": batch / (ms * 1e-3)}


def run(only=None, quick=False):
    flush = torch.empty(128 * 1024 * 1024, dtype=torch.float32, device="cuda")      # 512 MB > 50 MB L2
    out = {"l2_flush": "512 MB write between iterations"}
    Ms = [8192, 131072] if not quick else [131072]
    cases = [
        # cfg-2 size (L2-resident), cfg-3 size (142 MB, ~3x L2), and 570 MB (~11x L2: a DRAM steady-state measurement)
        ("gae", "gae", lambda: [gae_case(128, 4096, -1, flush), gae_case(512, 16384, 1, flush),
                                gae_case(512, 16384, 0, flush), gae_case(2048, 16384, 1, flush)]),
        ("fc1", "fc1", lambda: [fc1_case(M, k, flush) for M in Ms for k in ("fwd", "dgrad", "wgrad")]),
        ("gae", "gae_cpu", lambda: [gae_cpu_case(128, 4096), gae_cpu_case(512, 16384)]),
        ("per", "per", lambda: per_case(flush)),
        ("per", "replay_gather", lambda: replay_gather_case(flush)),
        ("dqn", "dqn", lambda: dqn_case(flush)),
    ]
    for group, key, fn in cases:                      # one failing case must not take the others with it
        if only not in (None, group):
            continue
        try:
            out[key] = fn()
        except Exception as ex:                       # noqa: BLE001
            out[key] = {"error": repr(ex)}
        torch.cuda.empty_cache()
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default=None)
    ap.add_argument("--quick", action="store_true", help="fc1 at M=131072 only")
    a = ap.parse_args()
    print(json.dumps(run(a.only, a.quick)))
