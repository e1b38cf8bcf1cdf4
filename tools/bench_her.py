"""Time the HER train step (sample, relabel, encode, forward / backward, Adam), store_episode with its normaliser
update, and update_target_net on the GPU, beside a torch-CPU float32 arm of the same step; one JSON line.

  python tools/bench_her.py [--iters 200]

Shapes: FetchReach (o 10, g 3, u 4) and FetchPush (o 25, g 3, u 4), T = 50, 3 x 256 networks, batch 256 and 1024,
rollout batch 2 and 32.  Each device time is the mean over `iters` calls after warm-up, from CUDA events around the
calls."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def make_agent(dimo, dimg, dimu, B, rbs, T=50):
    """DEFAULT_PARAMS' agent (3 x 256, polyak 0.95, action_l2 1) for a Fetch-shaped task with the sparse distance
    reward on the device; room for 2000 episodes of T transitions."""
    from baselines_b200.her.ddpg import DDPG
    from baselines_b200.her.experiment.config import simple_goal_subtract
    from baselines_b200.her.her_sampler import make_sample_her_transitions

    def reward_fun(ag_2, g, info):
        return -(np.linalg.norm(ag_2 - g, axis=-1) > 0.05).astype(np.float32)
    sampler = make_sample_her_transitions('future', 4, reward_fun)
    sampler.device_reward = ('sparse', 0.05)
    gamma = 1. - 1. / (T + 1)
    return DDPG(input_dims={'o': dimo, 'g': dimg, 'u': dimu, 'info_is_success': 1}, buffer_size=2000 * (T + 1),
                hidden=256, layers=3, network_class='baselines.her.actor_critic:ActorCritic', polyak=0.95,
                batch_size=B, Q_lr=1e-3, pi_lr=1e-3, norm_eps=0.01, norm_clip=5, max_u=1.0, action_l2=1.0,
                clip_obs=200., scope='ddpg', T=T + 1, rollout_batch_size=rbs, subtract_goals=simple_goal_subtract,
                relative_goals=False, clip_pos_returns=True, clip_return=1. / (1. - gamma), bc_loss=0, q_filter=0,
                num_demo=0, demo_batch_size=0, prm_loss_weight=0, aux_loss_weight=0, sample_transitions=sampler,
                gamma=gamma, seed=0)


def episodes(agent, rng, n):
    """n float32 episodes of random values, as RolloutWorker returns them."""
    T, d = agent.T - 1, agent.input_dims
    ep = {'o': rng.randn(n, T + 1, d['o']), 'ag': rng.randn(n, T + 1, d['g']), 'g': rng.randn(n, T, d['g']),
          'u': rng.uniform(-1, 1, (n, T, d['u'])), 'info_is_success': rng.randint(0, 2, (n, T, 1))}
    return {k: v.astype(np.float32) for k, v in ep.items()}


def timed(fn, iters):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / iters


def cpu_step(dimo, dimg, dimu, B, iters):
    """The same step in torch on the CPU, float32: the target, the critic loss and its gradient, the actor loss and its
    gradient (both at the step's starting parameters), Adam on each network.  10 untimed steps first."""
    torch.manual_seed(0)
    mk = lambda nin, nout: torch.nn.Sequential(torch.nn.Linear(nin, 256), torch.nn.ReLU(), torch.nn.Linear(256, 256),
                                               torch.nn.ReLU(), torch.nn.Linear(256, 256), torch.nn.ReLU(),
                                               torch.nn.Linear(256, nout))
    pi, Q = mk(dimo + dimg, dimu), mk(dimo + dimg + dimu, 1)
    tpi, tQ = mk(dimo + dimg, dimu), mk(dimo + dimg + dimu, 1)
    opt_pi, opt_Q = torch.optim.Adam(pi.parameters(), 1e-3), torch.optim.Adam(Q.parameters(), 1e-3)
    og, og2, u, r = (torch.randn(B, dimo + dimg), torch.randn(B, dimo + dimg), torch.rand(B, dimu) * 2 - 1,
                     -torch.rand(B, 1).round())

    def step():
        with torch.no_grad():
            y = (r + 0.98 * tQ(torch.cat([og2, torch.tanh(tpi(og2))], 1))).clamp(-50., 0.)
        q_loss = ((y - Q(torch.cat([og, u], 1))) ** 2).mean()
        q_grads = torch.autograd.grad(q_loss, list(Q.parameters()))
        a = torch.tanh(pi(og))
        pi_loss = -Q(torch.cat([og, a], 1)).mean() + (a ** 2).mean()
        pi_grads = torch.autograd.grad(pi_loss, list(pi.parameters()))
        for p_, g_ in zip(Q.parameters(), q_grads):
            p_.grad = g_
        for p_, g_ in zip(pi.parameters(), pi_grads):
            p_.grad = g_
        opt_pi.step()
        opt_Q.step()
    for _ in range(10):
        step()
    t0 = time.perf_counter()
    for _ in range(iters):
        step()
    return (time.perf_counter() - t0) * 1e6 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_her needs a CUDA device")
    from baselines_b200 import build_ext
    build_ext.build()
    rng = np.random.RandomState(0)
    out = {"gpu": torch.cuda.get_device_name(0), "threads_cpu": torch.get_num_threads(), "results": []}
    for name, dimo in (("FetchReach", 10), ("FetchPush", 25)):
        for B in (256, 1024):
            agent = make_agent(dimo, 3, 4, B, 2)
            for _ in range(10):
                agent.store_episode(episodes(agent, rng, 2))
            train_us = timed(agent.train_device, args.iters)
            target_us = timed(agent.update_target_net, args.iters)
            cpu_us = cpu_step(dimo, 3, 4, B, max(20, args.iters // 5))
            out["results"].append(dict(shape=name, B=B, train_us=round(train_us, 1),
                                       update_target_net_us=round(target_us, 1), torch_cpu_f32_step_us=round(cpu_us, 1)))
        for rbs in (2, 32):
            agent = make_agent(dimo, 3, 4, 256, rbs)
            eps = [episodes(agent, rng, rbs) for _ in range(4)]
            k = [0]

            def store():
                agent.store_episode(eps[k[0] % 4])
                k[0] += 1
            us = timed(store, max(10, args.iters // 4))
            out["results"].append(dict(shape=name, rollout_batch=rbs, store_episode_us=round(us, 1)))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
