"""CPU: the MultiDiscrete / MultiBinary space stand-ins, the oracle of their action distributions (tests/_action_oracle.py)
against float64 finite differences and the reference's own distribution identities, and MultiDiscreteIdentityEnv."""
import math

import numpy as np
import pytest
import torch

from oracle import nets
import _action_oracle as ao


# ------------------------------------------------------------------------------------------------ spaces
def test_multidiscrete_space():
    from baselines_b200.common import spaces
    sp = spaces.MultiDiscrete([3, 1, 5])
    assert sp.shape == (3,) and sp.dtype == np.int64 and list(sp.nvec) == [3, 1, 5]
    sp.seed(0)
    xs = np.array([sp.sample() for _ in range(2000)])
    assert xs.dtype == np.int64 and xs.shape == (2000, 3)
    assert all(sp.contains(x) for x in xs)
    assert set(xs[:, 0]) == {0, 1, 2} and set(xs[:, 1]) == {0} and set(xs[:, 2]) == set(range(5))
    sp.seed(0)
    assert np.array_equal(sp.sample(), xs[0])                       # seeded stream repeats
    assert not sp.contains(np.array([3, 0, 0])) and not sp.contains(np.array([0, 0])) and not sp.contains([-1, 0, 0])
    for bad in ([], [2, 0], [-1], [[2, 2]]):
        with pytest.raises(ValueError):
            spaces.MultiDiscrete(bad)
    assert spaces.is_multi_discrete(sp) and not spaces.is_discrete(sp) and not spaces.is_multi_binary(sp)


def test_multibinary_space_is_not_taken_for_discrete():
    from baselines_b200.common import spaces
    sp = spaces.MultiBinary(4)
    assert sp.n == 4 and sp.shape == (4,) and sp.dtype == np.int8
    sp.seed(1)
    xs = np.array([sp.sample() for _ in range(500)])
    assert xs.dtype == np.int8 and set(np.unique(xs)) == {0, 1}
    assert all(sp.contains(x) for x in xs) and not sp.contains(np.array([0, 2, 0, 0])) and not sp.contains([0, 1])
    assert spaces.is_multi_binary(sp) and not spaces.is_discrete(sp) and not spaces.is_multi_discrete(sp)
    # duck typing also sorts gym-like objects (gym's MultiBinary has .n and shape (n,); Discrete has shape ())
    d = spaces.Discrete(4)
    assert spaces.is_discrete(d) and not spaces.is_multi_binary(d)

    class GymMultiBinary:
        n, shape = 3, (3,)
    assert spaces.is_multi_binary(GymMultiBinary()) and not spaces.is_discrete(GymMultiBinary())
    with pytest.raises(ValueError):
        spaces.MultiBinary(0)


def test_segment_table_rejects_empty_components():
    from baselines_b200 import ops
    assert ops.segment_table([3, 1, 2], "cpu").tolist() == [0, 3, 4, 6]
    assert ops.segment_table([3, 1, 2], "cpu").dtype == torch.int32
    for bad in ([], [2, 0, 1], [-3]):
        with pytest.raises(ValueError):
            ops.segment_table(bad, "cpu")


# ------------------------------------------------------------------------------------------------ finite differences
def _fd_check(loss_fn, tp, n_probe, rng, h=1e-6):
    """max relative error between autograd and central differences over n_probe random coordinates per tensor."""
    for t in tp.values():
        t.requires_grad_(True)
    loss = loss_fn()
    grads = torch.autograd.grad(loss, list(tp.values()), allow_unused=True)
    for t in tp.values():
        t.requires_grad_(False)
    worst = 0.0
    for (k, t), g in zip(tp.items(), grads):
        g = torch.zeros_like(t) if g is None else g
        flat = t.view(-1)
        for i in rng.choice(flat.numel(), size=min(n_probe, flat.numel()), replace=False):
            old = float(flat[i])
            flat[i] = old + h
            lp = float(loss_fn())
            flat[i] = old - h
            lm = float(loss_fn())
            flat[i] = old
            fd = (lp - lm) / (2 * h)
            an = float(g.reshape(-1)[i])
            worst = max(worst, abs(fd - an) / max(1e-6, abs(fd) + abs(an)))
    return worst


@pytest.mark.parametrize("pd,arg,vn", [("mcat", [3, 1, 4], None), ("mcat", [2, 5], "copy"), ("bern", 5, None),
                                       ("bern", 3, "copy")])
def test_ppo_loss_gradient_vs_float64_finite_differences(pd, arg, vn):
    rng = np.random.RandomState(7)
    np.random.seed(8)
    p = ao.init_policy_params("mlp", (5,), pd, arg, value_network=vn, num_hidden=16)
    # scale the pi head up so the distributions are far from uniform (the 0.01 init makes every p ~ 1/n)
    p["ppo2_model/pi/w:0"] = p["ppo2_model/pi/w:0"] * 100.0
    tp = nets.to_torch(p, torch.float64)
    B = 16
    obs = torch.tensor(rng.randn(B, 5))
    if pd == "mcat":
        acts = torch.tensor(np.stack([rng.randint(0, n, B) for n in arg], 1))
    else:
        acts = torch.tensor((rng.rand(B, arg) < 0.5).astype(np.float64))
    advs, rets, oldv = torch.tensor(rng.randn(B)), torch.tensor(rng.randn(B)), torch.tensor(rng.randn(B))
    nvec = arg if pd == "mcat" else None
    with torch.no_grad():
        pi, _, _ = nets.policy_forward(tp, "mlp", obs, vn)
        nlp = ao.neglogp(pd, pi, None, acts, nvec)
    oldnlp = nlp + torch.tensor(rng.randn(B) * 0.05)
    fn = lambda: ao.ppo_loss(tp, "mlp", obs, acts, advs, rets, oldnlp, oldv, 0.2, 0.3, 0.5, vn, pd, nvec)[0]
    worst = _fd_check(fn, tp, 12, rng)
    assert worst < 2e-5, (pd, arg, worst)


def test_entropy_gradient_of_each_head_in_closed_form():
    """The kernels' closed forms: d(sum_s H_s)/dl_j = -p_j (log p_j + H_s) with the SEGMENT's entropy; for Bernoulli
    (differentiated through the labels p too) dH/dl_j = -l_j p_j (1 - p_j)."""
    rng = np.random.RandomState(0)
    nvec = [1, 2, 3, 4]
    l = torch.tensor(rng.randn(5, sum(nvec)) * 2, requires_grad=True)
    g, = torch.autograd.grad(ao.mcat_entropy(l, nvec).sum(), l)
    want = []
    for blk in torch.split(l.detach(), nvec, dim=1):
        lp = torch.log_softmax(blk, 1)
        Hs = -(lp.exp() * lp).sum(1, keepdim=True)
        want.append(-lp.exp() * (lp + Hs))
    assert torch.allclose(g, torch.cat(want, 1), atol=1e-12)
    b = torch.tensor(rng.randn(5, 6) * 3, requires_grad=True)
    g, = torch.autograd.grad(ao.bern_entropy(b).sum(), b)
    p = torch.sigmoid(b.detach())
    assert torch.allclose(g, -b.detach() * p * (1 - p), atol=1e-12)


# ------------------------------------------------------------------------------------------------ distribution identities
def _validate(neglogp, entropy, kl, sample, pdparam, nuni, rng):
    """common/distributions.py:321-348 (validate_probtype): E[-log p] = H and KL[p, q] = -H - E_p[log q], 3 sigma."""
    N = 100000
    M = torch.tensor(np.repeat(pdparam[None], N, 0))
    X = sample(M, torch.tensor(rng.rand(N, nuni)))
    ll = -neglogp(M, X).numpy()
    ent = float(entropy(M).mean())
    assert abs(ent - (-ll.mean())) < 3 * ll.std() / math.sqrt(N)
    q = pdparam + rng.randn(pdparam.size) * 0.1
    M2 = torch.tensor(np.repeat(q[None], N, 0))
    klv = float(kl(M, M2).mean())
    ll2 = -neglogp(M2, X).numpy()
    assert abs(klv - (-ent - ll2.mean())) < 3 * ll2.std() / math.sqrt(N)


def test_reference_probtype_identities_on_the_oracle():
    rng = np.random.RandomState(0)
    nvec = [1, 2, 3]
    _validate(lambda m, x: ao.mcat_neglogp(m, x, nvec), lambda m: ao.mcat_entropy(m, nvec),
              lambda m, o: ao.mcat_kl(m, o, nvec), lambda m, u: ao.mcat_sample(m, u, nvec),
              np.array([-.2, .3, .5, .1, 1, -.1]), 6, rng)
    _validate(ao.bern_neglogp, ao.bern_entropy, ao.bern_kl, ao.bern_sample, np.array([-.2, .3, .5]), 3, rng)


def test_multidiscrete_observation_encoding():
    oh = ao.encode_multidiscrete(np.array([[2, 0], [0, 1]]), [3, 2]).numpy()
    assert np.array_equal(oh, np.array([[0, 0, 1, 1, 0], [1, 0, 0, 0, 1]], np.float32))


# ------------------------------------------------------------------------------------------------ env
def test_multidiscrete_identity_env():
    from baselines_b200 import envs
    env = envs.make("MultiDiscreteIdentity-v0")
    assert env.spec.env_type == "identity"
    assert list(env.action_space.nvec) == [3, 3] and env.observation_space is env.action_space
    env.seed(0)
    ob = env.reset()
    assert ob.shape == (2,) and ob.dtype == np.int64
    steps, done = 0, False
    while not done:
        if steps % 2:
            act = ob.copy()
            act[steps % 4 // 2] = (act[steps % 4 // 2] + 1) % 3         # one component off: no reward
            want = 0
        else:
            act, want = ob.copy(), 1                                    # every component matches: reward 1
        ob, r, done, _ = env.step(act)
        assert r == want and ob.shape == (2,) and env.observation_space.contains(ob)
        steps += 1
    assert steps == 100                                               # episode_len = 100
    env2 = envs.MultiDiscreteIdentityEnv((2, 4), episode_len=3, delay=1)
    env2.seed(3)
    o0 = env2.reset()
    o1, r, _, _ = env2.step(o0)
    assert r == 0                                                     # the first `delay` rewards are zero
    _, r, _, _ = env2.step(o0)                                        # reward compares with the obs `delay` steps back
    assert r == 1
