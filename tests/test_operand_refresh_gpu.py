"""Every network's fp16 operand refresh, eagerly and replayed from a CUDA graph: after random fp32 master weights, each
fp16 operand equals the torch cast of its master bit for bit (padding zero), the pixel-shuffle operands wdg equal an
eager ops.dgrad_weights, and the refresh is 1 + (convs with wdg) library launches, the first one included.  The
expected operands come from the layer layouts, not from the networks' cast declarations; dropping any one cast from a
plan must show."""
import gc
from collections import namedtuple

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)

# name -> (ob_shape, uint8 observations, action space, network, value_network, network kwargs)
PPO = {
    "cnn_shared": ((84, 84, 4), True, ("cat", 6), "cnn", None, {}),
    "cnn_copy": ((84, 84, 4), True, ("cat", 6), "cnn", "copy", {}),
    "cnn_implicit_copy": ((64, 64, 4), True, ("cat", 6), "cnn", "copy", {}),
    "mlp_copy_fuse0": ((17,), False, ("gauss", 6), "mlp", "copy", {}),
    "mlp_identity_head": ((5,), False, ("cat", 8), "mlp", None, dict(num_hidden=8)),
    "lstm": ((7,), False, ("cat", 4), "lstm", None, dict(nlstm=64)),
    "cnn_lstm": ((84, 84, 4), True, ("cat", 6), "cnn_lstm", None, {}),
    "mlp_layer_norm_copy": ((9,), False, ("cat", 3), "mlp", "copy", dict(layer_norm=True)),
}
# name -> (ob_shape, network, QNet kwargs, param_noise)
DQN = {
    "mlp_dueling_param_noise": ((8,), "mlp", dict(dueling=True), True),
    "mlp_layer_norm": ((8,), "mlp", dict(dueling=False, layer_norm=True), False),
    "cnn_dueling_param_noise": ((84, 84, 4), "cnn", dict(dueling=True), True),
    "cnn_implicit": ((64, 64, 4), "cnn", dict(dueling=False), False),
    "conv_only_dueling": ((84, 84, 4), "conv_only", dict(dueling=True), False),
}

# one refresh of something that owns fp16 operands: what it reads, how it refreshes, what it must produce, the library
# launches one refresh makes, and where its plan lives
Subject = namedtuple("Subject", "name params refresh expect launches owner plan_attr jobs")


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def _cast(w, scale=1.0):
    return (w * torch.tensor(scale, dtype=torch.float32, device=w.device)).half()


def _fwd(l):
    """w_fwd [N, Kf]: W^T (both halves of a split_in layer's [hi | lo] input), zero elsewhere."""
    e = torch.zeros(l.N, l.Kf, dtype=torch.float16, device=DEV)
    wt = _cast(l.w, l.in_scale).t()
    e[:, :l.K] = wt
    if l.split_in:
        e[:, l.Kp:l.Kp + l.K] = wt
    return e


def _linear(l, name):
    bwd = torch.zeros(l.K, l.Np, dtype=torch.float16, device=DEV)
    bwd[:, :l.N] = _cast(l.w, l.in_scale)
    return [(name + ".w_fwd", l.w_fwd, _fwd(l)), (name + ".w_bwd", l.w_bwd, bwd)]


def _tower(t, name):
    from baselines_b200 import ops
    out = []
    for l in t.layers:
        out += _linear(l, f"{name}.{l.name}")
    for c in t.convs:
        if c.wdg is not None:
            ref = torch.zeros_like(c.wdg)
            ops.dgrad_weights(c.w, ref, c.rf, c.rf, c.C, c.nf, c.stride, c.ld_wdg)
            out.append((f"{name}.{c.name}.wdg", c.wdg, ref))
    if t.shift_mode:
        for c, g, wd in zip(t.convs[1:], t.sg[1:], t.wd[1:]):
            taps = g["k"] * g["k"]                      # tap blocks of the master weight side by side
            e = c.w.view(taps, g["Cg"], c.nf).permute(1, 0, 2).reshape(g["Cg"], taps * c.nf).half()
            out.append((f"{name}.{c.name}.wd", wd, e))
    if t.lstm is not None:
        out += _linear(t.lstm.wx, f"{name}.lstm.wx")
        out += [(f"{name}.lstm.wh16", t.lstm.wh16, t.lstm.wh.half()),
                (f"{name}.lstm.whT16", t.lstm.whT16, t.lstm.wh.t().half())]
    return out


def _policy_expect(net):
    out = _tower(net.tower_pi, "pi") + (_tower(net.tower_vf, "vf") if net.tower_vf else [])
    heads = [net.head] if net.head is not None else [net.head_pi, net.head_vf]
    for h in heads:
        out += _linear(h, h.name)
    if net.fuse0:
        a, b = net.tower_pi.fcs[0], net.tower_vf.fcs[0]
        out += [("w0cat", net.w0cat, torch.cat([_fwd(a), _fwd(b)])), ("b0cat", net.b0cat, torch.cat([a.b, b.b]))]
    return out


def _qnet_expect(q):
    out = _tower(q.trunk, "trunk")
    cat = torch.zeros_like(q.w_cat_bwd)
    for si, layers in enumerate(q.streams):
        for l in layers:
            out += _linear(l, l.name)
        l0, o = layers[0], q.cat_off[si]
        cat[:, o:o + l0.N] = l0.w.half()
    return out + [("w_cat_bwd", q.w_cat_bwd, cat)]


def _copy_expect(c):
    return [(f"{c.scope}.{l.name}.w_fwd", l.w_fwd, _fwd(l)) for layers in c.streams for l in layers]


def _nwdg(*towers):
    return sum(c.wdg is not None for t in towers if t is not None for c in t.convs)


def _launches_of(fn):
    from baselines_b200 import _lib
    before = _lib.LAUNCHES
    out = fn()
    return out, _lib.LAUNCHES - before


def _ppo_subjects(name):
    from baselines_b200.common import spaces
    from baselines_b200.common.policies import PolicyBuilder, PolicyNet
    ob_shape, u8, (ak, na), kind, vf, kw = PPO[name]
    ob = spaces.Box(0, 255, ob_shape, np.uint8) if u8 else spaces.Box(-5, 5, ob_shape, np.float32)
    ac = spaces.Discrete(na) if ak == "cat" else spaces.Box(-1, 1, (na,), np.float32)
    np.random.seed(0)
    net, first = _launches_of(lambda: PolicyNet(PolicyBuilder(ob, ac, kind, value_network=vf, **kw), 16, DEV))
    n = 1 + _nwdg(net.tower_pi, net.tower_vf)
    assert first == n                                 # construction launches nothing but its refresh
    assert net.fuse0 == (name == "mlp_copy_fuse0") and net.pi_identity == (name == "mlp_identity_head")
    return [Subject(name, net.store.params, net.refresh, lambda: _policy_expect(net), n, net, "cast_plan",
                    net.cast_jobs())]


def _dqn_subjects(name):
    from baselines_b200.deepq.build_graph import ParamNoise, QNet
    ob_shape, kind, kw, pn = DQN[name]
    q, first = _launches_of(lambda: QNet(ob_shape, 5, kind, 16, DEV, np.random.RandomState(1), **kw))
    n = 1 + _nwdg(q.trunk)
    assert first == n
    subs = [Subject(name, q.store.params, q.refresh, lambda: _qnet_expect(q), n, q, "cast_plan", q.cast_jobs())]
    if pn:
        p = ParamNoise(q, 5)
        for c in (p.perturbed, p.adaptive):
            subs.append(Subject(f"{name}.{c.scope}", c.params, lambda c=c: c.cast.run(), lambda c=c: _copy_expect(c), 1,
                                c, "cast", c.cast_jobs()))
    return subs


def _subjects(case):
    kind, name = case.split(":")
    return _ppo_subjects(name) if kind == "ppo" else _dqn_subjects(name)


CASES = [f"ppo:{k}" for k in PPO] + [f"dqn:{k}" for k in DQN]


def _randomise(s, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    s.params.copy_(torch.randn(s.params.shape, generator=g, device=DEV))


def _stale(s):
    """Names of the operands that differ from the cast of their masters."""
    exp = s.expect()
    torch.cuda.synchronize()
    return [nm for nm, got, e in exp if got.shape != e.shape or not torch.equal(_bits(got), _bits(e))]


@pytest.mark.parametrize("case", CASES)
def test_refresh_writes_every_operand(case):
    for s in _subjects(case):
        _randomise(s, 1)
        _, n = _launches_of(s.refresh)
        assert n == s.launches, (s.name, n)
        assert _stale(s) == [], s.name
        # the same refresh captured once and replayed over new masters
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        gc.disable()
        try:
            with torch.cuda.graph(graph):
                _, n = _launches_of(s.refresh)
        finally:
            gc.enable()
        assert n == s.launches, (s.name, n)
        for seed in (2, 3):
            _randomise(s, seed)
            graph.replay()
            assert _stale(s) == [], (s.name, seed)


@pytest.mark.parametrize("case", CASES)
def test_dropping_any_cast_shows(case):
    from baselines_b200 import ops
    for s in _subjects(case):
        full = getattr(s.owner, s.plan_attr)
        assert full.n == len(s.jobs)
        for i in range(len(s.jobs)):
            setattr(s.owner, s.plan_attr, ops.CastPlan(s.jobs[:i] + s.jobs[i + 1:], DEV))
            _randomise(s, 10 + i)
            s.refresh()
            assert _stale(s), f"{s.name}: the plan without job {i} still passes the operand check"
        setattr(s.owner, s.plan_attr, full)
        _randomise(s, 1)
        s.refresh()
        assert _stale(s) == [], s.name
