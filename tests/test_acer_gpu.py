"""ACER on the GPU: each kernel against exact or float64 restatements, whole train steps against the float64 mirror
(tests/_acer_refs.py), graph replay, determinism, checkpoints, the CLI and the reference's CartPole learning test."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import _acer_refs as AR
from baselines_b200 import ops
from baselines_b200.acer import acer as A
from baselines_b200.acer.buffer import Segment
from baselines_b200.common import spaces
from baselines_b200.common.policies import build_policy

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
dev = "cuda"


def test_acer_step_samples_the_cat_step_bits_and_mu_is_softmax():
    rng = np.random.RandomState(0)
    for nA in (2, 6, 18):
        B = 4099
        logits = torch.from_numpy(rng.randn(B, nA).astype(np.float32) * 3).to(dev)
        a1 = torch.zeros(B, dtype=torch.int64, device=dev)
        a2 = torch.zeros(B, dtype=torch.int64, device=dev)
        mu = torch.zeros(B, nA, device=dev)
        v, nlp = torch.zeros(B, device=dev), torch.zeros(B, device=dev)
        for off in (0, 7):
            ops.acer_step(logits, nA, nA, a1, mu, B, seed=1234, offset=off)
            ops.cat_step(logits, nA, nA, logits, nA, a2, v, nlp, B, seed=1234, offset=off)
            assert torch.equal(a1, a2)
        np.testing.assert_allclose(mu.cpu().numpy(), AR.softmax(logits.cpu().numpy()), rtol=2e-6, atol=1e-7)
    # frequencies of one row sampled many times
    nA, B = 6, 200000
    row = np.array([0.5, -1.0, 2.0, 0.0, 1.0, -3.0], np.float32)
    logits = torch.from_numpy(np.tile(row, (B, 1))).to(dev)
    a = torch.zeros(B, dtype=torch.int64, device=dev)
    ops.acer_step(logits, nA, nA, a, mu.new_zeros(B, nA), B, seed=9)
    freq = np.bincount(a.cpu().numpy(), minlength=nA) / B
    p = AR.softmax(row)
    assert np.abs(freq - p).max() < 5 * np.sqrt(p.max() / B)


def _ring(rng, slots, nenv, T, nstack, frame, nc, dtype):
    seg = Segment(slots, nenv, T, nstack, frame, nc, dtype, 3, dev)
    shape = seg.enc_obs.shape
    host = rng.randint(0, 256, shape).astype(np.uint8) if dtype == np.uint8 else \
        rng.randn(*shape).astype(np.float32)
    seg.enc_obs.copy_(torch.from_numpy(host))
    d = rng.rand(slots, nenv, T) < 0.25
    d[:, :, 0] |= rng.rand(slots, nenv) < 0.5
    d[:, :, -1] |= rng.rand(slots, nenv) < 0.5
    seg.dones.copy_(torch.from_numpy(d.astype(np.uint8)))
    return seg, host, d


@pytest.mark.parametrize("nstack,nc,dtype,frame,nenv", [(4, 1, np.uint8, (5, 3), 3), (1, 4, np.float32, (), 5),
                                                         (4, 2, np.float32, (3,), 2), (3, 1, np.uint8, (2, 2), 4),
                                                         (4, 1, np.uint8, (84, 84), 16)])
def test_stack_obs_bit_for_bit(nstack, nc, dtype, frame, nenv):
    rng = np.random.RandomState(nstack * 10 + nc)
    T, slots = 20, 7
    seg, host, d = _ring(rng, slots, nenv, T, nstack, frame, nc, dtype)
    idx = rng.randint(0, slots, nenv)
    idx[0] = slots - 1                                         # the slot written last before the ring wraps
    out = torch.zeros((nenv * (T + 1),) + frame + (nstack * nc,), dtype=seg.enc_obs.dtype, device=dev)
    ops.acer_stack_obs(seg.enc_obs, torch.from_numpy(idx).to(dev), nenv, T, nstack, seg.dones, out)
    enc = np.stack([host[idx[e], e] for e in range(nenv)])
    dn = np.stack([d[idx[e], e] for e in range(nenv)])
    want = AR.stack_obs(enc, dn, T).reshape(out.shape)
    got = out.cpu().numpy()
    assert got.tobytes() == want.tobytes()


def _head_case(rng, nenv, T, nA, mu_tiny=False, big_q=False):
    R = nenv * (T + 1)
    pi = (rng.randn(R, nA) * 2).astype(np.float32)
    q = (rng.randn(R, nA) * (30 if big_q else 1)).astype(np.float32)
    pol = (pi + rng.randn(R, nA) * 0.5).astype(np.float32)
    a = rng.randint(0, nA, nenv * T)
    r = rng.randn(nenv * T).astype(np.float32)
    dn = rng.rand(nenv, T) < 0.2
    dn[0, 0] = dn[min(1, nenv - 1), T - 1] = True
    mus = AR.softmax(rng.randn(nenv * T, nA) * 2).astype(np.float32)
    if mu_tiny:
        mus[np.arange(0, nenv * T, 3), a[::3]] = 1e-9             # rho far above c
    return pi, q, pol, a, r, dn.reshape(-1), mus


def _run_head(case, nenv, T, nA, tr, delta=1.0):
    pi, q, pol, a, r, dn, mus = case
    R = nenv * (T + 1)
    t = lambda x, dt=torch.float32: torch.from_numpy(np.ascontiguousarray(x)).to(dev, dt)
    dpi = torch.zeros(R, nA, dtype=torch.float16, device=dev)
    dq = torch.zeros(R, nA, dtype=torch.float16, device=dev)
    st = torch.zeros(12, dtype=torch.float64, device=dev)
    f = torch.zeros(R, nA, device=dev)
    v = torch.zeros(R, device=dev)
    qret = torch.zeros(nenv * T, device=dev)
    ops.acer_loss(t(pi), nA, t(q), nA, t(pol), nA, t(a, torch.int64), t(r), t(dn.astype(np.uint8), torch.uint8),
                  t(mus), nenv, T, nA, 0.99, 10.0, delta, 0.5, 0.01, tr, dpi, nA, dq, nA, st, f, v, qret)
    return (dpi.float().cpu().numpy(), dq.float().cpu().numpy(), st.cpu().numpy(), f.cpu().numpy(),
            v.cpu().numpy(), qret.cpu().numpy())


@pytest.mark.parametrize("nA", [2, 6, 18])
@pytest.mark.parametrize("tr", [True, False])
def test_loss_head_against_float64(nA, tr):
    rng = np.random.RandomState(nA + 100 * tr)
    nenv, T = 16, 20
    mutants = [dict(bc_drop_f=True), dict(shift_dones=True)] + ([dict(no_adj_max=True)] if tr else [])
    caught = [False] * len(mutants)
    for kw in (dict(), dict(mu_tiny=True), dict(big_q=True)):
        case = _head_case(rng, nenv, T, nA, **kw)
        delta = 0.05 if kw.get("big_q") else 1.0
        dpi, dq, st, f, v, qret = _run_head(case, nenv, T, nA, tr, delta=delta)
        ref = AR.head(*case, nenv, T, trust_region=tr, delta=delta)
        if tr and kw.get("big_q"):
            assert (ref.adj > 0).any() and (ref.adj == 0).any()
        tol_pi = 3e-3 * (np.abs(ref.dpi).max() + 1e-3)
        tol_q = 3e-3 * (np.abs(ref.dq).max() + 1e-3)
        np.testing.assert_allclose(dpi, ref.dpi, atol=tol_pi, rtol=2e-3)
        np.testing.assert_allclose(dq, ref.dq, atol=tol_q, rtol=2e-3)
        np.testing.assert_allclose(st, ref.stats, rtol=2e-4, atol=1e-5)
        # the mistakes a port tends to make fall outside these bounds in at least one of the cases
        for i, mut in enumerate(mutants):
            m = AR.head(*case, nenv, T, trust_region=tr, delta=delta, **mut)
            caught[i] |= bool(np.abs(m.dpi - dpi).max() > tol_pi + 2e-3 * np.abs(dpi).max()
                              or np.abs(m.dq - dq).max() > tol_q + 2e-3 * np.abs(dq).max()
                              or not np.allclose(st, m.stats, rtol=2e-4, atol=1e-5))
    assert all(caught), [m for m, c in zip(mutants, caught) if not c]


def test_retrace_bit_for_bit_in_float32():
    rng = np.random.RandomState(3)
    nenv, T, nA = 8, 20, 6
    case = _head_case(rng, nenv, T, nA, mu_tiny=True)
    _, _, _, f, v, qret = _run_head(case, nenv, T, nA, True)
    pi, q, pol, a, r, dn, mus = case
    f32 = np.float32
    F, Q = f.reshape(nenv, T + 1, nA), q.reshape(nenv, T + 1, nA)
    V = np.zeros((nenv, T + 1), f32)
    for j in range(nA):
        V = V + F[..., j] * Q[..., j]
    assert V.reshape(-1).tobytes() == v.tobytes()
    A_ = a.reshape(nenv, T)
    q_i = np.take_along_axis(Q[:, :T], A_[..., None], -1)[..., 0]
    f_i = np.take_along_axis(F[:, :T], A_[..., None], -1)[..., 0]
    mu_i = np.take_along_axis(mus.reshape(nenv, T, nA), A_[..., None], -1)[..., 0]
    rho_i = f_i / (mu_i + f32(1e-6))
    R_, D = r.reshape(nenv, T), dn.reshape(nenv, T).astype(f32)
    qr = V[:, T].copy()
    out = np.zeros((nenv, T), f32)
    for i in range(T - 1, -1, -1):
        qr = R_[:, i] + f32(0.99) * qr * (f32(1.0) - D[:, i])
        out[:, i] = qr
        qr = (np.minimum(f32(1.0), rho_i[:, i]) * (qr - q_i[:, i])) + V[:, i]
    assert out.reshape(-1).tobytes() == qret.tobytes()


@pytest.mark.parametrize("clip,ms0", [(0.0, "ones"), (1e6, "ones"), (0.5, "ones"), (0.0, "small")])
def test_clip_rmsprop_ema_against_float64(clip, ms0):
    rng = np.random.RandomState(4)
    n = 100003
    p, g, sh = (rng.randn(n).astype(np.float32) for _ in range(3))
    # "small": slots of a long run with small gradients, where eps is not negligible against ms
    ms = np.ones(n, np.float32) if ms0 == "ones" else (10.0 ** rng.uniform(-6, -3, n)).astype(np.float32)
    if ms0 == "small":
        g *= np.float32(1e-3)
    t = lambda x: torch.from_numpy(x.copy()).to(dev)
    P, G, M, S = t(p), t(g), t(ms), t(sh)
    lr = torch.tensor([7e-4], dtype=torch.float32, device=dev)
    ss = torch.zeros(1, dtype=torch.float64, device=dev)
    ops.sumsq(G, ss)
    ops.clip_rmsprop_ema(P, G, M, S, lr, clip, ss, 0.99, 1e-5, 0.99)
    rp, rms, rsh = AR.rmsprop_ema(p, g, ms, sh, float(np.float32(7e-4)), clip)
    for got, want in ((P, rp), (M, rms), (S, rsh)):
        np.testing.assert_allclose(got.cpu().numpy(), want, rtol=2e-6, atol=2e-7)
    # the moving average taken before the step (visible where the step is not clipped to a tiny one), and ms starting
    # at 0, fall outside these bounds
    if clip != 0.5:
        _, _, bsh = AR.rmsprop_ema(p, g, ms, sh, float(np.float32(7e-4)), clip, ema_first=True)
        assert not np.allclose(S.cpu().numpy(), bsh, rtol=2e-6, atol=2e-7)
    if ms0 == "ones":
        bp, bms, _ = AR.rmsprop_ema(p, g, np.zeros(n), sh, float(np.float32(7e-4)), clip)
        assert not np.allclose(P.cpu().numpy(), bp, rtol=2e-6, atol=2e-7)
        assert not np.allclose(M.cpu().numpy(), bms, rtol=2e-6, atol=2e-7)
    else:                                         # eps outside the square root
        bp, _, _ = AR.rmsprop_ema(p, g, ms, sh, float(np.float32(7e-4)), clip, eps_outside=True)
        assert not np.allclose(P.cpu().numpy(), bp, rtol=2e-6, atol=2e-7)


class _Env:
    def __init__(self, ob, nA, n):
        self.observation_space, self.action_space, self.num_envs = ob, spaces.Discrete(nA), n


def _model(kind, copy, nenv, T, nA, tr=True, ob=None, seed=0, delta=1, **kw):
    np.random.seed(seed)
    torch.manual_seed(seed)
    ob = ob or (spaces.Box(0, 255, (84, 84, 4), np.uint8) if kind == "cnn" else spaces.Box(-1, 1, (5,), np.float32))
    pol = build_policy(_Env(ob, nA, nenv), kind, value_network="copy" if copy else None, estimate_q=True, **kw)
    return A.Model(policy=pol, ob_space=ob, ac_space=spaces.Discrete(nA), nenvs=nenv, nsteps=T, ent_coef=0.01,
                   q_coef=0.5, gamma=0.99, max_grad_norm=10, lr=7e-4, rprop_alpha=0.99, rprop_epsilon=1e-5,
                   total_timesteps=10000, lrschedule='linear', c=10.0, trust_region=tr, alpha=0.99, delta=delta)


def _batch(rng, model, nenv, T, nA):
    R = nenv * (T + 1)
    if model.net.tower_pi.in_u8:
        obs = rng.randint(0, 256, (R,) + model.ob_shape).astype(np.uint8)
    else:
        obs = rng.randn(R, *model.ob_shape).astype(np.float32)
    a = rng.randint(0, nA, nenv * T)
    r = rng.randn(nenv * T).astype(np.float32)
    d = rng.rand(nenv * T) < 0.1
    mus = AR.softmax(rng.randn(nenv * T, nA)).astype(np.float32)
    return obs, a, r, d, mus


@pytest.mark.parametrize("copy", [False, True])
@pytest.mark.parametrize("tr", [True, False])
def test_mlp_train_steps_against_float64(copy, tr):
    nenv, T, nA = 4, 5, 3
    model = _model("mlp", copy, nenv, T, nA, tr)
    rng = np.random.RandomState(7)
    names = list(model.get_params())
    p = model.get_params()
    sh = model.get_polyak_params()
    ms = {k: np.ones_like(v) for k, v in p.items()}
    for call in range(3):
        obs, a, r, d, mus = _batch(rng, model, nenv, T, nA)
        lr = float(np.float32(model.lr.value_steps(call * 40)))
        p1, ms1, sh1, st_ref, _ = AR.train_step(p, sh, ms, obs, a, r, d, mus, nenv, T, lr, copy, trust_region=tr,
                                                names=names)
        names_ops, vals = model.train(obs, a, r, d, mus, None, None, call * 40)
        assert names_ops == A.NAMES + (A.NAMES_TR if tr else [])
        got = model.get_params()
        for k in names:
            dg, dr = got[k] - p[k], p1[k] - p[k]
            assert np.abs(dg - dr).max() <= 0.02 * np.abs(dr).max() + 1e-7, (k, call)
        gsh = model.get_polyak_params()
        for k in names:
            np.testing.assert_allclose(gsh[k], sh1[k], atol=2e-6 + 0.02 * np.abs(sh1[k] - sh[k]).max())
        np.testing.assert_allclose(np.asarray(vals), st_ref[:len(vals)], rtol=0.02, atol=2e-4)
        p, sh, ms = got, gsh, ms1


def _perturb_shadow(model, scale, seed):
    """Move the Polyak shadow visibly away from the parameters (and refresh the Polyak net's fp16 operands)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    p = model.net.store.params
    noise = torch.randn(p.shape, generator=g).to(p.device) * scale * p.abs().mean()
    model.shadow.copy_(p + noise * (p != 0))
    model.polyak.refresh()


def _check_step(model, p, sh, ms, batch, nenv, T, copy, tr, delta, steps, got_vals, names):
    obs, a, r, d, mus = batch
    lr = float(np.float32(model.lr.value_steps(steps)))
    p1, ms1, sh1, st_ref, h = AR.train_step(p, sh, ms, obs, a, r, d, mus, nenv, T, lr, copy, trust_region=tr,
                                            names=names, delta=delta)
    got = model.get_params()
    worst = {}
    for k in names:
        dg, dr = got[k] - p[k], p1[k] - p[k]
        bound = 0.02 * np.abs(dr).max() + 1e-7
        assert np.abs(dg - dr).max() <= bound, k
        worst[k] = bound
    np.testing.assert_allclose(np.asarray(got_vals), st_ref[:len(got_vals)], rtol=0.02, atol=2e-4)
    gsh = model.get_polyak_params()
    for k in names:
        np.testing.assert_allclose(gsh[k], sh1[k], atol=2e-6 + 0.02 * np.abs(sh1[k] - sh[k]).max())
    return got, worst, h


@pytest.mark.parametrize("copy", [False, True])
def test_polyak_network_drives_the_trust_region(copy):
    """With the shadow well apart from the parameters and delta small enough that the constraint binds, the update
    follows f_pol of the Polyak net: the mirror fed the live parameters as the Polyak net (f_pol from the live net, or
    a stale Polyak forward) falls outside the bounds."""
    nenv, T, nA, delta = 4, 5, 3, 0.01
    model = _model("mlp", copy, nenv, T, nA, True, delta=delta)
    _perturb_shadow(model, 0.5, 1)
    rng = np.random.RandomState(17)
    names = list(model.get_params())
    p, sh = model.get_params(), model.get_polyak_params()
    assert max(np.abs(p[k] - sh[k]).max() for k in names) > 0.01
    ms = {k: np.ones_like(v) for k, v in p.items()}
    batch = _batch(rng, model, nenv, T, nA)
    _, vals = model.train(*batch, None, None, 0)
    got, worst, h = _check_step(model, p, sh, ms, batch, nenv, T, copy, True, delta, 0, vals, names)
    assert (h.adj > 0).any()
    lr = float(np.float32(model.lr.value_steps(0)))
    live, _, _, _, _ = AR.train_step(p, p, ms, *batch, nenv, T, lr, copy, trust_region=True, names=names, delta=delta)
    assert any(np.abs((got[k] - p[k]) - (live[k] - p[k])).max() > worst[k] for k in names)


@pytest.mark.parametrize("copy", [False, True])
def test_replay_train_call_against_float64(copy):
    """A replay call (ring + slots from sample_slots) trains on the slots' re-stacked segments, as the mirror does
    with the reference's stacking rule; two replay calls in a row, with the shadow apart from the parameters."""
    from baselines_b200.acer.buffer import Buffer
    nenv, T, nA = 4, 5, 3
    model = _model("mlp", copy, nenv, T, nA, True)
    _perturb_shadow(model, 0.3, 2)

    class Env:
        observation_space, action_space, num_envs, nstack = spaces.Box(-1, 1, (5,), np.float32), \
            spaces.Discrete(nA), nenv, 1
    buf = Buffer(Env, T, size=T * 4)
    rng = np.random.RandomState(5)
    segs = []
    for i in range(6):                                            # 6 puts into 4 slots: the ring has wrapped
        enc = rng.randn(nenv, T + 1, 5).astype(np.float32)
        d = rng.rand(nenv, T) < 0.2
        seg = (enc, rng.randint(0, nA, (nenv, T)), rng.randn(nenv, T).astype(np.float32),
               AR.softmax(rng.randn(nenv, T, nA)).astype(np.float32), d,
               np.concatenate([rng.rand(nenv, 1) < 0.2, d], 1))
        buf.put(*seg)
        segs.append(seg)
    slots = {s: segs[i] for i, s in ((i, i % 4) for i in range(6))}
    names = list(model.get_params())
    p, sh = model.get_params(), model.get_polyak_params()
    ms = {k: np.ones_like(v) for k, v in p.items()}
    np.random.seed(3)
    for call in range(2):
        idx = buf.sample_slots()
        h, s = model.train_device(buf.ring, idx, 40 * call)
        vals = model.values_of(h, s)
        ix = idx.cpu().numpy()
        enc = np.stack([slots[ix[e]][0][e] for e in range(nenv)])
        take = lambda j: np.stack([slots[ix[e]][j][e] for e in range(nenv)])
        obs = AR.stack_obs(enc, take(4), T)
        batch = (obs.reshape(nenv * (T + 1), 5), take(1).reshape(-1), take(2).reshape(-1), take(4).reshape(-1),
                 take(3).reshape(-1, nA))
        p, _, _ = _check_step(model, p, sh, ms, batch, nenv, T, copy, True, 1.0, 40 * call, vals, names)
        sh = model.get_polyak_params()
        ms = _ms_of(model, names)


def _ms_of(model, names):
    """The RMSProp slots in TF naming (the store's second flat buffer)."""
    st = model.net.store
    views = st._views_of(model.ms)
    out = {}
    for tf_name in names:
        internal, sl, shape = st.tf_map[tf_name]
        v = views[internal]
        if sl is not None:
            v = v[..., sl]
        out[tf_name] = v.cpu().numpy().reshape(shape).copy()
    return out


def test_cnn_train_and_polyak_forwards_against_float64():
    """cfg-2 shape (nenv 16, nsteps 20, NatureCNN, nA 6): the train net's [pi | q] and the Polyak net's logits of a
    replayed train call against the float64 network at the parameters and at the (perturbed) shadow."""
    nenv, T, nA = 16, 20, 6
    model = _model("cnn", False, nenv, T, nA)
    _perturb_shadow(model, 0.3, 3)
    rng = np.random.RandomState(9)
    obs, a, r, d, mus = _batch(rng, model, nenv, T, nA)
    p, sh = model.get_params(), model.get_polyak_params()
    model.train(obs, a, r, d, mus, None, None, 0)
    R = nenv * (T + 1)
    pi = model.net.pi_out[:R, :nA].cpu().numpy()
    q = model.net.v_out[:R, :nA].cpu().numpy()
    pol = model.polyak.pi_out[:R, :nA].cpu().numpy()
    with torch.no_grad():
        rpi, rq, _, _ = (t.cpu().numpy() if torch.is_tensor(t) else t for t in AR.acer_net(p, False, obs, kind="cnn",
                                                                                         dev="cuda"))
        rpol = AR.acer_net(sh, False, obs, kind="cnn", dev="cuda")[0].cpu().numpy()
    for got, want in ((pi, rpi), (q, rq), (pol, rpol)):
        np.testing.assert_allclose(got, want, atol=2e-2 * np.abs(want).max(), rtol=0)
    assert np.abs(pol - rpi).max() > 2e-2 * np.abs(rpol).max()


def test_statistics_do_not_change_the_update_and_graph_replay_equals_eager():
    nenv, T, nA = 16, 20, 6
    rng = np.random.RandomState(8)
    batches = [_batch(rng, _model("cnn", False, 1, 1, nA), nenv, T, nA) for _ in range(3)]
    runs = []
    for with_stats, graphs_on in ((True, True), (False, True), (True, False)):
        model = _model("cnn", False, nenv, T, nA)
        os.environ["B200RL_NO_GRAPHS"] = "0" if graphs_on else "1"
        try:
            for i, (obs, a, r, d, mus) in enumerate(batches):
                model.obs_buf.copy_(torch.from_numpy(obs).reshape(model.obs_buf.shape))
                for buf, x in ((model.a_buf, a), (model.r_buf, r), (model.d_buf, d.astype(np.uint8)),
                               (model.mu_buf, mus)):
                    buf.copy_(torch.from_numpy(np.ascontiguousarray(x)).reshape(buf.shape))
                h, s = model.train_device(None, None, i * 320, with_stats=with_stats)
                assert np.isfinite(h.cpu().numpy()).all()
        finally:
            os.environ.pop("B200RL_NO_GRAPHS", None)
        runs.append((model.net.store.params.cpu().numpy(), model.shadow.cpu().numpy(), model.ms.cpu().numpy()))
    for other in runs[1:]:
        for x, y in zip(runs[0], other):
            assert x.tobytes() == y.tobytes()


def _cartpole(nenv=2):
    from baselines_b200.common.cmd_util import make_vec_env
    return make_vec_env('CartPole-v0', 'classic_control', nenv, 0)


def test_two_seeded_learn_runs_are_bit_identical_and_checkpoints_round_trip(tmp_path):
    out = []
    for _ in range(2):
        env = _cartpole()
        m = A.learn('mlp', env, seed=3, total_timesteps=1200, replay_start=200, log_interval=10,
                    value_network='copy')
        out.append((m.net.store.params.cpu().numpy().copy(), m.shadow.cpu().numpy().copy()))
        env.close()
    assert out[0][0].tobytes() == out[1][0].tobytes() and out[0][1].tobytes() == out[1][1].tobytes()
    path = str(tmp_path / "acer.ckpt")
    m.save(path)
    import joblib
    d = joblib.load(path)
    assert "acer_model/q/w:0" in d and "acer_model/pi/w:0" in d and "acer_model/vf/mlp_fc0/w:0" in d
    assert not any("ExponentialMovingAverage" in k or "RMSProp" in k for k in d)
    env = _cartpole()
    m2 = A.learn('mlp', env, seed=4, total_timesteps=0, value_network='copy', load_path=path)
    env.close()
    for k, v in m.get_params().items():
        assert np.array_equal(m2.get_params()[k], v)
    # only trainable variables are saved: the shadow and the RMSProp slots keep their initial values
    assert not np.array_equal(m2.shadow.cpu().numpy(), m2.net.store.params.cpu().numpy())
    assert float(m2.ms.min()) == 1.0 and float(m2.ms.max()) == 1.0


def test_variable_names_order_and_numpy_stream():
    m = _model("mlp", True, 1, 20, 2, seed=0)
    names = list(m.get_params())
    assert names == ['acer_model/pi/mlp_fc0/w:0', 'acer_model/pi/mlp_fc0/b:0', 'acer_model/pi/mlp_fc1/w:0',
                     'acer_model/pi/mlp_fc1/b:0', 'acer_model/vf/mlp_fc0/w:0', 'acer_model/vf/mlp_fc0/b:0',
                     'acer_model/vf/mlp_fc1/w:0', 'acer_model/vf/mlp_fc1/b:0', 'acer_model/pi/w:0',
                     'acer_model/pi/b:0', 'acer_model/q/w:0', 'acer_model/q/b:0']
    assert m.get_params()['acer_model/q/w:0'].shape == (64, 2)
    # the Polyak net draws nothing from numpy's global stream: it continues right after the ortho_init draws
    np.random.seed(0)
    _model("mlp", True, 1, 20, 2, seed=0)
    after = np.random.rand()
    np.random.seed(0)
    build = build_policy(_Env(spaces.Box(-1, 1, (5,), np.float32), 2, 1), "mlp", value_network="copy",
                         estimate_q=True)
    from baselines_b200.common.policies import PolicyNet
    PolicyNet(build, 2, torch.device(dev), rng=np.random, scope="acer_model")
    assert np.random.rand() == after


@pytest.mark.parametrize("env_args", [["--env=CartPole-v0", "--network=mlp", "--value_network=copy",
                                       "--gamma=1.0", "--num_timesteps=3e3"],
                                      ["--env=SyntheticAtari-v0", "--num_env=16", "--num_timesteps=2e4",
                                       "--replay_start=1000", "--buffer_size=4000"]])
def test_cli(env_args, tmp_path):
    cmd = [sys.executable, "-m", "baselines_b200.run", "--alg=acer", "--seed=0",
           f"--save_path={tmp_path / 'acer.ckpt'}"] + env_args
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900,
                       env=dict(os.environ, OPENAI_LOGDIR=str(tmp_path)))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert (tmp_path / "acer.ckpt").exists()


def test_cartpole_learns():
    """common/tests/test_cartpole.py['acer'] as util.reward_per_episode_test runs it: learn on a one-env DummyVecEnv
    of CartPole-v0 seeded 0, then roll out N_TRIALS = 100 episodes through the same DummyVecEnv with model.step."""
    from baselines_b200.common.vec_env import DummyVecEnv
    from baselines_b200.envs import make

    def env_fn():
        e = make('CartPole-v0')
        e.seed(0)
        return e
    env = DummyVecEnv([env_fn])
    model = A.learn('mlp', env, seed=0, total_timesteps=30000, gamma=1.0, value_network='copy')
    rewards = []
    for _ in range(100):
        obs = env.reset()
        ep = 0.0
        while True:
            action = model.step(obs)[0]
            obs, rew, done, _ = env.step(action)
            ep += float(rew[0])
            if done[0]:
                break
        rewards.append(ep)
    env.close()
    assert sum(rewards) / 100 > 100, rewards
