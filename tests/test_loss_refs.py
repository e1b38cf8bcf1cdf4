"""CPU self-test of the float64 references in tests/_loss_refs.py: gradients against float64 central differences,
values and gradients against the oracle's formulation (oracle/nets.py), and each mutant differing from the reference
where it should."""
import math

import numpy as np
import pytest
import torch

import _loss_refs as lr
from oracle import nets


def _loss(ref, ent_coef, vf_coef):
    return ref.stats[0] - ent_coef * ref.stats[2] + vf_coef * ref.stats[1]


def _ppo_case(pd, B=8, n=5, seed=0, clip=0.2):
    """Rows away from every branch boundary (ratio, value clip, l1 vs l2), so central differences are exact to h^2."""
    rng = np.random.RandomState(seed)
    head = rng.randn(B, n) * 1.2
    v = rng.randn(B)
    logstd = rng.randn(n) * 0.3 if pd == "gauss" else None
    acts = (head + rng.randn(B, n) * np.exp(logstd)) if pd == "gauss" else rng.randint(0, n, B)
    nlp = lr.ppo_ref(pd, head, v, acts, np.zeros(B), np.zeros(B), np.zeros(B), np.zeros(B), clip, 0, 0,
                     logstd=logstd).nlp
    r = np.array([0.6, 1.0, 1.4, 0.9, 0.7, 1.1, 1.35, 1.05])[:B]            # below / inside / above the interval
    oldnlp = nlp + np.log(r)
    oldv = v - np.array([0.05, 0.5, -0.6, 0.1, -0.9, 0.4, 0.0, 1.1])[:B]       # unclipped and both clipped sides
    R = oldv + np.array([1.0, -1.5, 1.2, -0.8, 2.0, 3.0, -1.1, -2.0])[:B]
    adv = np.array([1.0, -1.0, 0.5, -2.0, 1.5, -0.7, 1.2, 0.9])[:B]
    return head, v, acts, R, oldv, oldnlp, adv, logstd


@pytest.mark.parametrize("pd", ["cat", "gauss"])
def test_ppo_ref_gradients_match_central_differences(pd):
    clip, ent, vfc = 0.2, 0.3, 0.5
    head, v, acts, R, oldv, oldnlp, adv, logstd = _ppo_case(pd)
    ref = lr.ppo_ref(pd, head, v, acts, R, oldv, oldnlp, adv, clip, ent, vfc, logstd=logstd)
    assert not ref.near.any()
    for z in ("ratio_below", "ratio_inside", "ratio_above", "v_unclipped", "v_low", "v_high", "l1_lt_l2"):
        assert ref.zones[z].any(), z
    f = lambda hd, vv, ls: _loss(lr.ppo_ref(pd, hd, vv, acts, R, oldv, oldnlp, adv, clip, ent, vfc, logstd=ls),
                                 ent, vfc)
    h = 1e-6
    fd = np.zeros_like(head)
    for idx in np.ndindex(*head.shape):
        e = np.zeros_like(head)
        e[idx] = h
        fd[idx] = (f(head + e, v, logstd) - f(head - e, v, logstd)) / (2 * h)
    assert np.allclose(ref.dhead, fd, rtol=1e-6, atol=1e-7)
    fdv = np.array([(f(head, v + h * np.eye(len(v))[i], logstd) - f(head, v - h * np.eye(len(v))[i], logstd)) / (2 * h)
                    for i in range(len(v))])
    assert np.allclose(ref.dv, fdv, rtol=1e-6, atol=1e-7)
    if pd == "gauss":
        fdl = np.array([(f(head, v, logstd + h * np.eye(len(logstd))[j]) - f(head, v, logstd - h * np.eye(len(logstd))[j]))
                        / (2 * h) for j in range(len(logstd))])
        assert np.allclose(ref.dlogstd_rows.sum(0), fdl, rtol=1e-6, atol=1e-7)


@pytest.mark.parametrize("pd", ["cat", "gauss"])
def test_ppo_ref_matches_oracle_loss(pd):
    """The same loss written with oracle/nets.py's distributions and torch.maximum (ppo_loss of nets, mean scaling):
    away from ties the two agree, in value and gradient."""
    clip, ent, vfc = 0.2, 0.3, 0.5
    head, v, acts, R, oldv, oldnlp, adv, logstd = _ppo_case(pd)
    ref = lr.ppo_ref(pd, head, v, acts, R, oldv, oldnlp, adv, clip, ent, vfc, logstd=logstd)
    B = head.shape[0]
    t = lambda x: torch.tensor(np.asarray(x), dtype=torch.float64)
    mt, vp = t(head).requires_grad_(True), t(v).requires_grad_(True)
    lst = t(logstd)[None].requires_grad_(True) if pd == "gauss" else None
    if pd == "gauss":
        nl, H = nets.gauss_neglogp(mt, lst, t(acts)), nets.gauss_entropy(mt, lst).mean()
    else:
        nl, H = nets.cat_neglogp(mt, torch.tensor(acts)), nets.cat_entropy(mt).mean()
    A, Rt, OV, ONLP = t(adv), t(R), t(oldv), t(oldnlp)
    vclip = OV + torch.clamp(vp - OV, -clip, clip)
    vf = 0.5 * torch.maximum((vp - Rt) ** 2, (vclip - Rt) ** 2).mean()
    ratio = torch.exp(ONLP - nl)
    pg = torch.maximum(-A * ratio, -A * torch.clamp(ratio, 1 - clip, 1 + clip)).mean()
    loss = pg - H * ent + vf * vfc
    loss.backward()
    want = [float(x.detach()) for x in (pg, vf, H, 0.5 * ((nl - ONLP) ** 2).mean(),
                                        ((ratio - 1).abs() > clip).double().mean())]
    assert np.allclose(ref.stats / B, want, rtol=1e-12, atol=1e-14)
    assert np.allclose(ref.dhead / B, mt.grad.numpy(), rtol=1e-12, atol=1e-14)
    assert np.allclose(ref.dv / B, vp.grad.numpy(), rtol=1e-12, atol=1e-14)
    if pd == "gauss":
        assert np.allclose(ref.dlogstd_rows.sum(0) / B, lst.grad.numpy()[0], rtol=1e-12, atol=1e-14)


def test_ppo_ref_mutants_differ_where_they_should():
    clip, ent, vfc = 0.2, 0.3, 0.5
    head, v, acts, R, oldv, oldnlp, adv, _ = _ppo_case("cat")
    ref = lr.ppo_ref("cat", head, v, acts, R, oldv, oldnlp, adv, clip, ent, vfc)
    z = ref.zones
    mut = lambda m: lr.ppo_ref("cat", head, v, acts, R, oldv, oldnlp, adv, clip, ent, vfc, mutant=m)
    # clipped surrogate active outside the interval: (adv > 0, ratio above) and (adv < 0, ratio below)
    active = (z["adv_pos"] & z["ratio_above"]) | (z["adv_neg"] & z["ratio_below"])
    assert active.any()
    diff = np.abs(mut("pg_clip_passes").dhead - ref.dhead).max(1) > 0
    assert np.array_equal(diff, active)
    vdiff = np.abs(mut("vf_wrong_branch").dv - ref.dv) > 0
    assert vdiff.any() and not vdiff[z["v_unclipped"]].any()
    vdiff = np.abs(mut("vf_clip_passes").dv - ref.dv) > 0
    assert np.array_equal(vdiff, ~z["v_unclipped"] & z["l1_lt_l2"])
    assert np.abs(mut("no_entropy").dhead - ref.dhead).max() > 1e-3


def test_mcat_drop_last_entropy_mutant():
    rng = np.random.RandomState(1)
    nvec = [2, 3]
    head = rng.randn(4, 5)
    acts = np.stack([rng.randint(0, n, 4) for n in nvec], 1)
    z = np.zeros(4)
    full = lr.ppo_ref("mcat", head, z, acts, z, z, z, z, 0.2, 1.0, 0.0, nvec=nvec)
    drop = lr.ppo_ref("mcat", head, z, acts, z, z, z, z, 0.2, 1.0, 0.0, nvec=nvec, mutant="drop_last_entropy")
    assert np.allclose(full.dhead[:, :2], drop.dhead[:, :2]) and not np.allclose(full.dhead[:, 2:], drop.dhead[:, 2:])


@pytest.mark.parametrize("double_q", [True, False])
@pytest.mark.parametrize("dueling", [True, False])
def test_dqn_ref_matches_central_differences_and_oracle(double_q, dueling):
    rng = np.random.RandomState(2)
    B, nA, gamma = 7, 4, 0.9
    qa, on_a, tg_a = rng.randn(B, nA) * 2, rng.randn(B, nA), rng.randn(B, nA)
    qs, on_s, tg_s = (rng.randn(B), rng.randn(B), rng.randn(B)) if dueling else (None, None, None)
    act, rew = rng.randint(0, nA, B), rng.randn(B)
    done, w = (rng.rand(B) < 0.3).astype(float), rng.rand(B) + 0.1
    ref = lr.dqn_ref(qa, qs, on_a, on_s, tg_a, tg_s, act, rew, done, w, gamma, double_q)
    assert np.any(np.abs(ref.td) < 1) and np.any(np.abs(ref.td) > 1)
    f = lambda a, s: lr.dqn_ref(a, s, on_a, on_s, tg_a, tg_s, act, rew, done, w, gamma, double_q).loss
    h = 1e-6
    fd = np.zeros_like(qa)
    for idx in np.ndindex(*qa.shape):
        e = np.zeros_like(qa)
        e[idx] = h
        fd[idx] = (f(qa + e, qs) - f(qa - e, qs)) / (2 * h)
    assert np.allclose(ref.d_a, fd, rtol=1e-6, atol=1e-7)
    if dueling:
        fds = np.array([(f(qa, qs + h * np.eye(B)[i]) - f(qa, qs - h * np.eye(B)[i])) / (2 * h) for i in range(B)])
        assert np.allclose(ref.d_s, fds, rtol=1e-6, atol=1e-7)
    # oracle/nets.py: DQNOracle.td_and_loss's target and nets.huber
    t = lambda x: torch.tensor(np.asarray(x), dtype=torch.float64)
    q = lambda a, s: lr.dueling_q(t(a), None if s is None else t(s))
    q_tg = q(tg_a, tg_s)
    best = q_tg.gather(1, q(on_a, on_s).argmax(1, keepdim=True))[:, 0] if double_q else q_tg.max(1).values
    td = q(qa, qs).gather(1, torch.tensor(act)[:, None])[:, 0] - (t(rew) + gamma * (1 - t(done)) * best)
    assert np.allclose(ref.td, td.numpy(), rtol=1e-14, atol=1e-14)
    assert math.isclose(ref.loss, float((t(w) * nets.huber(td)).sum()), rel_tol=1e-14)


def test_dqn_ref_argmax_tie_takes_the_first_index():
    on_a = np.array([[2.0, 5.0, 5.0, 1.0]])
    tg_a = np.array([[0.0, 1.0, 3.0, -2.0]])
    args = (np.zeros((1, 4)), None, on_a, None, tg_a, None, [0], [0.0], [0.0], [1.0], 0.5, True)
    assert lr.dqn_ref(*args).td[0] == -0.5                     # target 0.5 * q_tg[1]
    assert lr.dqn_ref(*args, mutant="last_max").td[0] == -1.5  # target 0.5 * q_tg[2]


def test_adam_and_moments_helpers():
    rng = np.random.RandomState(3)
    p, g = rng.randn(50), rng.randn(50) * 1e-3
    m, v = np.zeros(50), np.zeros(50)
    pt, mt, vt = torch.tensor(p), torch.tensor(m), torch.tensor(v)
    for t in range(1, 4):
        lr_t = 1e-3 * math.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t)
        p, m, v = lr.adam_tf(p, g * t, m, v, lr_t, 0.9, 0.999, 1e-5)
        pt, mt, vt = nets.adam_tf(pt, torch.tensor(g * t), mt, vt, t, 1e-3, eps=1e-5)
    assert np.allclose(p, pt.numpy(), rtol=1e-14) and np.allclose(m, mt.numpy(), rtol=1e-14)
    assert np.allclose(v, vt.numpy(), rtol=1e-14)
    R, V = rng.randn(1000).astype(np.float32), rng.randn(1000).astype(np.float32)
    mean, std = lr.adv_moments(R, V)
    d = (R - V).astype(np.float64)
    assert math.isclose(mean, d.mean(), rel_tol=1e-13) and math.isclose(std, d.std(), rel_tol=1e-13)
    assert lr.clip_scale(25.0, 5.0) == 1.0 and lr.clip_scale(100.0, 5.0) == 0.5 and lr.clip_scale(1e9, 0.0) == 1.0


def test_philox_helper_known_answers_and_uniform_layout():
    """Philox4x32-10 known-answer vectors (Salmon et al., SC'11, Random123 kat_vectors), then the u01 mapping."""
    got = lr.philox4x32_10(0, [0], 0, 0)[0]
    assert [int(v) for v in got] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    c = 0xFFFFFFFF
    got = lr.philox4x32_10(c | (c << 32), [c | (c << 32)], c, c)[0]
    assert [int(v) for v in got] == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]
    u = lr.philox_uniforms(7, 3, 6, 2)
    w = lr.philox4x32_10(7, [1], 1, 2)[0]
    assert u[1, 5] == np.float32(((int(w[1]) >> 8) + 0.5) / 2 ** 24)
    assert u.dtype == np.float32 and (u > 0).all() and (u < 1).all()


def test_dqn_act_draws_helper():
    u, r = lr.dqn_act_draws(123, 4, 64, 6)
    assert ((u > 0) & (u < 1)).all() and ((r >= 0) & (r < 6)).all()
    u2, r2 = lr.dqn_act_draws(123, 5, 64, 6)
    assert not np.array_equal(r, r2)                     # the stream moves with the step
