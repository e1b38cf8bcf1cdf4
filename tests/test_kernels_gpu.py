"""GPU parity tests of every C-ABI kernel against the CPU oracle / golden fixtures.

Integer / index / float64 work is bit-exact; fp16-operand GEMM work is compared with an fp32 evaluation
of the SAME fp16-rounded operands (tolerance stated per test)."""
import os

import numpy as np
import pytest
import torch

import _refs

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def ops():
    from baselines_b200 import ops as _ops
    return _ops


@pytest.fixture(autouse=True)
def _fp32_references_without_tf32():
    """fp32 references are true fp32: TF32 is off for torch matmuls and cudnn convolutions."""
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def dev(x, dtype=None):
    t = torch.as_tensor(np.ascontiguousarray(x))
    if dtype is not None:
        t = t.to(dtype)
    return t.cuda()


# ------------------------------------------------------------------------------------------ GAE
def _run_gae(ops, rew, val, dones_before, last_val, last_dones, gamma, lam, variant):
    T, N = rew.shape
    adv = torch.empty(T, N, dtype=torch.float32, device="cuda")
    ret = torch.empty_like(adv)
    ops.gae_scan(dev(rew), dev(val), dev(dones_before.astype(np.uint8)), dev(last_val),
                 dev(last_dones.astype(np.uint8)), adv, ret, gamma, lam, variant)
    torch.cuda.synchronize()
    return adv.cpu().numpy(), ret.cpu().numpy()


@pytest.mark.parametrize("name", ["gae_small.npz", "gae_medium.npz", "gae_two_rollouts.npz", "gae_alldone.npz"])
def test_gae_bit_exact_vs_reference_golden(ops, name):
    from oracle.gae import sf01
    g = np.load(os.path.join(GOLDEN, name))
    T, N, K = int(g["T"]), int(g["N"]), int(g["nrollouts"])
    for k in range(K):
        rew, val = g["REW"][k * T:(k + 1) * T], g["VAL"][k * T:(k + 1) * T]
        dones_before = np.concatenate([g[f"first_dones{k}"][None], g["DONE"][k * T:(k + 1) * T - 1]], 0)
        variants = [0] + ([1] if N % 32 == 0 else [])
        for variant in variants:
            adv, ret = _run_gae(ops, rew, val, dones_before, g["VAL"][(k + 1) * T], g["DONE"][(k + 1) * T - 1],
                                float(g["gamma"]), float(g["lam"]), variant)
            assert np.array_equal(sf01(ret), g[f"returns{k}"]), (name, variant)


@pytest.mark.parametrize("T,N", [(128, 4096), (37, 96), (512, 1024), (5, 7),
                                 (161, 64), (33, 32)])          # T % 32 != 0: the partial chunk comes first
def test_gae_bit_exact_vs_oracle_random(ops, T, N):
    from oracle.gae import gae_reference_order
    rng = np.random.RandomState(T * 1000 + N)
    rew = rng.randn(T, N).astype(np.float32)
    val = rng.randn(T, N).astype(np.float32)
    dones = rng.rand(T, N) < 0.03
    last_val = rng.randn(N).astype(np.float32)
    last_dones = rng.rand(N) < 0.03
    adv_o, ret_o = gae_reference_order(rew, val, dones, last_val, last_dones, 0.99, 0.95)
    for variant in ([0, 1, -1] if N % 32 == 0 else [0, -1]):
        adv, ret = _run_gae(ops, rew, val, dones, last_val, last_dones, 0.99, 0.95, variant)
        assert np.array_equal(adv, adv_o), variant
        assert np.array_equal(ret, ret_o), variant


# ------------------------------------------------------------------------------------------ GEMM
def _gemm_ref(A, B, mn):
    A32, B32 = A.float(), B.float()
    return (A32.t() @ B32) if mn else (A32 @ B32.t())


@pytest.mark.parametrize("M,N,K", [(128, 64, 64), (300, 48, 200), (4096, 512, 3136), (1000, 32, 256),
                                   (777, 64, 576), (129, 16, 512), (2048, 256, 128), (64, 7, 24)])
def test_gemm_kmajor_vs_fp32(ops, M, N, K):
    torch.manual_seed(M + N + K)
    lda = (K + 7) // 8 * 8
    A = torch.zeros(M, lda, dtype=torch.float16, device="cuda")
    B = torch.zeros(N, lda, dtype=torch.float16, device="cuda")
    A[:, :K] = torch.randn(M, K, device="cuda") * 0.5
    B[:, :K] = torch.randn(N, K, device="cuda") * 0.5
    bias = torch.randn(N, device="cuda")
    ref = _gemm_ref(A[:, :K], B[:, :K], False)
    # fp32 store + bias
    ldc = N + 3
    C = torch.full((M, ldc), -7.0, dtype=torch.float32, device="cuda")
    ops.gemm(A, B, C, M=M, N=N, K=K, lda=lda, ldb=lda, ldc=ldc, bias=bias, mode=ops.MODE_F32_STORE)
    torch.cuda.synchronize()
    tol = 2e-3 * (K ** 0.5) * 0.25 + 1e-4
    assert torch.allclose(C[:, :N], ref + bias, atol=tol, rtol=1e-3), float((C[:, :N] - ref - bias).abs().max())
    assert torch.all(C[:, N:] == -7.0)                      # padding columns untouched
    # fp16 relu epilogue
    ldc16 = (N + 7) // 8 * 8
    C16 = torch.zeros(M, ldc16, dtype=torch.float16, device="cuda")
    ops.gemm(A, B, C16, M=M, N=N, K=K, lda=lda, ldb=lda, ldc=ldc16, bias=bias, mode=ops.MODE_F16_ACT,
             act=ops.ACT_RELU)
    torch.cuda.synchronize()
    want = torch.relu(ref + bias)
    assert torch.allclose(C16[:, :N].float(), want, atol=tol + 4e-3 * float(want.abs().max()), rtol=2e-3)
    # dact epilogue (relu mask from saved activation)
    saved = (torch.randn(M, ldc16, device="cuda")).half()
    D16 = torch.zeros(M, ldc16, dtype=torch.float16, device="cuda")
    ops.gemm(A, B, D16, M=M, N=N, K=K, lda=lda, ldb=lda, ldc=ldc16, saved=saved, ld_saved=ldc16,
             mode=ops.MODE_F16_DACT, act=ops.ACT_RELU, alpha=0.5)
    torch.cuda.synchronize()
    want = 0.5 * ref * (saved[:, :N].float() > 0)
    assert torch.allclose(D16[:, :N].float(), want, atol=tol + 4e-3 * float(want.abs().max()), rtol=2e-3)


def test_gemm_tanh_epilogues(ops):
    M, N, K = 512, 64, 376
    torch.manual_seed(0)
    A = (torch.randn(M, K, device="cuda") * 0.2).half()
    B = (torch.randn(N, K, device="cuda") * 0.2).half()
    C = torch.zeros(M, N, dtype=torch.float16, device="cuda")
    ops.gemm(A, B, C, M=M, N=N, K=K, lda=K, ldb=K, ldc=N, mode=ops.MODE_F16_ACT, act=ops.ACT_TANH)
    ref = torch.tanh(_gemm_ref(A, B, False))
    assert torch.allclose(C.float(), ref, atol=3e-3)
    D = torch.zeros(M, N, dtype=torch.float16, device="cuda")
    ops.gemm(A, B, D, M=M, N=N, K=K, lda=K, ldb=K, ldc=N, saved=C, ld_saved=N, mode=ops.MODE_F16_DACT,
             act=ops.ACT_TANH)
    want = _gemm_ref(A, B, False) * (1 - C.float() ** 2)
    assert torch.allclose(D.float(), want, atol=1e-2, rtol=1e-2)


@pytest.mark.parametrize("Kred,M,N,split", [(64, 128, 64, 1), (1000, 256, 32, 3), (20000, 576, 64, 16),
                                            (4096, 3136, 512, 4), (333, 64, 7, 2), (8192, 512, 64, 148)])
def test_gemm_mnmajor_splitk_atomic(ops, Kred, M, N, split):
    torch.manual_seed(Kred + M)
    lda, ldb = (M + 7) // 8 * 8, (N + 7) // 8 * 8
    A = torch.zeros(Kred, lda, dtype=torch.float16, device="cuda")
    B = torch.zeros(Kred, ldb, dtype=torch.float16, device="cuda")
    A[:, :M] = torch.randn(Kred, M, device="cuda") * 0.5
    B[:, :N] = torch.randn(Kred, N, device="cuda") * 0.5
    C = torch.ones(M, N, dtype=torch.float32, device="cuda")
    ops.gemm(A, B, C, M=M, N=N, K=Kred, lda=lda, ldb=ldb, ldc=N, mn_major=True, mode=ops.MODE_F32_ATOMIC,
             alpha=0.25, split_k=split)
    torch.cuda.synchronize()
    ref = 1.0 + 0.25 * _gemm_ref(A[:, :M], B[:, :N], True)
    tol = 2e-3 * (Kred ** 0.5) * 0.25 * 0.25 + 1e-4
    assert torch.allclose(C, ref, atol=tol, rtol=1e-3), float((C - ref).abs().max())


# ------------------------------------------------------------------------------------------ conv lowering
@pytest.mark.parametrize("B,H,W,C,rf,stride,same,u8", [(5, 84, 84, 4, 8, 4, False, True), (3, 20, 20, 32, 4, 2, False, False),
                                                       (4, 9, 9, 64, 3, 1, False, False), (2, 84, 84, 4, 8, 4, True, True),
                                                       (3, 21, 21, 32, 4, 2, True, False), (2, 11, 11, 64, 3, 1, True, False)])
def test_im2col_col2im_vs_torch(ops, B, H, W, C, rf, stride, same, u8):
    import torch.nn.functional as F
    torch.manual_seed(1)
    if u8:
        x = torch.randint(0, 256, (B, H, W, C), dtype=torch.uint8, device="cuda")
    else:
        x = torch.randn(B, H, W, C, device="cuda").half()
    if same:
        OH, OW = -(-H // stride), -(-W // stride)
        ph, pw = max((OH - 1) * stride + rf - H, 0), max((OW - 1) * stride + rf - W, 0)
        pad = (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2)
    else:
        OH, OW = (H - rf) // stride + 1, (W - rf) // stride + 1
        pad = (0, 0, 0, 0)
    K = rf * rf * C
    cols = torch.zeros(B * OH * OW, K, dtype=torch.float16, device="cuda")
    idx = torch.randperm(B, device="cuda")
    ops.im2col(x, cols, B, H, W, C, rf, stride, same, src_idx=idx)
    torch.cuda.synchronize()
    xp = F.pad(x[idx].float().permute(0, 3, 1, 2), pad)
    un = F.unfold(xp, rf, stride=stride)                       # [B, C*rf*rf, L] with (c, ky, kx) order
    un = un.view(B, C, rf, rf, OH * OW).permute(0, 4, 2, 3, 1).reshape(B * OH * OW, K)
    assert torch.equal(cols.float(), un)
    if not u8:
        dcols = torch.randn(B * OH * OW, K, device="cuda").half()
        dx = torch.zeros(B, H, W, C, dtype=torch.float16, device="cuda")
        ops.col2im(dcols, x, dx, B, H, W, C, rf, stride, same, act=ops.ACT_RELU)
        torch.cuda.synchronize()
        d = dcols.float().view(B, OH * OW, rf, rf, C).permute(0, 4, 2, 3, 1).reshape(B, K, OH * OW)
        folded = F.fold(d, (H + pad[2] + pad[3], W + pad[0] + pad[1]), rf, stride=stride)
        folded = folded[:, :, pad[2]:pad[2] + H, pad[0]:pad[0] + W].permute(0, 2, 3, 1)
        want = folded * (x.float() > 0)
        assert torch.allclose(dx.float(), want, atol=2e-2, rtol=2e-3)


@pytest.mark.parametrize("rows,C", [(1000, 32), (5000, 64), (333, 512), (700, 7), (100000, 64)])
def test_colsum(ops, rows, C):
    torch.manual_seed(2)
    ld = (C + 7) // 8 * 8
    dz = torch.randn(rows, ld, device="cuda").half()
    db = torch.ones(C, dtype=torch.float32, device="cuda")
    ops.colsum(dz, db, rows, C, ld, alpha=0.5)
    want = 1.0 + 0.5 * dz[:, :C].float().sum(0)
    assert torch.allclose(db, want, atol=1e-2 + 1e-4 * rows ** 0.5, rtol=1e-4)


# ------------------------------------------------------------------------------------------ heads / loss
def test_cat_step_matches_oracle(ops):
    from oracle import nets
    B, nA, ld = 1000, 6, 16
    rng = np.random.RandomState(0)
    head = np.zeros((B, ld), np.float32)
    head[:, :nA + 1] = rng.randn(B, nA + 1) * 2
    u = rng.rand(B, nA).astype(np.float32) * 0.998 + 0.001
    hd = dev(head)
    a = torch.zeros(B, dtype=torch.int64, device="cuda")
    v = torch.zeros(B, dtype=torch.float32, device="cuda")
    nlp = torch.zeros(B, dtype=torch.float32, device="cuda")
    ops.cat_step(hd, ld, nA, hd[:, nA:], ld, a, v, nlp, B, uniforms=dev(u))
    lg = torch.tensor(head[:, :nA])
    a_o = nets.cat_sample(lg, torch.tensor(u))
    assert np.array_equal(a.cpu().numpy(), a_o.numpy())
    assert np.allclose(nlp.cpu().numpy(), nets.cat_neglogp(lg, a_o).numpy(), atol=2e-6)
    assert np.array_equal(v.cpu().numpy(), head[:, nA])
    # Philox path: valid actions, empirical frequencies follow softmax
    Bb = 200000
    hb = torch.zeros(Bb, ld, device="cuda")
    hb[:, :nA] = torch.tensor([0.0, 1.0, -1.0, 0.5, 2.0, -2.0])
    a2 = torch.zeros(Bb, dtype=torch.int64, device="cuda")
    ops.cat_step(hb, ld, nA, hb[:, nA:], ld, a2, torch.zeros(Bb, device="cuda"), torch.zeros(Bb, device="cuda"), Bb,
                 seed=123, offset=5)
    freq = torch.bincount(a2, minlength=nA).float() / Bb
    p = torch.softmax(hb[0, :nA], 0)
    assert torch.allclose(freq, p, atol=5e-3)


def test_cat_loss_and_gradient_vs_autograd(ops):
    from oracle import nets
    B, nA, ld, ldd = 4096, 6, 16, 64
    rng = np.random.RandomState(3)
    head = np.zeros((B, ld), np.float32)
    head[:, :nA + 1] = rng.randn(B, nA + 1)
    actions = rng.randint(0, nA, B).astype(np.int64)
    returns = rng.randn(B).astype(np.float32)
    oldv = (returns + rng.randn(B) * 0.5).astype(np.float32)
    oldnlp = (np.log(nA) + rng.randn(B) * 0.3).astype(np.float32)
    perm = rng.permutation(B).astype(np.int64)             # rollout arrays are gathered through src_idx
    clip, ent, vfc = 0.1, 0.01, 0.5
    st = torch.zeros(2, dtype=torch.float64, device="cuda")
    inv = np.argsort(perm)
    ops.adv_stats(dev(returns[inv]), dev(oldv[inv]), dev(perm), B, st)
    adv_np = nets.normalize_advs(returns, oldv)
    assert abs(float(st[0]) - float((returns - oldv).mean())) < 1e-6
    assert abs(float(st[1]) - float((returns - oldv).std())) < 1e-6
    dout = torch.zeros(B, ldd, dtype=torch.float16, device="cuda")
    stats = torch.zeros(5, dtype=torch.float64, device="cuda")
    hd = dev(head)
    ops.cat_loss(hd, ld, nA, hd[:, nA:], ld, dev(actions[inv]), dev(perm), dev(returns[inv]), dev(oldv[inv]),
                 dev(oldnlp[inv]), st, clip, ent, vfc, dout, ldd, dout[:, nA:], ldd, stats, B)
    torch.cuda.synchronize()
    lg = torch.tensor(head[:, :nA], requires_grad=True)
    vp = torch.tensor(head[:, nA], requires_grad=True)
    nlp = nets.cat_neglogp(lg, torch.tensor(actions))
    entropy = nets.cat_entropy(lg).mean()
    advs, R, OV, ONLP = map(torch.tensor, (adv_np, returns, oldv, oldnlp))
    vclip = OV + torch.clamp(vp - OV, -clip, clip)
    vf_loss = 0.5 * torch.maximum((vp - R) ** 2, (vclip - R) ** 2).mean()
    ratio = torch.exp(ONLP - nlp)
    pg = torch.maximum(-advs * ratio, -advs * torch.clamp(ratio, 1 - clip, 1 + clip)).mean()
    loss = pg - entropy * ent + vf_loss * vfc
    loss.backward()
    got = stats.cpu().numpy() / B
    want = [float(pg), float(vf_loss), float(entropy), float(0.5 * ((nlp - ONLP) ** 2).mean()),
            float(((ratio - 1).abs() > clip).float().mean())]
    assert np.allclose(got, want, atol=2e-6, rtol=1e-5), (got, want)
    g = dout.float().cpu().numpy() / B                           # kernel emits sum-scaled gradients
    assert np.allclose(g[:, :nA], lg.grad.numpy(), atol=2e-3 / B + 1e-9, rtol=2e-3)
    assert np.allclose(g[:, nA], vp.grad.numpy(), atol=2e-3 / B + 1e-9, rtol=2e-3)
    assert np.all(g[:, nA + 1:] == 0)


def test_gauss_step_and_loss_vs_autograd(ops):
    from oracle import nets
    B, d, ld, ldd = 2048, 17, 32, 64
    rng = np.random.RandomState(4)
    mean = np.zeros((B, ld), np.float32)
    mean[:, :d] = rng.randn(B, d)
    vcol = rng.randn(B).astype(np.float32)
    logstd = (rng.randn(d) * 0.2).astype(np.float32)
    normals = rng.randn(B, d).astype(np.float32)
    a = torch.zeros(B, d, device="cuda")
    v = torch.zeros(B, device="cuda")
    nlp = torch.zeros(B, device="cuda")
    md, vd, lsd = dev(mean), dev(vcol), dev(logstd)
    ops.gauss_step(md, ld, lsd, d, vd, 1, a, v, nlp, B, normals=dev(normals))
    mt, lst = torch.tensor(mean[:, :d]), torch.tensor(logstd)[None]
    a_o = nets.gauss_sample(mt, lst, torch.tensor(normals))
    assert np.allclose(a.cpu().numpy(), a_o.numpy(), atol=1e-6)
    assert np.allclose(nlp.cpu().numpy(), nets.gauss_neglogp(mt, lst, a_o).numpy(), atol=2e-5)
    # loss
    actions = (mean[:, :d] + rng.randn(B, d) * 0.9).astype(np.float32)
    returns = rng.randn(B).astype(np.float32)
    oldv = (returns + rng.randn(B) * 0.5).astype(np.float32)
    oldnlp = nets.gauss_neglogp(mt, lst, torch.tensor(actions)).numpy() + (rng.randn(B) * 0.2).astype(np.float32)
    clip, ent, vfc = 0.2, 0.003, 0.5
    st = torch.zeros(2, dtype=torch.float64, device="cuda")
    ops.adv_stats(dev(returns), dev(oldv), None, B, st)
    dmean = torch.zeros(B, ldd, dtype=torch.float16, device="cuda")
    dv = torch.zeros(B, 8, dtype=torch.float16, device="cuda")
    dls = torch.zeros(d, dtype=torch.float32, device="cuda")
    stats = torch.zeros(5, dtype=torch.float64, device="cuda")
    ops.gauss_loss(md, ld, lsd, d, vd, 1, dev(actions), None, dev(returns), dev(oldv), dev(oldnlp), st, clip, ent,
                   vfc, dmean, ldd, dv, 8, dls, 1.0 / B, stats, B)
    torch.cuda.synchronize()
    mt = torch.tensor(mean[:, :d], requires_grad=True)
    lst = torch.tensor(logstd[None], requires_grad=True)
    vp = torch.tensor(vcol, requires_grad=True)
    nl = nets.gauss_neglogp(mt, lst, torch.tensor(actions))
    entropy = nets.gauss_entropy(mt, lst).mean()
    advs, R, OV, ONLP = map(torch.tensor, (nets.normalize_advs(returns, oldv), returns, oldv, oldnlp))
    vclip = OV + torch.clamp(vp - OV, -clip, clip)
    vf_loss = 0.5 * torch.maximum((vp - R) ** 2, (vclip - R) ** 2).mean()
    ratio = torch.exp(ONLP - nl)
    pg = torch.maximum(-advs * ratio, -advs * torch.clamp(ratio, 1 - clip, 1 + clip)).mean()
    (pg - entropy * ent + vf_loss * vfc).backward()
    got = stats.cpu().numpy() / B
    want = [float(pg), float(vf_loss), float(entropy), float(0.5 * ((nl - ONLP) ** 2).mean()),
            float(((ratio - 1).abs() > clip).float().mean())]
    assert np.allclose(got, want, atol=1e-5, rtol=1e-5), (got, want)
    assert np.allclose(dmean.float().cpu().numpy()[:, :d] / B, mt.grad.numpy(), atol=2e-3 / B, rtol=2e-3)
    assert np.allclose(dv.float().cpu().numpy()[:, 0] / B, vp.grad.numpy(), atol=2e-3 / B, rtol=2e-3)
    assert np.allclose(dls.cpu().numpy(), lst.grad.numpy()[0], atol=1e-5, rtol=1e-4)


# ------------------------------------------------------------------------------------------ optimiser
def test_sumsq_clip_adam_vs_oracle(ops):
    from oracle import nets
    n = 1687719                                          # NatureCNN/6 actions parameter count (SURVEY 8a)
    torch.manual_seed(5)
    p = torch.randn(n, device="cuda")
    g = torch.randn(n, device="cuda") * 1e-3
    m = torch.zeros(n, device="cuda")
    v = torch.zeros(n, device="cuda")
    po, mo, vo = p.cpu().clone(), m.cpu().clone(), v.cpu().clone()
    ss = torch.zeros(1, dtype=torch.float64, device="cuda")
    lr, clip = 2.5e-4, 0.5
    for t in range(1, 4):
        gt = g * t
        ops.sumsq(gt, ss)
        assert abs(float(ss[0]) - float((gt.double() ** 2).sum())) < 1e-9 * float(ss[0]) + 1e-12
        lr_t = lr * np.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t)
        ops.clip_adam(p, gt, m, v, lr_t, 0.9, 0.999, 1e-5, clip, ss)
        gc, _ = nets.clip_by_global_norm([gt.cpu()], clip)
        po, mo, vo = nets.adam_tf(po, gc[0], mo, vo, t, lr, eps=1e-5)
    torch.cuda.synchronize()
    assert torch.allclose(p.cpu(), po, atol=1e-6, rtol=1e-6)
    assert torch.allclose(m.cpu(), mo, atol=1e-9, rtol=1e-5)
    assert torch.allclose(v.cpu(), vo, atol=1e-12, rtol=1e-5)


def test_segment_clip_and_casts(ops):
    torch.manual_seed(6)
    sizes = [100, 3000, 17, 512 * 7]
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    n = int(off[-1])
    g = torch.randn(n, device="cuda") * torch.tensor(np.repeat([0.01, 1.0, 5.0, 0.2], sizes), device="cuda").float()
    ss = torch.zeros(len(sizes), dtype=torch.float64, device="cuda")
    ops.seg_sumsq(g, dev(off), len(sizes), ss)
    want = [float((g[off[i]:off[i + 1]].double() ** 2).sum()) for i in range(len(sizes))]
    assert np.allclose(ss.cpu().numpy(), want, rtol=1e-10)
    p = torch.zeros(n, device="cuda"); m = torch.zeros(n, device="cuda"); v = torch.zeros(n, device="cuda")
    ops.clip_adam(p, g, m, v, 1.0, 0.0, 0.0, 1.0, 10.0, ss, seg_off=dev(off), nseg=len(sizes))
    # with beta1=beta2=0: m = g_clipped
    for i in range(len(sizes)):
        seg = g[off[i]:off[i + 1]]
        nrm = float(seg.norm())
        assert torch.allclose(m[off[i]:off[i + 1]], seg * (10.0 / max(nrm, 10.0)), rtol=1e-5, atol=1e-7)
    R, C = 300, 70
    src = torch.randn(R, C, device="cuda")
    d1 = torch.zeros(R, 72, dtype=torch.float16, device="cuda")
    d2 = torch.zeros(C, 304, dtype=torch.float16, device="cuda")
    ops.cast_transpose(src, R, C, d1, 72, d2, 304, scale=0.5)
    assert torch.equal(d1[:, :C], (src * 0.5).half()) and torch.equal(d2[:, :R], (src * 0.5).half().t())
    d3 = torch.zeros(R, 72, dtype=torch.float16, device="cuda")
    ops.cast_f32_f16(src, d3, R, C, C, 72)
    assert torch.equal(d3[:, :C], src.half())


# ------------------------------------------------------------------------------------------ replay
def test_segment_tree_trace_bit_exact(ops):
    g = np.load(os.path.join(GOLDEN, "segment_tree_trace.npz"))
    cap = int(g["capacity"])
    s = torch.zeros(2 * cap, dtype=torch.float64, device="cuda")
    m = torch.full((2 * cap,), float("inf"), dtype=torch.float64, device="cuda")
    out = torch.zeros(1, dtype=torch.float64, device="cuda")
    for kind, a, b, res in g["ops"]:
        kind = int(kind)
        if kind == 0:
            ops.tree_set(s, m, cap, dev(np.array([int(a)], np.int64)), dev(np.array([b], np.float64)))
        elif kind == 1:
            ops.tree_range_sum(s, cap, int(a), int(b), out)
            assert float(out[0]) == res
    assert np.array_equal(s.cpu().numpy(), g["final_sum"])
    assert np.array_equal(m.cpu().numpy(), g["final_min"])


def test_per_trace_vs_reference_golden(ops):
    g = np.load(os.path.join(GOLDEN, "per_trace.npz"))
    size, alpha, batch = int(g["size"]), float(g["alpha"]), int(g["batch"])
    cap = 1
    while cap < size:
        cap *= 2
    s = torch.zeros(2 * cap, dtype=torch.float64, device="cuda")
    m = torch.full((2 * cap,), float("inf"), dtype=torch.float64, device="cuda")
    state = {"next": 0, "n": 0, "maxp": 1.0}

    def add(k):
        idx = [(state["next"] + i) % size for i in range(k)]
        state["next"] = (state["next"] + k) % size
        state["n"] = min(state["n"] + k, size)
        ops.tree_set(s, m, cap, dev(np.array(idx, np.int64)), dev(np.full(k, state["maxp"] ** alpha, np.float64)))

    add(int(g["nadd1"]))
    for r in range(len(g["betas"])):
        assert state["n"] == int(g["nstored"][r])
        idx = torch.zeros(batch, dtype=torch.int64, device="cuda")
        w = torch.zeros(batch, dtype=torch.float64, device="cuda")
        ops.per_sample(s, m, cap, state["n"], dev(g["uniforms"][r]), float(g["betas"][r]), idx, w)
        assert np.array_equal(idx.cpu().numpy(), g["idxes"][r])                      # bit exact indices
        assert np.allclose(w.cpu().numpy(), g["weights"][r], rtol=1e-13, atol=0)     # pow() may differ by ulps
        pr = g["priorities"][r]
        # python-float pow like the reference (numpy's vectorised pow may differ by an ulp)
        ops.tree_set(s, m, cap, idx, dev(np.array([float(x) ** alpha for x in pr])))   # duplicates: last write wins
        state["maxp"] = max(state["maxp"], float(pr.max()))
        add(int(g["adds_after_round"][r]))
    assert np.array_equal(s.cpu().numpy(), g["final_sum"])
    assert np.array_equal(m.cpu().numpy(), g["final_min"])
    assert state["maxp"] == float(g["max_priority"])


def test_per_large_tree_vs_oracle_float32_priorities(ops):
    """Trees, indices and weights at 2^14 leaves against the oracle; new priorities from float32 TD errors are the
    float32 values fl32(|td| + fl32(eps)) of the reference's graph, powered with the correctly rounded pow."""
    from oracle.segment_tree import PrioritizedSampler
    from _replay_refs import cr_pow, leaf_values, reference_priorities
    size, batch = 1 << 14, 512
    rng = np.random.RandomState(8)
    per = PrioritizedSampler(size, 0.6)
    pri = np.abs(rng.randn(size)) + 1e-6
    for i in range(size):
        per.add()
    per.update_priorities(list(range(size)), pri)
    cap = size
    s = torch.zeros(2 * cap, dtype=torch.float64, device="cuda")
    m = torch.full((2 * cap,), float("inf"), dtype=torch.float64, device="cuda")
    ops.tree_set(s, m, cap, dev(np.arange(size, dtype=np.int64)), dev(np.array([float(x) ** 0.6 for x in pri])))
    torch.cuda.synchronize()
    assert np.array_equal(s.cpu().numpy(), per.sum_tree.value)
    assert np.array_equal(m.cpu().numpy(), per.min_tree.value)
    u = rng.rand(batch)
    idx = torch.zeros(batch, dtype=torch.int64, device="cuda")
    w = torch.zeros(batch, dtype=torch.float64, device="cuda")
    wf = torch.zeros(batch, dtype=torch.float32, device="cuda")
    ops.per_sample(s, m, cap, size, dev(u), 0.4, idx, w, wf)
    want = per.sample_idx(u)
    assert np.array_equal(idx.cpu().numpy(), want)
    assert np.allclose(w.cpu().numpy(), per.weights(want, 0.4), rtol=1e-13)    # the oracle's weights use libm pow
    total = per.sum_tree.sum()
    want_w = (cr_pow(np.array([per.sum_tree.get(i) for i in want]) / total * size, -0.4)
              / cr_pow(per.min_tree.min() / total * size, -0.4))
    assert np.array_equal(w.cpu().numpy(), want_w) and np.array_equal(wf.cpu().numpy(), want_w.astype(np.float32))
    td = torch.randn(batch, device="cuda")
    powered = torch.zeros(batch, dtype=torch.float64, device="cuda")
    maxp = torch.ones(1, dtype=torch.float64, device="cuda")
    bad = torch.zeros(1, dtype=torch.int32, device="cuda")
    ops.per_priorities(td, 1e-6, 0.6, powered, maxp, bad)
    pw = reference_priorities(td.cpu().numpy(), 1e-6)                                # float32 priorities
    assert np.array_equal(powered.cpu().numpy(), leaf_values(pw, 0.6))
    assert float(maxp[0]) == max(1.0, float(pw.max())) and int(bad[0]) == 0


def test_dqn_td_vs_oracle(ops):
    from oracle import nets
    B, nA, ld = 512, 6, 16
    rng = np.random.RandomState(9)

    def head():
        h = np.zeros((B, ld), np.float32)
        h[:, :nA + 1] = rng.randn(B, nA + 1)
        return h

    ht, hon, htg = head(), head(), head()
    act = rng.randint(0, nA, B).astype(np.int64)
    rew = rng.randn(B).astype(np.float32)
    done = (rng.rand(B) < 0.1).astype(np.float32)
    w = rng.rand(B).astype(np.float32)
    for dueling in (True, False):
        dt, don, dtg = dev(ht), dev(hon), dev(htg)
        td = torch.zeros(B, device="cuda")
        dA = torch.zeros(B, 64, dtype=torch.float16, device="cuda")
        loss = torch.zeros(1, dtype=torch.float64, device="cuda")
        sp = (lambda t: t[:, nA:]) if dueling else (lambda t: None)
        ops.dqn_td(dt, ld, sp(dt), ld, don, ld, sp(don), ld, dtg, ld, sp(dtg), ld, nA, None, dev(act), dev(rew),
                   dev(done), dev(w), 0.99, True, td, dA, 64, dA[:, nA:] if dueling else None, 64, loss, B)
        torch.cuda.synchronize()

        def q(h, a_req=False):
            A = torch.tensor(h[:, :nA], requires_grad=a_req)
            S = torch.tensor(h[:, nA], requires_grad=a_req)
            return (S[:, None] + (A - A.mean(1, keepdim=True)) if dueling else A), A, S

        qt, At, St = q(ht, True)
        qon, _, _ = q(hon)
        qtg, _, _ = q(htg)
        best = qtg.gather(1, qon.argmax(1, keepdim=True))[:, 0]
        target = torch.tensor(rew) + 0.99 * (1 - torch.tensor(done)) * best
        tdo = qt.gather(1, torch.tensor(act)[:, None])[:, 0] - target.detach()
        L = (torch.tensor(w) * nets.huber(tdo)).sum()
        L.backward()
        assert np.allclose(td.cpu().numpy(), tdo.detach().numpy(), atol=2e-6)
        assert abs(float(loss[0]) - float(L)) < 1e-3
        assert np.allclose(dA.float().cpu().numpy()[:, :nA], At.grad.numpy(), atol=2e-3, rtol=2e-3)
        if dueling:
            assert np.allclose(dA.float().cpu().numpy()[:, nA], St.grad.numpy(), atol=2e-3, rtol=2e-3)


# ------------------------------------------------------------------------------------------ implicit-GEMM conv
def _patches(x, R, S, sh, sw, ph, pw, OH, OW):
    """float64 patch matrix [B*OH*OW, R*S*C] of x [B,H,W,C], K ordered (r, s, c) (tests/_refs.py)."""
    return _refs.patches(x.double(), R, S, sh, sw, ph, pw, OH, OW)


CONV_CASES = [
    # name, B, H, W, C, R, S, sh, sw, N
    ("c1_superpixel", 5, 84, 21, 16, 8, 2, 4, 1, 32),
    ("c2", 7, 20, 20, 32, 4, 4, 2, 2, 64),
    ("c3", 11, 9, 9, 64, 3, 3, 1, 1, 64),
]


@pytest.mark.parametrize("name,B,H,W,C,R,S,sh,sw,N", CONV_CASES)
def test_conv_gemm_forward_and_wgrad(ops, name, B, H, W, C, R, S, sh, sw, N):
    torch.manual_seed(hash(name) % 1000)
    OH, OW = (H - R) // sh + 1, (W - S) // sw + 1
    x = (torch.randn(B, H, W, C, device="cuda") * 0.5).half()
    K = R * S * C
    wt = (torch.randn(N, K, device="cuda") * 0.2).half()
    bias = torch.randn(N, device="cuda")
    rows = B * OH * OW
    P = _patches(x.float(), R, S, sh, sw, 0, 0, OH, OW)
    out = torch.zeros(rows, N, dtype=torch.float16, device="cuda")
    ops.conv_gemm(x, B, H, W, C, R, S, sh, sw, 0, 0, OH, OW, wt, K, out, N, N, 0, ops.MODE_F16_ACT, act=ops.ACT_RELU,
                  bias=bias)
    torch.cuda.synchronize()
    want = torch.relu(P @ wt.double().t() + bias.double()).float()
    err = float((out.float() - want).abs().max())
    assert torch.allclose(out.float(), want, atol=2e-2, rtol=5e-3), (name, err)
    # wgrad: gw[K, N] += alpha * patches^T dz
    dz = (torch.randn(rows, N, device="cuda") * 0.5).half()
    gw = torch.ones(K, N, dtype=torch.float32, device="cuda")
    ops.conv_gemm(x, B, H, W, C, R, S, sh, sw, 0, 0, OH, OW, dz, N, gw, N, N, 1, ops.MODE_F32_ATOMIC, alpha=0.5,
                  split_k=3)
    torch.cuda.synchronize()
    want = (1.0 + 0.5 * (P.t() @ dz.double())).float()
    err = float((gw - want).abs().max())
    assert torch.allclose(gw, want, atol=2e-3 * rows ** 0.5, rtol=2e-3), (name, err)


@pytest.mark.parametrize("B,Hin,Cin,Cout,rf,s", [(7, 20, 32, 64, 4, 2), (11, 9, 64, 64, 3, 1), (3, 84, 16, 32, 8, 4)])
def test_conv_gemm_dgrad_pixel_shuffle(ops, B, Hin, Cin, Cout, rf, s):
    """dx = conv_transpose(dz, W) * relu'(h_in), computed as ONE implicit GEMM over dz with the rearranged
    weights and the pixel-shuffle epilogue; reference = the float64 transposed convolution of tests/_refs.py."""
    torch.manual_seed(Hin + Cin)
    OHc = (Hin - rf) // s + 1                                 # conv output size
    w = (torch.randn(rf, rf, Cin, Cout, device="cuda") * 0.2)
    h_in = torch.randn(B, Hin, Hin, Cin, device="cuda").half()   # saved activation of the layer below
    dz = (torch.randn(B, OHc, OHc, Cout, device="cuda") * 0.5).half()
    An = -(-rf // s)
    ldw = An * An * Cout
    wdg = torch.zeros(s * s * Cin, ldw, dtype=torch.float16, device="cuda")
    ops.dgrad_weights(w.contiguous(), wdg, rf, rf, Cin, Cout, s, ldw)
    G = -(-Hin // s)                                          # base-pixel grid of the GEMM rows
    dx = torch.zeros(B, Hin, Hin, Cin, dtype=torch.float16, device="cuda")
    ops.conv_gemm(dz, B, OHc, OHc, Cout, An, An, 1, 1, An - 1, An - 1, G, G, wdg, ldw, dx, 0, s * s * Cin, 0,
                  ops.MODE_F16_SHUFFLE, act=ops.ACT_RELU, saved=h_in, shuffle=(Hin, Hin, Cin, s))
    torch.cuda.synchronize()
    want = (_refs.conv2d_dgrad(dz, w.half(), Hin, Hin, (s, s), (0, 0)) * (h_in.double() > 0)).float()
    err = float((dx.float() - want).abs().max())
    assert torch.allclose(dx.float(), want, atol=3e-2, rtol=5e-3), err


# ------------------------------------------------------------------------------------------ shift-GEMM convolutions
SHIFT_CASES = [("c1_s2d", 5, 21, 21, 64, 2, 32), ("c2_s2d", 7, 10, 10, 128, 2, 64), ("c3", 11, 9, 9, 64, 3, 64)]


@pytest.mark.parametrize("name,B,Hg,Wg,C,R,N", SHIFT_CASES)
def test_conv_shift_forward_wgrad_dgrad(ops, name, B, Hg, Wg, C, R, N):
    """Stride-1 RxR VALID conv over a [B,Hg,Wg,C] grid: forward (compact output), wgrad and dgrad (dY stored
    zero-bordered on the input grid) against explicit patch matrices."""
    torch.manual_seed(len(name) + B)
    OH, OW = Hg - R + 1, Wg - R + 1
    taps = R * R
    shifts = [r * Wg + s for r in range(R) for s in range(R)]
    x = (torch.randn(B, Hg, Wg, C, device="cuda") * 0.5).half()
    K = taps * C
    wt = (torch.randn(N, K, device="cuda") * 0.1).half()
    bias = torch.randn(N, device="cuda")
    P = _patches(x.float(), R, R, 1, 1, 0, 0, OH, OW)                    # [B*OH*OW, (r,s,c)]
    # ---- forward -> compact [B,OH,OW,N]
    out = torch.full((B, OH, OW, N), 7.0, dtype=torch.float16, device="cuda")
    omap = (0, OH * OW * N, OW * N, N, 0, 0)
    ops.conv_shift_fwd(x, B, Hg, Wg, C, wt, K, N, shifts, OH, OW, out, omap, bias=bias, act=ops.ACT_RELU)
    torch.cuda.synchronize()
    want = torch.relu(P @ wt.double().t() + bias.double()).float().view(B, OH, OW, N)
    err = float((out.float() - want).abs().max())
    assert torch.allclose(out.float(), want, atol=3e-2, rtol=5e-3), (name, "fwd", err)
    # ---- wgrad: dY lives on the INPUT grid, zero outside the valid OHxOW window
    dz = torch.zeros(B, Hg, Wg, N, dtype=torch.float16, device="cuda")
    dzv = (torch.randn(B, OH, OW, N, device="cuda") * 0.5).half()
    dz[:, :OH, :OW] = dzv
    G = torch.ones(K, N, dtype=torch.float32, device="cuda")
    gb = torch.ones(N, dtype=torch.float32, device="cuda")
    ops.conv_shift_wgrad(x, B * Hg * Wg, C, dz, N, shifts, G, N, alpha=0.5, gbias=gb, alpha_b=0.25)
    torch.cuda.synchronize()
    want_gb = 1.0 + 0.25 * dzv.float().reshape(-1, N).sum(0)           # fused bias gradient
    assert torch.allclose(gb, want_gb, atol=1e-2, rtol=1e-3), (name, "gbias", float((gb - want_gb).abs().max()))
    wantG = (1.0 + 0.5 * (P.t() @ dzv.double().reshape(-1, N))).float()
    err = float((G - wantG).abs().max())
    assert torch.allclose(G, wantG, atol=3e-3 * (B * OH * OW) ** 0.5, rtol=3e-3), (name, "wgrad", err)
    # ---- dgrad: dX[m] = sum_t dY[m - sh_t] W_t, W_t = [C rows (c_in), N cols (c_out)] = rows t*C.. of W_hwio[K, N]
    if C == 64:
        w_hwio = (torch.randn(K, N, device="cuda") * 0.1).half()          # [(r,s,c_in), c_out]
        wd = torch.zeros(C, taps * N, dtype=torch.float16, device="cuda")  # [c_in, (t, c_out)] K-major operand
        for t in range(taps):
            wd[:, t * N:(t + 1) * N] = w_hwio[t * C:(t + 1) * C]
        saved = torch.randn(B, Hg, Wg, C, device="cuda").half()
        dx = torch.zeros(B, Hg, Wg, C, dtype=torch.float16, device="cuda")
        gmap = (0, Hg * Wg * C, Wg * C, C, 0, 0)
        if N in (64, 128):
            # the ReLU mask as 1 bit per element: bit k of word e/16 <-> saved element e+k > 0
            bits = ((saved.reshape(-1, 16) > 0).to(torch.int32) << torch.arange(16, device="cuda", dtype=torch.int32)
                    ).sum(1).to(torch.int16)                                  # two's complement wrap of bit 15
            ops.conv_shift_fwd(dz, B, Hg, Wg, N, wd, taps * N, C, [-s for s in shifts], Hg, Wg, dx, gmap, smap=gmap,
                               act=ops.ACT_RELU, dact=True, saved_bits=bits)
            torch.cuda.synchronize()
            # reference: dX = patches-transpose: scatter-add of dz_valid @ W_t^T
            dcols = dzv.float().reshape(-1, N) @ w_hwio.float().t()        # [B*OH*OW, (r,s,c)]
            ref = torch.zeros(B, Hg, Wg, C, device="cuda")
            dc = dcols.view(B, OH, OW, R, R, C)
            for r in range(R):
                for s in range(R):
                    ref[:, r:r + OH, s:s + OW] += dc[:, :, :, r, s]
            ref = ref * (saved.float() > 0)
            err = float((dx.float() - ref).abs().max())
            assert torch.allclose(dx.float(), ref, atol=3e-2, rtol=5e-3), (name, "dgrad", err)
    # ---- forward can emit that bit array for its own (ReLU) output
    bo = torch.zeros(B * OH * OW * N // 16, dtype=torch.int16, device="cuda")
    out2 = torch.empty_like(out)
    ops.conv_shift_fwd(x, B, Hg, Wg, C, wt, K, N, shifts, OH, OW, out2, omap, bias=bias, act=ops.ACT_RELU, bits_out=bo)
    torch.cuda.synchronize()
    assert torch.equal(out, out2)
    want_bits = ((out2.reshape(-1, 16) > 0).to(torch.int32) << torch.arange(16, device="cuda", dtype=torch.int32)
                 ).sum(1).to(torch.int16)
    assert torch.equal(bo, want_bits), (name, "fwd bits")


def test_conv_shift_address_maps(ops):
    """space->depth (mode 2) output map of conv1 -> h1 and depth->space (mode 1) map of conv2's dgrad."""
    torch.manual_seed(3)
    B, Hg, Wg, C, N = 3, 21, 21, 64, 32
    shifts = [0, 1, Wg, Wg + 1]
    x = (torch.randn(B, Hg, Wg, C, device="cuda") * 0.5).half()
    wt = (torch.randn(N, 4 * C, device="cuda") * 0.1).half()
    P = _patches(x.float(), 2, 2, 1, 1, 0, 0, 20, 20)
    want = (P @ wt.double().t()).float().view(B, 20, 20, N)
    h1 = torch.zeros(B, 10, 10, 4 * N, dtype=torch.float16, device="cuda")
    ops.conv_shift_fwd(x, B, Hg, Wg, C, wt, 4 * C, N, shifts, 20, 20, h1, (2, 100 * 4 * N, 10 * 4 * N, 4 * N, N, 2))
    torch.cuda.synchronize()
    s2d = want.view(B, 10, 2, 10, 2, N).permute(0, 1, 3, 2, 4, 5).reshape(B, 10, 10, 4 * N)
    assert torch.allclose(h1.float(), s2d, atol=3e-2, rtol=5e-3)
    # depth->space: GEMM columns (dy, dx, c) of row (n, Y, X) land at (2Y+dy, 2X+dx, c) of a 21x21x32 grid
    dz = torch.zeros(B, 10, 10, 64, dtype=torch.float16, device="cuda")
    dz[:, :9, :9] = (torch.randn(B, 9, 9, 64, device="cuda") * 0.5).half()
    wd = (torch.randn(128, 4 * 64, device="cuda") * 0.1).half()           # [(dy,dx,c), (t, c_out)]
    out = torch.zeros(B, 21, 21, 32, dtype=torch.float16, device="cuda")
    sh = [-(a * 10 + b) for a in range(2) for b in range(2)]
    ops.conv_shift_fwd(dz, B, 10, 10, 64, wd, 256, 128, sh, 10, 10, out, (1, 21 * 21 * 32, 21 * 32, 32, 32, 2),
                       dact=True)
    torch.cuda.synchronize()
    dzp = torch.zeros(B, 11, 11, 64, device="cuda")
    dzp[:, 1:, 1:] = dz.float()                                            # dY[m - (a*10+b)] == padded(Y-a, X-b)
    ref = torch.zeros(B, 10, 10, 128, device="cuda")
    for t, (a, b) in enumerate([(a, b) for a in range(2) for b in range(2)]):
        ref += dzp[:, 1 - a:11 - a, 1 - b:11 - b] @ wd.float()[:, t * 64:(t + 1) * 64].t()
    ref_sp = ref.view(B, 10, 10, 2, 2, 32).permute(0, 1, 3, 2, 4, 5).reshape(B, 20, 20, 32)
    assert torch.allclose(out[:, :20, :20].float(), ref_sp, atol=3e-2, rtol=5e-3)
    assert float(out[:, 20:].abs().max()) == 0 and float(out[:, :, 20:].abs().max()) == 0


def test_gemm_column_remap(ops):
    """fc1 dgrad writes its [B, 7*7*64] rows into the zero-bordered [B, 9, 9, 64] grid of conv3's dY."""
    torch.manual_seed(4)
    M, N, K = 300, 49 * 64, 128
    A = (torch.randn(M, K, device="cuda") * 0.3).half()
    W = (torch.randn(N, K, device="cuda") * 0.3).half()
    saved = torch.randn(M, N, device="cuda").half()
    out = torch.zeros(M, 81 * 64, dtype=torch.float16, device="cuda")
    ops.gemm(A, W, out, M=M, N=N, K=K, lda=K, ldb=K, ldc=81 * 64, saved=saved, ld_saved=N, mode=ops.MODE_F16_DACT,
             act=ops.ACT_RELU, remap=(64, 7, 9))
    torch.cuda.synchronize()
    ref = (A.float() @ W.float().t()) * (saved.float() > 0)
    grid = out.float().view(M, 9, 9, 64)
    assert torch.allclose(grid[:, :7, :7].reshape(M, -1), ref, atol=3e-2, rtol=5e-3)
    assert float(grid[:, 7:].abs().max()) == 0 and float(grid[:, :, 7:].abs().max()) == 0


@pytest.mark.parametrize("B,gather", [(3, False), (37, True), (700, True), (4000, True)])
def test_conv_shift_fused_uint8_source(ops, B, gather):
    """First conv layer straight from uint8 frames: the producer warps' gather + cast + space-to-depth tile must
    give the same forward (bit-exact: same fp16 operands, same MMA order) and the same wgrad (different
    reduction blocking -> tolerance) as s2d_gather followed by the fp16 TMA path."""
    torch.manual_seed(B)
    H = W = 84
    C, s, Hg, Wg, N = 4, 4, 21, 21, 32
    pool = 2 * B + 5
    frames = torch.randint(0, 256, (pool, H, W, C), dtype=torch.uint8, device="cuda")
    idx = torch.randperm(pool, device="cuda")[:B].contiguous() if gather else None
    x16 = torch.empty(B, Hg * Wg * 64, dtype=torch.float16, device="cuda")
    ops.s2d_gather(frames, x16, B, H, W, C, s, src_idx=idx)
    shifts = [0, 1, Wg, Wg + 1]
    wt = (torch.randn(N, 256, device="cuda") * 0.01).half()
    bias = torch.randn(N, device="cuda")
    omap = (2, 100 * 4 * N, 10 * 4 * N, 4 * N, N, 2)
    h_ref = torch.zeros(B, 10, 10, 4 * N, dtype=torch.float16, device="cuda")
    h_u8 = torch.zeros_like(h_ref)
    ops.conv_shift_fwd(x16, B, Hg, Wg, 64, wt, 256, N, shifts, 20, 20, h_ref, omap, bias=bias, act=ops.ACT_RELU)
    u8 = (frames, idx, H, W, C, s)
    ops.conv_shift_fwd(None, B, Hg, Wg, 64, wt, 256, N, shifts, 20, 20, h_u8, omap, bias=bias, act=ops.ACT_RELU, u8=u8)
    torch.cuda.synchronize()
    assert float(h_ref.float().abs().max()) > 0
    assert torch.equal(h_ref, h_u8)
    dz = torch.zeros(B, Hg, Wg, N, dtype=torch.float16, device="cuda")
    dz[:, :20, :20] = (torch.randn(B, 20, 20, N, device="cuda") * 0.5).half()
    G_ref = torch.zeros(256, N, dtype=torch.float32, device="cuda")
    G_u8 = torch.zeros_like(G_ref)
    gb_ref = torch.zeros(N, dtype=torch.float32, device="cuda")
    gb_u8 = torch.zeros_like(gb_ref)
    rows = B * Hg * Wg
    ops.conv_shift_wgrad(x16, rows, 64, dz, N, shifts, G_ref, N, alpha=1.0 / 255, gbias=gb_ref, alpha_b=1.0)
    ops.conv_shift_wgrad(None, rows, 64, dz, N, shifts, G_u8, N, alpha=1.0 / 255, gbias=gb_u8, alpha_b=1.0, u8=u8)
    torch.cuda.synchronize()
    scale = float(G_ref.abs().max())
    assert scale > 0
    assert float((G_ref - G_u8).abs().max()) <= 1e-5 * scale + 1e-3, float((G_ref - G_u8).abs().max())
    assert torch.allclose(gb_ref, gb_u8, atol=1e-3, rtol=1e-5)


@pytest.mark.parametrize("name", ["frame_stack_c1.npz", "frame_stack_c2.npz"])
def test_frame_stack_kernel_matches_reference_golden(ops, name):
    """b200rl_frame_stack against outputs of the reference VecFrameStack (golden) -- bit exact."""
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", name))
    frames, news, want = g["frames"], g["news"], g["stacked"]
    nstack, c = int(g["nstack"]), int(g["c"])
    cur = torch.zeros(want.shape[1:], dtype=torch.uint8, device="cuda")
    nxt = torch.empty_like(cur)
    ops.frame_stack(cur, torch.from_numpy(frames[0]).cuda(), torch.ones(want.shape[1], dtype=torch.uint8, device="cuda"),
                    nxt, nstack, c)
    assert np.array_equal(nxt.cpu().numpy(), want[0])
    for t in range(news.shape[0]):
        cur, nxt = nxt, cur
        ops.frame_stack(cur, torch.from_numpy(frames[t + 1]).cuda(), torch.from_numpy(news[t].astype(np.uint8)).cuda(),
                        nxt, nstack, c)
        assert np.array_equal(nxt.cpu().numpy(), want[t + 1]), t


def test_frame_stack_kernel_atari_shape_vs_oracle(ops):
    """84x84x(4x1) at 64 envs (vectorised 4-pixel path) and an unaligned view (scalar word path) vs the oracle."""
    from oracle import frame_stack as fs
    rng = np.random.RandomState(0)
    N = 64
    prev = rng.randint(0, 256, (N, 84, 84, 4)).astype(np.uint8)
    frames = rng.randint(0, 256, (N, 84, 84, 1)).astype(np.uint8)
    news = rng.rand(N) < 0.3
    want = fs.frame_stack_step(prev, frames, news)
    out = torch.empty(N, 84, 84, 4, dtype=torch.uint8, device="cuda")
    ops.frame_stack(torch.from_numpy(prev).cuda(), torch.from_numpy(frames).cuda(),
                    torch.from_numpy(news.astype(np.uint8)).cuda(), out, 4, 1)
    assert np.array_equal(out.cpu().numpy(), want)
    big = torch.empty(N * 84 * 84 * 4 + 4, dtype=torch.uint8, device="cuda")
    out2 = big[4:].view(N, 84, 84, 4)                      # 4-byte but not 16-byte aligned
    ops.frame_stack(torch.from_numpy(prev).cuda(), torch.from_numpy(frames).cuda(),
                    torch.from_numpy(news.astype(np.uint8)).cuda(), out2, 4, 1)
    assert np.array_equal(out2.cpu().numpy(), want)


# ------------------------------------------------------------------------------------------ x-folded shift-GEMM
XFOLD_CASES = [("c1", 67, 21, 21, 64, 2, 32), ("c2", 90, 10, 10, 128, 2, 64), ("c3", 130, 9, 9, 64, 3, 64),
               ("k2c64", 9, 12, 7, 64, 2, 64)]


@pytest.mark.parametrize("name,B,Hg,Wg,C,R,N", XFOLD_CASES)
def test_conv_shift_xfold_wgrad(ops, name, B, Hg, Wg, C, R, N):
    """kx = R weight gradient: the R taps of a filter row are N-chunks of the dY tile one row apart.  Checked against
    explicit patch matrices in fp32; several tiles per CTA and tile / warp / image boundaries at arbitrary phases (rows
    per image not a multiple of anything)."""
    torch.manual_seed(len(name) * 7 + B)
    OH, OW = Hg - R + 1, Wg - R + 1
    K = R * R * C
    yshifts = [r * Wg for r in range(R)]
    x = (torch.randn(B, Hg, Wg, C, device="cuda") * 0.5).half()
    P = _patches(x.float(), R, R, 1, 1, 0, 0, OH, OW)
    dz = torch.zeros(B, Hg, Wg, N, dtype=torch.float16, device="cuda")
    dzv = (torch.randn(B, OH, OW, N, device="cuda") * 0.5).half()
    dz[:, :OH, :OW] = dzv
    G = torch.ones(K, N, dtype=torch.float32, device="cuda")
    gb = torch.ones(N, dtype=torch.float32, device="cuda")
    ops.conv_shift_wgrad(x, B * Hg * Wg, C, dz, N, yshifts, G, N, alpha=0.5, gbias=gb, alpha_b=0.25, kx=R)
    torch.cuda.synchronize()
    want_gb = 1.0 + 0.25 * dzv.float().reshape(-1, N).sum(0)
    assert torch.allclose(gb, want_gb, atol=2e-2, rtol=1e-3), (name, "fold gbias", float((gb - want_gb).abs().max()))
    wantG = (1.0 + 0.5 * (P.t() @ dzv.double().reshape(-1, N))).float()
    err = float((G - wantG).abs().max())
    assert torch.allclose(G, wantG, atol=3e-3 * (B * OH * OW) ** 0.5, rtol=3e-3), (name, "fold wgrad", err)


@pytest.mark.parametrize("B,gather", [(5, False), (300, True), (3000, True)])
def test_conv_shift_xfold_wgrad_fused_uint8_source(ops, B, gather):
    """conv1 weight gradient with the x-fold straight from uint8 frames == the same folded kernel fed by s2d_gather, and
    == the un-folded kernel (to float-atomic order)."""
    torch.manual_seed(B)
    H = W = 84
    C, s, Hg, Wg, N = 4, 4, 21, 21, 32
    pool = 2 * B + 5
    frames = torch.randint(0, 256, (pool, H, W, C), dtype=torch.uint8, device="cuda")
    idx = torch.randperm(pool, device="cuda")[:B].contiguous() if gather else None
    x16 = torch.empty(B, Hg * Wg * 64, dtype=torch.float16, device="cuda")
    ops.s2d_gather(frames, x16, B, H, W, C, s, src_idx=idx)
    yshifts = [0, Wg]
    u8 = (frames, idx, H, W, C, s)
    dz = torch.zeros(B, Hg, Wg, N, dtype=torch.float16, device="cuda")
    dz[:, :20, :20] = (torch.randn(B, 20, 20, N, device="cuda") * 0.5).half()
    G_ref = torch.zeros(256, N, dtype=torch.float32, device="cuda")
    G_u8 = torch.zeros_like(G_ref)
    G_old = torch.zeros_like(G_ref)
    gb_ref = torch.zeros(N, dtype=torch.float32, device="cuda")
    gb_u8 = torch.zeros_like(gb_ref)
    rows = B * Hg * Wg
    ops.conv_shift_wgrad(x16, rows, 64, dz, N, yshifts, G_ref, N, alpha=1.0 / 255, gbias=gb_ref, alpha_b=1.0, kx=2)
    ops.conv_shift_wgrad(None, rows, 64, dz, N, yshifts, G_u8, N, alpha=1.0 / 255, gbias=gb_u8, alpha_b=1.0, u8=u8, kx=2)
    ops.conv_shift_wgrad(x16, rows, 64, dz, N, [0, 1, Wg, Wg + 1], G_old, N, alpha=1.0 / 255)
    torch.cuda.synchronize()
    scale = float(G_ref.abs().max())
    assert scale > 0
    assert float((G_ref - G_u8).abs().max()) <= 1e-5 * scale + 1e-3
    assert float((G_ref - G_old).abs().max()) <= 1e-5 * scale + 1e-3          # folded == un-folded wgrad
    assert torch.allclose(gb_ref, gb_u8, atol=1e-3, rtol=1e-5)


def test_gemm_dact_bit_mask_equals_fp16_mask(ops):
    """fc1 data gradient with the ReLU mask as 1 bit per element (as conv_shift_fwd emits it) == the same GEMM masked
    by the fp16 activation, incl. the column remap into conv3's zero-bordered grid; M spans many tiles per CTA."""
    torch.manual_seed(5)
    M, N, K = 20000, 49 * 64, 512
    A = (torch.randn(M, K, device="cuda") * 0.3).half()
    W = (torch.randn(N, K, device="cuda") * 0.3).half()
    saved = torch.relu(torch.randn(M, N, device="cuda")).half()
    bits = ((saved.reshape(-1, 16) > 0).to(torch.int32) << torch.arange(16, device="cuda", dtype=torch.int32)
            ).sum(1).to(torch.int16)
    out_a = torch.zeros(M, 81 * 64, dtype=torch.float16, device="cuda")
    out_b = torch.zeros_like(out_a)
    ops.gemm(A, W, out_a, M=M, N=N, K=K, lda=K, ldb=K, ldc=81 * 64, saved=saved, ld_saved=N, mode=ops.MODE_F16_DACT,
             act=ops.ACT_RELU, remap=(64, 7, 9))
    ops.gemm(A, W, out_b, M=M, N=N, K=K, lda=K, ldb=K, ldc=81 * 64, saved_bits=bits, ld_saved=N, mode=ops.MODE_F16_DACT,
             act=ops.ACT_RELU, remap=(64, 7, 9))
    torch.cuda.synchronize()
    assert torch.equal(out_a, out_b)
    ref = (A[:512].float() @ W.float().t()) * (saved[:512].float() > 0)
    grid = out_b[:512].float().view(512, 9, 9, 64)
    assert torch.allclose(grid[:, :7, :7].reshape(512, -1), ref, atol=5e-2, rtol=5e-3)


@pytest.mark.parametrize("n,T,N", [(1, 0, 0), (7, 0, 0), (4096, 0, 0), (524288, 128, 4096), (100003, 0, 0),
                                   (8 * 1024 * 1024 + 5, 0, 0)])
def test_shuffle_indices_is_a_keyed_permutation(ops, n, T, N):
    """ops.shuffle_indices (ppo2.py:160 on the device): a bijection of [0, n) for any n, different for different keys,
    composed with the env-major -> buffer offset map of sf01 when (T, N) are given; positions look uniform."""
    out1 = torch.empty(n, dtype=torch.int64, device="cuda")
    out2 = torch.empty(n, dtype=torch.int64, device="cuda")
    ops.shuffle_indices(out1, n, 0x1234567890ABCDEF, T, N)
    ops.shuffle_indices(out2, n, 0x0FEDCBA987654321, T, N)
    torch.cuda.synchronize()
    assert torch.equal(torch.sort(out1).values, torch.arange(n, device="cuda"))
    assert torch.equal(torch.sort(out2).values, torch.arange(n, device="cuda"))
    if n >= 4096:
        assert float((out1 == out2).float().mean()) < 0.01
        # a uniform permutation has E[pi(i)] = (n-1)/2 over any block of positions; |corr(i, pi(i))| small
        x = out1.double()
        if T:
            e, t = x % N, torch.div(x, N, rounding_mode="floor")           # undo offset t*N + e -> flat e*T + t
            x = e * T + t
        i = torch.arange(n, device="cuda", dtype=torch.float64)
        corr = float(((x - x.mean()) * (i - i.mean())).mean() / (x.std() * i.std()))
        assert abs(corr) < 0.02, corr
        first = x[: n // 16].mean() / ((n - 1) / 2.0)
        assert abs(float(first) - 1.0) < 0.05
    out3 = torch.empty(n, dtype=torch.int64, device="cuda")
    ops.shuffle_indices(out3, n, 0x1234567890ABCDEF, T, N)
    assert torch.equal(out1, out3)                                         # reproducible given the key


def test_weight_gradient_reductions_repeat_bit_for_bit(ops):
    """Cross-CTA reductions (split-K GEMM weight gradient, shift-conv weight and bias gradients, bias column sums,
    gradient sum of squares) add their per-CTA parts in a fixed order: the same inputs give the same bits on every
    call, so a training run repeats exactly."""
    torch.manual_seed(7)
    Kred, M, N = 20000, 576, 64
    A = (torch.randn(Kred, M, device="cuda") * 0.5).half()
    B = (torch.randn(Kred, N, device="cuda") * 0.5).half()
    B_, Hg, Wg, Nc = 64, 21, 21, 32
    x16 = (torch.randn(B_ * Hg * Wg, 64, device="cuda")).half()
    dz = torch.zeros(B_, Hg, Wg, Nc, dtype=torch.float16, device="cuda")
    dz[:, :20, :20] = (torch.randn(B_, 20, 20, Nc, device="cuda") * 0.5).half()
    g = torch.randn(1 << 20, device="cuda")

    def run():
        C = torch.zeros(M, N, device="cuda")
        ops.gemm(A, B, C, M=M, N=N, K=Kred, lda=M, ldb=N, ldc=N, mn_major=True, mode=ops.MODE_F32_ATOMIC,
                 alpha=0.25, split_k=16)
        G = torch.zeros(256, Nc, device="cuda")
        gb = torch.zeros(Nc, device="cuda")
        ops.conv_shift_wgrad(x16, B_ * Hg * Wg, 64, dz, Nc, [0, 1, Wg, Wg + 1], G, Nc, alpha=1.0 / 255, gbias=gb)
        db = torch.zeros(N, device="cuda")
        ops.colsum(B, db, Kred, N, N)
        ss = torch.zeros(1, dtype=torch.float64, device="cuda")
        ops.sumsq(g, ss)
        torch.cuda.synchronize()
        return C, G, gb, db, ss

    first = run()
    assert float(first[0].abs().max()) > 0 and float(first[1].abs().max()) > 0
    for _ in range(3):
        for a, b in zip(first, run()):
            assert torch.equal(a, b)
