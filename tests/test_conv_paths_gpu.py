"""Every convolution path of nn.Tower against a float64 reference.

The conv paths are chosen by shape and by environment switches (INTEGRATION.md section 6).  For each configuration a
NatureCNN tower for (84, 84, 4) uint8 observations -- and the DQN conv_only trunk (SAME padding, xavier init) -- runs
forward and backward from a fixed d(latent), at a small odd batch and at a batch that gives every persistent CTA
several tiles.  The latent activations and every weight and bias gradient are compared with float64 autograd of the
same network: the weights are the fp16-rounded operands the kernels see (c1 with 1/255 folded in, then rounded) and
the stored activations are rounded to fp16.  The reference follows the kernels' ReLU decisions (a mask taken from
the kernels' own activations); the test asserts that the two disagree only where the float64 pre-activation lies
within the error bound of zero.

Bound: per element, |got - ref| <= g * S + r * |ref|, where S is the same network evaluated on |x|, |W|, |b| with the
same masks (the network analogue of |A| @ |B|) and, for gradients, the float64 gradient of that absolute network.
Every comparison also checks that the bound rejects the reference computed with one image dropped (gradients) or
with one c1 tap zeroed (latent).

G_LAT / G_GRAD were set from an H100 run, at 3.5x the observed maxima (see their definitions).
"""
import numpy as np
import pytest
import torch

import _refs as R

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")


def _is_default(t):
    g = t.sg
    assert t.shift_mode and t.fused_u8
    assert [s["kx"] for s in g] == [2, 2, 3] and [s["kx_fwd"] for s in g] == [1, 1, 1]
    assert all(b is not None for b in t.hbits)


def _no_xfold(t):
    assert t.shift_mode and t.fused_u8 and [s["kx"] for s in t.sg] == [1, 1, 1]


def _xfold_fwd(t):
    assert t.shift_mode and not t.fused_u8 and [s["kx_fwd"] for s in t.sg] == [2, 2, 3]


def _no_fused(t):
    assert t.shift_mode and not t.fused_u8 and t.x16 is not None and [s["kx_fwd"] for s in t.sg] == [1, 1, 1]


def _no_bits(t):
    assert t.shift_mode and all(b is None for b in t.hbits)


def _implicit_s2d(t):
    c1, c2, c3 = t.convs
    assert not t.shift_mode and c1.implicit and c1.s2d and c2.implicit and c3.implicit
    assert c2.implicit_dgrad and c3.implicit_dgrad and c1.geom[2] == 64


def _implicit_superpixel(t):
    c1, c2, c3 = t.convs
    assert not t.shift_mode and c1.implicit and not c1.s2d and c1.geom[2] == 16 and c1.geom[4] == 2
    assert c2.implicit and c3.implicit and c2.implicit_dgrad


def _explicit(t):
    assert not t.shift_mode and not any(c.implicit for c in t.convs) and all(c is not None for c in t.cols)


def _dqn_conv_only(t):
    c1, c2, c3 = t.convs
    assert not t.shift_mode and all(c.same for c in t.convs)
    assert not c1.implicit and c2.implicit and c3.implicit                    # explicit c1, padded implicit c2 / c3
    assert not c2.implicit_dgrad and not c3.implicit_dgrad                    # col2im data gradients


CONFIGS = {
    "default": ({}, _is_default),
    "no_xfold": ({"B200RL_NO_XFOLD": "1"}, _no_xfold),
    "xfold_fwd_no_fused_u8": ({"B200RL_XFOLD_FWD": "1", "B200RL_NO_FUSED_U8": "1"}, _xfold_fwd),
    "no_fused_u8": ({"B200RL_NO_FUSED_U8": "1"}, _no_fused),
    "no_relu_bits": ({"B200RL_NO_RELU_BITS": "1"}, _no_bits),
    "no_shift": ({"B200RL_NO_SHIFT": "1"}, _implicit_s2d),
    "no_shift_no_s2d": ({"B200RL_NO_SHIFT": "1", "B200RL_NO_S2D": "1"}, _implicit_superpixel),
    "explicit_conv": ({"B200RL_EXPLICIT_CONV": "1"}, _explicit),
    "dqn_conv_only": ({}, _dqn_conv_only),
}
SWITCHES = ("B200RL_NO_XFOLD", "B200RL_XFOLD_FWD", "B200RL_NO_FUSED_U8", "B200RL_NO_RELU_BITS", "B200RL_NO_SHIFT",
            "B200RL_NO_S2D", "B200RL_EXPLICIT_CONV")

# g per compared tensor and batch: 3.5x the maximum observed on an H100 80GB HBM3 (700 W) over the configurations
# (floor 1e-8).  Latent: 2.1e-7 (dqn_conv_only; 8e-9 on the NatureCNN paths).  Gradients below, per layer (weights),
# then per layer (biases).  One g per tensor: the network's |W| scale S over-estimates the error of the deep layers'
# gradients (c1's by ~100x against c3's bias), and a single g loose enough for c3's bias would accept c1's gradient
# computed with an image dropped.
G_LAT = 7e-7         # latent activations (fp16 outputs, r = 2^-11 on top)
_OBSERVED = {
    ("cnn", 37): ([8.42e-7, 1.56e-6, 1.59e-6, 1.21e-6], [1.39e-7, 1.80e-6, 2.14e-5, 0.0]),
    ("cnn", 300): ([4.06e-7, 1.57e-6, 9.69e-7, 1.25e-6], [2.36e-7, 5.21e-6, 3.74e-5, 2.31e-8]),
    ("conv_only", 37): ([6.97e-6, 5.32e-6, 1.23e-6], [6.97e-6, 4.31e-6, 9.35e-9]),
    ("conv_only", 300): ([2.72e-6, 6.80e-6, 5.49e-7], [1.88e-6, 1.57e-6, 1.76e-8]),
}
G_GRAD = {k: [3.5 * max(v, 1e-8) for v in w + b] for k, (w, b) in _OBSERVED.items()}   # fp32 outputs


def _build(name, B, monkeypatch):
    from baselines_b200 import nn as bnn
    env, check = CONFIGS[name]
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    rng = np.random.RandomState(11)
    store = bnn.ParamStore(DEV)
    if name == "dqn_conv_only":
        tower = bnn.Tower(store, "conv_only", (84, 84, 4), "trunk", "q", rng, B, init="xavier", same_pad=True,
                          tf_style="contrib")
    else:
        tower = bnn.Tower(store, "cnn", (84, 84, 4), "pi", "m/pi", rng, B)
    store.finalize()
    tower.materialize()
    check(tower)                                  # the intended path was taken (a silent fall-back fails here)
    for l in tower.layers:                        # biases away from zero so the ReLU masks matter
        l.b.copy_(torch.from_numpy(rng.randn(l.N).astype(np.float32) * 0.05).to(DEV))
    tower.refresh()
    return tower, store, rng


def _kernel_act(tower, i, B):
    """NHWC [B, OH, OW, nf] view of the kernels' stored activation of conv i."""
    c = tower.convs[i]
    h = tower.hconv[i]
    if tower.shift_mode and i + 1 < len(tower.convs) and tower.convs[i + 1].stride > 1:
        s = tower.convs[i + 1].stride
        return R.depth_to_space(h[:B].view(B, c.OH // s, c.OW // s, s * s * c.nf), s)
    return h.reshape(-1)[:B * c.P * c.nf].view(B, c.OH, c.OW, c.nf)


def _pads(c):
    if not c.same:
        return 0, 0
    return max((c.OH - 1) * c.stride + c.rf - c.H, 0) // 2, max((c.OW - 1) * c.stride + c.rf - c.W, 0) // 2


def _reference(tower, imgs, Ws, bs, masks, dlat, B, rnd=True):
    """float64 forward through the conv stack (+ fc1) with the given weights and ReLU masks; returns the last layer's
    pre-activation and the pre-activations of every conv.  Backward: d(sum(pre_last * dlat) / B)."""
    a = imgs
    pres = []
    nconv = len(tower.convs)
    for i, c in enumerate(tower.convs):
        pre = R.conv2d(a, Ws[i], (c.stride, c.stride), _pads(c), c.OH, c.OW) + bs[i]
        pres.append(pre)
        if i + 1 == nconv and not tower.fcs:
            return pre.reshape(B, -1), pres
        a = pre * masks[i]
        if rnd:                                   # the kernels store activations in fp16
            a = a + (a.half().double() - a).detach()
    flat = a.reshape(B, -1)
    return flat @ Ws[nconv] + bs[nconv], pres


@pytest.mark.parametrize("B", [37, 300])
@pytest.mark.parametrize("name", list(CONFIGS))
def test_conv_path_vs_float64(name, B, monkeypatch):
    """Observed g on an H100 80GB HBM3 (700 W), latent / worst gradient:
         shift-GEMM paths (default, no_xfold, xfold_fwd_no_fused_u8, no_fused_u8, no_relu_bits)  8.3e-9 / 3.7e-5
         no_shift, no_shift_no_s2d, explicit_conv                                                 8.3e-9 / 3.7e-5
         dqn_conv_only                                                                            2.1e-7 / 7.0e-6
    The worst gradient is c3's bias at B = 300 on every NatureCNN path; per-tensor values are above G_GRAD, and
    each run prints its own numbers."""
    tower, store, rng = _build(name, B, monkeypatch)
    pool = torch.from_numpy(rng.randint(0, 256, (2 * B + 3, 84, 84, 4)).astype(np.uint8)).to(DEV)
    idx = torch.from_numpy(rng.permutation(2 * B + 3)[:B].astype(np.int64)).to(DEV)
    h, ldh = tower.forward(pool, B, idx)
    L = tower.latent_dim
    lat = h.reshape(-1)[:B * ldh].view(B, ldh)[:, :L].double().clone()
    g = torch.from_numpy(rng.randn(B, L).astype(np.float32) * 0.1).to(DEV)
    dlat16 = (g * (lat > 0).float()).half()
    ldd = tower.ld_dlatent
    tower.dlatent.reshape(-1)[:B * ldd].view(B, ldd)[:, :L].copy_(dlat16)
    store.grads.zero_()
    tower.backward(B, 1.0 / B)
    torch.cuda.synchronize()
    masks = [(_kernel_act(tower, i, B) > 0).double() for i in range(len(tower.convs))]
    grads = store.export_tf("grads")
    params = store.export_tf("params")
    names = list(store.tf_map)                                # (w, b) per layer, in layer order
    wn, bn = names[0::2], names[1::2]
    scale1 = torch.tensor(1.0 / 255.0, dtype=torch.float32)
    w32 = [torch.from_numpy(params[n]) for n in wn]
    Ws = [((w32[0] * scale1) if i == 0 else w32[i]).half().double().to(DEV) for i in range(len(wn))]
    bs = [torch.from_numpy(params[n]).reshape(-1).double().to(DEV) for n in bn]
    imgs = pool[idx].double()
    dlat = dlat16.double()

    def run(Wl, bl, x, d, rnd=True):
        Wl = [w.clone().requires_grad_(True) for w in Wl]
        bl = [b.clone().requires_grad_(True) for b in bl]
        out, pres = _reference(tower, x, Wl, bl, masks, d, B, rnd)
        (out * d).sum().mul(1.0 / B).backward()
        gr = [w.grad / 255.0 if i == 0 else w.grad for i, w in enumerate(Wl)] + [b.grad for b in bl]
        return out.detach(), [p.detach() for p in pres], gr

    ref, pres, gref = run(Ws, bs, imgs, dlat)
    S, pres_abs, gS = run([w.abs() for w in Ws], [b.abs() for b in bs], imgs, dlat.abs(), rnd=False)
    Ws_tap = [w.clone() for w in Ws]
    Ws_tap[0][0, 0] = 0.0                                    # one c1 tap zeroed
    ref_tap, _, _ = run(Ws_tap, bs, imgs, dlat)
    d_drop = dlat.clone()
    d_drop[0] = 0.0                                          # image 0 dropped from the reductions
    _, _, g_drop = run(Ws, bs, imgs, d_drop)

    # the kernels' ReLU decisions differ from float64 only where the pre-activation is within the bound of zero
    for i, (p, pa, m) in enumerate(zip(pres, pres_abs, masks)):
        off = m != (p > 0).double()
        worst = float((p.abs()[off] / pa[off]).max()) if bool(off.any()) else 0.0
        print(f"  {name} B={B} conv{i + 1}: {int(off.sum())} ReLU decisions differ, max |pre|/S there {worst:.2e}")
        assert worst <= G_LAT, (name, B, i, worst)

    lat_ref = ref * (lat > 0).double()
    lat_S = S * (lat > 0).double()
    gl = R.excess(lat, lat_ref, lat_S, R.R_F16)
    gg = {n: R.excess(torch.from_numpy(grads[n]).to(DEV).double().reshape(gref[k].shape), gref[k], gS[k], R.R_F32)
          for k, n in enumerate(wn + bn)}
    print(f"  {name} B={B}: latent g {gl:.2e}; grads g " + " ".join(f"{n.split('/')[-2]}:{v:.2e}" for n, v in gg.items()))
    R.assert_within(lat, lat_ref, lat_S, G_LAT, R.R_F16, {"c1 tap zeroed": ref_tap * (lat > 0).double()},
                    what=f"{name} B={B} latent")
    gmax = G_GRAD[(tower.kind, B)]
    for k, n in enumerate(wn + bn):
        got = torch.from_numpy(grads[n]).to(DEV).double().reshape(gref[k].shape)
        R.assert_within(got, gref[k], gS[k], gmax[k], R.R_F32, {"image 0 dropped": g_drop[k]}, what=f"{name} B={B} {n}")
