"""Every convolution path of nn.Tower against a float64 reference.

The conv paths are chosen from the shapes (nn.plan_conv_stack).  For each configuration -- a cnn tower (NatureCNN convs
unless stated) for uint8 observations of one shape, or the DQN conv_only trunk (SAME padding, xavier init) -- a tower runs
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
from _net_refs import kernel_act as _kernel_act, reference as _reference

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")


def _is_default(t):
    g = t.sg
    assert t.shift_mode and t.fused_u8
    assert [s["kx"] for s in g] == [2, 2, 3]
    assert all(b is not None for b in t.hbits)


def _shift_unfused(t):                                                        # c1 from s2d_gather, unfolded c1 wgrad
    assert t.shift_mode and not t.fused_u8 and t.x16 is not None and [s["kx"] for s in t.sg] == [1, 2, 3]


def _implicit_s2d(t):
    c1, c2, c3 = t.convs
    assert not t.shift_mode and c1.implicit and c1.s2d and c2.implicit and c3.implicit
    assert c2.implicit_dgrad and c3.implicit_dgrad and c1.geom[2] == 64 and c2.geom[2] == 32


def _implicit_superpixel(t):
    c1, c2, c3 = t.convs
    assert not t.shift_mode and c1.implicit and not c1.s2d and c1.geom[2] == 16 and c1.geom[4] == 2
    assert c2.implicit and c3.implicit and c2.implicit_dgrad


def _implicit_merged(t):                                                      # 4 pixels of 16 channels per tap
    c1, c2, c3 = t.convs
    assert not t.shift_mode and c1.implicit and not c1.s2d and c1.geom[2] == 64 and c1.geom[4] == 2
    assert c2.implicit_dgrad and c3.implicit_dgrad


def _explicit_c1(t):
    c1, c2, c3 = t.convs
    assert not t.shift_mode and not c1.implicit and t.cols[0] is not None
    assert c2.implicit and c3.implicit and c2.implicit_dgrad and c3.implicit_dgrad


def _explicit_c2_c3(t):
    c1, c2, c3 = t.convs
    assert not t.shift_mode and c1.implicit and c1.s2d
    assert not c2.implicit and not c3.implicit and all(d is not None for d in t.dcols[1:])   # GEMM + col2im dgrads


def _dqn_conv_only(t):
    c1, c2, c3 = t.convs
    assert not t.shift_mode and all(c.same for c in t.convs)
    assert not c1.implicit and c2.implicit and c3.implicit                    # explicit c1, padded implicit c2 / c3
    assert not c2.implicit_dgrad and not c3.implicit_dgrad                    # col2im data gradients


def _dqn_conv_only_superpixel(t):
    c1, c2, c3 = t.convs
    assert not t.shift_mode and c1.implicit and c1.geom[2] == 16 and c2.implicit and c3.implicit
    assert not c2.implicit_dgrad and not c3.implicit_dgrad


def _dqn_conv_only_plain16(t):                                               # 16 channels per tap, padded
    c1, c2, c3 = t.convs
    assert not t.shift_mode and c1.implicit and c1.geom[2] == 16 and c1.geom[4] == 8 and c2.implicit and c3.implicit
    assert not c2.implicit_dgrad and not c3.implicit_dgrad


C48 = (("c1", 48, 8, 4), ("c2", 48, 4, 2), ("c3", 64, 3, 1))
# name: (observation shape, tower kind, convs (None: NatureCNN), check of the planned path)
CONFIGS = {
    "default": ((84, 84, 4), "cnn", None, _is_default),
    "shift_unfused_60x60x8": ((60, 60, 8), "cnn", None, _shift_unfused),
    "implicit_s2d_64x64x4": ((64, 64, 4), "cnn", None, _implicit_s2d),
    "implicit_superpixel_85x84x4": ((85, 84, 4), "cnn", None, _implicit_superpixel),
    "implicit_merged_84x84x16": ((84, 84, 16), "cnn", None, _implicit_merged),
    "explicit_c1_84x84x6": ((84, 84, 6), "cnn", None, _explicit_c1),
    "explicit_c2_c3_48_filters": ((84, 84, 4), "cnn", C48, _explicit_c2_c3),
    "dqn_conv_only": ((84, 84, 4), "conv_only", None, _dqn_conv_only),
    "dqn_conv_only_84x84x8": ((84, 84, 8), "conv_only", None, _dqn_conv_only_superpixel),
    "dqn_conv_only_84x84x16": ((84, 84, 16), "conv_only", None, _dqn_conv_only_plain16),
}

# g per compared tensor and batch: 3.5x the maximum observed on an H100 80GB HBM3 (700 W) (floor 1e-8).  Latent
# activations: per configuration, over both batches and the ReLU-decision check below; default and dqn_conv_only share
# one value from their maximum, 2.1e-7 (dqn_conv_only; 8e-9 on default).  Gradients below, per layer (weights), then
# per layer (biases).  One g per tensor: the network's |W| scale S over-estimates the error of the deep layers'
# gradients (c1's by ~100x against c3's bias), and a single g loose enough for c3's bias would accept c1's gradient
# computed with an image dropped.
_OBSERVED_LAT = {
    "shift_unfused_60x60x8": 1.75e-8,
    "implicit_s2d_64x64x4": 1.88e-8,
    "implicit_superpixel_85x84x4": 7.16e-7,       # a ReLU decision of c2 at B = 300
    "implicit_merged_84x84x16": 5.66e-8,
    "explicit_c1_84x84x6": 2.25e-8,
    "explicit_c2_c3_48_filters": 2.85e-8,
    "dqn_conv_only_84x84x8": 2.79e-7,
    "dqn_conv_only_84x84x16": 2.73e-7,
}
# fp16 outputs, r = 2^-11 on top
G_LAT = {"default": 7e-7, "dqn_conv_only": 7e-7, **{k: 3.5 * v for k, v in _OBSERVED_LAT.items()}}
_OBSERVED = {
    ("default", 37): ([8.42e-7, 1.56e-6, 1.59e-6, 1.21e-6], [1.39e-7, 1.80e-6, 2.14e-5, 0.0]),
    ("default", 300): ([4.06e-7, 1.57e-6, 9.69e-7, 1.25e-6], [2.36e-7, 5.21e-6, 3.74e-5, 2.31e-8]),
    ("dqn_conv_only", 37): ([6.97e-6, 5.32e-6, 1.23e-6], [6.97e-6, 4.31e-6, 9.35e-9]),
    ("dqn_conv_only", 300): ([2.72e-6, 6.80e-6, 5.49e-7], [1.88e-6, 1.57e-6, 1.76e-8]),
    ("shift_unfused_60x60x8", 37): ([1.22e-7, 3.85e-7, 3.53e-7, 7.90e-7], [8.34e-8, 9.57e-7, 1.19e-5, 0.0]),
    ("shift_unfused_60x60x8", 300): ([1.69e-6, 2.97e-7, 4.03e-7, 5.73e-7], [5.88e-7, 6.00e-7, 3.77e-5, 2.32e-8]),
    ("implicit_s2d_64x64x4", 37): ([2.66e-7, 3.35e-6, 4.18e-7, 1.17e-6], [2.66e-7, 1.09e-5, 1.69e-5, 0.0]),
    ("implicit_s2d_64x64x4", 300): ([5.51e-7, 1.00e-6, 4.73e-7, 1.18e-6], [9.10e-8, 1.76e-6, 1.77e-5, 1.86e-8]),
    ("implicit_superpixel_85x84x4", 37): ([6.48e-7, 9.11e-7, 3.43e-7, 1.25e-6], [6.48e-7, 2.83e-6, 6.80e-6, 7.44e-9]),
    ("implicit_superpixel_85x84x4", 300): ([5.47e-7, 6.71e-7, 3.10e-7, 1.22e-6], [1.89e-7, 2.22e-6, 4.08e-6, 2.50e-8]),
    ("implicit_merged_84x84x16", 37): ([7.74e-8, 1.93e-7, 1.31e-7, 5.51e-7], [3.59e-8, 1.36e-6, 7.40e-6, 0.0]),
    ("implicit_merged_84x84x16", 300): ([9.58e-8, 3.54e-7, 1.19e-7, 5.56e-7], [9.57e-8, 7.64e-7, 4.38e-6, 1.65e-8]),
    ("explicit_c1_84x84x6", 37): ([6.06e-7, 9.09e-7, 3.95e-7, 6.43e-7], [1.87e-7, 4.45e-6, 1.09e-5, 0.0]),
    ("explicit_c1_84x84x6", 300): ([6.07e-7, 3.58e-7, 2.19e-7, 6.47e-7], [4.00e-7, 6.91e-7, 5.96e-6, 3.65e-8]),
    ("explicit_c2_c3_48_filters", 37): ([2.22e-7, 5.62e-7, 3.48e-7, 7.76e-7], [1.21e-7, 1.51e-6, 2.05e-5, 0.0]),
    ("explicit_c2_c3_48_filters", 300): ([5.85e-8, 7.58e-7, 2.14e-7, 7.54e-7], [2.15e-8, 1.51e-6, 6.83e-6, 1.95e-8]),
    ("dqn_conv_only_84x84x8", 37): ([4.60e-6, 5.99e-6, 2.53e-6], [2.36e-6, 2.94e-5, 1.32e-8]),
    ("dqn_conv_only_84x84x8", 300): ([3.14e-6, 7.97e-6, 4.93e-7], [4.17e-7, 2.38e-5, 1.44e-8]),
    ("dqn_conv_only_84x84x16", 37): ([2.20e-6, 2.53e-6, 2.88e-6], [5.99e-7, 7.86e-6, 7.63e-9]),
    ("dqn_conv_only_84x84x16", 300): ([1.23e-6, 2.14e-6, 1.22e-6], [2.30e-7, 2.52e-6, 8.59e-9]),
}
G_GRAD = {k: [3.5 * max(v, 1e-8) for v in w + b] for k, (w, b) in _OBSERVED.items()}   # fp32 outputs


def _build(name, B):
    from baselines_b200 import nn as bnn
    ob_shape, kind, convs, check = CONFIGS[name]
    kw = {} if convs is None else dict(convs=convs)
    rng = np.random.RandomState(11)
    store = bnn.ParamStore(DEV)
    if kind == "conv_only":
        tower = bnn.Tower(store, "conv_only", ob_shape, "trunk", "q", rng, B, init="xavier", same_pad=True,
                          tf_style="contrib", **kw)
    else:
        tower = bnn.Tower(store, "cnn", ob_shape, "pi", "m/pi", rng, B, **kw)
    store.finalize()
    tower.materialize()
    check(tower)                                  # the intended path was taken (a silent fall-back fails here)
    for l in tower.layers:                        # biases away from zero so the ReLU masks matter
        l.b.copy_(torch.from_numpy(rng.randn(l.N).astype(np.float32) * 0.05).to(DEV))
    tower.refresh()
    return tower, store, rng


@pytest.mark.parametrize("B", [37, 300])
@pytest.mark.parametrize("name", list(CONFIGS))
def test_conv_path_vs_float64(name, B):
    """Observed g on an H100 80GB HBM3 (700 W), latent / worst gradient:
         default, shift_unfused_60x60x8, implicit_*, explicit_*      3.6e-9 .. 1.9e-8 / 4.1e-6 .. 3.8e-5
         dqn_conv_only, dqn_conv_only_84x84x{8,16}                    9.1e-8 .. 2.8e-7 / 2.5e-6 .. 2.9e-5
    The worst gradient is c3's bias (conv_only: Conv_1's weights or bias); per-tensor values are above G_GRAD, and
    each run prints its own numbers."""
    tower, store, rng = _build(name, B)
    pool = torch.from_numpy(rng.randint(0, 256, (2 * B + 3,) + CONFIGS[name][0]).astype(np.uint8)).to(DEV)
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
        assert worst <= G_LAT[name], (name, B, i, worst)

    lat_ref = ref * (lat > 0).double()
    lat_S = S * (lat > 0).double()
    gl = R.excess(lat, lat_ref, lat_S, R.R_F16)
    gg = {n: R.excess(torch.from_numpy(grads[n]).to(DEV).double().reshape(gref[k].shape), gref[k], gS[k], R.R_F32)
          for k, n in enumerate(wn + bn)}
    print(f"  {name} B={B}: latent g {gl:.2e}; grads g " + " ".join(f"{n.split('/')[-2]}:{v:.2e}" for n, v in gg.items()))
    R.assert_within(lat, lat_ref, lat_S, G_LAT[name], R.R_F16, {"c1 tap zeroed": ref_tap * (lat > 0).double()},
                    what=f"{name} B={B} latent")
    gmax = G_GRAD[(name, B)]
    for k, n in enumerate(wn + bn):
        got = torch.from_numpy(grads[n]).to(DEV).double().reshape(gref[k].shape)
        R.assert_within(got, gref[k], gS[k], gmax[k], R.R_F32, {"image 0 dropped": g_drop[k]}, what=f"{name} B={B} {n}")
