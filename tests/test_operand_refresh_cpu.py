"""The fp16 operand declarations of nn.Tower (cast_jobs, operand_launches), read on towers built on the CPU: no kernel
runs.  Every cast reads the fp32 master weights, and together the casts write every element of every fp16 operand the
tower owns exactly once, padding excepted."""
import numpy as np
import pytest
import torch

from baselines_b200 import _lib, nn, ops

C48 = (("c1", 48, 8, 4), ("c2", 48, 4, 2), ("c3", 64, 3, 1))

# name -> (kind, ob_shape, Tower keyword arguments, expected conv paths)
TOWERS = {
    "mlp": ("mlp", (11,), {}, None),
    "mlp_layer_norm": ("mlp", (11,), dict(layer_norm=True, num_hidden=24), None),
    "shift_84x84x4": ("cnn", (84, 84, 4), {}, ["shift"] * 3),
    "shift_unfused_60x60x8": ("cnn", (60, 60, 8), {}, ["shift"] * 3),
    "implicit_s2d_64x64x4": ("cnn", (64, 64, 4), {}, ["implicit"] * 3),
    "implicit_superpixel_85x84x4": ("cnn", (85, 84, 4), {}, ["implicit"] * 3),
    "implicit_merged_84x84x16": ("cnn", (84, 84, 16), {}, ["implicit"] * 3),
    "explicit_c1_84x84x6": ("cnn", (84, 84, 6), {}, ["explicit", "implicit", "implicit"]),
    "explicit_48_filters": ("cnn", (84, 84, 4), dict(convs=C48), ["implicit", "explicit", "explicit"]),
    "conv_only_same_84x84x4": ("conv_only", (84, 84, 4), dict(same_pad=True, init="xavier", tf_style="contrib"),
                               ["explicit", "implicit", "implicit"]),
    "conv_only_same_84x84x8": ("conv_only", (84, 84, 8), dict(same_pad=True, init="xavier", tf_style="contrib"),
                               ["implicit"] * 3),
    "lstm": ("lstm", (7,), dict(nlstm=64), None),
    "cnn_lstm": ("cnn_lstm", (84, 84, 4), {}, ["shift"] * 3),
}


def _tower(name):
    kind, ob_shape, kw, paths = TOWERS[name]
    store = nn.ParamStore("cpu")
    tower = nn.Tower(store, kind, ob_shape, "pi", "m/pi", np.random.RandomState(3), 4, **kw)
    store.finalize()
    tower.materialize()
    assert paths is None or [l.path for l in tower.plan.layers] == paths
    return tower, store


def _operands(tower):
    """(name, fp16 tensor, bool mask of its non-padding elements) of every cast operand the tower owns, from the layer
    layouts alone."""
    out = []

    def linear(l):
        fwd = torch.zeros(l.N, l.Kf, dtype=torch.bool)
        fwd[:, :l.K] = True
        if l.split_in:                                 # [W^T | W^T] for the [hi | lo] input rows
            fwd[:, l.Kp:l.Kp + l.K] = True
        bwd = torch.zeros(l.K, l.Np, dtype=torch.bool)
        bwd[:, :l.N] = True
        out.extend([(l.name + ".w_fwd", l.w_fwd, fwd), (l.name + ".w_bwd", l.w_bwd, bwd)])

    for l in tower.layers:
        linear(l)
    if tower.shift_mode:
        for c, wd in zip(tower.convs[1:], tower.wd[1:]):
            out.append((c.name + ".wd", wd, torch.ones(wd.shape, dtype=torch.bool)))
    if tower.lstm is not None:
        lstm = tower.lstm
        linear(lstm.wx)
        out.append(("lstm.wh16", lstm.wh16, torch.ones(lstm.wh16.shape, dtype=torch.bool)))
        out.append(("lstm.whT16", lstm.whT16, torch.ones(lstm.whT16.shape, dtype=torch.bool)))
    return out


def _writes(jobs, operands):
    """Per operand: how many times the jobs write each of its elements.  Fails on a write outside every operand."""
    counts = [torch.zeros(t.numel(), dtype=torch.int64) for _, t, _ in operands]
    for j in jobs:
        r = torch.arange(j.R).view(-1, 1)
        c = torch.arange(j.C).view(1, -1)
        for out, idx in ((j.dst, r * j.ld_dst + c), (j.dstT, c * j.ld_t + r)):
            if out is None:
                continue
            assert out.dtype == torch.float16
            addr = out.data_ptr() + 2 * idx.reshape(-1)
            hit = False
            for (name, t, _), cnt in zip(operands, counts):
                lo = t.data_ptr()
                if lo <= addr.min() and addr.max() < lo + 2 * t.numel():
                    cnt.index_add_(0, (addr - lo) // 2, torch.ones_like(addr))
                    hit = True
                    break
            assert hit, f"a cast of [{j.R}, {j.C}] writes outside the tower's operands"
    return counts


@pytest.mark.parametrize("name", list(TOWERS))
def test_casts_cover_every_operand_once(name):
    tower, store = _tower(name)
    launches = _lib.LAUNCHES
    jobs = tower.cast_jobs()
    assert _lib.LAUNCHES == launches
    p0, p1 = store.params.data_ptr(), store.params.data_ptr() + 4 * store.params.numel()
    for j in jobs:
        assert isinstance(j, ops.CastJob)
        assert j.src.dtype == torch.float32 and j.src.is_contiguous()
        assert p0 <= j.src.data_ptr() and j.src.data_ptr() + 4 * j.R * j.C <= p1, "a cast reads outside store.params"
    operands = _operands(tower)
    for (nm, t, mask), cnt in zip(operands, _writes(jobs, operands)):
        cnt = cnt.view(t.shape)
        assert torch.equal(cnt[mask], torch.ones_like(cnt[mask])), f"{nm}: a non-padding element is not written once"
        assert not cnt[~mask].any(), f"{nm}: a padding element is written"


@pytest.mark.parametrize("name", list(TOWERS))
def test_non_cast_launches_write_each_wdg(name):
    tower, _ = _tower(name)
    launches = _lib.LAUNCHES
    decl = tower.operand_launches()
    assert _lib.LAUNCHES == launches
    wdg = [c for c in tower.convs if c.wdg is not None]
    assert len(decl) == len(wdg)
    for f, c in zip(decl, wdg):
        assert f.func is ops.dgrad_weights and f.args[0] is c.w and f.args[1] is c.wdg
