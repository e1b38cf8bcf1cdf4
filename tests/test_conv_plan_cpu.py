"""nn.plan_conv_stack: the convolution path of every layer, from the shapes alone (no GPU)."""
import pytest

from baselines_b200.nn import NATURE_CONVS, plan_conv_stack

C48 = (("c1", 48, 8, 4), ("c2", 48, 4, 2), ("c3", 64, 3, 1))


def _plan(ob_shape, convs=NATURE_CONVS, same_pad=False, has_fc=True):
    return plan_conv_stack(ob_shape, convs, same_pad, has_fc)


def test_default_is_shift_gemm_from_uint8():
    p = _plan((84, 84, 4))
    assert p.shift and p.fused_u8
    assert [l.path for l in p.layers] == ["shift"] * 3
    assert [l.kx for l in p.layers] == [2, 2, 3]                 # x-folded weight gradients
    assert [l.s2d for l in p.layers] == [True, True, False]


def test_shift_unfused_first_layer():
    # 128 space-to-depth channels in c1: s2d_gather feeds the TMA path, and c1's weight gradient is not folded
    p = _plan((60, 60, 8))
    assert p.shift and not p.fused_u8 and [l.kx for l in p.layers] == [1, 2, 3]


def test_shift_span_limit_of_128_channel_inputs():
    # c1 over 8 channels of 84x84: space-to-depth gives C = 128 and a 22-row shift span, past the 16 rows
    # b200rl_conv_shift_fwd takes for C = 128; nor can c1 run space-to-depth'ed as an implicit GEMM
    # (b200rl_conv_gemm takes at most 64 channels per tap), so it reads 16-channel super-pixels
    p = _plan((84, 84, 8))
    assert not p.shift
    c1, c2, c3 = p.layers
    assert c1.path == "implicit" and not c1.s2d and c1.geom[2] == 16
    assert c2.implicit_dgrad and c3.implicit_dgrad


@pytest.mark.parametrize("ob_shape", [(64, 64, 4), (72, 72, 4), (80, 80, 4), (96, 96, 4)])
def test_implicit_s2d(ob_shape):
    p = _plan(ob_shape)
    assert not p.shift and not p.fused_u8
    c1, c2, c3 = p.layers
    assert [l.path for l in p.layers] == ["implicit"] * 3
    assert c1.s2d and c1.geom[2] == 64 and not c1.implicit_dgrad
    assert c2.geom[2] == 32 and c2.implicit_dgrad and c3.geom[2] == 64 and c3.implicit_dgrad


def test_implicit_superpixel():
    c1, c2, c3 = _plan((85, 84, 4)).layers
    assert c1.path == "implicit" and not c1.s2d and c1.geom[2] == 16 and c1.geom[4] == 2
    assert c2.path == c3.path == "implicit" and c2.implicit_dgrad and c3.implicit_dgrad


@pytest.mark.parametrize("C", [1, 3, 6])
def test_explicit_first_layer(C):
    p = _plan((84, 84, C))
    c1, c2, c3 = p.layers
    assert not p.shift and c1.path == "explicit" and c1.geom is None and not c1.s2d
    assert c2.path == "implicit" and c2.geom[2] == 64 and c2.implicit_dgrad
    assert c3.path == "implicit" and c3.geom[2] == 64 and c3.implicit_dgrad


def test_implicit_merged_pixels():
    c1, c2, c3 = _plan((84, 84, 16)).layers
    assert c1.path == "implicit" and not c1.s2d and c1.geom[2] == 64
    assert c2.implicit_dgrad and c3.implicit_dgrad


def test_48_filters():
    p = _plan((84, 84, 4), C48)
    c1, c2, c3 = p.layers
    assert not p.shift and c1.path == "implicit" and c1.s2d
    assert c2.path == c3.path == "explicit" and not c2.implicit_dgrad and not c3.implicit_dgrad


@pytest.mark.parametrize("C,c1_geom_c", [(1, None), (3, None), (4, None), (8, 16), (16, 16)])
def test_conv_only_same(C, c1_geom_c):
    p = _plan((84, 84, C), same_pad=True, has_fc=False)
    c1, c2, c3 = p.layers
    assert not p.shift and not c1.s2d
    assert c1.path == ("explicit" if c1_geom_c is None else "implicit")
    assert c1_geom_c is None or c1.geom[2] == c1_geom_c
    assert c2.path == "implicit" and c2.geom[2] == 32 and not c2.implicit_dgrad      # col2im data gradients
    assert c3.path == "implicit" and c3.geom[2] == 64 and not c3.implicit_dgrad


def test_conv_only_valid_shift_stack_raises():
    with pytest.raises(NotImplementedError, match="shift-mode conv_only towers"):
        _plan((84, 84, 4), has_fc=False)
