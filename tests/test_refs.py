"""CPU tests of the float64 references and the error bound in tests/_refs.py (no GPU needed)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import _refs as R


def _nchw_conv(x, w_hwio, stride, pad_lo, pad_hi):
    xp = F.pad(x.permute(0, 3, 1, 2), (pad_lo[1], pad_hi[1], pad_lo[0], pad_hi[0]))
    return F.conv2d(xp, w_hwio.permute(3, 2, 0, 1), stride=stride).permute(0, 2, 3, 1)


@pytest.mark.parametrize("B,H,W,C,Rr,S,st,pad,N", [(2, 9, 7, 3, 3, 3, (1, 1), (0, 0), 5), (3, 21, 21, 4, 4, 4, (2, 2), (1, 1), 6),
                                                  (1, 84, 84, 4, 8, 8, (4, 4), (2, 2), 8), (2, 11, 13, 2, 8, 2, (4, 1), (0, 0), 3),
                                                  (2, 10, 10, 5, 5, 5, (2, 2), (2, 2), 4)])
def test_conv_refs_match_float64_conv2d(B, H, W, C, Rr, S, st, pad, N):
    g = torch.Generator().manual_seed(B * 100 + H)
    x = torch.randn(B, H, W, C, generator=g, dtype=torch.float64)
    w = torch.randn(Rr, S, C, N, generator=g, dtype=torch.float64)
    OH, OW = (H + 2 * pad[0] - Rr) // st[0] + 1, (W + 2 * pad[1] - S) // st[1] + 1
    hi = (max((OH - 1) * st[0] + Rr - pad[0] - H, 0), max((OW - 1) * st[1] + S - pad[1] - W, 0))
    want = _nchw_conv(x, w, st, pad, hi)
    got = R.conv2d(x, w, st, pad, OH, OW)
    assert got.shape == want.shape and torch.allclose(got, want, rtol=1e-12, atol=1e-12)
    # gradients against autograd of the same float64 conv
    dz = torch.randn(B, OH, OW, N, generator=g, dtype=torch.float64)
    xr, wr = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    (_nchw_conv(xr, wr, st, pad, hi) * dz).sum().backward()
    assert torch.allclose(R.conv2d_wgrad(x, dz, Rr, S, st, pad), wr.grad.reshape(-1, N), rtol=1e-12, atol=1e-11)
    assert torch.allclose(R.conv2d_dgrad(dz, w, H, W, st, pad), xr.grad, rtol=1e-12, atol=1e-11)


def test_shift_conv_is_the_convolution_on_valid_positions():
    g = torch.Generator().manual_seed(1)
    B, Hg, Wg, C, N, k = 3, 9, 11, 4, 5, 3
    x = torch.randn(B, Hg, Wg, C, generator=g, dtype=torch.float64)
    w = torch.randn(k, k, C, N, generator=g, dtype=torch.float64)
    Wt = w.reshape(k * k * C, N).t()
    shifts = [a * Wg + b for a in range(k) for b in range(k)]
    OH, OW = Hg - k + 1, Wg - k + 1
    out = R.shift_conv(x.reshape(-1, C), shifts, Wt).view(B, Hg, Wg, N)
    assert torch.allclose(out[:, :OH, :OW], R.conv2d(x, w, (1, 1), (0, 0), OH, OW), rtol=1e-12, atol=1e-12)
    # wgrad over a zero-bordered dY == the convolution's weight gradient; dgrad by negative shifts == transposed conv
    dz = torch.randn(B, OH, OW, N, generator=g, dtype=torch.float64)
    dY = torch.zeros(B, Hg, Wg, N, dtype=torch.float64)
    dY[:, :OH, :OW] = dz
    G = R.shift_wgrad(x.reshape(-1, C), dY.reshape(-1, N), shifts)
    assert torch.allclose(G, R.conv2d_wgrad(x, dz, k, k, (1, 1), (0, 0)), rtol=1e-12, atol=1e-11)
    Wd = torch.cat([w[a, b] for a in range(k) for b in range(k)], 1)              # [C, (t, n)]: the dgrad operand
    dX = R.shift_conv(dY.reshape(-1, N), [-s for s in shifts], Wd)
    assert torch.allclose(dX.view(B, Hg, Wg, C), R.conv2d_dgrad(dz, w, Hg, Wg, (1, 1), (0, 0)), rtol=1e-12, atol=1e-11)


def test_space_to_depth_round_trip_and_relu_bits():
    x = torch.arange(2 * 8 * 4 * 3, dtype=torch.float64).view(2, 8, 4, 3)
    y = R.space_to_depth(x, 2)
    assert y.shape == (2, 4, 2, 12)
    assert float(y[1, 3, 1, (1 * 2 + 0) * 3 + 2]) == float(x[1, 7, 2, 2])        # channel (dy, dx, c)
    assert torch.equal(R.depth_to_space(y, 2), x)
    v = torch.tensor([1.0, -1.0, 0.0, 2.0] * 4 + [0.0] * 15 + [3.0])
    b = R.relu_bits(v)
    assert b.tolist() == [0b1001100110011001 - 65536, -32768]


def test_small_ints_and_probe_rows():
    g = torch.Generator().manual_seed(0)
    v = R.small_ints((1000, 50), 0.3, g)
    assert set(v.unique().tolist()) <= {-2.0, -1.0, 0.0, 1.0, 2.0} and 0.2 < float((v != 0).double().mean()) < 0.4
    rows = R.probe_rows(1000, tile=128, kblock=64, ends=[333, 1000], shifts=[3], n_random=4, seed=1)
    s = set(rows.tolist())
    for t0 in range(0, 1000, 128):
        assert t0 in s and min(t0 + 127, 999) in s
    assert all(min(k + 63, 999) in s for k in range(0, 1000, 64))
    assert {332, 999, 128 - 3, 256 - 3 - 1}.issubset(s) and rows.tolist() == sorted(s)
    valid = torch.arange(1000) % 2 == 0
    assert all(r % 2 == 0 for r in R.probe_rows(1000, kblock=64, valid=valid).tolist())
    Z = R.rows_only(torch.ones(10, 3), torch.tensor([2, 7]))
    assert float(Z.sum()) == 6 and float(Z[2].sum()) == 3


def test_exact_precondition_and_bound_self_check():
    A = torch.full((4, 600), 2.0, dtype=torch.float64)
    B = torch.full((3, 600), 2.0, dtype=torch.float64)
    with pytest.raises(AssertionError):
        R.assert_exact_ok(A.abs() @ B.abs().t())                                   # 2400 > 2048
    assert R.assert_exact_ok(A[:, :500].abs() @ B[:, :500].abs().t()) == 2000
    # bound: a perturbation of relative size 1e-4 of |A|@|B| passes g = 4e-4 and fails g = 5e-5
    g = torch.Generator().manual_seed(3)
    A = torch.randn(64, 300, generator=g, dtype=torch.float64)
    B = torch.randn(32, 300, generator=g, dtype=torch.float64)
    ref, scale = R.gemm(A, B), A.abs() @ B.abs().t()
    got = ref + 1e-4 * scale * torch.sign(torch.randn(ref.shape, generator=g, dtype=torch.float64))
    assert abs(R.excess(got, ref, scale, 0.0) - 1e-4) < 1e-12
    drop_row = ref - A[:, -1:] @ B[:, -1:].t()
    zero_tap = ref - A[:, :10] @ B[:, :10].t()
    R.assert_within(got, ref, scale, 4e-4, 0.0, {"row dropped": drop_row, "tap zeroed": zero_tap})
    with pytest.raises(AssertionError):
        R.assert_within(got, ref, scale, 5e-5, 0.0, {"row dropped": drop_row})
    # a bound so loose that it accepts a dropped row fails the self-check
    with pytest.raises(AssertionError, match="accepts the reference with row dropped"):
        R.assert_within(got, ref, scale, 1.0, 0.0, {"row dropped": drop_row})
    with pytest.raises(AssertionError):
        R.assert_within(got, ref, scale, 4e-4, 0.0, {})
    bad = got.clone()
    bad[0, 0] = float("nan")
    with pytest.raises(AssertionError, match="non-finite"):
        R.assert_within(bad, ref, scale, 4e-4, 0.0, {"row dropped": drop_row})
