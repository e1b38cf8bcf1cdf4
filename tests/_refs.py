"""Plain float64 references for the GEMM / convolution kernels, the per-element error bound the tolerance-based tests
use, and the inputs of the exact-arithmetic tests.

Every function here is ordinary torch arithmetic: it runs on the CPU or the GPU, in float64, and never calls a kernel
of the project.

Exact arithmetic.  Operands that are small integers (|v| <= 2) and power-of-two scale factors give products and partial
sums that are integers (or dyadic fractions) far below 2^24: as long as max(|A| @ |B|) <= 2048 every partial sum in
every summation order, at any accumulator width of 12 or more significant bits, and every fp16 output are exact.
Kernels can then be compared with torch.equal -- a dropped, duplicated or misplaced row, tap or split changes some
output by at least 1.

Tolerance bound.  For data that cannot be exact, |got - ref| <= g * (|A| @ |B|) + r * |ref| + tiny per element, with
r = 2^-11 for fp16 outputs (one rounding of the result).  `assert_within` checks that bound and also that the same
bound REJECTS references built with one reduction row (or image) dropped and with one tap's weights zeroed: a
tolerance that would accept those is too loose to say anything about the kernel.
"""
import numpy as np
import torch
import torch.nn.functional as F

EXACT_LIMIT = 2048.0
R_F16 = 2.0 ** -11           # relative rounding of an fp16 output
R_F32 = 2.0 ** -23


# ------------------------------------------------------------------------------------------------ exact operands
def small_ints(shape, density=0.5, gen=None, device="cpu", lo=-2, hi=2):
    """float64 tensor of integers in [lo, hi] \\ {0}, nonzero with probability `density` (zero elsewhere)."""
    vals = torch.randint(lo, hi, shape, generator=gen, dtype=torch.int64)
    vals = vals + (vals >= 0).to(torch.int64) if lo < 0 <= hi else vals        # skip 0: {-2,-1,1,2}
    keep = torch.rand(shape, generator=gen) < density
    return (vals * keep).to(torch.float64).to(device)


def probe_rows(M, tile=128, kblock=None, ends=(), shifts=(), n_random=16, seed=0, valid=None):
    """Rows where a row-wise reduction goes wrong first: the first and last row of every `tile`-row tile, the last row
    of every `kblock`-row block, the row before each end in `ends` (e.g. each CTA's k-range), the rows a tap shifted by
    s reads past a tile's end (row m with m + s the first row of the next tile), the last row, and a few random rows.
    valid: optional bool tensor [M]; rows where it is False are dropped.  Returns a sorted int64 tensor."""
    rows = {0, M - 1}
    for t0 in range(0, M, tile):
        rows.update((t0, min(t0 + tile, M) - 1))
        for s in shifts:
            rows.update((t0 + tile - s, t0 + tile - 1 - s))
    if kblock:
        for k0 in range(0, M, kblock):
            rows.add(min(k0 + kblock, M) - 1)
    rows.update(e - 1 for e in ends)
    rng = np.random.RandomState(seed)
    rows.update(int(v) for v in rng.randint(0, M, n_random))
    out = torch.tensor(sorted(r for r in rows if 0 <= r < M), dtype=torch.int64)
    if valid is not None:
        out = out[valid.cpu()[out]]
    return out


def rows_only(X, rows):
    """X with every row outside `rows` zeroed (rows: int64 tensor)."""
    Z = torch.zeros_like(X)
    r = rows.to(X.device)
    Z[r] = X[r]
    return Z


def assert_exact_ok(absprod, extra=0.0, what=""):
    """The precondition of an exact comparison: every output's |A| @ |B| (+ |extra| terms) is <= 2048."""
    m = float(absprod.max()) + float(extra)
    assert m <= EXACT_LIMIT, f"{what}: max |A|@|B| = {m} > {EXACT_LIMIT}: the exact comparison would not be exact"
    return m


# ------------------------------------------------------------------------------------------------ float64 references
def gemm(A, B):
    """A [M, K] @ B[N, K]^T in float64."""
    return A.double() @ B.double().t()


def patches(x, R, S, sh, sw, ph, pw, OH, OW):
    """x [B, H, W, C] -> [B*OH*OW, R*S*C] with K ordered (r, s, c); zero padding (ph, pw) on the low side and whatever
    is needed on the high side.  Keeps x's dtype."""
    B, H, W, C = x.shape
    hi_h = max((OH - 1) * sh + R - ph - H, 0)
    hi_w = max((OW - 1) * sw + S - pw - W, 0)
    xp = F.pad(x.permute(0, 3, 1, 2), (pw, hi_w, ph, hi_h))
    un = F.unfold(xp, (R, S), stride=(sh, sw))                        # [B, C*R*S, L]
    oh_full = (xp.shape[2] - R) // sh + 1
    ow_full = (xp.shape[3] - S) // sw + 1
    un = un.view(B, C, R, S, oh_full, ow_full)[:, :, :, :, :OH, :OW]
    return un.permute(0, 4, 5, 2, 3, 1).reshape(B * OH * OW, R * S * C)


def conv2d(x, w_hwio, stride, pad, OH, OW):
    """NHWC x [B,H,W,C] (*) HWIO w [R,S,C,N], low-side padding pad = (ph, pw) -> [B, OH, OW, N] float64."""
    R, S, C, N = w_hwio.shape
    P = patches(x.double(), R, S, stride[0], stride[1], pad[0], pad[1], OH, OW)
    return (P @ w_hwio.double().reshape(R * S * C, N)).view(x.shape[0], OH, OW, N)


def conv2d_wgrad(x, dz, R, S, stride, pad):
    """d/dW of sum(conv2d(x, W) * dz): [R*S*C, N] float64 (rows (r, s, c)); dz [B, OH, OW, N]."""
    B, OH, OW, N = dz.shape
    P = patches(x.double(), R, S, stride[0], stride[1], pad[0], pad[1], OH, OW)
    return P.t() @ dz.double().reshape(-1, N)


def conv2d_dgrad(dz, w_hwio, H, W, stride, pad):
    """d/dx of sum(conv2d(x, W) * dz) for x [B, H, W, C]: the transposed convolution, float64 [B, H, W, C]."""
    R, S, C, N = w_hwio.shape
    B, OH, OW, _ = dz.shape
    cols = dz.double().reshape(-1, N) @ w_hwio.double().reshape(R * S * C, N).t()      # [B*OH*OW, (r, s, c)]
    cols = cols.view(B, OH * OW, R, S, C).permute(0, 4, 2, 3, 1).reshape(B, C * R * S, OH * OW)
    Hp = max((OH - 1) * stride[0] + R, H + pad[0])
    Wp = max((OW - 1) * stride[1] + S, W + pad[1])
    full = F.fold(cols, (Hp, Wp), (R, S), stride=stride)                                # [B, C, Hp, Wp]
    return full[:, :, pad[0]:pad[0] + H, pad[1]:pad[1] + W].permute(0, 2, 3, 1)


def shift_conv(X, shifts, Wt, M=None):
    """Shift-GEMM form of a stride-1 convolution over a flattened grid: out[m] = sum_t X[m + shifts[t]] @ Wt_t^T with
    X [rows, C], Wt [N, taps*C] (K order (tap, c)) and rows outside [0, rows) reading zeros.  At grid positions whose
    filter window lies inside the image this is the convolution; the others are wrapped rows a kernel discards."""
    X = X.double()
    rows, C = X.shape
    M = rows if M is None else M
    out = torch.zeros(M, Wt.shape[0], dtype=torch.float64, device=X.device)
    for t, s in enumerate(shifts):
        lo, hi = max(0, -s), min(M, rows - s)
        if hi > lo:
            out[lo:hi] += X[lo + s:hi + s] @ Wt[:, t * C:(t + 1) * C].double().t()
    return out


def shift_wgrad(X, dY, shifts):
    """G [taps*C, N] = sum_m X[m + shifts[t]]^T dY[m] (rows outside X read zeros), float64."""
    X, dY = X.double(), dY.double()
    rows, C = X.shape
    G = torch.zeros(len(shifts) * C, dY.shape[1], dtype=torch.float64, device=X.device)
    for t, s in enumerate(shifts):
        lo, hi = max(0, -s), min(dY.shape[0], rows - s)
        if hi > lo:
            G[t * C:(t + 1) * C] = X[lo + s:hi + s].t() @ dY[lo:hi]
    return G


def space_to_depth(x, s):
    """[B, H, W, C] -> [B, H/s, W/s, s*s*C] with channel order (dy, dx, c)."""
    B, H, W, C = x.shape
    return x.view(B, H // s, s, W // s, s, C).permute(0, 1, 3, 2, 4, 5).reshape(B, H // s, W // s, s * s * C)


def depth_to_space(x, s):
    """Inverse of space_to_depth: [B, h, w, s*s*C] with channels (dy, dx, c) -> [B, s*h, s*w, C]."""
    B, h, w, Cs = x.shape
    C = Cs // (s * s)
    return x.view(B, h, w, s, s, C).permute(0, 1, 3, 2, 4, 5).reshape(B, h * s, w * s, C)


def relu_bits(x):
    """1 bit per element (x > 0), bit k of int16 word e/16 <-> element e + k (two's complement wrap of bit 15)."""
    w = (x.reshape(-1, 16) > 0).to(torch.int32) << torch.arange(16, device=x.device, dtype=torch.int32)
    return w.sum(1).to(torch.int16)


# ------------------------------------------------------------------------------------------------ tolerance bound
def excess(got, ref, scale, r):
    """Observed g: max over elements of (|got - ref| - r |ref|) / scale (elements with scale == 0 excluded)."""
    got, ref, scale = got.double(), ref.double(), scale.double()
    e = ((got - ref).abs() - r * ref.abs()).clamp_min(0.0)
    nz = scale > 0
    return float((e[nz] / scale[nz]).max()) if bool(nz.any()) else 0.0


def within(got, ref, scale, g, r, tiny=1e-30):
    """Per element: |got - ref| <= g * scale + r * |ref| + tiny."""
    got, ref, scale = got.double(), ref.double(), scale.double()
    return bool(((got - ref).abs() <= g * scale + r * ref.abs() + tiny).all())


def assert_within(got, ref, scale, g, r, mutants, what="", tiny=1e-30):
    """Assert the bound for `got` and that it rejects every mutated reference in `mutants` (name -> tensor, built from
    `ref` with one reduction row / image dropped, one tap zeroed, ...).  Returns the observed g."""
    assert bool(torch.isfinite(got.double()).all()), f"{what}: non-finite output"
    seen = excess(got, ref, scale, r)
    assert within(got, ref, scale, g, r, tiny), f"{what}: observed g = {seen:.3e} > allowed {g:.3e}"
    assert mutants, f"{what}: a tolerance comparison needs its self-check mutants"
    for name, mref in mutants.items():
        # the kernel's output would have to be this mutant: is it inside the same bound around the true reference?
        assert not within(mref, ref, scale, g, r, tiny), \
            f"{what}: the bound g = {g:.1e}, r = {r:.1e} also accepts the reference with {name}: it cannot see that bug"
    return seen
