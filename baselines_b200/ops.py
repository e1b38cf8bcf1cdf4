"""Torch-tensor front end of the C-ABI: tensors only supply device pointers and the current stream.

Every function launches hand-written sm_90a kernels from libb200rl.so; nothing here computes with
torch ops (torch is plumbing: allocation, streams, torch.distributed).
"""
from collections import namedtuple

import torch

from . import _lib

MODE_F16_ACT, MODE_F32_STORE, MODE_F32_ATOMIC, MODE_F16_DACT, MODE_F16_SHUFFLE = 0, 1, 2, 3, 4
ACT_NONE, ACT_RELU, ACT_TANH = 0, 1, 2
ACT_CODES = {None: ACT_NONE, "none": ACT_NONE, "relu": ACT_RELU, "tanh": ACT_TANH}


def _ptr(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


_SMS = {}


def num_sms():
    """Streaming multiprocessors of the current device (132 on an H100 SXM); split-K factors aim at two CTAs per SM."""
    d = torch.cuda.current_device()
    if d not in _SMS:
        _SMS[d] = torch.cuda.get_device_properties(d).multi_processor_count
    return _SMS[d]


def _chk(t, dtype, name):
    if t is None:
        return
    if not t.is_cuda:
        raise RuntimeError(f"{name}: expected a CUDA tensor (the hot path has no CPU fallback)")
    if t.dtype != dtype:
        raise RuntimeError(f"{name}: expected {dtype}, got {t.dtype}")


def gae_scan(rewards, values, dones, last_values, last_dones, advs, returns, gamma, lam, variant=-1):
    """rewards/values/advs/returns float32 [T,N]; dones uint8 [T,N]; last_* [N]."""
    T, N = rewards.shape
    for t, dt, nm in ((rewards, torch.float32, "rewards"), (values, torch.float32, "values"),
                      (dones, torch.uint8, "dones"), (last_values, torch.float32, "last_values"),
                      (last_dones, torch.uint8, "last_dones"), (advs, torch.float32, "advs"),
                      (returns, torch.float32, "returns")):
        _chk(t, dt, nm)
        assert t.is_contiguous(), nm
    _lib.call("b200rl_gae_scan", _ptr(rewards), _ptr(values), _ptr(dones), _ptr(last_values), _ptr(last_dones),
              _ptr(advs), _ptr(returns), T, N, float(gamma), float(lam), int(variant), _stream(),
              label="gae_scan", nbytes=17.0 * T * N + 5.0 * N)


def gemm(A, B, C, *, M, N, K, lda, ldb, ldc, bias=None, saved=None, ld_saved=0, mn_major=False,
         mode=MODE_F16_ACT, act=ACT_NONE, alpha=1.0, split_k=1, max_ctas=0, tag=None, remap=(0, 0, 0), saved_bits=None):
    _chk(A, torch.float16, "A")
    _chk(B, torch.float16, "B")
    _chk(bias, torch.float32, "bias")
    _chk(saved, torch.float16, "saved")
    _chk(saved_bits, torch.int16, "saved_bits")
    _lib.call("b200rl_gemm_f16", _ptr(A), _ptr(B), _ptr(C), _ptr(bias), _ptr(saved), int(M), int(N), int(K),
              int(lda), int(ldb), int(ldc), int(ld_saved), int(bool(mn_major)), int(mode), int(act), float(alpha),
              int(split_k), int(max_ctas), int(remap[0]), int(remap[1]), int(remap[2]), _ptr(saved_bits), _stream(),
              label="gemm." + (tag or ("wgrad" if mn_major else "tn")),
              flops=2.0 * M * N * K,
              nbytes=2.0 * (M * K + N * K) + M * N * (2 if mode in (MODE_F16_ACT, MODE_F16_DACT) else 4)
              + ((0.125 if saved_bits is not None else 2.0) * M * N if mode == MODE_F16_DACT else 0))


def conv_gemm(x, B, H, W, C, R, S, stride_h, stride_w, pad_h, pad_w, OH, OW, wt_or_dz, ldb, out, ldc, N, kind,
              mode, act=ACT_NONE, alpha=1.0, bias=None, saved=None, ld_saved=0, split_k=1, shuffle=None, tag=None):
    """Implicit-GEMM convolution (TMA im2col A operand).  kind 0: forward / data-gradient form; kind 1: wgrad."""
    _chk(x, torch.float16, "x")
    _chk(wt_or_dz, torch.float16, "wt_or_dz")
    sh = shuffle or (0, 0, 0, 0)
    rows = B * OH * OW
    _lib.call("b200rl_conv_gemm", _ptr(x), int(B), H, W, C, R, S, stride_h, stride_w, pad_h, pad_w, OH, OW,
              _ptr(wt_or_dz), int(ldb), _ptr(out), int(ldc), _ptr(bias), _ptr(saved), int(ld_saved), int(N), int(kind),
              int(mode), int(act), float(alpha), int(split_k), int(sh[0]), int(sh[1]), int(sh[2]), int(sh[3]),
              _stream(), label="conv." + (tag or str(kind)), flops=2.0 * rows * N * R * S * C,
              nbytes=2.0 * B * H * W * C + 2.0 * R * S * C * N + rows * N * (2.0 if kind == 0 else 2.0))


import ctypes as _C


def _iarr(vals, ctype):
    return (ctype * len(vals))(*[int(v) for v in vals])


def _u8_args(u8):
    """u8 = (images uint8 [.., H, W, C], src_idx or None, H, W, C, s) or None."""
    if u8 is None:
        return None, None, 0, 0, 0, 0
    x, idx, H, W, C, s = u8
    _chk(x, torch.uint8, "u8 images")
    _chk(idx, torch.int64, "u8 src_idx")
    return _ptr(x), _ptr(idx), int(H), int(W), int(C), int(s)


def conv_shift_fwd(X, B, Hg, Wg, C, W, ldw, N, shifts, vy, vx, out, omap, *, smap=None, bias=None,
                   act=ACT_NONE, dact=False, alpha=1.0, tag=None, u8=None, bits_out=None, saved_bits=None,
                   useful_rows=None):
    """Shift-GEMM convolution (forward, or data gradient with dact=True, masked by the ReLU bits saved_bits of the
    saved activation when given).  omap / smap: 6-tuples (mode, sN, sY, sX, Cq, s).  useful_rows (accounting only): positions that are real conv outputs -- the kernel
    also computes (and discards) the grid positions that are not; reported flops / bytes count the useful ones."""
    _chk(X, torch.float16, "X")
    _chk(W, torch.float16, "W")
    _chk(out, torch.float16, "out")
    u8a = _u8_args(u8)
    _chk(bits_out, torch.int16, "bits_out")
    _chk(saved_bits, torch.int16, "saved_bits")
    sh = _iarr(shifts, _C.c_int)
    om = _iarr(omap, _C.c_longlong)
    sm = _iarr(smap, _C.c_longlong) if smap is not None else None
    rows = B * Hg * Wg
    useful = float(useful_rows) if useful_rows is not None else float(B) * vy * vx
    if dact:      # data gradient: reads the valid dY rows, writes every dX position, reads the activation mask
        nbytes = 2.0 * useful * C + 2.0 * rows * N
        nbytes += 0.0 if saved_bits is None else 0.125 * rows * N
    else:         # forward: reads every input position, writes the valid outputs (+ 1 bit per element of mask)
        nbytes = (1.0 if u8 is not None else 2.0) * rows * C + 2.0 * useful * N + (0.125 * useful * N if bits_out is not None else 0.0)
    _lib.call("b200rl_conv_shift_fwd", _ptr(X), int(B), Hg, Wg, C, _ptr(W), int(ldw), int(N), len(shifts), sh, vy, vx,
              _ptr(out), om, sm, _ptr(bias), int(act), int(bool(dact)), float(alpha), *u8a,
              _ptr(bits_out), _ptr(saved_bits), _stream(),
              label="convs." + (tag or "fwd"), flops=2.0 * useful * N * len(shifts) * C, nbytes=nbytes)


def conv_shift_wgrad(X, rows, C, dY, N, shifts, G, ldg, alpha=1.0, max_ctas=0, tag=None, gbias=None, alpha_b=1.0,
                     u8=None, useful_rows=None, kx=1):
    _chk(X, torch.float16, "X")
    _chk(dY, torch.float16, "dY")
    _chk(G, torch.float32, "G")
    sh = _iarr(shifts, _C.c_int)
    _chk(gbias, torch.float32, "gbias")
    u8a = _u8_args(u8)
    _lib.call("b200rl_conv_shift_wgrad", _ptr(X), int(rows), C, _ptr(dY), int(N), len(shifts), sh, _ptr(G), int(ldg),
              float(alpha), _ptr(gbias), float(alpha_b), int(max_ctas), *u8a, int(kx), _stream(),
              label="convs." + (tag or "wgrad"),
              flops=2.0 * (float(useful_rows) if useful_rows is not None else rows) * N * len(shifts) * kx * C,
              nbytes=rows * (1.0 if u8 is not None else 2.0) * C +
              2.0 * N * (float(useful_rows) if useful_rows is not None else rows))


def dgrad_weights(w, out, R, S, Cin, Cout, s, ld):
    _chk(w, torch.float32, "w")
    _chk(out, torch.float16, "out")
    _lib.call("b200rl_dgrad_weights", _ptr(w), _ptr(out), R, S, Cin, Cout, s, int(ld), _stream())


def _conv_out(H, W, rf, stride, same_pad):
    if same_pad:
        return -(-H // stride), -(-W // stride)
    return (H - rf) // stride + 1, (W - rf) // stride + 1


def im2col(x, cols, B, H, W, C, rf, stride, same_pad=False, src_idx=None, tag=None):
    _chk(src_idx, torch.int64, "src_idx")
    _chk(cols, torch.float16, "cols")
    src_u8 = x.dtype == torch.uint8
    if not src_u8:
        _chk(x, torch.float16, "x")
    OH, OW = _conv_out(H, W, rf, stride, same_pad)
    _lib.call("b200rl_im2col", _ptr(x), int(src_u8), _ptr(src_idx), _ptr(cols), int(B), H, W, C, rf, stride,
              int(bool(same_pad)), _stream(), label="im2col." + (tag or ("u8" if src_u8 else "f16")),
              nbytes=float(B) * H * W * C * (1 if src_u8 else 2) + 2.0 * B * OH * OW * rf * rf * C)


def frame_stack(prev, frame, news, out, nstack, c):
    """out = VecFrameStack update of prev with the new frames (vec_frame_stack.py:17-25); uint8 [N, ..., nstack*c]."""
    for t, nm in ((prev, "prev"), (frame, "frame"), (news, "news"), (out, "out")):
        _chk(t, torch.uint8, nm)
    N = out.shape[0]
    pixels = out[0].numel() // (nstack * c)
    if prev.numel() != out.numel() or frame.numel() != N * pixels * c or news.numel() != N:
        raise RuntimeError("frame_stack: shape mismatch")
    _lib.call("b200rl_frame_stack", _ptr(prev), _ptr(frame), _ptr(news), _ptr(out), int(N), int(pixels), int(nstack),
              int(c), _stream(), label="frame_stack", nbytes=float(2 * out.numel() + frame.numel()))


def s2d_gather(x, out, B, H, W, C, s, src_idx=None):
    _chk(x, torch.uint8, "x")
    _chk(out, torch.float16, "out")
    _chk(src_idx, torch.int64, "src_idx")
    _lib.call("b200rl_s2d_gather", _ptr(x), _ptr(src_idx), _ptr(out), int(B), H, W, C, s, _stream(),
              label="s2d_gather", nbytes=3.0 * B * H * W * C)


def col2im(dcols, saved, dx, B, H, W, C, rf, stride, same_pad=False, act=ACT_NONE, tag=None):
    _chk(dcols, torch.float16, "dcols")
    _chk(dx, torch.float16, "dx")
    OH, OW = _conv_out(H, W, rf, stride, same_pad)
    _lib.call("b200rl_col2im", _ptr(dcols), _ptr(saved), _ptr(dx), int(B), H, W, C, rf, stride, int(bool(same_pad)),
              int(act), _stream(), label="col2im." + (tag or ""),
              nbytes=2.0 * B * OH * OW * rf * rf * C + 2.0 * B * H * W * C * (2 if saved is not None else 1))


def colsum(dz, db, rows, C, ld, alpha=1.0):
    _chk(dz, torch.float16, "dz")
    _chk(db, torch.float32, "db")
    _lib.call("b200rl_colsum", _ptr(dz), _ptr(db), int(rows), int(C), int(ld), float(alpha), _stream(),
              label="colsum", nbytes=2.0 * rows * C)


def segment_table(nvec, device):
    """int32 device tensor [len(nvec) + 1] of the offsets of MultiDiscrete components in a row: 0, n0, n0 + n1, ...
    (the seg_off argument of cat_step / cat_loss / obs_encode).  Every component needs at least one value
    (distributions.py:79 asserts the same)."""
    import numpy as np
    nv = np.asarray(nvec, dtype=np.int64).reshape(-1)
    if nv.size == 0 or np.any(nv < 1):
        raise ValueError(f"MultiDiscrete nvec entries must be >= 1, got {list(nv)}")
    off = np.concatenate([[0], np.cumsum(nv)]).astype(np.int32)
    return torch.from_numpy(off).to(device)


def _seg_args(seg_off):
    if seg_off is None:
        return None, 0
    _chk(seg_off, torch.int32, "seg_off")
    return _ptr(seg_off), seg_off.numel() - 1


def cat_step(logits, ld, nA, vpred, ldv, actions, values, neglogp, B, uniforms=None, seed=0, offset=0,
             offset_dev=None, seg_off=None):
    """Categorical sample + neglogp; with seg_off (segment_table(nvec), nA = sum(nvec)) one categorical per
    MultiDiscrete component: actions int64 [B, len(nvec)], neglogp their sum."""
    _chk(logits, torch.float32, "logits")
    _chk(actions, torch.int64, "actions")
    _chk(uniforms, torch.float32, "uniforms")
    _chk(offset_dev, torch.int64, "offset_dev")
    so, nseg = _seg_args(seg_off)
    _lib.call("b200rl_cat_step", _ptr(logits), int(ld), int(nA), so, nseg, _ptr(vpred), int(ldv), _ptr(uniforms),
              int(seed), int(offset), _ptr(offset_dev), _ptr(actions), _ptr(values), _ptr(neglogp), int(B), _stream(),
              **({} if so is None else dict(label="mcat_step", nbytes=float(B) * (4.0 * nA + 8.0 * nseg + 12.0))))


def bern_step(logits, ld, n, vpred, ldv, actions, values, neglogp, B, uniforms=None, seed=0, offset=0,
              offset_dev=None):
    """Bernoulli (MultiBinary) sample + neglogp: actions float32 [B, n] of 0 / 1."""
    _chk(logits, torch.float32, "logits")
    _chk(actions, torch.float32, "actions")
    _chk(uniforms, torch.float32, "uniforms")
    _chk(offset_dev, torch.int64, "offset_dev")
    _lib.call("b200rl_bern_step", _ptr(logits), int(ld), int(n), _ptr(vpred), int(ldv), _ptr(uniforms), int(seed),
              int(offset), _ptr(offset_dev), _ptr(actions), _ptr(values), _ptr(neglogp), int(B), _stream(),
              label="bern_step", nbytes=float(B) * (8.0 * n + 12.0))


def gauss_step(mean, ld, logstd, d, vpred, ldv, actions, values, neglogp, B, normals=None, seed=0, offset=0,
               offset_dev=None):
    _chk(mean, torch.float32, "mean")
    _chk(actions, torch.float32, "actions")
    _chk(normals, torch.float32, "normals")
    _chk(offset_dev, torch.int64, "offset_dev")
    _lib.call("b200rl_gauss_step", _ptr(mean), int(ld), _ptr(logstd), int(d), _ptr(vpred), int(ldv), _ptr(normals),
              int(seed), int(offset), _ptr(offset_dev), _ptr(actions), _ptr(values), _ptr(neglogp), int(B), _stream())


def set_scalars(dst, *vals):
    """dst[0..len(vals)) = vals (float32 device tensor): values travel as kernel arguments."""
    _chk(dst, torch.float32, "dst")
    v = [float(x) for x in vals] + [0.0] * (4 - len(vals))
    _lib.call("b200rl_set_scalars", _ptr(dst), len(vals), v[0], v[1], v[2], v[3], _stream())


def shuffle_indices(out, n, key, T=0, N=0):
    """out[:n] = buffer offsets of a keyed pseudo-random permutation of the n rollout samples (ppo2.py:160)."""
    _chk(out, torch.int64, "out")
    _lib.call("b200rl_shuffle_indices", _ptr(out), int(n), int(key) & 0xFFFFFFFFFFFFFFFF, int(T), int(N), _stream(),
              label="shuffle_indices", nbytes=8.0 * n)


def counter_add(ctr, inc=1):
    _chk(ctr, torch.int64, "ctr")
    _lib.call("b200rl_counter_add", _ptr(ctr), int(inc), _stream())


def adv_stats(returns, values, src_idx, M, out):
    _chk(out, torch.float64, "out")
    _chk(src_idx, torch.int64, "src_idx")
    _lib.call("b200rl_adv_stats", _ptr(returns), _ptr(values), _ptr(src_idx), int(M), _ptr(out), _stream())


def cat_loss(logits, ld, nA, vpred, ldv, actions, src_idx, returns, old_values, old_neglogp, adv_st, cliprange,
             ent_coef, vf_coef, dlogits, ld_dl, dv, ld_dv, stats, B, cliprange_dev=None, seg_off=None):
    """Categorical PPO loss + logit gradient; with seg_off (segment_table(nvec)) the MultiCategorical one, actions
    int64 [*, len(nvec)]."""
    _chk(actions, torch.int64, "actions")
    _chk(stats, torch.float64, "stats")
    so, nseg = _seg_args(seg_off)
    _lib.call("b200rl_cat_loss", _ptr(logits), int(ld), int(nA), so, nseg, _ptr(vpred), int(ldv), _ptr(actions),
              _ptr(src_idx), _ptr(returns), _ptr(old_values), _ptr(old_neglogp), _ptr(adv_st), float(cliprange),
              float(ent_coef), float(vf_coef), _ptr(dlogits), int(ld_dl), _ptr(dv), int(ld_dv), _ptr(stats), int(B),
              _ptr(cliprange_dev), _stream(),
              **({} if so is None else dict(label="mcat_loss", nbytes=float(B) * (6.0 * nA + 8.0 * nseg + 28.0))))


def bern_loss(logits, ld, n, vpred, ldv, actions, src_idx, returns, old_values, old_neglogp, adv_st, cliprange,
              ent_coef, vf_coef, dlogits, ld_dl, dv, ld_dv, stats, B, cliprange_dev=None):
    """Bernoulli (MultiBinary) PPO loss + logit gradient; actions float32 [*, n]."""
    _chk(actions, torch.float32, "actions")
    _chk(stats, torch.float64, "stats")
    _lib.call("b200rl_bern_loss", _ptr(logits), int(ld), int(n), _ptr(vpred), int(ldv), _ptr(actions), _ptr(src_idx),
              _ptr(returns), _ptr(old_values), _ptr(old_neglogp), _ptr(adv_st), float(cliprange), float(ent_coef),
              float(vf_coef), _ptr(dlogits), int(ld_dl), _ptr(dv), int(ld_dv), _ptr(stats), int(B), _ptr(cliprange_dev),
              _stream(), label="bern_loss", nbytes=float(B) * (10.0 * n + 28.0))


def gauss_loss(mean, ld, logstd, d, vpred, ldv, actions, src_idx, returns, old_values, old_neglogp, adv_st,
               cliprange, ent_coef, vf_coef, dmean, ld_dm, dv, ld_dv, dlogstd, inv_M, stats, B, cliprange_dev=None):
    _chk(actions, torch.float32, "actions")
    _lib.call("b200rl_gauss_loss", _ptr(mean), int(ld), _ptr(logstd), int(d), _ptr(vpred), int(ldv), _ptr(actions),
              _ptr(src_idx), _ptr(returns), _ptr(old_values), _ptr(old_neglogp), _ptr(adv_st), float(cliprange),
              float(ent_coef), float(vf_coef), _ptr(dmean), int(ld_dm), _ptr(dv), int(ld_dv), _ptr(dlogstd),
              float(inv_M), _ptr(stats), int(B), _ptr(cliprange_dev), _stream())


def sumsq(g, out):
    _chk(g, torch.float32, "g")
    _chk(out, torch.float64, "out")
    _lib.call("b200rl_sumsq", _ptr(g), g.numel(), _ptr(out), _stream(), label="sumsq", nbytes=4.0 * g.numel())


def seg_sumsq(g, seg_off, nseg, out):
    _chk(seg_off, torch.int64, "seg_off")
    _lib.call("b200rl_seg_sumsq", _ptr(g), _ptr(seg_off), int(nseg), _ptr(out), _stream())


def clip_adam(p, g, m, v, lr_t, beta1, beta2, eps, clip, sumsq_buf, seg_off=None, nseg=0, lr_t_dev=None):
    for t, nm in ((p, "p"), (g, "g"), (m, "m"), (v, "v")):
        _chk(t, torch.float32, nm)
    _lib.call("b200rl_clip_adam", _ptr(p), _ptr(g), _ptr(m), _ptr(v), p.numel(), float(lr_t), float(beta1),
              float(beta2), float(eps), float(clip if clip else 0.0), _ptr(sumsq_buf), _ptr(seg_off), int(nseg),
              _ptr(lr_t_dev), _stream(), label="clip_adam", nbytes=28.0 * p.numel())


def clip_accumulate(g, acc, clip, weight, sumsq_buf):
    _chk(g, torch.float32, "g")
    _chk(acc, torch.float32, "acc")
    _lib.call("b200rl_clip_accumulate", _ptr(g), _ptr(acc), g.numel(), float(clip if clip else 0.0), float(weight),
              _ptr(sumsq_buf), _stream(), label="clip_accumulate", nbytes=12.0 * g.numel())


def soft_update(t0, s0, keep, mix, t1=None, s1=None):
    """Soft target update t <- float32(keep) * t + float32(mix) * s of (t0, s0) and, when given, (t1, s1), one launch."""
    for t, nm in ((t0, "t0"), (s0, "s0"), (t1, "t1"), (s1, "s1")):
        _chk(t, torch.float32, nm)
    if s0.numel() != t0.numel() or (t1 is not None and s1.numel() != t1.numel()):
        raise RuntimeError("soft_update: source and target sizes differ")
    _lib.call("b200rl_soft_update", _ptr(t0), _ptr(s0), t0.numel(), _ptr(t1), _ptr(s1),
              0 if t1 is None else t1.numel(), float(keep), float(mix), _stream(), label="soft_update",
              nbytes=12.0 * (t0.numel() + (0 if t1 is None else t1.numel())))


CastJob = namedtuple("CastJob", "src R C dst ld_dst dstT ld_t scale")
CastJob.__doc__ = """One fp32 -> fp16 operand cast (struct CastJob of csrc/optim.cu): dst[r, c] = fp16(src[r, c] * scale)
(row pitch ld_dst) and dstT[c, r] likewise (row pitch ld_t) for the contiguous float32 [R, C] src; dst or dstT may be
None.  The fields are cast_transpose's arguments, in its order."""


def cast_transpose(src, R, C, dst, ld_dst, dstT, ld_t, scale=1.0):
    _chk(src, torch.float32, "src")
    _lib.call("b200rl_cast_transpose", _ptr(src), int(R), int(C), _ptr(dst), int(ld_dst), _ptr(dstT), int(ld_t),
              float(scale), _stream())


class CastPlan:
    """A list of CastJobs (the fp16 operand casts of a whole network) as ONE launch: a device table of the jobs, built
    once.  Building it copies to the device, so it cannot happen inside a graph capture; running it can."""

    def __init__(self, jobs, device):
        import numpy as np
        jobs = list(jobs)
        self.n = len(jobs)
        self.keep = jobs                                   # keeps the tensors (and their storage) alive
        rec = np.zeros(max(self.n, 1), dtype=np.dtype([("src", "<u8"), ("dst", "<u8"), ("dstT", "<u8"), ("ld_dst", "<i8"),
                                                        ("ld_t", "<i8"), ("R", "<i4"), ("C", "<i4"), ("scale", "<f4"),
                                                        ("pad", "<i4")]))
        assert rec.dtype.itemsize == 56
        for i, (src, Rr, Cc, dst, ld_dst, dstT, ld_t, scale) in enumerate(jobs):
            _chk(src, torch.float32, "src")
            rec[i] = (src.data_ptr(), 0 if dst is None else dst.data_ptr(), 0 if dstT is None else dstT.data_ptr(),
                      ld_dst, ld_t, Rr, Cc, scale, 0)
        self.table = torch.from_numpy(rec.view(np.uint8).copy()).to(device)
        self.max_r = max([j.R for j in jobs], default=1)
        self.max_c = max([j.C for j in jobs], default=1)

    def run(self):
        if self.n:
            _lib.call("b200rl_cast_transpose_batch", _ptr(self.table), self.n, self.max_r, self.max_c, _stream(),
                      label="cast_transpose_batch")


def cast_f32_f16(src, dst, rows, cols, ld_src, ld_dst, scale=1.0):
    _chk(src, torch.float32, "src")
    _chk(dst, torch.float16, "dst")
    _lib.call("b200rl_cast_f32_f16", _ptr(src), _ptr(dst), int(rows), int(cols), int(ld_src), int(ld_dst),
              float(scale), _stream())


def obs_encode(x, out, B, raw_dim, in_dim, in_pad, src_idx=None, mean=None, inv_std=None, clip=(-5.0, 5.0), onehot_n=0,
               seg_off=None, overflow=None):
    """float32 observation rows -> fp16 [hi | lo] operand rows (input.py:43-63, policies.py:182-185, ppo2.py:165).
    onehot_n with seg_off (segment_table(nvec)): MultiDiscrete rows of len(nvec) integers -> concatenated one-hot.
    overflow: optional int32 device scalar, set to 1 when an encoded value has |v| >= 65520 (beyond fp16)."""
    _chk(x, torch.float32, "x")
    _chk(out, torch.float16, "out")
    _chk(src_idx, torch.int64, "src_idx")
    _chk(mean, torch.float32, "mean")
    _chk(inv_std, torch.float32, "inv_std")
    _chk(overflow, torch.int32, "overflow")
    so, nseg = _seg_args(seg_off)
    _lib.call("b200rl_obs_encode", _ptr(x), _ptr(src_idx), int(B), int(raw_dim), int(in_dim), int(in_pad), _ptr(mean),
              _ptr(inv_std), float(clip[0]), float(clip[1]), int(onehot_n), so, nseg, _ptr(out), _ptr(overflow),
              _stream(),
              label="obs_encode", nbytes=float(B) * (4.0 * raw_dim + 4.0 * in_pad))


def tree_set(sum_tree, min_tree, capacity, idx, vals):
    _chk(sum_tree, torch.float64, "sum_tree")
    _chk(idx, torch.int64, "idx")
    _chk(vals, torch.float64, "vals")
    _lib.call("b200rl_tree_set", _ptr(sum_tree), _ptr(min_tree), int(capacity), _ptr(idx), _ptr(vals), idx.numel(),
              _stream())


def tree_range_sum(tree, capacity, start, end, out):
    _lib.call("b200rl_tree_range_sum", _ptr(tree), int(capacity), int(start), int(end), _ptr(out), _stream())


def per_sample(sum_tree, min_tree, capacity, n_stored, uniforms, beta, idx_out, w_out, w_out_f32=None, bad=None):
    """bad: optional int32 device scalar, set to 1 when the tree holds a priority that is not > 0 (the slot that would
    leave the stored range returns index 0)."""
    _chk(uniforms, torch.float64, "uniforms")
    _chk(idx_out, torch.int64, "idx_out")
    _chk(w_out, torch.float64, "w_out")
    _chk(bad, torch.int32, "bad")
    _lib.call("b200rl_per_sample", _ptr(sum_tree), _ptr(min_tree), int(capacity), int(n_stored), _ptr(uniforms),
              uniforms.numel(), float(beta), _ptr(idx_out), _ptr(w_out), _ptr(w_out_f32), _ptr(bad), _stream())


def per_priorities(td, eps, alpha, powered, max_priority, bad):
    """p = float32(|td| + float32(eps)); powered = p ** alpha (float64); max_priority = max(max_priority, p).
    bad: int32 device scalar, set to 1 when some p is not > 0 (NaN or zero)."""
    _chk(td, torch.float32, "td")
    _chk(powered, torch.float64, "powered")
    _chk(max_priority, torch.float64, "max_priority")
    _chk(bad, torch.int32, "bad")
    _lib.call("b200rl_per_priorities", _ptr(td), td.numel(), float(eps), float(alpha), _ptr(powered),
              _ptr(max_priority), _ptr(bad), _stream())


def per_pow(x, y, out):
    """out = x ** y (float64), correctly rounded: the pow of the replay leaves and weights."""
    _chk(x, torch.float64, "x")
    _chk(out, torch.float64, "out")
    _lib.call("b200rl_per_pow", _ptr(x), x.numel(), float(y), _ptr(out), _stream())


def dqn_td(a_t, lda_t, s_t, lds_t, a_on, lda_on, s_on, lds_on, a_tg, lda_tg, s_tg, lds_tg, nA, idx, actions,
           rewards, dones, weights, gamma, double_q, td_out, d_a, ld_da, d_s, ld_ds, loss_sum, B):
    _lib.call("b200rl_dqn_td", _ptr(a_t), int(lda_t), _ptr(s_t), int(lds_t), _ptr(a_on), int(lda_on), _ptr(s_on),
              int(lds_on), _ptr(a_tg), int(lda_tg), _ptr(s_tg), int(lds_tg), int(nA), _ptr(idx), _ptr(actions),
              _ptr(rewards), _ptr(dones), _ptr(weights), float(gamma), int(bool(double_q)), _ptr(td_out), _ptr(d_a),
              int(ld_da), _ptr(d_s), int(ld_ds), _ptr(loss_sum), int(B), _stream())


def dqn_act(a, lda, s, lds, nA, eps, seed, step, actions, B, eps_dev=None, step_dev=None):
    _chk(eps_dev, torch.float32, "eps_dev")
    _chk(step_dev, torch.int64, "step_dev")
    _lib.call("b200rl_dqn_act", _ptr(a), int(lda), _ptr(s), int(lds), int(nA), float(eps), int(seed), int(step),
              _ptr(eps_dev), _ptr(step_dev), _ptr(actions), int(B), _stream())


def lstm_seq_fwd(xg, ldxg, wh, masks, state_in, h_out, ldh, T, B, H, *, mask_idx=None, state_idx=None, state_out=None,
                 hprev_out=None, gates_out=None, c_out=None):
    """LSTM recurrence (a2c/utils.py:84-97) over T time-major steps of B environments: xg float32 [T*B, ldxg] (x.Wx + b),
    wh fp16 [H, 4H], masks uint8 (done before the step; gathered through mask_idx), state_in float32 [*, 2H] = [c | h]
    (gathered through state_idx).  See include/b200rl.h for the optional outputs."""
    for t, dt, nm in ((xg, torch.float32, "xg"), (wh, torch.float16, "wh"), (masks, torch.uint8, "masks"),
                      (mask_idx, torch.int64, "mask_idx"), (state_in, torch.float32, "state_in"),
                      (state_idx, torch.int64, "state_idx"), (state_out, torch.float32, "state_out"),
                      (h_out, torch.float16, "h_out"), (hprev_out, torch.float16, "hprev_out"),
                      (gates_out, torch.float32, "gates_out"), (c_out, torch.float32, "c_out")):
        _chk(t, dt, nm)
    rows = T * B
    _lib.call("b200rl_lstm_seq_fwd", _ptr(xg), int(ldxg), _ptr(wh), _ptr(masks), _ptr(mask_idx), _ptr(state_in),
              _ptr(state_idx), _ptr(state_out), _ptr(h_out), int(ldh), _ptr(hprev_out), _ptr(gates_out), _ptr(c_out),
              int(T), int(B), int(H), _stream(), label="lstm_seq_fwd",
              flops=8.0 * rows * H * H,
              nbytes=16.0 * rows * H + 8.0 * H * H * -(-B // 8) + 2.0 * rows * H
              + (2.0 * rows * H + 16.0 * rows * H + 4.0 * rows * H if gates_out is not None else 0))


def lstm_seq_bwd(dh, lddh, gates, c, masks, state_in, whT, dz, lddz, T, B, H, *, mask_idx=None, state_idx=None):
    """Backward of lstm_seq_fwd: dz fp16 [T*B, lddz] = d loss / d (pre-activation gates) from dh fp16 [T*B, lddh]
    (d loss / d h_t) and the forward's gates / c, walking t downwards with the dh carry through whT fp16 [4H, H]."""
    for t, dt, nm in ((dh, torch.float16, "dh"), (gates, torch.float32, "gates"), (c, torch.float32, "c"),
                      (masks, torch.uint8, "masks"), (mask_idx, torch.int64, "mask_idx"),
                      (state_in, torch.float32, "state_in"), (state_idx, torch.int64, "state_idx"),
                      (whT, torch.float16, "whT"), (dz, torch.float16, "dz")):
        _chk(t, dt, nm)
    rows = T * B
    _lib.call("b200rl_lstm_seq_bwd", _ptr(dh), int(lddh), _ptr(gates), _ptr(c), _ptr(masks), _ptr(mask_idx),
              _ptr(state_in), _ptr(state_idx), _ptr(whT), _ptr(dz), int(lddz), int(T), int(B), int(H), _stream(),
              label="lstm_seq_bwd", flops=8.0 * rows * H * H,
              nbytes=2.0 * rows * H + 16.0 * rows * H + 8.0 * rows * H + 8.0 * rows * H + 8.0 * H * H * -(-B // 8))


def ln_fwd(z, ld_z, gamma, beta, y, ld_y, rows, N, act, eps):
    """y fp16 = act(gamma * (z - mean) / sqrt(var + eps) + beta) per row of z float32 [rows, ld_z] (biased variance)."""
    for t, dt, nm in ((z, torch.float32, "z"), (gamma, torch.float32, "gamma"), (beta, torch.float32, "beta"),
                      (y, torch.float16, "y")):
        _chk(t, dt, nm)
    _lib.call("b200rl_ln_fwd", _ptr(z), int(ld_z), _ptr(gamma), _ptr(beta), _ptr(y), int(ld_y), int(rows), int(N),
              int(act), float(eps), _stream(), label="ln_fwd", nbytes=6.0 * rows * N)


def ln_bwd(du, ld_du, z, ld_z, gamma, dz, ld_dz, dgamma, dbeta, rows, N, alpha, eps):
    """Backward of ln_fwd from du fp16 = d loss / d (gamma * xhat + beta): dz fp16 (may be du), dgamma += alpha *
    sum_r du * xhat, dbeta += alpha * sum_r du (deterministic)."""
    for t, dt, nm in ((du, torch.float16, "du"), (z, torch.float32, "z"), (gamma, torch.float32, "gamma"),
                      (dz, torch.float16, "dz"), (dgamma, torch.float32, "dgamma"), (dbeta, torch.float32, "dbeta")):
        _chk(t, dt, nm)
    _lib.call("b200rl_ln_bwd", _ptr(du), int(ld_du), _ptr(z), int(ld_z), _ptr(gamma), _ptr(dz), int(ld_dz),
              _ptr(dgamma), _ptr(dbeta), int(rows), int(N), float(alpha), float(eps), _stream(), label="ln_bwd",
              nbytes=8.0 * rows * N)


def param_perturb(src, dst, jobs, njobs, max_len, scale_dev, seed, offset_dev, normals=None):
    """dst <- src (+ scale_dev[0] * N(0, 1) on the jobs marked perturb) per record {src_off, dst_off, len, perturb} of
    the int64 device table `jobs`; the noise is the Philox stream at *offset_dev, or `normals` (indexed like dst)."""
    for t, dt, nm in ((src, torch.float32, "src"), (dst, torch.float32, "dst"), (jobs, torch.int64, "jobs"),
                      (scale_dev, torch.float32, "scale_dev"), (normals, torch.float32, "normals"),
                      (offset_dev, torch.int64, "offset_dev")):
        _chk(t, dt, nm)
    _lib.call("b200rl_param_perturb", _ptr(src), _ptr(dst), _ptr(jobs), int(njobs), int(max_len), _ptr(scale_dev),
              _ptr(normals), int(seed), _ptr(offset_dev), _stream(), label="param_perturb")


def dqn_param_noise_adapt(q, q_adapt, ld, nA, dueling, B, scale_dev, threshold_dev, mean_kl_dev):
    """mean_kl_dev[0] = mean KL(softmax(Q) || softmax(Q_adapt)) over B rows; scale_dev[0] *= or /= 1.01 against the
    threshold (build_graph.py:279-287)."""
    for t, nm in ((q, "q"), (q_adapt, "q_adapt"), (scale_dev, "scale_dev"), (threshold_dev, "threshold_dev"),
                  (mean_kl_dev, "mean_kl_dev")):
        _chk(t, torch.float32, nm)
    _lib.call("b200rl_dqn_param_noise_adapt", _ptr(q), _ptr(q_adapt), int(ld), int(nA), int(bool(dueling)), int(B),
              _ptr(scale_dev), _ptr(threshold_dev), _ptr(mean_kl_dev), _stream(), label="dqn_param_noise_adapt")


_VN_DTYPES = {torch.float32: 0, torch.float64: 1}


def _vn_dtype(t, name):
    if not t.is_cuda:
        raise RuntimeError(f"{name}: expected a CUDA tensor (the hot path has no CPU fallback)")
    if t.dtype not in _VN_DTYPES:
        raise RuntimeError(f"{name}: expected float32 or float64, got {t.dtype}")
    if not t.is_contiguous():
        raise RuntimeError(f"{name}: expected a contiguous tensor")
    return _VN_DTYPES[t.dtype]


def vecnorm_moments(x, ws):
    """ws float64 [2D] = (np.mean(x, 0), np.var(x, 0)) of x [N, ...] float32 / float64, in numpy's summation order."""
    f64 = _vn_dtype(x, "x")
    _chk(ws, torch.float64, "ws")
    N, D = x.shape[0], x[0].numel()
    if ws.numel() < 2 * D:
        raise RuntimeError("vecnorm_moments: ws needs 2 * D elements")
    _lib.call("b200rl_vecnorm_moments", _ptr(x), f64, int(N), int(D), _ptr(ws), _stream(),
              label="vecnorm_moments." + ("col" if D > 1 else "pairwise"), flops=4.0 * N * D,
              nbytes=2.0 * x.numel() * x.element_size())


def vecnorm_combine(rms, ws, N, eps, ws_f32):
    """rms float64 [3D + 1] = (mean, var, std, count) updated with the batch moments ws of N rows (ws_f32: the batch
    was float32, so bvar * N is a float32 product as in numpy)."""
    _chk(rms, torch.float64, "rms")
    _chk(ws, torch.float64, "ws")
    D = (rms.numel() - 1) // 3
    if rms.numel() != 3 * D + 1 or ws.numel() < 2 * D:
        raise RuntimeError("vecnorm_combine: rms must hold 3 * D + 1 and ws 2 * D elements")
    _lib.call("b200rl_vecnorm_combine", _ptr(rms), _ptr(ws), int(bool(ws_f32)), int(N), int(D), float(eps), _stream(),
              label="vecnorm_combine", nbytes=56.0 * D)


def vecnorm_normalize(x, rms, clip, out):
    """out float32 [N, D] = clip((x - mean) / std, +-clip) in float64 (rms None: out = float32(x))."""
    f64 = _vn_dtype(x, "x")
    _chk(rms, torch.float64, "rms")
    _chk(out, torch.float32, "out")
    N, D = x.shape[0], x[0].numel()
    if out.numel() != N * D or not out.is_contiguous():
        raise RuntimeError("vecnorm_normalize: out must be contiguous with N * D elements")
    if rms is not None and rms.numel() != 3 * D + 1:
        raise RuntimeError("vecnorm_normalize: rms must hold 3 * D + 1 elements")
    _lib.call("b200rl_vecnorm_normalize", _ptr(x), f64, int(N), int(D), _ptr(rms), float(clip), _ptr(out), _stream(),
              label="vecnorm_normalize", nbytes=float(x.numel() * (x.element_size() + 4)))


def vecnorm_rewards(rew, news, ret, rms, gamma, eps, cliprew, out):
    """ret = ret * gamma + rew; with rms (float64 [4]): update it with ret's moments and out = clip(rew / std);
    without: out = float32(rew); then ret = 0 where news (uint8 [N] or None)."""
    f64 = _vn_dtype(rew, "rew")
    _chk(news, torch.uint8, "news")
    _chk(ret, torch.float64, "ret")
    _chk(rms, torch.float64, "rms")
    _chk(out, torch.float32, "out")
    N = rew.numel()
    if ret.numel() != N or out.numel() != N or (news is not None and news.numel() != N) or \
            (rms is not None and rms.numel() != 4):
        raise RuntimeError("vecnorm_rewards: shape mismatch")
    _lib.call("b200rl_vecnorm_rewards", _ptr(rew), f64, _ptr(news), int(N), _ptr(ret), _ptr(rms), float(gamma),
              float(eps), float(cliprew), _ptr(out), _stream(), label="vecnorm_rewards",
              nbytes=float(N * (rew.element_size() + 1 + 24 + 4)))


def vecnorm_add_latency(f64, n, out):
    """out float64 [2]: out[0] = SM cycles per dependent add (float64 if f64), over n adds in one thread."""
    _chk(out, torch.float64, "out")
    _lib.call("b200rl_vecnorm_add_latency", int(bool(f64)), int(n), _ptr(out), _stream(), label="vecnorm_add_latency")


# ---- DDPG (csrc/ddpg.cu) ---------------------------------------------------------------------------------------------
def ddpg_encode(obs, out, B, obs_dim, in_pad, sel=None, limit=0, mean=None, std=None, clip=5.0, act=None, act_sel=False,
                nA=0, overflow=None):
    """[clip(normalize(obs), +-clip) | action] -> fp16 [hi | lo] operand rows out [B, 2 * in_pad]; rows at the ring
    selection sel ([start, idx...], int64) or row b; act: float32 [*, nA] rows (ring rows when act_sel) or None."""
    for t, dt, nm in ((obs, torch.float32, "obs"), (out, torch.float16, "out"), (sel, torch.int64, "sel"),
                      (mean, torch.float32, "mean"), (std, torch.float32, "std"), (act, torch.float32, "act"),
                      (overflow, torch.int32, "overflow")):
        _chk(t, dt, nm)
    _lib.call("b200rl_ddpg_encode", _ptr(obs), _ptr(sel), int(limit), int(B), int(obs_dim), _ptr(mean), _ptr(std),
              float(clip), _ptr(act), int(bool(act_sel)), int(nA), int(in_pad), _ptr(out), _ptr(overflow), _stream(),
              label="ddpg_encode", nbytes=float(B) * (4.0 * (obs_dim + nA) + 4.0 * in_pad))


def ddpg_tanh(z, ldz, mu, B, nA):
    _chk(z, torch.float32, "z")
    _chk(mu, torch.float32, "mu")
    _lib.call("b200rl_ddpg_tanh", _ptr(z), int(ldz), _ptr(mu), int(B), int(nA), _stream(), label="ddpg_tanh")


def ddpg_denorm(q, ldq, mean, std, out, B):
    for t, nm in ((q, "q"), (mean, "mean"), (std, "std"), (out, "out")):
        _chk(t, torch.float32, nm)
    _lib.call("b200rl_ddpg_denorm", _ptr(q), int(ldq), _ptr(mean), _ptr(std), _ptr(out), int(B), _stream(),
              label="ddpg_denorm")


def ddpg_target(q1, ldq, sel, limit, rewards, terminals, mean, std, gamma, y, B):
    for t, nm in ((q1, "q1"), (rewards, "rewards"), (terminals, "terminals"), (mean, "mean"), (std, "std"), (y, "y")):
        _chk(t, torch.float32, nm)
    _chk(sel, torch.int64, "sel")
    _lib.call("b200rl_ddpg_target", _ptr(q1), int(ldq), _ptr(sel), int(limit), _ptr(rewards), _ptr(terminals),
              _ptr(mean), _ptr(std), float(gamma), _ptr(y), int(B), _stream(), label="ddpg_target")


def ddpg_loss(q, ldq, y, mean, std, B, dq, lddq, losses):
    for t, nm in ((q, "q"), (y, "y"), (mean, "mean"), (std, "std"), (losses, "losses")):
        _chk(t, torch.float32, nm)
    _chk(dq, torch.float16, "dq")
    _lib.call("b200rl_ddpg_loss", _ptr(q), int(ldq), _ptr(y), _ptr(mean), _ptr(std), int(B), _ptr(dq), int(lddq),
              _ptr(losses), _stream(), label="ddpg_loss")


def ddpg_actor_dz(g, ldg, mu, B, nA, dz, lddz):
    _chk(g, torch.float32, "g")
    _chk(mu, torch.float32, "mu")
    _chk(dz, torch.float16, "dz")
    _lib.call("b200rl_ddpg_actor_dz", _ptr(g), int(ldg), _ptr(mu), int(B), int(nA), _ptr(dz), int(lddz), _stream(),
              label="ddpg_actor_dz")


def ddpg_l2(w, g, segs, reg, loss):
    """segs: int64 device [nseg, 2] of (offset, length) into the flat w / g."""
    for t, nm in ((w, "w"), (g, "g"), (loss, "loss")):
        _chk(t, torch.float32, nm)
    _chk(segs, torch.int64, "segs")
    _lib.call("b200rl_ddpg_l2", _ptr(w), _ptr(g), _ptr(segs), int(segs.shape[0]), float(reg), _ptr(loss), _stream(),
              label="ddpg_l2")


def ddpg_obs_rms(x, pos0, limit, n, D, st, mean, std):
    _chk(x, torch.float32, "x")
    _chk(st, torch.float64, "st")
    _chk(mean, torch.float32, "mean")
    _chk(std, torch.float32, "std")
    _lib.call("b200rl_ddpg_obs_rms", _ptr(x), int(pos0), int(limit), int(n), int(D), _ptr(st), _ptr(mean), _ptr(std),
              _stream(), label="ddpg_obs_rms")


def ddpg_ret_rms(y, B, st, mean, std, popart=None):
    """popart: (w0, b0, w1, b1) float32 device views of the critic's and the target critic's output layers, or None."""
    _chk(y, torch.float32, "y")
    _chk(st, torch.float64, "st")
    w0 = b0 = w1 = b1 = None
    if popart is not None:
        w0, b0, w1, b1 = popart
        for t, nm in ((w0, "w0"), (b0, "b0"), (w1, "w1"), (b1, "b1")):
            _chk(t, torch.float32, nm)
    _lib.call("b200rl_ddpg_ret_rms", _ptr(y), int(B), _ptr(st), _ptr(mean), _ptr(std), _ptr(w0), _ptr(b0), _ptr(w1),
              _ptr(b1), 0 if w0 is None else w0.numel(), _stream(), label="ddpg_ret_rms")


def ddpg_pn_adapt(mu, mu_adapt, n, desired, stddev, stddev32, dist):
    _chk(mu, torch.float32, "mu")
    _chk(mu_adapt, torch.float32, "mu_adapt")
    _chk(stddev, torch.float64, "stddev")
    _chk(stddev32, torch.float32, "stddev32")
    _chk(dist, torch.float32, "dist")
    _lib.call("b200rl_ddpg_pn_adapt", _ptr(mu), _ptr(mu_adapt), int(n), float(desired), _ptr(stddev), _ptr(stddev32),
              _ptr(dist), _stream(), label="ddpg_pn_adapt")


# ---- HER (csrc/her.cu) ----------------------------------------------------------------------------------------------
def her_sample(ring, sel, B, relative, clip_obs, o_mean, o_std, g_mean, g_std, norm_clip, max_u, reward_type,
               threshold, r, xa, xta, pad_a, xc, xtc, pad_c, ag2_out=None, g_out=None, info_out=None):
    """ring: (o, ag, g, u, info) float64 device tensors [S, T+1 or T, dim]; sel: int64 [B, 3] (episode, t, future_t)."""
    o, ag, g, u, info = ring
    for t, nm in ((o, "o"), (ag, "ag"), (g, "g"), (u, "u"), (info, "info"), (ag2_out, "ag2_out"), (g_out, "g_out"),
                  (info_out, "info_out")):
        _chk(t, torch.float64, nm)
    for t, nm in ((o_mean, "o_mean"), (o_std, "o_std"), (g_mean, "g_mean"), (g_std, "g_std"), (max_u, "max_u"),
                  (r, "r")):
        _chk(t, torch.float32, nm)
    for t, nm in ((xa, "xa"), (xta, "xta"), (xc, "xc"), (xtc, "xtc")):
        _chk(t, torch.float16, nm)
    _chk(sel, torch.int64, "sel")
    T, ninfo = g.shape[1], (0 if info is None else info.shape[2])
    _lib.call("b200rl_her_sample", _ptr(o), _ptr(ag), _ptr(g), _ptr(u), _ptr(info), int(T), int(o.shape[2]),
              int(g.shape[2]), int(u.shape[2]), int(ninfo), _ptr(sel), int(B), int(bool(relative)), float(clip_obs),
              _ptr(o_mean), _ptr(o_std), _ptr(g_mean), _ptr(g_std), float(norm_clip), _ptr(max_u), int(reward_type),
              float(threshold), _ptr(r), _ptr(xa), _ptr(xta), int(pad_a), _ptr(xc), _ptr(xtc), int(pad_c),
              _ptr(ag2_out), _ptr(g_out), _ptr(info_out), _stream(), label="her_sample")


def her_obs_encode(o, g, n, o_mean, o_std, g_mean, g_std, norm_clip, xa, pad_a, xc=None, pad_c=0):
    for t, nm in ((o, "o"), (g, "g"), (o_mean, "o_mean"), (o_std, "o_std"), (g_mean, "g_mean"), (g_std, "g_std")):
        _chk(t, torch.float32, nm)
    _chk(xa, torch.float16, "xa")
    _chk(xc, torch.float16, "xc")
    _lib.call("b200rl_her_obs_encode", _ptr(o), _ptr(g), int(n), int(o.shape[1]), int(g.shape[1]), _ptr(o_mean),
              _ptr(o_std), _ptr(g_mean), _ptr(g_std), float(norm_clip), _ptr(xa), int(pad_a), _ptr(xc), int(pad_c),
              _stream(), label="her_obs_encode")


def her_pi(z, ldz, B, dimu, max_u, pi, xc=None, pad_c=0, col0=0):
    for t, nm in ((z, "z"), (max_u, "max_u"), (pi, "pi")):
        _chk(t, torch.float32, nm)
    _chk(xc, torch.float16, "xc")
    _lib.call("b200rl_her_pi", _ptr(z), int(ldz), int(B), int(dimu), _ptr(max_u), _ptr(pi), _ptr(xc), int(pad_c),
              int(col0), _stream(), label="her_pi")


def her_target(q, ldq, r, B, gamma, lo, hi, y):
    for t, nm in ((q, "q"), (r, "r"), (y, "y")):
        _chk(t, torch.float32, nm)
    _lib.call("b200rl_her_target", _ptr(q), int(ldq), _ptr(r), int(B), float(gamma), float(lo), float(hi), _ptr(y),
              _stream(), label="her_target")


def her_loss(q, ldq, y, B, dq, lddq, loss, q_pi):
    for t, nm in ((q, "q"), (y, "y"), (loss, "loss"), (q_pi, "q_pi")):
        _chk(t, torch.float32, nm)
    _chk(dq, torch.float16, "dq")
    _lib.call("b200rl_her_loss", _ptr(q), int(ldq), _ptr(y), int(B), _ptr(dq), int(lddq), _ptr(loss), _ptr(q_pi),
              _stream(), label="her_loss")


def her_actor_dz(g, ldg, z, ldz, pi, B, dimu, max_u, action_l2, dz, lddz):
    for t, nm in ((g, "g"), (z, "z"), (pi, "pi"), (max_u, "max_u")):
        _chk(t, torch.float32, nm)
    _chk(dz, torch.float16, "dz")
    _lib.call("b200rl_her_actor_dz", _ptr(g), int(ldg), _ptr(z), int(ldz), _ptr(pi), int(B), int(dimu), _ptr(max_u),
              float(action_l2), _ptr(dz), int(lddz), _stream(), label="her_actor_dz")


def her_norm(o, ag, g, sel, N, relative, clip_obs, f32_o, f32_g, o_stats, g_stats, eps):
    """o / ag / g: float64 episode arrays [S, T+1 or T, dim]; *_stats: (state [2D + 1], mean [D], std [D]) float32."""
    for t, nm in ((o, "o"), (ag, "ag"), (g, "g")):
        _chk(t, torch.float64, nm)
    for t in tuple(o_stats) + tuple(g_stats):
        _chk(t, torch.float32, "stats")
    _chk(sel, torch.int64, "sel")
    _lib.call("b200rl_her_norm", _ptr(o), _ptr(ag), _ptr(g), int(g.shape[1]), int(o.shape[2]), int(g.shape[2]),
              _ptr(sel), int(N), int(bool(relative)), float(clip_obs), int(bool(f32_o)), int(bool(f32_g)),
              _ptr(o_stats[0]), _ptr(o_stats[1]), _ptr(o_stats[2]), _ptr(g_stats[0]), _ptr(g_stats[1]),
              _ptr(g_stats[2]), float(eps), _stream(), label="her_norm")


def acer_step(logits, ld, nA, actions, mu, B, seed=0, offset=0, offset_dev=None):
    """ACER act: actions int64 [B] (the cat_step sampler's bits) and mu float32 [B, nA] = softmax(logits)."""
    _chk(logits, torch.float32, "logits")
    _chk(actions, torch.int64, "actions")
    _chk(mu, torch.float32, "mu")
    _chk(offset_dev, torch.int64, "offset_dev")
    _lib.call("b200rl_acer_step", _ptr(logits), int(ld), int(nA), int(seed), int(offset), _ptr(offset_dev),
              _ptr(actions), _ptr(mu), int(B), _stream(), label="acer_step", nbytes=float(B) * (8.0 * nA + 8.0))


def acer_stack_obs(ring, idx, nenv, nsteps, nstack, dones_ring, out):
    """_stack_obs of ring slot idx[e] of every env e (idx None: slot 0).  ring [slots, nenv, nsteps+nstack, *frame, nc]
    uint8 / float32, dones_ring uint8 [slots, nenv, nsteps], out [nenv * (nsteps + 1), *frame, nstack * nc]."""
    if ring.dtype not in (torch.uint8, torch.float32) or out.dtype != ring.dtype:
        raise RuntimeError("acer_stack_obs: uint8 or float32 frames, and out of the same dtype")
    _chk(dones_ring, torch.uint8, "dones_ring")
    _chk(idx, torch.int64, "idx")
    nc = int(ring.shape[-1])
    F = int(ring[0, 0, 0].numel()) // nc
    if ring.shape[1] != nenv or ring.shape[2] != nsteps + nstack or out.numel() != nenv * (nsteps + 1) * F * nstack * nc:
        raise RuntimeError("acer_stack_obs: ring / out shapes do not match nenv, nsteps, nstack")
    _lib.call("b200rl_acer_stack_obs", _ptr(ring), int(ring.dtype == torch.float32), int(ring[0].numel()), _ptr(idx),
              int(nenv), int(nsteps), int(nstack), F, nc, _ptr(dones_ring), _ptr(out), _stream(),
              label="acer_stack_obs", nbytes=float(out.numel() * out.element_size()) * 2.0)


def acer_take(idx, nenv, nsteps, nA, rings, outs):
    """Buffer.take of the per-step arrays: rings / outs = (actions int64, rewards f32, mus f32, dones u8, masks u8)."""
    for ts in (rings, outs):
        for t, dt, nm in zip(ts, (torch.int64, torch.float32, torch.float32, torch.uint8, torch.uint8),
                             ("actions", "rewards", "mus", "dones", "masks")):
            _chk(t, dt, nm)
    _chk(idx, torch.int64, "idx")
    _lib.call("b200rl_acer_take", _ptr(idx), int(nenv), int(nsteps), int(nA), *[_ptr(t) for t in rings],
              *[_ptr(t) for t in outs], _stream(), label="acer_take")


def acer_loss(pi, ldpi, q, ldq, pol, ldpol, actions, rewards, dones, mus, nenv, nsteps, nA, gamma, c, delta, q_coef,
              ent_coef, trust_region, dpi, lddpi, dq, lddq, stats, f_out=None, v_out=None, qret_out=None):
    """acer.py:103-178 for nenv * (nsteps + 1) head rows; see include/b200rl.h."""
    for t, nm in ((pi, "pi"), (q, "q"), (pol, "pol"), (rewards, "rewards"), (mus, "mus"), (f_out, "f_out"),
                  (v_out, "v_out"), (qret_out, "qret_out")):
        _chk(t, torch.float32, nm)
    _chk(actions, torch.int64, "actions")
    _chk(dones, torch.uint8, "dones")
    _chk(dpi, torch.float16, "dpi")
    _chk(dq, torch.float16, "dq")
    _chk(stats, torch.float64, "stats")
    _lib.call("b200rl_acer_loss", _ptr(pi), int(ldpi), _ptr(q), int(ldq), _ptr(pol), int(ldpol), _ptr(actions),
              _ptr(rewards), _ptr(dones), _ptr(mus), int(nenv), int(nsteps), int(nA), float(gamma), float(c),
              float(delta), float(q_coef), float(ent_coef), int(bool(trust_region)), _ptr(dpi), int(lddpi), _ptr(dq),
              int(lddq), _ptr(stats), _ptr(f_out), _ptr(v_out), _ptr(qret_out), _stream(), label="acer_loss")


def clip_rmsprop_ema(p, g, ms, shadow, lr_dev, clip, sumsq_buf, decay, eps, alpha):
    """Global-norm clip + TF RMSProp (momentum 0) + Polyak moving average of the updated parameters, one pass."""
    for t, nm in ((p, "p"), (g, "g"), (ms, "ms"), (shadow, "shadow"), (lr_dev, "lr_dev")):
        _chk(t, torch.float32, nm)
    if not (p.numel() == g.numel() == ms.numel() == shadow.numel()):
        raise RuntimeError("clip_rmsprop_ema: buffer sizes differ")
    _lib.call("b200rl_clip_rmsprop_ema", _ptr(p), _ptr(g), _ptr(ms), _ptr(shadow), p.numel(), _ptr(lr_dev),
              float(clip if clip else 0.0), _ptr(sumsq_buf), float(decay), float(eps), float(alpha), _stream(),
              label="clip_rmsprop_ema", nbytes=20.0 * p.numel())
