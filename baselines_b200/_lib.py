"""ctypes binding of libb200rl.so (the C-ABI declared in include/b200rl.h).

There is NO fallback: if the shared library is missing or a call fails, a RuntimeError is raised --
the product path never routes through the CPU oracle or plain PyTorch ops.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200rl.so")

_p, _i, _ll, _f, _d, _ull = C.c_void_p, C.c_int, C.c_longlong, C.c_float, C.c_double, C.c_ulonglong

# name -> argtypes (all return int); must mirror include/b200rl.h exactly (checked by tests/test_cabi.py)
SIGNATURES = {
    "b200rl_gae_scan": [_p, _p, _p, _p, _p, _p, _p, _i, _i, _d, _d, _i, _p],
    "b200rl_gemm_f16": [_p, _p, _p, _p, _p, _i, _i, _i, _ll, _ll, _ll, _ll, _i, _i, _i, _f, _i, _i, _i, _i, _i, _p, _p],
    "b200rl_conv_shift_fwd": [_p, _ll, _i, _i, _i, _p, _ll, _i, _i, _p, _i, _i, _p, _p, _p, _p, _i, _i, _f,
                              _p, _p, _i, _i, _i, _i, _p, _p, _p],
    "b200rl_conv_shift_wgrad": [_p, _ll, _i, _p, _i, _i, _p, _p, _ll, _f, _p, _f, _i, _p, _p, _i, _i, _i, _i, _i, _p],
    "b200rl_conv_gemm": [_p, _ll, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _p, _ll, _p, _ll, _p, _p, _ll, _i, _i, _i,
                         _i, _f, _i, _i, _i, _i, _i, _p],
    "b200rl_dgrad_weights": [_p, _p, _i, _i, _i, _i, _i, _ll, _p],
    "b200rl_im2col": [_p, _i, _p, _p, _ll, _i, _i, _i, _i, _i, _i, _p],
    "b200rl_s2d_gather": [_p, _p, _p, _ll, _i, _i, _i, _i, _p],
    "b200rl_frame_stack": [_p, _p, _p, _p, _ll, _ll, _i, _i, _p],
    "b200rl_col2im": [_p, _p, _p, _ll, _i, _i, _i, _i, _i, _i, _i, _p],
    "b200rl_colsum": [_p, _p, _ll, _i, _ll, _f, _p],
    "b200rl_cat_step": [_p, _ll, _i, _p, _i, _p, _ll, _p, _ull, _ull, _p, _p, _p, _p, _ll, _p],
    "b200rl_bern_step": [_p, _ll, _i, _p, _ll, _p, _ull, _ull, _p, _p, _p, _p, _ll, _p],
    "b200rl_gauss_step": [_p, _ll, _p, _i, _p, _ll, _p, _ull, _ull, _p, _p, _p, _p, _ll, _p],
    "b200rl_set_scalars": [_p, _i, _f, _f, _f, _f, _p],
    "b200rl_shuffle_indices": [_p, _ll, _ull, _ll, _ll, _p],
    "b200rl_counter_add": [_p, _ull, _p],
    "b200rl_adv_stats": [_p, _p, _p, _ll, _p, _p],
    "b200rl_cat_loss": [_p, _ll, _i, _p, _i, _p, _ll, _p, _p, _p, _p, _p, _p, _f, _f, _f, _p, _ll, _p, _ll, _p, _ll, _p,
                        _p],
    "b200rl_bern_loss": [_p, _ll, _i, _p, _ll, _p, _p, _p, _p, _p, _p, _f, _f, _f, _p, _ll, _p, _ll, _p, _ll, _p, _p],
    "b200rl_gauss_loss": [_p, _ll, _p, _i, _p, _ll, _p, _p, _p, _p, _p, _p, _f, _f, _f, _p, _ll, _p, _ll, _p, _f,
                          _p, _ll, _p, _p],
    "b200rl_sumsq": [_p, _ll, _p, _p],
    "b200rl_seg_sumsq": [_p, _p, _i, _p, _p],
    "b200rl_clip_adam": [_p, _p, _p, _p, _ll, _f, _f, _f, _f, _f, _p, _p, _i, _p, _p],
    "b200rl_clip_accumulate": [_p, _p, _ll, _f, _f, _p, _p],
    "b200rl_cast_transpose": [_p, _i, _i, _p, _ll, _p, _ll, _f, _p],
    "b200rl_cast_transpose_batch": [_p, _i, _i, _i, _p],
    "b200rl_cast_f32_f16": [_p, _p, _ll, _i, _ll, _ll, _f, _p],
    "b200rl_obs_encode": [_p, _p, _ll, _i, _i, _i, _p, _p, _f, _f, _i, _p, _i, _p, _p, _p],
    "b200rl_tree_set": [_p, _p, _ll, _p, _p, _i, _p],
    "b200rl_tree_range_sum": [_p, _ll, _ll, _ll, _p, _p],
    "b200rl_per_sample": [_p, _p, _ll, _ll, _p, _i, _d, _p, _p, _p, _p, _p],
    "b200rl_per_priorities": [_p, _i, _d, _d, _p, _p, _p, _p],
    "b200rl_per_pow": [_p, _i, _d, _p, _p],
    "b200rl_dqn_td": [_p, _ll, _p, _ll, _p, _ll, _p, _ll, _p, _ll, _p, _ll, _i, _p, _p, _p, _p, _p, _f, _i, _p, _p,
                      _ll, _p, _ll, _p, _i, _p],
    "b200rl_dqn_act": [_p, _ll, _p, _ll, _i, _f, _ull, _ull, _p, _p, _p, _i, _p],
    "b200rl_lstm_seq_fwd": [_p, _ll, _p, _p, _p, _p, _p, _p, _p, _ll, _p, _p, _p, _i, _i, _i, _p],
    "b200rl_lstm_seq_bwd": [_p, _ll, _p, _p, _p, _p, _p, _p, _p, _p, _ll, _i, _i, _i, _p],
    "b200rl_ln_fwd": [_p, _ll, _p, _p, _p, _ll, _ll, _i, _i, _f, _p],
    "b200rl_ln_bwd": [_p, _ll, _p, _ll, _p, _p, _ll, _p, _p, _ll, _i, _f, _f, _p],
    "b200rl_param_perturb": [_p, _p, _p, _i, _ll, _p, _p, _ull, _p, _p],
    "b200rl_dqn_param_noise_adapt": [_p, _p, _ll, _i, _i, _i, _p, _p, _p, _p],
    "b200rl_vecnorm_moments": [_p, _i, _ll, _i, _p, _p],
    "b200rl_vecnorm_combine": [_p, _p, _i, _ll, _i, _d, _p],
    "b200rl_vecnorm_normalize": [_p, _i, _ll, _i, _p, _d, _p, _p],
    "b200rl_vecnorm_rewards": [_p, _i, _p, _ll, _p, _p, _d, _d, _d, _p, _p],
    "b200rl_vecnorm_add_latency": [_i, _ll, _p, _p],
}

_lib = None


def load():
    """Load (once) and return the ctypes handle; raises if the extension has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"libb200rl.so not found at {LIB_PATH}: build it with `python -m baselines_b200.build_ext` "
            "(or __graft_entry__.build()). There is no CPU / PyTorch fallback for the hot path.")
    lib = C.CDLL(LIB_PATH)
    lib.b200rl_last_error.restype = C.c_char_p
    lib.b200rl_last_error.argtypes = []
    lib.b200rl_version.restype = C.c_int
    lib.b200rl_version.argtypes = []
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if a declared symbol is not exported
        fn.argtypes = argtypes
        fn.restype = C.c_int
    _lib = lib
    return lib


LAUNCHES = 0          # library kernels launched by this process, eagerly or inside graph replays (bench.py reports the delta)
REPLAYS = 0           # CUDA-graph replays (graphs.py)
_prof = None          # list of (label, start_event, end_event, flops, bytes) while profiling
phase = ""            # profile-label suffix ("@act" / "@train"): the same kernel runs at two very different sizes


def call(name, *args, label=None, flops=0, nbytes=0):
    global LAUNCHES
    lib = load()
    LAUNCHES += 1
    if _prof is not None:
        import torch
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        rc = getattr(lib, name)(*args)
        e1.record()
        _prof.append(((label or name) + phase, e0, e1, flops, nbytes))
    else:
        rc = getattr(lib, name)(*args)
    if rc != 0:
        raise RuntimeError(f"{name} failed (rc={rc}): {lib.b200rl_last_error().decode()}")


def profile_begin():
    """Start timing every C-ABI call with CUDA events on the launching stream (no host sync is added)."""
    global _prof
    _prof = []


def profile_end():
    """-> {label: [total_ms, calls, algorithmic_flops, algorithmic_bytes]}"""
    global _prof
    import torch
    torch.cuda.synchronize()
    out = {}
    for label, e0, e1, flops, nbytes in _prof:
        acc = out.setdefault(label, [0.0, 0, 0.0, 0.0])
        acc[0] += e0.elapsed_time(e1)
        acc[1] += 1
        acc[2] += flops
        acc[3] += nbytes
    _prof = None
    return out
