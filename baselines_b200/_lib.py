"""ctypes binding of libb200rl.so (the C-ABI declared in include/b200rl.h).

There is NO fallback: if the shared library is missing or a call fails, a RuntimeError is raised --
the product path never routes through the CPU oracle or plain PyTorch ops.
"""
import ctypes as C
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200rl.so")
HEADER = os.path.join(_HERE, "..", "include", "b200rl.h")

# C parameter type -> ctypes type; every pointer passes as c_void_p
_CTYPES = {"int": C.c_int, "long long": C.c_longlong, "unsigned long long": C.c_ulonglong, "float": C.c_float,
           "double": C.c_double}


def _ctype(param):
    """ctypes type of one C parameter declaration ("const float* x", "long long ld", ...); raises on a type without
    a mapping rather than guess one."""
    if "*" in param:
        return C.c_void_p
    typ = " ".join(param.split()[:-1])
    if typ not in _CTYPES:
        raise ValueError(f"include/b200rl.h: no ctypes mapping for parameter {param!r}")
    return _CTYPES[typ]


def _signatures():
    """name -> argtypes of every entry point the header declares, except the two argument-less ones load() binds."""
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    decls = re.findall(r"\b(?:int|const char\*)\s+(b200rl_\w+)\s*\(([^;]*?)\)\s*;", src, flags=re.S)
    return {name: [_ctype(a.strip()) for a in args.split(",")] for name, args in decls
            if name not in ("b200rl_last_error", "b200rl_version")}


# all entry points return int; parsed once per process
SIGNATURES = _signatures()

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
