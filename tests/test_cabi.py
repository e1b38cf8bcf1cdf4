"""CPU: the C-ABI library loads and exports every symbol include/b200rl.h declares (no compute)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "b200rl.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    decls = re.findall(r"\b(?:int|const char\*)\s+(b200rl_\w+)\s*\(([^;]*?)\)\s*;", src, flags=re.S)
    return {name: args for name, args in decls}


def _lib_path():
    from baselines_b200 import build_ext
    if build_ext.needs_build():
        build_ext.build()
    return build_ext.LIB


def test_library_exports_every_declared_symbol():
    decl = _declared()
    assert len(decl) >= 20
    lib = ctypes.CDLL(_lib_path())
    for name in decl:
        assert hasattr(lib, name), f"{name} declared in include/b200rl.h but not exported"


def test_binding_table_covers_every_header_parameter():
    """_lib.SIGNATURES is derived from the header: one row per int-returning declaration, one ctypes type per
    parameter, and every parameter type of the header has a mapping."""
    from baselines_b200 import _lib
    decl = _declared()
    assert set(_lib.SIGNATURES) == set(decl) - {"b200rl_last_error", "b200rl_version"}
    known = {ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_ulonglong, ctypes.c_float, ctypes.c_double}
    for name, argtypes in _lib.SIGNATURES.items():
        nargs = len([a for a in decl[name].split(",") if a.strip() and a.strip() != "void"])
        assert nargs == len(argtypes), f"{name}: header has {nargs} args, binding has {len(argtypes)}"
        assert all(t in known for t in argtypes), name
        assert decl[name].split(",")[-1].strip() == "void* stream", f"{name}: the stream is the last parameter"


def test_binding_rows_match_hand_written_ones():
    """Two derived rows against hand-written ones (gae_scan is the ctypes stub of INTEGRATION.md section 3), and a
    parameter type without a mapping is refused rather than guessed."""
    from baselines_b200 import _lib
    p, i, ll, f, d = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_float, ctypes.c_double
    assert _lib.SIGNATURES["b200rl_gae_scan"] == [p] * 7 + [i, i, d, d, i, p]
    assert _lib.SIGNATURES["b200rl_gemm_f16"] == [p] * 5 + [i] * 3 + [ll] * 4 + [i] * 3 + [f] + [i] * 5 + [p, p]
    assert _lib._ctype("unsigned long long seed") is ctypes.c_ulonglong
    for bad in ("size_t n", "const int n", "long n", "unsigned n"):
        with pytest.raises(ValueError):
            _lib._ctype(bad)


def test_version_and_error_string():
    from baselines_b200 import _lib
    lib = _lib.load()
    assert lib.b200rl_version() >= 100
    assert isinstance(lib.b200rl_last_error(), bytes)


def test_ops_refuse_cpu_tensors():
    """The hot path must fail loudly instead of falling back when tensors are not on the GPU."""
    import torch
    from baselines_b200 import ops
    a = torch.zeros(8, 8, dtype=torch.float16)
    with pytest.raises(RuntimeError):
        ops.gemm(a, a, a, M=8, N=8, K=8, lda=8, ldb=8, ldc=8)


def test_rebuild_decision_follows_source_content_not_file_times(tmp_path):
    """build_ext.needs_build(): a GPU box receives the tree with arbitrary file times, so the decision is a content hash
    of csrc/ + include/b200rl.h + the nvcc flags, stamped beside the library."""
    from baselines_b200 import build_ext
    _lib_path()
    assert not build_ext.needs_build()
    src = os.path.join(build_ext.CSRC, "gae.cu")
    st = os.stat(build_ext.LIB)
    os.utime(src, (st.st_atime + 1000, st.st_mtime + 1000))            # "newer" source, same content
    assert not build_ext.needs_build()
    stamp = open(build_ext.STAMP).read()
    try:
        open(build_ext.STAMP, "w").write("0" * 64 + "\n")              # stale stamp = sources changed since the build
        assert build_ext.needs_build()
    finally:
        open(build_ext.STAMP, "w").write(stamp)
    assert not build_ext.needs_build()
