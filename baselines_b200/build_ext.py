"""Build libb200rl.so in-tree with nvcc for sm_90a (no torch dependency in the library)."""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libb200rl.so")
SOURCES = ["api.cu", "gemm_wgmma.cu", "conv_shift.cu", "gae.cu", "conv_lowering.cu", "policy_heads.cu", "optim.cu", "replay.cu", "obs_encode.cu",
           "lstm.cu", "layer_norm.cu", "param_noise.cu", "vec_normalize.cu", "ddpg.cu",
           "her.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; libb200rl needs the CUDA toolkit to build")


STAMP = LIB + ".srchash"


def _source_hash():
    """Content hash of everything the library is built from.  (File times do not survive the copy to a GPU box in
    order, so an mtime comparison rebuilt the library there at random -- a minute of nvcc inside a measurement run.)"""
    import hashlib
    h = hashlib.sha256(" ".join(NVCC_FLAGS + SOURCES).encode())
    deps = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC)) + [os.path.join(HERE, "..", "include", "b200rl.h")]
    for d in deps:
        h.update(os.path.basename(d).encode())
        with open(d, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def needs_build():
    if not os.path.exists(LIB) or not os.path.exists(STAMP):
        return True
    with open(STAMP) as f:
        return f.read().strip() != _source_hash()


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    nvcc = _nvcc()
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write(f"--- nvcc {src}\n{out}\n")
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed building libb200rl")
    cmd = [nvcc] + NVCC_FLAGS[:2] + ["-shared", "-o", LIB] + objs + ["-lcudart"]
    subprocess.check_call(cmd)
    with open(STAMP, "w") as f:
        f.write(_source_hash() + "\n")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
