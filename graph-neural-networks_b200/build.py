"""Builds libb200gf.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

`python graph-neural-networks_b200/build.py` or `__graft_entry__.build()`.  The .so and the objects under build/ are
git-ignored build products.  nvcc cross-compiles without a GPU.
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libb200gf.so")
SOURCES = ["plan.cu", "spmm.cu", "taps.cu", "layout.cu", "lsigf.cu", "tc_contract.cu", "ev.cu", "layer.cu", "dmma_contract.cu",
           "egate.cu", "nv/nv.cu", "arma/arma.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC,-O3,-Wall", "--expt-relaxed-constexpr"]


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build_library(force=False, verbose=False):
    srcs = [os.path.join(CSRC, s) for s in SOURCES]
    missing = [s for s in srcs if not os.path.exists(s)]
    if missing:
        raise FileNotFoundError("b200gf: listed CUDA sources do not exist: %s" % ", ".join(missing))
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(os.path.dirname(HERE), "include", "b200gf.h"))
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    nvcc = _nvcc()
    objs = []
    procs = []
    for s in srcs:
        o = os.path.join(objdir, os.path.basename(s) + ".o")
        objs.append(o)
        if force or _stale(o, [s] + headers):
            cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", s, "-o", o]
            procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write("nvcc failed on %s:\n%s\n" % (s, out))
        elif verbose or out.strip():
            sys.stderr.write(out)
    if failed:
        raise RuntimeError("b200gf: CUDA build failed")
    if force or procs or _stale(LIB, objs):
        cmd = [nvcc, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart"]
        subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build_library(force="--force" in sys.argv, verbose="-v" in sys.argv))
