"""What every kernel dispatch table shares: inputs, canaries, launch tracing and the GPU check of one row.

A table is a list of rows (case id, fn, kernel regexes).  fn runs one launch branch of the library and returns a
Result; the regexes name the kernels that branch must launch (on the demangled name, template arguments included, see
_norm).  check_case holds a row to every check: the expected launches, each output within its componentwise fp64
bound, canaries intact, no NaN leaked from input pads, and bit-identical reruns.  Tables trace their launches either in
the pytest process (_launched) or in a child process of their own (child_traced).  tests/test_dispatch_tables.py
checks on the CPU that the tables together cover every __global__ function of the package.
"""
import functools
import json
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import lsigf_oracle as orc

SENT = -7.125e30            # canary value: exactly representable in fp32 and fp64, never produced by these inputs
F32, F64 = torch.float32, torch.float64
NPD = {F32: np.float32, F64: np.float64}


def _lib():
    import gnn_b200
    return gnn_b200._cabi, gnn_b200._cabi.load()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _check(rc):
    cabi, lib = _lib()
    assert rc == 0, lib.b200gf_strerror(rc)


def _padded(C, dtype):
    q = 32 // torch.empty(0, dtype=dtype).element_size()
    return (C + q - 1) // q * q


class Result:
    """What a case run hands back: outputs (tensors, compared bit-for-bit across runs), checks (name, out, ref, bound;
    ref None when the case asserted the output exact itself, or a callable returning (ref, bound) that check_case calls
    when it checks the row, so a costly reference is computed once and outside traced runs), canaries (name, tensor that must equal SENT, or 0x5A for
    integer buffers, bit-for-bit), finite (name, tensor that must be all finite), same (name, a, b: bit-identical) and
    nondeterministic (the outputs' last bits may change between runs: only the bounds are checked)."""

    def __init__(self):
        self.outputs, self.checks, self.canaries, self.finite, self.same = [], [], [], [], []
        self.nondeterministic = False


@functools.lru_cache(maxsize=None)
def _graph(kind, N, seed=0):
    """Row lengths 0, 1, S*U-1 .. S*U+1 of every lane mapping (S*U = 4, 8, 16, 32), 31..65, 127..129, a self-loop, a
    neighbour in column N-1, and (N > 20000) a hub row of 20 000 entries; the transpose gets the same lengths through
    the long columns added at the end."""
    rng = np.random.default_rng(seed + N)
    special = [0, 1, 3, 4, 5, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129]
    if kind == "tiny":
        special = special[:N]
    lens = list(rng.integers(0, 9, N))
    for i, L in enumerate(special[:N]):
        lens[i] = min(L, N)
    if N > 20000:
        lens[N // 2] = 20000
    rows, cols = [], []
    for r, L in enumerate(lens):
        rows += [r] * int(L)
        cols += list(rng.choice(N, size=int(L), replace=False))
    # long columns (rows of S^T) of the same lengths, in columns N-1, N-2, ...
    for i, L in enumerate(special[:N] + ([20000] if N > 20000 else [])):
        if N >= 60:
            rows += list(rng.choice(N, size=min(L, N), replace=False))
            cols += [N - 1 - i] * min(L, N)
    rows += [min(3, N - 1), min(5, N - 1)]
    cols += [min(3, N - 1), N - 1]                       # self-loop, neighbour N-1
    m = sp.coo_matrix((rng.standard_normal(len(rows)), (rows, cols)), shape=(N, N)).tocsr()
    m.sum_duplicates()
    if kind == "sym":
        m = sp.triu(m, 1) + sp.triu(m, 1).T + sp.diags(m.diagonal())
        m = sp.csr_matrix(m)
    m.sort_indices()
    return m


def _from_node_major(t, B, C, N):
    return t[:N, :B * C].reshape(N, B, C).permute(1, 2, 0)


def _norm(name):
    """Demangled kernel name without casts and spaces: 'spmm_hop_kernel<float, (int)4, ...' -> 'spmm_hop_kernel<float,4,...'."""
    name = re.sub(r"\((?:int|bool|unsigned int|long)\)", "", name)
    return name.replace(" ", "").replace("true", "1").replace("false", "0")


def _bits(t):
    t = t.detach().contiguous()
    return t.view(torch.int32 if t.element_size() == 4 else torch.int64) if t.is_floating_point() else t


def kernel_names(cases):
    """The __global__ function names a table's regexes refer to."""
    return {re.match(r"\w+", k).group(0) for _, _, ks in cases for k in ks}


@functools.lru_cache(maxsize=None)
def library_kernels():
    """The normalised demangled names of every kernel compiled into libb200gf.so, or None without the library or
    cuobjdump / cu++filt."""
    import gnn_b200
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    filt = shutil.which("cu++filt") or "/usr/local/cuda/bin/cu++filt"
    lib = gnn_b200._cabi.LIB_PATH
    if not (os.path.exists(tool) and os.path.exists(filt) and os.path.exists(lib)):
        return None
    syms = subprocess.run([tool, "-symbols", lib], capture_output=True, text=True, check=True).stdout
    mangled = re.findall(r"STT_FUNC\s+.*?\s(\S+)\s*$", syms, flags=re.M)
    return [_norm(n) for n in subprocess.run([filt], input="\n".join(mangled), capture_output=True, text=True,
                                              check=True).stdout.splitlines()]


# ------------------------------------------------------------------------------------------------------- tracing
def _launched(fn):
    """fn's Result and the names of the CUDA activities of that run, traced in this process."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        res = fn()
        torch.cuda.synchronize()
    names = [_norm(e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return res, names


def _profiled(fn, kernels, tries=4):
    """The demangled names of the CUDA activities of one run of fn under torch.profiler.  A session can come back
    without its GPU records (seen with torch 2.11 on an H100 once a process had been profiling for about two minutes:
    alternate sessions empty, whatever they ran); fn is deterministic, so while some regex of `kernels` matches no
    traced name the case is profiled again, up to `tries` times.  The caller still requires every expected kernel."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(tries):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = [_norm(e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        if all(any(re.search(k, n) for n in names) for k in kernels):
            break
    return names


def trace_all(module, table, path):
    """Writes {case id: traced names} of every row of module.table to path (JSON); run in a process of its own by
    child_traced."""
    import importlib
    rows = getattr(importlib.import_module(module), table)
    with open(path, "w") as f:
        json.dump({cid: _profiled(fn, ks) for cid, fn, ks in rows}, f)


def child_traced(module, table):
    """A module-scoped fixture `traced`: {case id: kernels launched} of every row of module.table, traced in a fresh
    Python process.  The profiler degrades with the time since a process first used it (see _profiled); tracing in the
    pytest process would start that clock minutes before test_kernel_dispatch.py and test_nv_dispatch.py profile their
    own rows there.  A child process per table keeps its sessions inside its own first minute and leaves the pytest
    process's profiler untouched."""
    @pytest.fixture(scope="module")
    def traced(tmp_path_factory):
        path = tmp_path_factory.mktemp(module) / "names.json"
        here = os.path.dirname(os.path.abspath(__file__))
        root = os.path.dirname(here)
        env = dict(os.environ, PYTHONDONTWRITEBYTECODE="1",
                   PYTHONPATH=os.pathsep.join([here, os.path.join(root, "oracle"), root]
                                              + [p for p in os.environ.get("PYTHONPATH", "").split(os.pathsep) if p]))
        flags = ["-s"] if sys.flags.no_user_site else []
        subprocess.run([sys.executable] + flags + ["-c", "import sys, dispatch_harness as h; h.trace_all(*sys.argv[1:])",
                                                   module, table, str(path)], env=env, cwd=root, check=True, timeout=1800)
        with open(path) as f:
            return json.load(f)
    return traced


# ----------------------------------------------------------------------------------------------------- GPU check
def check_case(cid, fn, kernels, names, res1=None):
    """Holds one row to every check.  names: the kernels its run launched; res1: that run's Result when it was traced in
    this process (otherwise fn runs here)."""
    print("%s: %s" % (cid, sorted(set(n.split("(")[0] for n in names if "kernel" in n))))
    remaining = list(names)
    for k in kernels:   # a regex listed twice must match two launches
        hit = next((n for n in remaining if re.search(k, n)), None)
        assert hit is not None, "%s: expected %s among %s" % (cid, k, sorted(set(n.split("(")[0] for n in names)))
        remaining.remove(hit)
    if res1 is None:
        res1 = fn()
        torch.cuda.synchronize()
    worst = []
    for name, out, ref, bound in res1.checks:
        if ref is None:
            continue
        if callable(ref):
            ref, bound = ref()
        v = orc.bound_violation(out.detach().double().cpu().numpy(), ref, bound)
        worst.append("%s %.3g" % (name, v))
        assert v <= 1.0, "%s/%s: error %.3g x its bound" % (cid, name, v)
    print("%s: worst error / bound: %s" % (cid, ", ".join(worst) or ("exact" if res1.checks else "oracle tolerance")))
    for name, t in res1.canaries:
        assert torch.equal(_bits(t), _bits(torch.full_like(t, SENT if t.is_floating_point() else 0x5A))), \
            "%s: wrote outside its contract (%s)" % (cid, name)
    for name, t in res1.finite:
        assert bool(torch.isfinite(t).all()), "%s: non-finite %s (NaN in an input pad leaked)" % (cid, name)
    for name, a, b in res1.same:
        assert torch.equal(_bits(a), _bits(b)), "%s: %s" % (cid, name)
    if res1.nondeterministic:
        return
    res2 = fn()
    torch.cuda.synchronize()
    for a, b in zip(res1.outputs, res2.outputs):
        assert torch.equal(_bits(a), _bits(b)), "%s: two runs differ" % cid
