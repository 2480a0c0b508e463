#!/usr/bin/env python
"""Times the localized activations (MaxLocalActivation / MedianLocalActivation) on CUDA, and MaxPoolLocal's kernel
against another build of the library.  Writes one JSON file (default tools/results/local_activation_bench.json) with
the card's name and power limit, read in the same run.

    python tools/local_activation_bench.py [--out PATH] [--parent-lib PATH]

  * N = 100 000, degree 16 (16 uniform out-neighbours per node), B = 16, F = 32, K = 2, fp32: forward, and forward + backward
    (x and weight gradients), for Max and Median; CUDA events around `--reps` calls after a warm-up.
  * The same at N = 20 000 next to the torch path (index matrices padded to the widest neighbourhood, as the layers ran
    on CUDA tensors before; that path is reached through `_forward_torch`); "oom" where it does not fit.
  * The max forward's achieved bytes/s against its gather model: K-hop list entries x C x 4 bytes (every list entry
    gathers one node row of C values once; agg, arg and y writes are left out, so the rate is a lower bound).
  * MaxPoolLocal's forward kernel (b200gf_maxpool_forward, N = 100 000, the 1-hop matrix, C = 512) in this library
    and in `--parent-lib`, alternated call by call, to show what generalising the kernel in place cost it.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import scipy.sparse as sp
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def _time(fn, reps, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def _graph(N, deg, seed):
    """deg uniformly drawn out-neighbours per node (repeats merged)."""
    rng = np.random.default_rng(seed)
    return sp.csr_matrix((np.ones(N * deg), (np.repeat(np.arange(N), deg), rng.integers(0, N, N * deg))), shape=(N, N))


def _layer_times(kind, A, B, F, K, reps, torch_path=False):
    import gnn_b200
    from gnn_b200 import activations
    m = getattr(activations, kind + "LocalActivation")(K).cuda()
    m.addGSO(gnn_b200.SparseGSO.from_scipy([A]))
    N = A.shape[0]
    x = torch.randn(B, F, N, device="cuda", requires_grad=True)
    dy = torch.randn(B, F, N, device="cuda")
    fwd = (lambda: m._forward_torch(x)) if torch_path else (lambda: m(x))

    def fwd_bwd():
        y = fwd()
        torch.autograd.grad(y, [x, m.weight], dy)
    out = {}
    try:
        with torch.no_grad():
            out["forward_ms"] = _time(fwd, reps)
        out["forward_backward_ms"] = _time(fwd_bwd, reps)
    except torch.OutOfMemoryError:
        out["result"] = "oom"
    out["peak_gb"] = torch.cuda.max_memory_allocated() / 1e9
    out["list_entries"] = int(m._rings[0][-1])
    out["max_neighborhood_sizes"] = m.maxNeighborhoodSizes
    del m, x, dy
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    return out


def _maxpool_ab(parent_lib, N, C, reps):
    """ms per b200gf_maxpool_forward call, this library and parent_lib alternated, on one neighbourhood matrix."""
    import gnn_b200
    from gnn_b200.graphtools_sparse import compute_neighborhood
    libs = {"this": gnn_b200._cabi.load()}
    if parent_lib:
        p = ctypes.CDLL(parent_lib)
        name = "b200gf_maxpool_forward"
        getattr(p, name).restype, getattr(p, name).argtypes = gnn_b200._cabi._SIGNATURES[name]
        libs["parent"] = p
    nb = torch.tensor(compute_neighborhood(_graph(N, 16, 3), 1, outputType="matrix"), dtype=torch.int32,
                      device="cuda")
    x = torch.randn(N, C, device="cuda")
    out = torch.empty(N, C, device="cuda")
    arg = torch.empty(N, C, dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    res, ref = {k: [] for k in libs}, None
    for _ in range(5):
        for k, lib in libs.items():
            call = lambda: lib.b200gf_maxpool_forward(0, x.data_ptr(), C, N, C, nb.data_ptr(), N, nb.shape[1],  # noqa
                                                      out.data_ptr(), C, arg.data_ptr(), st)
            res[k].append(_time(call, reps))
            ref = out.clone() if ref is None else ref
            assert torch.equal(out, ref), "the two libraries' MaxPoolLocal results differ"
    return {"N": N, "C": C, "max_nb": int(nb.shape[1]),
            **{k + "_ms": {"median": float(np.median(v)), "min": float(np.min(v)), "all": v} for k, v in res.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "tools", "results", "local_activation_bench.json"))
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    B, F, K = 16, 32, 2
    C = B * F
    result = {"card": _card(), "dtype": "float32", "B": B, "F": F, "K": K, "runs": []}
    for N in (100_000, 20_000):
        A = _graph(N, 16, 1)
        for kind in ("Max", "Median"):
            r = {"N": N, "degree": 16, "kind": kind, "cuda": _layer_times(kind, A, B, F, K, a.reps)}
            if kind == "Max":
                r["cuda"]["max_forward_gather_GBps"] = r["cuda"]["list_entries"] * C * 4 / r["cuda"]["forward_ms"] / 1e6
            if N == 20_000:
                r["torch_path"] = _layer_times(kind, A, B, F, K, max(2, a.reps // 5), torch_path=True)
            result["runs"].append(r)
            print(json.dumps(r), flush=True)
    result["maxpool_local_forward"] = _maxpool_ab(a.parent_lib, 100_000, C, a.reps * 5)
    print(json.dumps(result["maxpool_local_forward"]), flush=True)
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(result, f, indent=1)
    print("wrote", a.out)


if __name__ == "__main__":
    main()
