#!/usr/bin/env python
"""Times the aggregation GNNs' graph product (aggregation.py) on CUDA and writes one JSON file,
tools/results/aggregation_bench_h100_<power limit>.json unless --out is given, with the card's name and power limit
read in the same run.

    python tools/aggregation_bench.py [--out PATH] [--reps R]

For every workload: the operator build time (R and R^T from the GSO's powers on the GPU, the level split and the level
plans, first call), the product's forward time and forward + backward time (input gradient; CUDA events around --reps
calls after a warm-up), the nnz of every level, and the bytes model: per level, the gathered rows (nnz x C x element
size) plus the column indices, values, 32-bit row offsets and the stored rows, over the measured time.  The forward
rate counts the R chain against the forward time; the forward + backward rate counts both chains against that time,
which also holds the layout passes, so it is a lower bound.

  * sourceloc: N = 100, nNodes = 1, maxN = N, B = 100, F = 1, float64 (examples/sourceLocGNN.py's aggregation GNN)
  * rand20k:   N = 20 000, 16 random out-neighbours per node, nNodes = 16, maxN = 5, B = 32, F = 4, float64
  * er1m:      N = 1 000 000, 32 random out-neighbours per node (average degree 32), nNodes = 16, maxN = 5, B = 32,
               F = 1, float32
The first two also run the reference's dense path on the same GPU, restated here: SN from dense numpy products
S @ delta on the host (its __init__), then torch.matmul(x [B,1,1,F,N], SN [1,nNodes,E,N,maxN]) and the same permutes
(its forward).  The er1m GSO would take 8 TB dense, so it runs on the sparse path only.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.sparse as sp
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = {
    "sourceloc": dict(N=100, deg=None, nNodes=1, maxN=100, B=100, F=1, dtype="float64", dense=True),
    "rand20k": dict(N=20_000, deg=16, nNodes=16, maxN=5, B=32, F=4, dtype="float64", dense=True),
    "er1m": dict(N=1_000_000, deg=32, nNodes=16, maxN=5, B=32, F=1, dtype="float32", dense=False),
}


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


def _graph(name, N, deg, seed=0):
    rng = np.random.default_rng(seed)
    if name == "sourceloc":          # sourceLocGNN's graph: a 5-community SBM (p = 0.8 inside, 0.2 across), normalised
        comm = np.repeat(np.arange(5), N // 5)
        W = np.triu(rng.random((N, N)) < np.where(comm[:, None] == comm[None, :], 0.8, 0.2), 1).astype(np.float64)
        W = W + W.T
        return sp.csr_matrix(W / np.abs(np.linalg.eigvalsh(W)).max())
    rows = np.repeat(np.arange(N), deg)   # deg uniformly drawn out-neighbours per node (repeats merged)
    A = sp.csr_matrix((np.ones(N * deg) / deg, (rows, rng.integers(0, N, N * deg))), shape=(N, N))
    A.sum_duplicates()
    return A


def _level_bytes(plans, C, es):
    """Bytes the chain of level plans moves for C columns: gathered rows, col + val, row offsets, stored rows."""
    total = 0
    for p in plans:
        total += p.nnz * (C * es + 4 + es) + (p.n_rows + 1) * 4 + p.n_rows * C * es
    return total


def _reference_dense(S, nNodes, maxN, B, F, dtype, reps):
    """The reference's graph arithmetic (architectures.py:3079-3094 and :3175-3192) on the same GPU."""
    N = S.shape[0]
    t0 = time.perf_counter()
    G = S.toarray()[None]
    delta = np.zeros([1, N, nNodes])
    for n in range(nNodes):
        delta[:, n, n] = 1.0
    SN = delta.copy().reshape([1, 1, N, nNodes])
    for _ in range(1, maxN):
        delta = G @ delta
        SN = np.concatenate((SN, delta.reshape([1, 1, N, nNodes])), axis=1)
    SN = torch.tensor(SN.transpose(3, 0, 2, 1)).to(device="cuda", dtype=dtype)
    torch.cuda.synchronize()
    init_s = time.perf_counter() - t0
    x = torch.randn(B, F, N, dtype=dtype, device="cuda", requires_grad=True)

    def fwd():
        z = torch.matmul(x.reshape([B, 1, 1, F, N]), SN.reshape([1, nNodes, 1, N, maxN]))
        z = z.permute(2, 3, 4, 0, 1).reshape([1, F, maxN, B * nNodes])
        return z.permute(3, 2, 0, 1).reshape([B * nNodes, maxN, F]).permute(0, 2, 1)

    dz = torch.randn(B * nNodes, F, maxN, dtype=dtype, device="cuda")
    out = dict(init_s=init_s, sn_bytes=SN.numel() * SN.element_size(), gso_dense_bytes=N * N * 8,
               forward_ms=_time(lambda: fwd(), reps), forward_backward_ms=_time(lambda: fwd().backward(dz), reps))
    return out, SN, x


def run(name, reps):
    import gnn_b200
    from gnn_b200 import aggregation
    w = WORKLOADS[name]
    dtype = getattr(torch, w["dtype"])
    es = torch.empty(0, dtype=dtype).element_size()
    N, B, F, nNodes, maxN = w["N"], w["B"], w["F"], w["nNodes"], w["maxN"]
    A = _graph(name, N, w["deg"])
    gso = gnn_b200.SparseGSO.from_scipy([A])
    dev = torch.device("cuda")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    op = aggregation.AggregationOperator(gso, np.arange(nNodes), maxN)
    fwd_plans, bwd_plans = op.levels(dev, dtype)
    torch.cuda.synchronize()
    build_s = time.perf_counter() - t0
    x = torch.randn(B, F, N, dtype=dtype, device=dev, requires_grad=True)
    z = aggregation._aggregate_cuda(op, x)
    dz = torch.randn_like(z)
    fwd_ms = _time(lambda: aggregation._aggregate_cuda(op, x), reps)
    fb_ms = _time(lambda: aggregation._aggregate_cuda(op, x).backward(dz), reps)
    C = B * F
    fb, bb = _level_bytes(fwd_plans, C, es), _level_bytes(bwd_plans, C, es)
    res = dict(workload=dict(w, nnz_S=int(A.nnz)), build_s=build_s, forward_ms=fwd_ms, forward_backward_ms=fb_ms,
               nnz_R=int(op.host(dev)[0][0][-1]),
               levels_forward=[dict(n_rows=p.n_rows, n_cols=p.n_cols, nnz=p.nnz) for p in fwd_plans],
               levels_backward=[dict(n_rows=p.n_rows, n_cols=p.n_cols, nnz=p.nnz) for p in bwd_plans],
               bytes_forward=fb, bytes_backward=bb,
               forward_tb_s=fb / (fwd_ms * 1e-3) / 1e12, forward_backward_tb_s=(fb + bb) / (fb_ms * 1e-3) / 1e12)
    if w["dense"]:
        ref, SN, xr = _reference_dense(A, nNodes, maxN, B, F, dtype, reps)
        with torch.no_grad():                          # the same x through both paths: same z up to rounding
            xr.copy_(x)
            zr = torch.matmul(xr.reshape([B, 1, 1, F, N]), SN.reshape([1, nNodes, 1, N, maxN]))
            zr = zr.permute(2, 3, 4, 0, 1).reshape([1, F, maxN, B * nNodes]).permute(3, 2, 0, 1)
            zr = zr.reshape([B * nNodes, maxN, F]).permute(0, 2, 1)
            ref["max_abs_diff_z"] = float((zr - z.detach()).abs().max())
        res["reference_dense"] = ref
        del SN, xr
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("aggregation_bench: needs a CUDA device")
    card = _card()
    out = dict(card=card, torch=torch.__version__, results={})
    for name in args.workloads.split(","):
        out["results"][name] = run(name, args.reps)
        print(name, json.dumps(out["results"][name]), flush=True)
    path = args.out
    if path is None:
        limit = card.split(",")[1].strip().split(".")[0].split(" ")[0] if "," in card else "unknown"
        path = os.path.join(ROOT, "tools", "results", "aggregation_bench_h100_%sw.json" % limit)
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", path)


if __name__ == "__main__":
    main()
