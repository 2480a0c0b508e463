"""Times the node-variant graph filter (gnn_b200.NodeVariantGF, csrc/nv/nv.cu) on the GPU with CUDA events.

    python tools/nv_bench.py [--iters 20] [--quick]

For each shape: forward, forward + backward, and each new kernel (torch.profiler, a separate pass), then GraphFilter at
the same shape.  The contraction's gather-model bytes are T*N*B*G*s (the T shifted signals) + N*B*F*s (y) + N*T*G*F*s
(each node reads its tap block), and the achieved bandwidth is reported against the H100 SXM data sheet's 3.35 TB/s.
Prints the card, its power limit and SM clock first, then one JSON line per shape.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import scipy.sparse as sp
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import gnn_b200  # noqa: E402

HBM_BYTES_PER_S = 3.35e12

SHAPES = [  # (name, N, degree, B, G, F, K, M)
    ("N100k-deg16-B32-G32-F32-K3-M=N", 100_000, 16, 32, 32, 32, 3, 100_000),
    ("N100k-deg16-B32-G32-F32-K3-M1000", 100_000, 16, 32, 32, 32, 3, 1000),
    ("N1M-deg32-B1-G64-F64-K5-M1000", 1_000_000, 32, 1, 64, 64, 5, 1000),
]


def er_gso(N, deg, seed):
    rng = np.random.default_rng(seed)
    nnz = N * deg
    m = sp.csr_matrix((rng.standard_normal(nnz).astype(np.float32), (rng.integers(0, N, nnz), rng.integers(0, N, nnz))),
                      shape=(N, N))
    m.sum_duplicates()
    m = sp.csr_matrix(sp.diags(1.0 / np.maximum(np.abs(m).sum(axis=1).A.ravel(), 1.0)) @ m, dtype=np.float32)
    m.sort_indices()
    return gnn_b200.SparseGSO.from_scipy([m], dtype=torch.float32)


def timed(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def kernel_ms(fn, iters):
    """Mean device time per call of every nv_* kernel over `iters` calls of fn."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if "nv_" in e.key and "kernel" in e.key:
            name = e.key.replace("void ", "").replace("(anonymous namespace)::", "").split("(")[0]
            t = getattr(e, "device_time_total", None)
            if t is None:
                t = e.cuda_time_total
            out[name] = out.get(name, 0.0) + t / 1000.0 / iters
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--quick", action="store_true", help="first shape only")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("nv_bench: no CUDA device (this tool measures on the GPU only)")
    gnn_b200._cabi.load()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print("# card:", q.stdout.strip() or "nvidia-smi unavailable")
    for (name, N, deg, B, G, F, K, M) in SHAPES[:1] if args.quick else SHAPES:
        S = er_gso(N, deg, 7)
        torch.manual_seed(0)
        nv = gnn_b200.NodeVariantGF(G, F, K, M).cuda()
        nv.addGSO(S)
        gf = gnn_b200.GraphFilter(G, F, K).cuda()
        gf.addGSO(S)
        x = torch.randn(B, G, N, device="cuda")
        xg = x.clone().requires_grad_(True)
        dy = torch.randn(B, F, N, device="cuda")

        def nv_fwd():
            with torch.no_grad():
                nv(x)

        def nv_fb():
            nv(xg).backward(dy)

        def gf_fwd():
            with torch.no_grad():
                gf(x)

        def gf_fb():
            gf(xg).backward(dy)

        res = dict(shape=name, N=N, deg=deg, B=B, G=G, F=F, K=K, M=M)
        res["nv_forward_ms"] = timed(nv_fwd, args.iters)
        res["nv_fwd_bwd_ms"] = timed(nv_fb, args.iters)
        res["graphfilter_forward_ms"] = timed(gf_fwd, args.iters)
        res["graphfilter_fwd_bwd_ms"] = timed(gf_fb, args.iters)
        kf = kernel_ms(nv_fwd, 5)
        kb = kernel_ms(nv_fb, 5)
        res["kernels_forward_ms"] = kf
        res["kernels_fwd_bwd_ms"] = kb
        T, s = 1 + (K - 1), 4
        gather = T * N * B * G * s + N * B * F * s + N * T * G * F * s
        tc = sum(v for k, v in kf.items() if k.startswith("nv_contract_kernel"))
        res["contract_gather_bytes"] = gather
        if tc > 0:
            res["contract_ms"] = tc
            res["contract_TBps"] = gather / (tc * 1e-3) / 1e12
            res["contract_share_of_3.35TBps"] = gather / (tc * 1e-3) / HBM_BYTES_PER_S
        print(json.dumps(res))
        sys.stdout.flush()
        del nv, gf, S, x, xg, dy
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
