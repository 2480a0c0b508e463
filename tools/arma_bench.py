#!/usr/bin/env python
"""ARMA filter (gnn_b200.jARMA) timings on an Erdos-Renyi graph, with CUDA events.

Prints the card and its power limit, then for a zero-diagonal GSO (the constant-diagonal path: an LSIGF over S~^T with
tMax + 2 taps) and a combinatorial Laplacian L = D - A (a varying diagonal: the general path, csrc/arma/arma.cu):
forward and forward + backward ms; for the general path the wide hop's time, its gather-model bytes
nnz (4 + s) + (N + 1) 8 + nnz C s + N C s (C = 2 B F P G) and the rate they imply, and the share of the step spent in
arma.cu's element-wise kernels (torch.profiler, a run of its own); GraphFilter at the same G, F and K as a yardstick;
and the bytes of the reference's dense Sbar, SbarInv and SbarInvStilde.

    python tools/arma_bench.py [--n 100000] [--deg 16] [--b 4] [--g 8] [--f 8] [--p 2] [--k 3] [--tmax 5] [--out DIR]
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


def er(N, deg, seed):
    rng = np.random.default_rng(seed)
    nnz = N * deg
    A = sp.csr_matrix((np.ones(nnz), (rng.integers(0, N, nnz), rng.integers(0, N, nnz))), shape=(N, N))
    A = sp.csr_matrix(A - sp.diags(A.diagonal()))
    A.data[:] = 1.0
    A.eliminate_zeros()
    return A


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(steps):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000)
    ap.add_argument("--deg", type=int, default=16)
    ap.add_argument("--b", type=int, default=4)
    ap.add_argument("--g", type=int, default=8)
    ap.add_argument("--f", type=int, default=8)
    ap.add_argument("--p", type=int, default=2)
    ap.add_argument("--k", type=int, default=3)
    ap.add_argument("--tmax", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import gnn_b200
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("card: %s" % q)
    N, B, G, F, P, K, tMax = a.n, a.b, a.g, a.f, a.p, a.k, a.tmax
    s = 4
    A = er(N, a.deg, 0)
    deg = np.asarray(A.sum(axis=1)).ravel()
    dinv = 1.0 / np.sqrt(np.maximum(deg, 1.0))
    gsos = {"zero-diagonal (normalised adjacency, constant path)": sp.csr_matrix(sp.diags(dinv) @ A @ sp.diags(dinv)),
            "Laplacian D - A (general path)": sp.csr_matrix((sp.diags(deg) - A) / deg.max())}
    rng = np.random.default_rng(1)
    stdv = 1. / np.sqrt(G * P)
    mk = lambda shape, lo, hi: torch.tensor(rng.uniform(lo, hi, shape), dtype=torch.float32, device="cuda",  # noqa: E731
                                            requires_grad=True)
    psi, varphi = mk((F, 1, P, G), 1 + 1 / stdv, 1 + 2 / stdv), mk((F, 1, P, G), -stdv, stdv)
    phi, bias = mk((F, 1, K, G), -stdv, stdv), mk((F, 1), -stdv, stdv)
    x = torch.tensor(rng.standard_normal((B, G, N)), dtype=torch.float32, device="cuda", requires_grad=True)
    du = torch.ones((B, F, N), dtype=torch.float32, device="cuda")
    report = {"card": q, "shape": dict(N=N, deg=a.deg, B=B, G=G, F=F, P=P, K=K, tMax=tMax, dtype="fp32")}
    for name, m in gsos.items():
        S = gnn_b200.SparseGSO.from_scipy([m], dtype=torch.float32)
        op = gnn_b200.arma.arma_operator(S)             # the operator (and plans) jARMA itself uses

        def fwd():
            with torch.no_grad():
                gnn_b200.jARMA(psi, varphi, phi, S, x, bias, tMax=tMax)

        def fwd_bwd():
            gnn_b200.jARMA(psi, varphi, phi, S, x, bias, tMax=tMax).backward(du)

        row = dict(constant_path=bool(op.constant[0]), nnz=int(m.nnz),
                   forward_ms=timed(fwd, a.steps, a.warmup), forward_backward_ms=timed(fwd_bwd, a.steps, a.warmup))
        if not op.constant[0]:
            plan = op.plan([0], "cuda")
            lib = gnn_b200._cabi.load()
            nnz = plan.nnz
            C = 2 * B * F * P * G
            row["wide_hop_model_bytes"] = nnz * (4 + s) + (N + 1) * 8 + nnz * C * s + N * C * s
            lib.b200gf_profile_hops(plan.handle, 1 + tMax)
            fwd()
            buf = (ctypes.c_float * (1 + tMax))()
            n = lib.b200gf_profile_read(plan.handle, buf, 1 + tMax)
            lib.b200gf_profile_hops(plan.handle, 0)
            wide = sorted(list(buf)[1:n])
            row["wide_hop_ms_median"] = float(wide[len(wide) // 2]) if wide else None
            if wide:
                row["wide_hop_TBps"] = row["wide_hop_model_bytes"] / (row["wide_hop_ms_median"] * 1e-3) / 1e12
            from torch.profiler import ProfilerActivity, profile
            fwd_bwd()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(3):
                    fwd_bwd()
                torch.cuda.synchronize()
            tot = elem = 0.0
            for e in prof.key_averages():
                if e.device_type == torch.autograd.DeviceType.CUDA:
                    t = e.self_device_time_total
                    tot += t
                    if "arma_" in e.key:
                        elem += t
            row["elementwise_share_of_fwd_bwd"] = elem / tot if tot else None
        report[name] = row
    gf = gnn_b200.GraphFilter(G, F, K, 1).cuda()
    gf.addGSO(gnn_b200.SparseGSO.from_scipy([gsos["zero-diagonal (normalised adjacency, constant path)"]],
                                            dtype=torch.float32))

    def gf_fwd():
        with torch.no_grad():
            gf(x)

    def gf_fb():
        gf(x).backward(du)
    report["GraphFilter (same G, F, K)"] = dict(forward_ms=timed(gf_fwd, a.steps, a.warmup),
                                                forward_backward_ms=timed(gf_fb, a.steps, a.warmup))
    report["reference dense bytes, each of Sbar / SbarInv / SbarInvStilde"] = F * 1 * P * G * N * N * s
    print(json.dumps(report, indent=1))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "arma_bench.json"), "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
