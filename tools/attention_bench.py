#!/usr/bin/env python
"""Graph attention layer timings (GraphAttentional, GraphFilterAttentional, EdgeVariantAttentional) with CUDA events.

Prints the card, its power limit and clocks, then at two shapes, fp32, for each layer: forward and forward + backward
ms; per-kernel device time of one forward + backward (torch.profiler, a run of its own); and the gated hop's
gather-model bytes (DESIGN §4b: nnz (4 + s + 4) + nnz B_s (C + 1) s + N B_s C s) over its mean kernel time.

  big:   N = 100 000, degree 16, B = 16, G = F = 32, P = 4, E = 1, K = 3
  small: N = 2 000 (same degree and widths), where the dense formulation still fits.  Beside it, the dense formulation
         of the same layers (a B x P x E x N x N masked softmax and dense N x N hops, the algorithm of the reference's
         learnAttentionGSO / graphAttention*, restated in torch here because the reference itself is not installed
         with the package), labelled as such.

    python tools/attention_bench.py [--steps 10] [--warmup 3] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import scipy.sparse as sp
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def er(N, deg, seed):
    rng = np.random.default_rng(seed)
    nnz = N * deg
    A = sp.csr_matrix((rng.uniform(0.1, 1.0, nnz), (rng.integers(0, N, nnz), rng.integers(0, N, nnz))), shape=(N, N))
    A.sum_duplicates()
    A = sp.csr_matrix(A - sp.diags(A.diagonal()))
    A.eliminate_zeros()
    return sp.csr_matrix(sp.diags(1.0 / np.maximum(A.sum(axis=1).A.ravel(), 1e-9)) @ A)


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


def kernel_times(fn):
    """{kernel name: (calls, total ms)} of one call of fn."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if e.device_type == torch.autograd.DeviceType.CUDA and e.self_device_time_total > 0:
            out[e.key[:90]] = (int(e.count), e.self_device_time_total / 1e3)
    return dict(sorted(out.items(), key=lambda kv: -kv[1][1])[:12])


def dense_layer(kind, layer, S, x):
    """The dense formulation: attention as B x P x E x N x N masked softmax, dense hops (the reference's algorithm)."""
    E, N, _ = S.shape
    mask = (S + torch.eye(N, device=S.device)).abs().sum(0) > 1e-9

    def att(a, W):                                  # a [P, E, 2F], W [P, E, F, G] -> [B, P, E, N, N], Wx
        F = W.shape[2]
        Wx = torch.einsum("pefg,bgn->bpefn", W, x)
        s1 = torch.einsum("bpefn,pef->bpen", Wx, a[..., :F])
        s2 = torch.einsum("bpefn,pef->bpen", Wx, a[..., F:])
        e = nn.functional.leaky_relu(s1.unsqueeze(-2) + s2.unsqueeze(-1), 0.2)
        return torch.softmax(e.masked_fill(~mask, -float("inf")), -1).nan_to_num(0.0), Wx
    if kind == "GraphAttentional":
        al, Wx = att(layer.mixer, layer.weight)
        return torch.matmul(Wx, S * al).sum(2)
    if kind == "GraphFilterAttentional":
        al, _ = att(layer.mixer, layer.weight)
        P, E, F, G = layer.weight.shape
        K = layer.filterWeight.shape[1]
        h = layer.filterWeight.reshape(1, 1, E, K, 1) * layer.weight.permute(0, 3, 1, 2).reshape(P, F, E, 1, G)
        u = x.reshape(x.shape[0], 1, 1, G, N)
        zs = [u.expand(-1, P, E, G, N)]
        for _ in range(1, K):
            u = torch.matmul(u, al)
            zs.append(u)
        z = torch.stack(zs, 3)
        return torch.einsum("bpekgn,pfekg->bpfn", z, h) + layer.bias
    P, K, E, F, G = layer.weight.shape
    u = torch.einsum("pefg,bgn->bpefn", layer.weight[:, 0], x)
    y = 0
    for k in range(K):
        al, _ = att(layer.mixer[:, k], layer.weight[:, k])
        u = torch.matmul(u, S * al)
        y = y + u
    return y.sum(2) + layer.bias


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import gnn_b200
    if not torch.cuda.is_available():
        raise SystemExit("attention_bench: needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("card (name, power limit, SM clock, max SM clock): %s" % q)
    report = {"card": q}
    deg, B, G, F, P, E, K = 16, 16, 32, 32, 4, 1, 3
    for shape, N in (("big", 100_000), ("small", 2_000)):
        m = er(N, deg, 0)
        S = gnn_b200.SparseGSO.from_scipy([m], dtype=torch.float32)
        pat = gnn_b200.attention.pattern_for(S, "cuda")
        rng = np.random.default_rng(1)
        x = torch.tensor(rng.standard_normal((B, G, N)), dtype=torch.float32, device="cuda")
        rows = {"shape": dict(N=N, deg=deg, B=B, G=G, F=F, P=P, E=E, K=K, nnz_S=int(m.nnz), nnz_mask=pat.nnz)}
        torch.manual_seed(0)
        layers = {"GraphAttentional": gnn_b200.GraphAttentional(G, F, P, E, nn.functional.relu, False),
                  "GraphFilterAttentional": gnn_b200.GraphFilterAttentional(G, F, K, P, E, True,
                                                                            nn.functional.relu, False),
                  "EdgeVariantAttentional": gnn_b200.EdgeVariantAttentional(G, F, K, P, E, True,
                                                                            nn.functional.relu, False)}
        Sd = torch.tensor(m.toarray(), dtype=torch.float32, device="cuda").reshape(1, N, N) if shape == "small" else None
        for name, layer in layers.items():
            layer = layer.cuda()
            layer.addGSO(S)
            xg = x.clone().requires_grad_(True)

            def fwd():
                with torch.no_grad():
                    layer(x)

            def fb():
                layer(xg).sum().backward()
            row = dict(forward_ms=timed(fwd, a.steps, a.warmup), forward_backward_ms=timed(fb, a.steps, a.warmup))
            kt = kernel_times(fb)
            row["kernels_fwd_bwd (calls, ms)"] = kt
            hop = [v for k, v in kt.items() if "egate_hop_kernel" in k]
            if hop:
                calls, ms = hop[0]
                s = 4
                C = G if name == "GraphFilterAttentional" else F
                Bs = B * P * (E if name == "GraphFilterAttentional" else 1)
                nnz = pat.nnz if name == "GraphFilterAttentional" else int(m.nnz)   # the hop runs over the mask / S^T
                model = nnz * (4 + s + 4) + nnz * Bs * (C + 1) * s + N * Bs * C * s
                row["gated_hop_model_bytes"] = model
                row["gated_hop_mean_ms (forward and backward launches)"] = ms / calls
                row["gated_hop_TBps_model"] = model / (ms / calls * 1e-3) / 1e12
            if Sd is not None:
                def dfwd():
                    with torch.no_grad():
                        dense_layer(name, layer, Sd, x)

                def dfb():
                    dense_layer(name, layer, Sd, xg).sum().backward()
                row["dense formulation (reference algorithm, restated in torch): forward_ms"] = timed(dfwd, 3, 1)
                row["dense formulation (reference algorithm, restated in torch): forward_backward_ms"] = timed(dfb, 3, 1)
            rows[name] = row
            torch.cuda.empty_cache()
        report[shape] = rows
        print(json.dumps({shape: rows}, indent=1), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "attention_bench.json"), "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
