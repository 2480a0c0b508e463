"""Timing of the edge-gated recurrent layer (gnn_b200.EdgeGatedHiddenState, csrc/egate.cu) on the GPU.

    python tools/egate_bench.py [--reps 20] [--out egate_bench.json]

Two shapes: the epidemic example's layer (F = 1, H = 12, K = 5, B = 100, T = 8; examples/epidemicGRNN.py of the
reference) on a synthetic graph of N = 2 000 nodes, average degree 16, and N = 100 000, average degree 16, B = 16, T = 8.
Per shape: layer forward (inference) and forward + backward from CUDA events, and per-kernel times of the attention
(forward / backward) and the gated hop (forward / backward) at the two (samples, C) of the layer: the input filter
(B*T samples, C = F) and the hidden filter (B samples, C = H), next to the ungated b200gf_hop at the same batch and C.
Achieved GB/s use the gather model below (every gathered element counted once per use, no cache reuse), s = 4 bytes:
  attention fwd   N*Bs*s + nnz_m*(4 + 8) + nnz_m*Bs*(2 gathers of s + 2 writes + 1 read)*s
  attention bwd   nnz_m*Bs*s*(alpha, dalpha twice, 1 gather of s, dlogit write + read) + 2*N*Bs*s + nnz_m*8
  gated hop fwd   nnz*(4 + s + 4) + nnz*Bs*(C + 1)*s + N*Bs*C*s           (index, value, position; gate; src; dst)
  gated hop bwd   the same hop over S + the SDDMM: nnz_m*(4 + s) + nnz_m*Bs*(2*C + 1)*s
  ungated hop     nnz*(4 + s) + nnz*Bs*C*s + N*Bs*C*s
Prints the card name, power limit and clocks read in the same run, and one JSON object.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import gnn_b200  # noqa: E402
from gnn_b200 import _cabi  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return dict(zip(q.split(","), [v.strip() for v in out[0].split(",")])) if out else {}
    except Exception as e:                                   # the numbers below still stand; say what is missing
        return {"error": repr(e)}


def graph(N, deg, seed):
    import scipy.sparse as sp
    rng = np.random.default_rng(seed)
    nnz = N * deg
    m = sp.csr_matrix((rng.standard_normal(nnz), (rng.integers(0, N, nnz), rng.integers(0, N, nnz))), shape=(N, N))
    m.sum_duplicates()
    m = sp.csr_matrix(sp.diags(1.0 / np.maximum(np.abs(m).sum(axis=1).A.ravel(), 1.0)) @ m)
    m.sort_indices()
    return gnn_b200.SparseGSO([(m.indptr, m.indices, m.data.astype(np.float32))], N)


def timed(fn, reps, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), float(np.min(ts))


def shape_run(name, N, deg, B, T, F, H, K, reps):
    dev = torch.device("cuda")
    S = graph(N, deg, 5)
    torch.manual_seed(0)
    layer = gnn_b200.EdgeGatedHiddenState(F, H, K)
    layer.addGSO(S)
    layer = layer.to(dev)
    rng = np.random.default_rng(1)
    x = torch.tensor(rng.standard_normal((B, T, F, N)), dtype=torch.float32, device=dev)
    z0 = torch.tensor(rng.standard_normal((B, H, N)), dtype=torch.float32, device=dev)
    dz = torch.tensor(rng.standard_normal((B, T, H, N)), dtype=torch.float32, device=dev)
    res = {"shape": name, "N": N, "avg_degree": deg, "B": B, "T": T, "F": F, "H": H, "K": K}

    def fwd():
        with torch.no_grad():
            layer(x, z0)

    xg = x.clone().requires_grad_(True)

    def fwd_bwd():
        z, _ = layer(xg, z0)
        z.backward(dz)
    res["layer_forward_ms"], res["layer_forward_ms_min"] = timed(fwd, reps)
    res["layer_fwd_bwd_ms"], res["layer_fwd_bwd_ms_min"] = timed(fwd_bwd, reps)

    pat = layer.pattern.on(dev)
    nnz_s, nnz_m, s = int(pat.s_col.numel()), pat.nnz, 4
    lib = _cabi.load()
    plan = gnn_b200.plan_for(S)
    st = lambda: torch.cuda.current_stream().cuda_stream                     # noqa: E731
    kernels = []
    # attention at B*T samples
    Bs = B * T
    sv = torch.randn(N, Bs, device=dev)
    mixer = torch.tensor([0.5, -0.7], device=dev)
    alpha = torch.empty(nnz_m, Bs, device=dev)
    da, dl = torch.randn(nnz_m, Bs, device=dev), torch.empty(nnz_m, Bs, device=dev)
    d1, d2 = torch.empty(N, Bs, device=dev), torch.empty(N, Bs, device=dev)
    att_f = lambda: _cabi.check(lib.b200gf_egate_attention_forward(  # noqa: E731
        _cabi.F32, N, nnz_m, Bs, pat.m_rowptr.data_ptr(), pat.m_col.data_ptr(), sv.data_ptr(), mixer.data_ptr(),
        alpha.data_ptr(), st()))
    att_b = lambda: _cabi.check(lib.b200gf_egate_attention_backward(  # noqa: E731
        _cabi.F32, N, nnz_m, Bs, pat.m_rowptr.data_ptr(), pat.m_col.data_ptr(), pat.mT_rowptr.data_ptr(),
        pat.mT_perm.data_ptr(), sv.data_ptr(), mixer.data_ptr(), alpha.data_ptr(), da.data_ptr(), dl.data_ptr(),
        d1.data_ptr(), d2.data_ptr(), st()))
    kernels.append(("attention_forward", Bs, 1, att_f, N * Bs * s + nnz_m * 12 + 5 * nnz_m * Bs * s))
    kernels.append(("attention_backward", Bs, 1, att_b, 6 * nnz_m * Bs * s + 2 * N * Bs * s + nnz_m * 8))
    t_val, s_val, m_sval = pat.values(torch.float32)
    for label, Bs, C in (("input", B * T, F), ("hidden", B, H)):
        gate = torch.rand(nnz_m, Bs, device=dev)
        src = torch.randn(N, Bs * C, device=dev)
        dst = torch.empty(N, Bs * C, device=dev)
        dg = torch.empty(nnz_m, Bs, device=dev)
        hop_f = lambda Bs=Bs, C=C, gate=gate, src=src, dst=dst: _cabi.check(lib.b200gf_gated_hop_forward(  # noqa: E731
            _cabi.F32, N, Bs, C, pat.t_rowptr.data_ptr(), pat.t_col.data_ptr(), t_val.data_ptr(), pat.t_pos.data_ptr(),
            gate.data_ptr(), 1, Bs, src.data_ptr(), Bs * C, dst.data_ptr(), Bs * C, st()))
        hop_b = lambda Bs=Bs, C=C, gate=gate, src=src, dst=dst, dg=dg: _cabi.check(lib.b200gf_gated_hop_backward(  # noqa
            _cabi.F32, N, Bs, C, pat.s_rowptr.data_ptr(), pat.s_col.data_ptr(), s_val.data_ptr(), pat.s_pos.data_ptr(),
            pat.m_rowptr.data_ptr(), pat.m_col.data_ptr(), m_sval.data_ptr(), gate.data_ptr(), 1, Bs, src.data_ptr(),
            Bs * C, src.data_ptr(), Bs * C, dst.data_ptr(), Bs * C, dg.data_ptr(), 1, Bs, st()))
        hop_u = lambda Bs=Bs, C=C, src=src, dst=dst: _cabi.check(lib.b200gf_hop(  # noqa: E731
            plan.handle, 0, _cabi.HOP_FWD, src.data_ptr(), Bs * C, dst.data_ptr(), Bs * C, Bs * C, st()))
        hop_bytes = nnz_s * (4 + s + 4) + nnz_s * Bs * (C + 1) * s + N * Bs * C * s
        kernels.append(("gated_hop_forward_" + label, Bs, C, hop_f, hop_bytes))
        kernels.append(("gated_hop_backward_" + label, Bs, C, hop_b,
                        hop_bytes + nnz_m * (4 + s) + nnz_m * Bs * (2 * C + 1) * s))
        kernels.append(("ungated_hop_" + label, Bs, C, hop_u, nnz_s * (4 + s) + nnz_s * Bs * C * s + N * Bs * C * s))
    res["nnz_S"], res["nnz_mask"] = nnz_s, nnz_m
    res["kernels"] = []
    for kname, Bs, C, fn, nbytes in kernels:
        med, mn = timed(fn, max(reps, 20))
        res["kernels"].append({"kernel": kname, "samples": Bs, "C": C, "ms": med, "ms_min": mn,
                               "gather_model_bytes": int(nbytes), "GBps": nbytes / (med * 1e-3) / 1e9})
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("egate_bench: needs a CUDA device (nothing is measured without one)")
    out = {"card": card(), "runs": [shape_run("epidemic", 2000, 16, 100, 8, 1, 12, 5, args.reps),
                                    shape_run("n100k", 100_000, 16, 16, 8, 1, 12, 5, args.reps)]}
    out["card_after"] = card()
    for r in out["runs"]:
        print("%-9s N=%-7d B=%-3d T=%d  layer fwd %.3f ms  fwd+bwd %.3f ms" % (
            r["shape"], r["N"], r["B"], r["T"], r["layer_forward_ms"], r["layer_fwd_bwd_ms"]))
        for k in r["kernels"]:
            print("    %-28s samples=%-4d C=%-3d %8.4f ms  %8.1f GB/s" % (k["kernel"], k["samples"], k["C"], k["ms"],
                                                                         k["GBps"]))
    print("card:", out["card"])
    print(json.dumps(out))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
