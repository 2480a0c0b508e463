"""Feasibility probe for slab-major hop chains: one C = 64 hop of the headline graph (ER N = 1M, avgDeg 32, fp32) against
eight C = 8 hops over eight distinct 32 MB slabs [N][8], the slab-major way of doing the same gather.  Alternates the two
arms with CUDA events; prints the card and its power limit.

    python tools/l2_slab_probe.py [--reps 20]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as exc:  # noqa: BLE001
        return "unknown (%s)" % exc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--N", type=int, default=1_000_000)
    args = ap.parse_args()
    from gnn_b200 import graphs, _cabi
    lib = _cabi.load()
    dev = torch.device("cuda", 0)
    N = args.N
    gso = graphs.er_gso(N, 32, seed=1, E=1)
    plan = gso.plan(dev)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    g = torch.Generator(device=dev).manual_seed(0)
    x64 = torch.randn(N, 64, device=dev, generator=g)
    y64 = torch.empty(N, 64, device=dev)
    slabs = torch.randn(8, N, 8, device=dev, generator=g)
    out_slabs = torch.empty(8, N, 8, device=dev)

    def hop(src, src_ld, dst, dst_ld, C):
        rc = lib.b200gf_hop(plan.handle, 0, 0, ctypes.c_void_p(src), src_ld, ctypes.c_void_p(dst), dst_ld, C, st)
        assert rc == 0, rc

    def wide():
        hop(x64.data_ptr(), 64, y64.data_ptr(), 64, 64)

    def slab_major():   # destination slab-major too
        for s in range(8):
            hop(slabs[s].data_ptr(), 8, out_slabs[s].data_ptr(), 8, 8)

    def slab_to_node_major():   # destination = 32-byte column s of the node-major [N, 64] matrix
        for s in range(8):
            hop(slabs[s].data_ptr(), 8, y64.data_ptr() + 32 * s, 64, 8)

    def one_slab():
        hop(slabs[0].data_ptr(), 8, out_slabs[0].data_ptr(), 8, 8)

    arms = {"wide_C64": wide, "8x_slab_C8": slab_major, "8x_slab_C8_dst_node_major": slab_to_node_major,
            "1x_slab_C8": one_slab}
    for f in arms.values():
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(args.reps):
        for k, f in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1))
    # agreement: the slab arm's results equal the wide hop of the concatenated slabs
    x_cat = slabs.permute(1, 0, 2).reshape(N, 64).contiguous()
    hop(x_cat.data_ptr(), 64, y64.data_ptr(), 64, 64)
    slab_major()
    torch.cuda.synchronize()
    diff = float((out_slabs.permute(1, 0, 2).reshape(N, 64) - y64).abs().max() / y64.abs().max())
    res = {"card": card(), "N": N, "nnz": gso.nnz(), "reps": args.reps, "max_rel_diff": diff}
    for k, v in times.items():
        a = np.array(v)
        res[k] = {"median_ms": float(np.median(a)), "min_ms": float(a.min()), "max_ms": float(a.max())}
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
