"""L2-sized column chunks of the hop: LSIGF forward, and forward + backward, of the bench workloads with the plan's L2
size at 0 (every hop takes the chunk width of its row width) against the device's L2 size (the library's choice), and
optionally against L2 sizes that force a given chunk width.  Arms alternate; prints the card and power limit, the
median and spread of ms per step and per hop, and the largest relative difference of every output against arm "off".

    python tools/l2_chunk_bench.py [--workloads er1m,cfg2,cfg4,er2m,sbm1m] [--f64 er1m] [--rounds 5] [--force]
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

import bench  # noqa: E402  (workload table and graph builders)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as exc:  # noqa: BLE001
        return "unknown (%s)" % exc


def forced_l2(N, L):
    """An L2 size that holds a chunk of L lanes x 32 bytes of N rows but not one of 2L lanes."""
    return N * L * 32


def run(name, w, dtype, rounds, force, lib):
    import gnn_b200
    dev = torch.device("cuda", 0)
    tdt = torch.float64 if dtype == "f64" else torch.float32
    es = 8 if dtype == "f64" else 4
    E, K, G, F, B, N = w["E"], w["K"], w["G"], w["F"], w["B"], w["N"]
    gso = bench.make_gso(w).astype(tdt)
    h_cpu, b_cpu = bench.seeded_taps(w, tdt)
    h, b = h_cpu.to(dev), b_cpu.to(dev)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, G, N, generator=g).to(dev, tdt)
    dy = torch.randn(B, F, N, generator=g).to(dev, tdt)
    plan = gso.plan(dev)
    dev_l2 = int(lib.b200gf_plan_info(plan.handle, 7))
    arms = {"off": 0, "default": dev_l2}
    if force:
        for L in (4, 8, 16):
            if B * G * es > L * 32:
                arms["L%d" % L] = forced_l2(N, L)
    xg, hg, bg = (t.clone().requires_grad_(True) for t in (x, h, b))

    def fwd():
        return gnn_b200.LSIGF(h, gso, x, b)

    def fwd_bwd():
        xg.grad = hg.grad = bg.grad = None
        gnn_b200.LSIGF(hg, gso, xg, bg).backward(dy)

    def timed(fn, steps):
        fn()
        torch.cuda.synchronize()
        hops = E * (K - 1) * steps * 2
        lib.b200gf_profile_hops(plan.handle, hops)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        buf = (ctypes.c_float * hops)()
        got = lib.b200gf_profile_read(plan.handle, buf, hops)
        lib.b200gf_profile_hops(plan.handle, 0)
        return e0.elapsed_time(e1) / steps, float(np.mean([buf[i] for i in range(got)])) if got > 0 else None

    res = {k: {"fwd": [], "fwd_hop": [], "fb": [], "fb_hop": []} for k in arms}
    outs = {}
    with torch.no_grad():
        for k, v in arms.items():   # warm-up + outputs
            lib.b200gf_plan_set_l2_bytes(plan.handle, v)
            outs[k] = [fwd().detach().clone()]
    for k, v in arms.items():
        lib.b200gf_plan_set_l2_bytes(plan.handle, v)
        fwd_bwd()
        torch.cuda.synchronize()
        outs[k] += [xg.grad.clone(), hg.grad.clone(), bg.grad.clone()]
    for _ in range(rounds):
        for k, v in arms.items():
            lib.b200gf_plan_set_l2_bytes(plan.handle, v)
            with torch.no_grad():
                ms, hop = timed(fwd, 3)
            res[k]["fwd"].append(ms)
            res[k]["fwd_hop"].append(hop)
            ms, hop = timed(fwd_bwd, 2)
            res[k]["fb"].append(ms)
            res[k]["fb_hop"].append(hop)
    out = {"workload": bench.describe(w, dtype), "device_l2_bytes": dev_l2, "arms": {}}
    for k in arms:
        r = {"l2_bytes": arms[k]}
        for m, v in res[k].items():
            a = np.array([t for t in v if t is not None])
            if len(a):
                r[m] = {"median_ms": float(np.median(a)), "min_ms": float(a.min()), "max_ms": float(a.max())}
        r["max_rel_vs_off"] = {n: float((o.double() - ref.double()).abs().max() / ref.double().abs().max())
                               for n, o, ref in zip(("y", "dx", "dh", "db"), outs[k], outs["off"])}
        out["arms"][k] = r
    lib.b200gf_plan_set_l2_bytes(plan.handle, dev_l2)
    del outs, xg, hg, bg
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="er1m,cfg2,cfg4,er2m,sbm1m")
    ap.add_argument("--f64", default="er1m", help="workloads also run in fp64")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--force", action="store_true", help="also time L2 sizes that force 4, 8 and 16-lane chunks")
    ap.add_argument("--out", help="also write the report as JSON here")
    args = ap.parse_args()
    from gnn_b200 import _cabi
    lib = _cabi.load()
    report = {"card": card(), "runs": []}
    jobs = [(n, "f32") for n in args.workloads.split(",") if n] + [(n, "f64") for n in args.f64.split(",") if n]
    for name, dtype in jobs:
        r = run(name, bench.WORKLOADS[name], dtype, args.rounds, args.force, lib)
        report["runs"].append(r)
        print(json.dumps(r), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(report, f, indent=1)
    print("card:", report["card"])
    print("%-46s %-8s %10s %7s %10s %7s %10s %9s" % ("workload", "arm", "fwd ms", "spread", "fwd+bwd", "spread",
                                                   "hop ms", "max rel"))
    for r in report["runs"]:
        for k, a in r["arms"].items():
            sp = lambda m: (a[m]["max_ms"] - a[m]["min_ms"]) if m in a else float("nan")  # noqa: E731
            print("%-46s %-8s %10.3f %7.3f %10.3f %7.3f %10.3f %9.2e" % (
                r["workload"][:46], k, a["fwd"]["median_ms"], sp("fwd"), a["fb"]["median_ms"], sp("fb"),
                a["fwd_hop"]["median_ms"], max(a["max_rel_vs_off"].values())))


if __name__ == "__main__":
    main()
