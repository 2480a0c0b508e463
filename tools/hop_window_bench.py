"""Windowed hop (b200gf_plan_set_hop_windows): source windows off against on, alternated, with CUDA events.

Part 1, hops: one forward hop of the workload's graph (C = B * G columns) with the plan's window copy dropped (today's
hop) against window copies of R rows, for every R of --rows and every library given with --libs (builds of the library
whose windowed hop has another geometry or L2 policy, see --variants).  Part 2, layers: LSIGF forward and forward +
backward of the --fwd workloads on two plans of one graph, one without windows and one with the default window rule,
and every output's largest relative difference between them.  Prints the card, power limit and clocks, medians and
spreads (min, max) in ms.

    python tools/hop_window_bench.py [--hops er1m] [--f64-hops er1m] [--rows 125000,200000,250000,333000]
                                     [--libs a.so,b.so] [--fwd er1m,er2m] [--f64 er1m] [--rounds 5] [--out r.json]
    python tools/hop_window_bench.py --variants DIR   # builds the GS x U x HINT variant libraries into DIR and exits
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

import bench  # noqa: E402  (workload table and graph builders)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as exc:  # noqa: BLE001
        return "unknown (%s)" % exc


VARIANTS = [(gs, u, hint) for gs in (4, 8) for u in (2, 4) for hint in (1, 3)]


def build_variants(outdir):
    """Relinks the library once per windowed-hop geometry (B200GF_HOP_WIN_GS / _U / _HINT); only spmm.cu differs."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("b200gf_build", os.path.join(ROOT, "graph-neural-networks_b200", "build.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    b.build_library()
    objdir = os.path.join(b.HERE, "build")
    others = [os.path.join(objdir, os.path.basename(s) + ".o") for s in b.SOURCES if s != "spmm.cu"]
    os.makedirs(outdir, exist_ok=True)
    for gs, u, hint in VARIANTS:
        tag = "gs%d_u%d_h%d" % (gs, u, hint)
        o = os.path.join(outdir, "spmm_%s.o" % tag)
        subprocess.check_call([b._nvcc()] + b.NVCC_FLAGS + ["-DB200GF_HOP_WIN_GS=%d" % gs, "-DB200GF_HOP_WIN_U=%d" % u,
                                                            "-DB200GF_HOP_WIN_HINT=%d" % hint, "-c",
                                                            os.path.join(b.CSRC, "spmm.cu"), "-o", o])
        subprocess.check_call([b._nvcc(), "-shared", "-o", os.path.join(outdir, "libb200gf_%s.so" % tag), o] + others +
                              ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart"])
        print(tag, flush=True)


def load_lib(path):
    from gnn_b200 import _cabi
    lib = ctypes.CDLL(path)
    for name, (res, args) in _cabi._SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    return lib


def check(lib, rc):
    if rc != 0:
        raise RuntimeError(lib.b200gf_strerror(int(rc)).decode())


def stats(v):
    a = np.array(v)
    return {"median_ms": float(np.median(a)), "min_ms": float(a.min()), "max_ms": float(a.max())}


def hop_sweep(name, dtype, libs, rows, rounds, reps=10):
    import torch
    from gnn_b200 import _cabi
    w = bench.WORKLOADS[name]
    tdt = torch.float64 if dtype == "f64" else torch.float32
    N, C = w["N"], w["B"] * w["G"]
    gso = bench.make_gso(w).astype(tdt)
    r, c, v = gso.csr[0]
    r = np.ascontiguousarray(r, np.int64); c = np.ascontiguousarray(c, np.int32)
    v = np.ascontiguousarray(v, np.float64 if dtype == "f64" else np.float32)
    dev = torch.device("cuda", 0)
    g = torch.Generator().manual_seed(3)
    src = torch.randn(N, C, generator=g).to(dev, tdt)
    dst = torch.empty(N, C, device=dev, dtype=tdt)
    ref = torch.empty_like(dst)
    st = torch.cuda.current_stream().cuda_stream
    out = {"workload": bench.describe(w, dtype), "C": C, "libs": {}}
    for path in libs:
        lib = load_lib(path)
        plans = []
        for _ in range(2):
            h = ctypes.c_void_p()
            check(lib, lib.b200gf_plan_create(ctypes.byref(h), 0, N, 1, _cabi.ptr_array([r.ctypes.data]),
                                              _cabi.ptr_array([c.ctypes.data]), _cabi.ptr_array([v.ctypes.data]),
                                              _cabi.F64 if dtype == "f64" else _cabi.F32))
            plans.append(h)
        off, on = plans
        check(lib, lib.b200gf_plan_set_hop_windows(off, 0))

        def hop(p, o=dst):
            check(lib, lib.b200gf_hop(p, 0, _cabi.HOP_FWD, src.data_ptr(), C, o.data_ptr(), C, C, st))

        def timed(p):
            hop(p)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                hop(p)
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / reps

        hop(off, ref)
        res = {"default_rows": int(lib.b200gf_plan_info(on, 8)), "arms": {}}
        for R in rows:
            check(lib, lib.b200gf_plan_set_hop_windows(on, R))
            hop(on)
            torch.cuda.synchronize()
            rel = float((dst.double() - ref.double()).abs().max() / ref.double().abs().max())
            t_off, t_on = [], []
            for _ in range(rounds):
                t_off.append(timed(off))
                t_on.append(timed(on))
            res["arms"][str(R)] = {"off": stats(t_off), "on": stats(t_on), "max_rel_vs_off": rel}
            print(json.dumps({"workload": name, "dtype": dtype, "lib": os.path.basename(path), "R": R,
                              **res["arms"][str(R)]}), flush=True)
        for p in plans:
            lib.b200gf_plan_destroy(p)
        out["libs"][os.path.basename(path)] = res
    del src, dst, ref
    torch.cuda.empty_cache()
    return out


def layer_ab(name, dtype, rounds):
    import torch
    import gnn_b200
    from gnn_b200 import _cabi
    from gnn_b200.gso import Plan
    lib = _cabi.load()
    w = bench.WORKLOADS[name]
    dev = torch.device("cuda", 0)
    tdt = torch.float64 if dtype == "f64" else torch.float32
    E, K, N = w["E"], w["K"], w["N"]
    gso = bench.make_gso(w).astype(tdt)
    h_cpu, b_cpu = bench.seeded_taps(w, tdt)
    h, b = h_cpu.to(dev), b_cpu.to(dev)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(w["B"], w["G"], N, generator=g).to(dev, tdt)
    dy = torch.randn(w["B"], w["F"], N, generator=g).to(dev, tdt)
    plans = {"off": Plan.from_host_csr(gso.csr, N, tdt, dev), "on": Plan.from_host_csr(gso.csr, N, tdt, dev)}
    check(lib, lib.b200gf_plan_set_hop_windows(plans["off"].handle, 0))
    default_rows = int(lib.b200gf_plan_info(plans["on"].handle, 8))
    xg, hg, bg = (t.clone().requires_grad_(True) for t in (x, h, b))

    def fwd(p):
        return gnn_b200.LSIGF(h, p, x, b)

    def fwd_bwd(p):
        xg.grad = hg.grad = bg.grad = None
        gnn_b200.LSIGF(hg, p, xg, bg).backward(dy)

    def timed(fn, p, steps):
        fn(p)
        torch.cuda.synchronize()
        hops = E * (K - 1) * steps * 2
        lib.b200gf_profile_hops(p.handle, hops)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn(p)
        e1.record()
        torch.cuda.synchronize()
        buf = (ctypes.c_float * hops)()
        got = lib.b200gf_profile_read(p.handle, buf, hops)
        lib.b200gf_profile_hops(p.handle, 0)
        return e0.elapsed_time(e1) / steps, float(np.mean([buf[i] for i in range(got)])) if got > 0 else None

    outs = {}
    for k, p in plans.items():
        with torch.no_grad():
            outs[k] = [fwd(p).detach().clone()]
        fwd_bwd(p)
        torch.cuda.synchronize()
        outs[k] += [xg.grad.clone(), hg.grad.clone(), bg.grad.clone()]
    res = {k: {"fwd": [], "fwd_hop": [], "fb": [], "fb_hop": []} for k in plans}
    for _ in range(rounds):
        for k, p in plans.items():
            with torch.no_grad():
                ms, hop = timed(fwd, p, 3)
            res[k]["fwd"].append(ms)
            res[k]["fwd_hop"].append(hop)
            ms, hop = timed(fwd_bwd, p, 2)
            res[k]["fb"].append(ms)
            res[k]["fb_hop"].append(hop)
    out = {"workload": bench.describe(w, dtype), "default_rows": default_rows, "arms": {}}
    for k in plans:
        out["arms"][k] = {m: stats([t for t in v if t is not None]) for m, v in res[k].items()}
    out["max_rel_on_vs_off"] = {n: float((o.double() - r.double()).abs().max() / r.double().abs().max())
                                for n, o, r in zip(("y", "dx", "dh", "db"), outs["on"], outs["off"])}
    print(json.dumps(out), flush=True)
    del outs, xg, hg, bg, plans
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hops", default="er1m", help="workloads of the fp32 hop sweep")
    ap.add_argument("--f64-hops", default="", help="workloads of the fp64 hop sweep")
    ap.add_argument("--rows", default="125000,200000,250000,333000")
    ap.add_argument("--libs", default="", help="comma-separated variant libraries for the hop sweep (default: the built one)")
    ap.add_argument("--fwd", default="er1m", help="workloads of the LSIGF off/on comparison")
    ap.add_argument("--f64", default="", help="workloads of the fp64 LSIGF off/on comparison")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--variants", help="build the variant libraries into this directory and exit")
    ap.add_argument("--out", help="also write the report as JSON here")
    args = ap.parse_args()
    if args.variants:
        build_variants(args.variants)
        return
    from gnn_b200 import _cabi
    _cabi.load()
    libs = [p for p in args.libs.split(",") if p] or [_cabi.LIB_PATH]
    rows = [int(s) for s in args.rows.split(",") if s]
    report = {"card": card(), "hops": [], "layers": []}
    print("card:", report["card"], flush=True)
    for names, dtype in ((args.hops, "f32"), (args.f64_hops, "f64")):
        for n in (s for s in names.split(",") if s):
            report["hops"].append(hop_sweep(n, dtype, libs if dtype == "f32" else [_cabi.LIB_PATH], rows, args.rounds))
    for names, dtype in ((args.fwd, "f32"), (args.f64, "f64")):
        for n in (s for s in names.split(",") if s):
            report["layers"].append(layer_ab(n, dtype, args.rounds))
    report["card_after"] = card()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(report, f, indent=1)
    print("card:", report["card_after"])
    for hs in report["hops"]:
        for lib, r in hs["libs"].items():
            for R, a in r["arms"].items():
                print("%-44s %-26s R=%-7s off %.3f [%.3f,%.3f]  on %.3f [%.3f,%.3f]  rel %.1e" % (
                    hs["workload"], lib, R, a["off"]["median_ms"], a["off"]["min_ms"], a["off"]["max_ms"],
                    a["on"]["median_ms"], a["on"]["min_ms"], a["on"]["max_ms"], a["max_rel_vs_off"]))
    for ls in report["layers"]:
        for k, a in ls["arms"].items():
            print("%-44s %-3s fwd %.3f [%.3f,%.3f] fwd+bwd %.3f [%.3f,%.3f] hop %.3f" % (
                ls["workload"], k, a["fwd"]["median_ms"], a["fwd"]["min_ms"], a["fwd"]["max_ms"], a["fb"]["median_ms"],
                a["fb"]["min_ms"], a["fb"]["max_ms"], a["fwd_hop"]["median_ms"]))
        print("  max rel on vs off:", ls["max_rel_on_vs_off"])


if __name__ == "__main__":
    main()
