"""Do the wide-row hop's 16-byte half-lane loads cost one L2 request per half sector?  Parent library against this one,
and a control, alternated in one process with CUDA events.

Part 1, libraries: one er1m forward hop (b200gf_hop, C = 64) through each library given with --libs, with the plan's
window copy (the default) and without it (b200gf_plan_set_hop_windows(plan, 0)), fp32 and fp64.  Median and spread of
--rounds rounds of --reps hops each, and whether every library's output is bitwise equal to the first one's.

Part 2, control (fp32, windows of the plan's default size, built here from the same CSR): the windowed gather of
tools/hop_sector_probe.cu with adjacent halves (the old mapping), the same with only the first 16-byte half of each lane
loaded (same sectors, half the load instructions, wrong sums), and with split halves (LaneMap).  If the first-half-only
form runs about as fast as the adjacent one, the sectors bound the gather and splitting the halves cannot help; if it
runs close to twice as fast, each half-sector load costs its own L2 request.

    python tools/hop_sector_probe.py --libs parent.so,new.so [--probe-so probe.so] [--rounds 5] [--reps 10] [--out r.json]

--probe-so defaults to compiling tools/hop_sector_probe.cu into a temporary directory.  Prints the card, power limit
and clocks before and after.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402

import bench  # noqa: E402
from hop_window_bench import card, check, load_lib, stats  # noqa: E402


def build_probe(out):
    nvcc = os.environ.get("NVCC") or "nvcc"
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-shared", "-Xcompiler",
                           "-fPIC", os.path.join(ROOT, "tools", "hop_sector_probe.cu"), "-o", out])
    return out


def timed(fn, reps):
    import torch
    fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def lib_ab(name, dtype, libs, rounds, reps):
    import torch
    from gnn_b200 import _cabi
    w = bench.WORKLOADS[name]
    tdt = torch.float64 if dtype == "f64" else torch.float32
    N, C = w["N"], w["B"] * w["G"]
    r, c, v = bench.make_gso(w).csr[0]
    r = np.ascontiguousarray(r, np.int64)
    c = np.ascontiguousarray(c, np.int32)
    v = np.ascontiguousarray(v, np.float64 if dtype == "f64" else np.float32)
    src = torch.randn(N, C, generator=torch.Generator().manual_seed(3), dtype=torch.float64).to("cuda", tdt)
    st = torch.cuda.current_stream().cuda_stream
    arms = {}
    for path in libs:
        lib = load_lib(path)
        for mode in ("on", "off"):
            h = ctypes.c_void_p()
            check(lib, lib.b200gf_plan_create(ctypes.byref(h), 0, N, 1, _cabi.ptr_array([r.ctypes.data]),
                                              _cabi.ptr_array([c.ctypes.data]), _cabi.ptr_array([v.ctypes.data]),
                                              _cabi.F64 if dtype == "f64" else _cabi.F32))
            if mode == "off":
                check(lib, lib.b200gf_plan_set_hop_windows(h, 0))
            arms[os.path.basename(path), mode] = {"lib": lib, "plan": h, "rows": int(lib.b200gf_plan_info(h, 8)),
                                                  "dst": torch.empty(N, C, device="cuda", dtype=tdt), "ms": []}

    def hop(a):
        check(a["lib"], a["lib"].b200gf_hop(a["plan"], 0, _cabi.HOP_FWD, src.data_ptr(), C, a["dst"].data_ptr(), C, C, st))

    for _ in range(rounds):
        for a in arms.values():
            a["ms"].append(timed(lambda: hop(a), reps))
    first = os.path.basename(libs[0])
    out = {"workload": bench.describe(w, dtype), "C": C, "arms": {}}
    for (lib, mode), a in arms.items():
        ref = arms[first, mode]["dst"]
        out["arms"]["%s windows=%s" % (lib, mode)] = {
            **stats(a["ms"]), "window_rows": a["rows"], "bitwise_equal_to_%s" % first: bool(torch.equal(a["dst"], ref))}
    for a in arms.values():
        a["lib"].b200gf_plan_destroy(a["plan"])
    print(json.dumps(out), flush=True)
    return out


def window_csr(r, c, v, N, R):
    """Window-major copy of a CSR: window w holds the entries whose column lies in [w*R, (w+1)*R), each row's entries in
    their order, as a full-height CSR whose offsets index one shared col/val array."""
    W = (N + R - 1) // R
    win = c.astype(np.int64) // R
    order = np.argsort(win, kind="stable")
    row = np.repeat(np.arange(N, dtype=np.int64), np.diff(r))
    counts = np.bincount(win * N + row, minlength=W * N).reshape(W, N)
    rp = np.zeros((W, N + 1), np.int64)
    rp[:, 1:] = np.cumsum(counts, axis=1)
    rp += np.concatenate([[0], np.cumsum(counts.sum(axis=1))[:-1]])[:, None]
    assert rp[-1, -1] < 2 ** 31
    return rp.astype(np.int32), c[order], v[order], W


def control(name, probe_path, rows, rounds, reps):
    import torch
    w = bench.WORKLOADS[name]
    N, C = w["N"], w["B"] * w["G"]
    r, c, v = bench.make_gso(w).csr[0]
    rp, wc, wv, W = window_csr(np.asarray(r, np.int64), np.asarray(c, np.int32), np.asarray(v, np.float32), N, rows)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    rp_d, c_d, v_d = dev(rp), dev(wc), dev(wv)
    src = torch.randn(N, C, generator=torch.Generator().manual_seed(3)).cuda()
    probe = ctypes.CDLL(probe_path)
    probe.probe_window_hop.restype = ctypes.c_int
    probe.probe_window_hop.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                       ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                       ctypes.c_int, ctypes.c_void_p]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    st = torch.cuda.current_stream().cuda_stream
    names = {0: "adjacent halves", 1: "adjacent, first half only (control)", 2: "split halves (LaneMap)"}
    dst = {k: torch.empty(N, C, device="cuda") for k in names}
    ms = {k: [] for k in names}

    def hop(k):
        rc = probe.probe_window_hop(k, rp_d.data_ptr(), W, c_d.data_ptr(), v_d.data_ptr(), src.data_ptr(), C,
                                    dst[k].data_ptr(), N, C, sms, st)
        if rc:
            raise RuntimeError("probe_window_hop(%d) failed" % k)

    for _ in range(rounds):
        for k in names:
            ms[k].append(timed(lambda: hop(k), reps))
    out = {"workload": bench.describe(w, "f32"), "window_rows": rows, "windows": W,
           "gathered_sector_bytes": int(len(wc)) * C * 4, "arms": {names[k]: stats(ms[k]) for k in names},
           "split_bitwise_equal_to_adjacent": bool(torch.equal(dst[0], dst[2]))}
    print(json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--libs", required=True, help="comma-separated libb200gf builds; the first is the baseline")
    ap.add_argument("--workload", default="er1m")
    ap.add_argument("--probe-so", default="", help="tools/hop_sector_probe.cu built as a shared library")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", help="also write the report as JSON here")
    args = ap.parse_args()
    import torch
    from gnn_b200 import _cabi
    _cabi.load()
    libs = [p for p in args.libs.split(",") if p]
    report = {"card": card(), "libs": [os.path.basename(p) for p in libs], "hops": []}
    print("card:", report["card"], flush=True)
    for dtype in ("f32", "f64"):
        report["hops"].append(lib_ab(args.workload, dtype, libs, args.rounds, args.reps))
        torch.cuda.empty_cache()
    rows = report["hops"][0]["arms"]["%s windows=on" % report["libs"][0]]["window_rows"]
    with tempfile.TemporaryDirectory() as tmp:
        probe = args.probe_so or build_probe(os.path.join(tmp, "hop_sector_probe.so"))
        report["control"] = control(args.workload, probe, rows, args.rounds, args.reps)
    report["card_after"] = card()
    print("card:", report["card_after"])
    if args.out:
        with open(args.out, "w") as f:
            json.dump(report, f, indent=1)
    for hs in report["hops"]:
        for k, a in hs["arms"].items():
            print("%-40s %-42s %.3f ms [%.3f, %.3f]" % (hs["workload"][:40], k, a["median_ms"], a["min_ms"], a["max_ms"]))
    for k, a in report["control"]["arms"].items():
        print("control %-40s %.3f ms [%.3f, %.3f]" % (k, a["median_ms"], a["min_ms"], a["max_ms"]))


if __name__ == "__main__":
    main()
