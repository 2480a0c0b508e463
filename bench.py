#!/usr/bin/env python
"""bench.py — LSIGF edge·feature ops/s on H100 (BASELINE.json `metric`), with roofline, parity check and CPU baseline.

  python bench.py [--gpus N] [--steps K] [--warmup W] [--workload er1m|cfg2|cfg3|cfg4|er2m|sbm1m] [--impl reference]

A "step" is one LSIGF forward (alegnn/utils/graphML.py:83-176 semantics) over one synthetic batch:
  value  = E * nnz * (K-1) * B * G / t_step     (one op = one multiply-add of one non-zero of S with one feature
           column for one hop; SURVEY.md §8d), inputs resident in HBM, timed with CUDA events around exactly K steps
           after a barrier + synchronize, max over ranks.  N = 1: x in the reference's [B,G,N] layout, the layout
           conversion is inside the step.  N > 1: every rank holds its shard of the node-major x (DESIGN.md §4).
  e2e    = same metric through the public API with pinned HOST x and y: every step's H2D and D2H copy inside the
           timed region, overlapped ACROSS steps on two copy streams (class E2EPipeline).
  roofline = the shift kernel: algorithmic bytes per launch (gather model, SURVEY.md §8d) divided by its average
           duration measured live with CUDA events around every hop launch inside the timed region (events recorded
           by the library on the launching stream), against MEASURED_PEAKS.json's HBM copy bandwidth when present, else
           the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s).
  parity_max_rel = max|y - y_ref| / max|y_ref| of the timed path's output against the fp64 CPU oracle
           (oracle/lsigf_oracle.py:lsigf_sparse_stream) at the FULL workload size, at every N (the ranks' rows are
           gathered); the run fails above 1e-4.  `selftest` (N > 1): forward AND backward of both shardings against the
           oracle on a small graph, over NCCL / NVLink on the same ranks.
  cpu_baseline = the reference's dense torch.matmul algorithm (oracle/lsigf_oracle.py:lsigf_dense_torch, a port: the
           reference is Python, cannot be pip-installed offline — DESIGN.md §6 — and is not part of this repository) on
           the GPU machine's host cores, bounded sample, thread count pinned and printed.
  configs = at N = 1 the other single-GPU configurations of BASELINE.json (cfg2, cfg3, cfg4; cfg4ev = config 4 as the
           reference's EdgeVariantGF layer) measured the same way in the same run (fewer steps), each with its own parity.
Default workload = the configuration the north_star target is quoted on: ER N=1M, avgDeg=32, K=5, G=F=64, B=1, fp32.
"""
import argparse
import json
import os
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

WORKLOADS = {
    # name: graph, N, deg, E, K, G, F, B, seed
    "er1m": dict(graph="er", N=1_000_000, deg=32, E=1, K=5, G=64, F=64, B=1, seed=1),
    "er2m": dict(graph="er", N=2_000_000, deg=32, E=1, K=5, G=64, F=64, B=1, seed=5),
    "cfg2": dict(graph="er", N=100_000, deg=16, E=1, K=5, G=64, F=64, B=32, seed=2),
    "cfg3": dict(graph="knn", N=1682, deg=10, E=1, K=5, G=64, F=64, B=32, seed=3),
    "cfg4": dict(graph="er", N=200_000, deg=16, E=4, K=3, G=32, F=32, B=32, seed=4),
    "tiny": dict(graph="er", N=20_000, deg=16, E=1, K=5, G=64, F=64, B=1, seed=9),
    # stochastic block model, 1000 communities of 1000 nodes, ~80 % of the edges inside a community (avgDeg ~ 32);
    # nodes are numbered community by community, so gathers have the locality a real graph ordering would give
    "sbm1m": dict(graph="sbm", N=1_000_000, deg=32, E=1, K=5, G=64, F=64, B=1, seed=6, communities=1000, intra=0.8),
}
PARITY_TOL = 1e-4      # north_star tolerance (fp32); fp64 runs are held to 1e-10
L2_BYTES = 50 * 2 ** 20  # H100 SXM L2


def describe(w, dtype="f32"):
    return "%s N=%d avgDeg=%d E=%d K=%d G=%d F=%d B=%d %s" % (
        {"er": "Erdos-Renyi", "knn": "kNN-like", "sbm": "SBM(%d communities)" % w.get("communities", 0)}[w["graph"]],
        w["N"], w["deg"], w["E"], w["K"], w["G"], w["F"], w["B"], "fp64" if dtype == "f64" else "fp32")


def make_gso(w):
    from gnn_b200 import graphs
    if w["graph"] == "er":
        return graphs.er_gso(w["N"], w["deg"], seed=w["seed"], E=w["E"])
    if w["graph"] == "sbm":
        C, n = w["communities"], w["N"] // w["communities"]
        p_in = w["deg"] * w["intra"] / (n - 1)
        p_out = w["deg"] * (1 - w["intra"]) / (w["N"] - n)
        return graphs.sbm_gso(w["N"], C, p_in, p_out, seed=w["seed"], E=w["E"])
    return graphs.knn_like_gso(w["N"], w["deg"], seed=w["seed"])


def hop_algorithmic_bytes(nnz, N, C, s=4):
    """Gather model, per hop and per S_e (SURVEY.md §8d): col idx + value per nnz, rowptr, one neighbour row of C
    columns per non-zero, one result row per node."""
    return nnz * (4 + s) + (N + 1) * 8 + nnz * C * s + N * C * s


def measured_peak_gbs():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        try:
            return float(json.load(open(p))["hbm_gbs"]), "measured (MEASURED_PEAKS.json)"
        except Exception:
            pass
    return 3350.0, "H100 SXM data sheet (HBM3, 3.35 TB/s)"


def usable_cores():
    """Host threads this process may really use: CPU affinity mask, capped by the cgroup CPU quota when there is one."""
    try:
        n = len(os.sched_getaffinity(0))
    except Exception:
        n = os.cpu_count() or 1
    for path in ("/sys/fs/cgroup/cpu.max", "/sys/fs/cgroup/cpu/cpu.cfs_quota_us"):
        try:
            txt = open(path).read().split()
            if path.endswith("cpu.max"):
                if txt[0] != "max":
                    n = min(n, max(1, int(float(txt[0]) / float(txt[1]))))
            else:
                q = int(txt[0])
                if q > 0:
                    per = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
                    n = min(n, max(1, q // per))
            break
        except Exception:
            continue
    return max(1, n)


class ClockSampler:
    """Samples SM clock and throttle reasons DURING the timed region (NVML every 10 ms; nvidia-smi fallback)."""

    NAMES = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]

    def __init__(self, index=0):
        self.index = index
        self.sm = []
        self.sm_max = None
        self.reasons = set()
        self._stop = threading.Event()
        self._t = None
        self._nvml = None
        try:
            import pynvml
            pynvml.nvmlInit()
            self._nvml = pynvml
            self._h = pynvml.nvmlDeviceGetHandleByIndex(index)  # all GPUs of the box are visible: NVML index == CUDA index
            self.sm_max = float(pynvml.nvmlDeviceGetMaxClockInfo(self._h, pynvml.NVML_CLOCK_SM))
        except Exception:
            self._nvml = None

    def _sample_nvml(self):
        n = self._nvml
        self.sm.append(float(n.nvmlDeviceGetClockInfo(self._h, n.NVML_CLOCK_SM)))
        try:
            r = n.nvmlDeviceGetCurrentClocksEventReasons(self._h)
        except Exception:
            r = n.nvmlDeviceGetCurrentClocksThrottleReasons(self._h)
        bits = {"hw_slowdown": 0x8, "hw_thermal_slowdown": 0x40, "sw_thermal_slowdown": 0x20, "sw_power_cap": 0x4}
        for k, b in bits.items():
            if r & b:
                self.reasons.add(k)

    def _sample_smi(self):
        import subprocess
        q = ("clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
             "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")
        out = subprocess.run(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + q, "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=5).stdout
        f = [v.strip() for v in out.strip().split(",")]
        if len(f) >= 6:
            self.sm.append(float(f[0]))
            self.sm_max = float(f[1])
            for i, k in enumerate(self.NAMES):
                if f[2 + i].lower().startswith("active"):
                    self.reasons.add(k)

    def _run(self):
        while not self._stop.is_set():
            try:
                if self._nvml is not None:
                    self._sample_nvml()
                else:
                    self._sample_smi()
            except Exception:
                pass
            self._stop.wait(0.01 if self._nvml is not None else 0.2)

    def __enter__(self):
        self._t = threading.Thread(target=self._run, daemon=True)
        self._t.start()
        return self

    def __exit__(self, *a):
        self._stop.set()
        self._t.join(timeout=6)

    def summary(self):
        if not self.sm:
            return {"sm_mhz": None, "sm_max_mhz": self.sm_max, "reasons": ["unsampled"]}
        sm = sorted(self.sm)
        return {"sm_mhz": sm[len(sm) // 2], "sm_max_mhz": self.sm_max, "reasons": sorted(self.reasons),
                "samples": len(sm), "source": "nvml" if self._nvml is not None else "nvidia-smi"}


# ------------------------------------------------------------------------------------------------------
# CPU legs: the reference's dense algorithm on a bounded sample (reference arm / cpu_baseline), a sparse restatement at
# the full size (labelled "not reference code"), and the fp64 oracle forward used by the parity check
# ------------------------------------------------------------------------------------------------------
def seeded_taps(w, tdt=torch.float32):
    g = torch.Generator().manual_seed(0)
    bound = 1.0 / np.sqrt(w["G"] * w["K"])
    h = ((torch.rand(w["F"], w["E"], w["K"], w["G"], generator=g) * 2 - 1) * bound).to(tdt)
    b = ((torch.rand(w["F"], 1, generator=g) * 2 - 1) * bound).to(tdt)
    return h, b


def cpu_dense_sample(w, n_dense, reps, threads):
    """Reference algorithm (dense E x N x N GSO, K-1 batched GEMMs + contraction; graphML.py:152-175) at N = n_dense with
    the workload's avgDeg/K/G/F/B.  `threads` host threads, one warm-up, median of `reps`.
    Returns (ops_per_s, seconds_per_forward, nnz, all_times)."""
    import lsigf_oracle as orc
    from gnn_b200 import graphs
    torch.set_num_threads(threads)
    gso = graphs.er_gso(n_dense, w["deg"], seed=w["seed"], E=w["E"]) if w["graph"] != "knn" else \
        graphs.knn_like_gso(n_dense, w["deg"], seed=w["seed"])
    S = gso.to_dense().float()
    h, b = seeded_taps(w)
    x = torch.randn(w["B"], w["G"], n_dense, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        orc.lsigf_dense_torch(h, S, x, b)  # warm-up
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            orc.lsigf_dense_torch(h, S, x, b)
            ts.append(time.perf_counter() - t0)
    t = float(np.median(ts))
    ops = float(gso.nnz()) * (w["K"] - 1) * w["B"] * w["G"]
    return ops / t, t, gso.nnz(), ts


def cpu_sparse_sample(w, gso, threads, reps=3):
    """The same filter at the workload's FULL size with torch.sparse CSR x dense products on the host cores
    (oracle/lsigf_oracle.py:lsigf_sparse_torch).  NOT reference code — the reference has no sparse path; it shows what a
    CPU could do with the sparse formulation, and it is the one CPU number taken at the same size as the GPU's."""
    import warnings
    import lsigf_oracle as orc
    torch.set_num_threads(threads)
    h, b = seeded_taps(w)
    x = torch.randn(w["B"], w["G"], w["N"], generator=torch.Generator().manual_seed(1))
    csr = [(r, c, v.astype(np.float32)) for (r, c, v) in gso.csr]
    ts = []
    with torch.no_grad(), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        prepared = orc.prepare_sparse_torch(csr, w["N"], torch.float32)     # format conversion: once, untimed
        for _ in range(reps):
            t0 = time.perf_counter()
            orc.lsigf_sparse_torch(h, csr, x, b, prepared=prepared)
            ts.append(time.perf_counter() - t0)
    t = float(np.median(ts))
    ops = float(gso.nnz()) * (w["K"] - 1) * w["B"] * w["G"]
    return {"value": ops / t, "unit": "edge-feature-op/s", "cores": threads, "kind": "port-sparse (not reference code)",
            "same_size_as_gpu": True,
            "sample": "full workload (N=%d, nnz=%d), torch.sparse CSR, median of %d forwards of %.2f s" % (w["N"], gso.nnz(), reps, t)}


def oracle_forward_nm(gso, h, b, x_nm, B, G):
    """fp64 oracle forward (oracle/lsigf_oracle.py:lsigf_sparse_stream, sparse products threaded over the host cores) of a
    node-major x [N, B*G]; returns y node-major [N, B*F] float64."""
    import scipy.sparse as sp
    import lsigf_oracle as orc
    torch.set_num_threads(usable_cores())       # torchrun exports OMP_NUM_THREADS=1; the check runs on rank 0 only
    N = gso.N
    S = [sp.csr_matrix((v.astype(np.float64), c, r), shape=(N, N)) for (r, c, v) in gso.csr]
    x = x_nm.double().numpy().reshape(N, B, G).transpose(1, 2, 0)                         # [B, G, N]
    y = orc.lsigf_sparse_stream(h.double().numpy(), S, x, None if b is None else b.double().numpy(), spmm=orc.threaded_spmm)
    F = h.shape[0]
    return np.ascontiguousarray(y.transpose(2, 0, 1).reshape(N, B * F))


def max_rel(got_nm, want_nm):
    """max|a - ref| / max|ref| with the comparison done on the GPU when the operands are large."""
    want = torch.from_numpy(want_nm)
    if got_nm.is_cuda:
        want = want.to(got_nm.device)
    d = (got_nm.double() - want).abs().max().item()
    return float(d / max(want.abs().max().item(), 1e-300))


def pick_dense_n(w):
    # dense work ~ 2*(K-1)*B*G*E*N^2 flop; keep one forward to a few seconds on a multi-core host
    flop_budget = 6e11
    n = int(np.sqrt(flop_budget / (2.0 * max(w["K"] - 1, 1) * w["B"] * w["G"] * w["E"])))
    return int(min(w["N"], max(1024, min(n, 16384))))


def cpu_baseline_block(w, reps):
    threads = usable_cores()
    n_dense = pick_dense_n(w)
    ops_s, t, nnz_d, ts = cpu_dense_sample(w, n_dense, reps, threads)
    # the dense algorithm does O(N^2) work for O(N) non-zeros: its op/s falls like 1/N.  Measured at smaller N too
    # (SURVEY.md §8d: "report the measured 1/N trend rather than extrapolating silently"); cheap next to the sample above.
    trend = []
    for n_small in (1682, 4096, 8192):
        if n_small < n_dense:
            o_, t_, z_, _ = cpu_dense_sample(w, n_small, min(3, reps), threads)
            trend.append({"N": n_small, "nnz": z_, "s_per_forward": t_, "ops_per_s": o_})
    trend.append({"N": n_dense, "nnz": nnz_d, "s_per_forward": t, "ops_per_s": ops_s})
    return ops_s, t, {"value": ops_s, "unit": "edge-feature-op/s", "cores": threads, "kind": "port",
                      "threads_pinned": threads, "host_cpus_visible": os.cpu_count(), "dense_trend": trend,
                      "sample": "reference dense torch.matmul algorithm at N=%d (nnz=%d), same avgDeg/K/G/F/B; 1 warm-up, "
                                "median of %d forwards (min %.2f s, median %.2f s, max %.2f s); the dense algorithm is "
                                "O(N^2) and cannot hold N=%d" % (n_dense, nnz_d, len(ts), min(ts), t, max(ts), w["N"])}


def run_reference_arm(args, w):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    t_start = time.time()
    ops_s, t, block = cpu_baseline_block(w, reps=max(1, min(args.steps, 7)))   # one "step" = one dense forward
    line = {
        "impl": "reference", "metric": "LSIGF edge-feature ops/s", "value": ops_s, "unit": "edge-feature-op/s",
        "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup, "ms_per_step": t * 1e3,
        "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": describe(w), "note": "CPU dense torch.matmul algorithm of the reference (port; the "
                   "reference package cannot be pip-installed offline: poetry-core build backend missing)"},
        "cpu_baseline": block,
        "e2e": {"value": ops_s, "unit": "edge-feature-op/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    if not args.no_full_size_cpu and w["B"] * w["G"] <= 256:
        try:   # the one CPU figure at the GPU arm's own size (sparse restatement, labelled as such)
            line["cpu_sparse_full_size"] = cpu_sparse_sample(w, make_gso(w), usable_cores())
        except Exception as exc:
            line["cpu_sparse_full_size"] = {"error": str(exc)[:200]}
    line["wall_s"] = time.time() - t_start
    print(json.dumps(line))


# ------------------------------------------------------------------------------------------------------
# GPU arm
# ------------------------------------------------------------------------------------------------------
class E2EPipeline:
    """End-to-end steps with the copies overlapped across steps: while step i computes, step i+1's input goes host ->
    device and step i-1's result device -> host on two copy streams (PCIe is full duplex).  Every step still copies ITS
    input from pinned host memory and ITS result back to pinned host memory; device inputs and host outputs are
    double-buffered, ordering is by CUDA events, nothing is skipped or cached."""

    def __init__(self, dev, xh, yh_shape, compute):
        self.xh, self.compute = xh, compute
        self.s_in, self.s_out = torch.cuda.Stream(dev), torch.cuda.Stream(dev)
        self.xd = [torch.empty(xh.shape, dtype=xh.dtype, device=dev) for _ in range(2)]
        self.yh = [torch.empty(yh_shape, dtype=xh.dtype).pin_memory() for _ in range(2)]
        self.ev_in = [torch.cuda.Event() for _ in range(2)]
        self.ev_cmp = [torch.cuda.Event() for _ in range(2)]
        self.i = 0

    def step(self):
        k = self.i & 1
        self.i += 1
        cur = torch.cuda.current_stream()
        with torch.cuda.stream(self.s_in):
            self.s_in.wait_event(self.ev_cmp[k])            # the compute of two steps ago has finished reading xd[k]
            self.xd[k].copy_(self.xh, non_blocking=True)
            self.ev_in[k].record(self.s_in)
        cur.wait_event(self.ev_in[k])
        y = self.compute(self.xd[k])                         # contiguous device result
        self.ev_cmp[k].record(cur)
        with torch.cuda.stream(self.s_out):
            self.s_out.wait_event(self.ev_cmp[k])
            self.yh[k].copy_(y, non_blocking=True)
        y.record_stream(self.s_out)


class _JsonOnlyStdout:
    """The driver reads ONE JSON line from stdout; NCCL / libraries print banners there.  Everything written to fd 1
    while this is active goes to stderr; `emit` writes the final line to the real stdout."""

    def __init__(self):
        sys.stdout.flush()
        self._real = os.dup(1)
        os.dup2(2, 1)

    def emit(self, text):
        sys.stdout.flush()
        os.write(self._real, (text + "\n").encode())


class Ctx:
    """Per-process measurement context (device, ranks, library handle, timing helper)."""

    def __init__(self, args):
        import torch.distributed as dist
        from gnn_b200 import _cabi
        self.args, self.dist = args, dist
        self.rank = int(os.environ.get("RANK", "0"))
        self.world = int(os.environ.get("WORLD_SIZE", "1"))
        self.local = int(os.environ.get("LOCAL_RANK", "0"))
        if not torch.cuda.is_available():
            raise SystemExit("bench.py: no CUDA device (the GPU arm has no CPU fallback)")
        torch.cuda.set_device(self.local)
        self.dev = torch.device("cuda", self.local)
        if self.world > 1:
            os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
            os.environ["NCCL_DEBUG"] = os.environ.get("B200GF_NCCL_DEBUG", "WARN")   # keep stdout to the one JSON line
            dist.init_process_group("nccl", device_id=self.dev)
        self.lib = _cabi.load()
        self.tdt = torch.float64 if args.dtype == "f64" else torch.float32
        self.es = 8 if args.dtype == "f64" else 4
        self.tol = 1e-10 if args.dtype == "f64" else PARITY_TOL
        self.peak, self.peak_src = measured_peak_gbs()

    def timed(self, fn, steps, warmup):
        """W warm-up calls, barrier + synchronize, exactly `steps` calls between two CUDA events, synchronize + barrier;
        max over ranks.  Returns (ms per step, library kernel launches inside the timed region on this rank)."""
        for _ in range(warmup):
            fn()
        if self.world > 1:
            self.dist.barrier()
        torch.cuda.synchronize()
        self.lib.b200gf_launch_count(1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        launches = int(self.lib.b200gf_launch_count(1))
        ms = torch.tensor([e0.elapsed_time(e1)], device=self.dev)
        if self.world > 1:
            self.dist.barrier()
            self.dist.all_reduce(ms, op=self.dist.ReduceOp.MAX)
        return float(ms.item()) / steps, launches


def ctypes_floats(lib, plan, n):
    import ctypes
    buf = (ctypes.c_float * n)()
    got = lib.b200gf_profile_read(plan.handle, buf, n)
    return [float(buf[i]) for i in range(max(0, got))]


def load_ncu_traffic(workload, dtype):
    """DRAM bytes per hop launch (dram__bytes_read.sum + dram__bytes_write.sum) from the committed `ncu --set full`
    capture of this workload / dtype / kernel version (profiles/ncu_traffic.json, when one is on file), or null."""
    p = os.path.join(ROOT, "profiles", "ncu_traffic.json")
    try:
        d = json.load(open(p))
        return d.get("%s:%s" % (workload, dtype), d.get(workload) if dtype == "f32" else None)
    except Exception:
        return None


def hop_compulsory_bytes(nnz, rows, C, es=4, src_rows=None):
    """Cache-ideal bytes of one hop (SURVEY.md §8d): 2*N*C*s + nnz*(4+s); a row shard reads all `src_rows` source rows
    and writes its own `rows`."""
    return (int(rows if src_rows is None else src_rows) + int(rows)) * int(C) * es + int(nnz) * (4 + es)


def hop_roofline(ctx, hop_ms, step_ms_total, nnz, rows, C, kernel, workload=None, src_rows=None):
    if not hop_ms:
        return None
    hop_bytes = hop_algorithmic_bytes(nnz, rows, C, ctx.es)
    avg = float(np.mean(hop_ms))
    achieved = hop_bytes / (avg * 1e-3) / 1e9
    traffic = load_ncu_traffic(workload, ctx.args.dtype) if workload else None
    out = {"bound": "hbm", "achieved": achieved, "peak": ctx.peak, "unit": "GB/s", "frac": achieved / ctx.peak,
           "traffic": traffic, "kernel": kernel, "bytes_per_launch": hop_bytes, "ms_per_launch": avg,
           "launches_timed": len(hop_ms), "peak_source": ctx.peak_src,
           "kernel_share_of_step": float(np.sum(hop_ms)) / step_ms_total}
    if traffic:
        out["dram_frac"] = traffic / (avg * 1e-3) / 1e9 / ctx.peak      # actual DRAM bytes / time / copy peak
    # SURVEY.md §8d secondary bound: what a kernel with perfect L2 reuse would move (every source row read once, every
    # result row written once, the indices and values once)
    out["compulsory_bytes"] = hop_compulsory_bytes(nnz, rows, C, ctx.es, src_rows)
    out["compulsory_frac"] = out["compulsory_bytes"] / (avg * 1e-3) / 1e9 / ctx.peak
    return out


def single_gpu_workload(ctx, name, w, steps, warmup, full, keep_last=False):
    """One workload on one GPU: timed forward (+ hop profile, parity; with `full` also e2e and forward+backward).
    keep_last: the output of the last timed step is returned as res["last_output"]."""
    import gnn_b200
    args, dev, tdt, es, lib = ctx.args, ctx.dev, ctx.tdt, ctx.es, ctx.lib
    E, K, G, F, B, N = w["E"], w["K"], w["G"], w["F"], w["B"], w["N"]
    gso = make_gso(w).astype(tdt)
    nnz_e = gso.nnz() // E
    ops_per_step = float(gso.nnz()) * (K - 1) * B * G
    h_cpu, b_cpu = seeded_taps(w, tdt)
    h, b = h_cpu.to(dev), b_cpu.to(dev)
    g = torch.Generator().manual_seed(1)
    x_cpu = torch.randn(B, G, N, generator=g).to(tdt)
    x = x_cpu.to(dev)                                         # reference layout, resident in HBM
    plan = gso.plan(dev)
    fwd = lambda: gnn_b200.LSIGF(h, gso, x, b)               # noqa: E731  (layout conversion inside the step)
    last = []

    def fwd_keep():
        last[:] = [fwd()]

    hops = E * (K - 1)
    cap = hops * (steps + warmup)
    lib.b200gf_profile_hops(plan.handle, cap)
    with torch.no_grad(), ClockSampler(ctx.local) as clk:
        ms, launches = ctx.timed(fwd_keep if keep_last else fwd, steps, warmup)
    hop_ms = ctypes_floats(lib, plan, cap)[hops * warmup:]   # launches inside the timed region only
    lib.b200gf_profile_hops(plan.handle, 0)
    rf = hop_roofline(ctx, hop_ms, ms * steps, nnz_e, N, B * G, "spmm_hop_v2_kernel" if B * G * es > 128
                      else "spmm_hop_multirow_kernel", workload=name)
    out = {"ms_per_step": ms, "value": ops_per_step / (ms * 1e-3), "unit": "edge-feature-op/s", "nnz": gso.nnz(),
           "ops_per_step": ops_per_step, "gpu_launches": launches, "clocks": clk.summary(), "roofline": rf}
    if keep_last:
        out["last_output"] = last[0]
    if not args.no_check:
        t0 = time.time()
        with torch.no_grad():
            y = fwd()                                        # [B, F, N] view of the node-major result
            y_nm = y.permute(2, 0, 1).reshape(N, B * F)
        x_nm = x_cpu.permute(2, 0, 1).reshape(N, B * G)
        want = oracle_forward_nm(gso, h_cpu, b_cpu, x_nm, B, G)
        out["parity_max_rel"] = max_rel(y_nm, want)
        out["parity_note"] = "all %d x %d outputs vs the fp64 CPU oracle at full size (%.1f s on the host)" % (N, B * F, time.time() - t0)
        del y, y_nm, want
    if full:
        # end-to-end through the public API with pinned host buffers
        xh = x_cpu.pin_memory()
        pipe = E2EPipeline(dev, xh, (B, F, N), lambda xd: gnn_b200.to_feature_major(gnn_b200.LSIGF(h, gso, xd, b)))
        yh = pipe.yh[0]
        with torch.no_grad():
            ms_e2e, _ = ctx.timed(pipe.step, steps, 3)
        out["e2e"] = {"value": ops_per_step / (ms_e2e * 1e-3), "unit": "edge-feature-op/s",
                      "h2d_bytes_per_step": xh.numel() * es, "d2h_bytes_per_step": yh.numel() * es, "ms_per_step": ms_e2e}
        del pipe
        # forward + backward (reported beside the headline; SURVEY.md §8d asks for both)
        xg = x.clone().requires_grad_(True)
        hg = h.clone().requires_grad_(True)
        bg = b.clone().requires_grad_(True)
        dy = torch.randn(B, F, N, generator=g).to(dev, tdt)

        def fwd_bwd():
            xg.grad = hg.grad = bg.grad = None
            gnn_b200.LSIGF(hg, gso, xg, bg).backward(dy)

        ms_fb, _ = ctx.timed(fwd_bwd, max(3, steps // 2), 2)
        out["fwd_bwd"] = {"ms_per_step": ms_fb, "unit": "edge-feature-op/s",
                          "value": float(gso.nnz()) * (K - 1) * B * (G + F) / (ms_fb * 1e-3),
                          "note": "forward hops on B*G columns + backward hops on B*F columns per step"}
    out["l2"] = ("inputs larger than L2 (x and every z_k are %d MB each; no flush needed)" % (N * B * G * es // 2 ** 20)
                 if N * B * G * es > L2_BYTES else "working set fits L2: numbers are L2-warm")
    return out, gso


def edge_variant_workload(ctx, steps, warmup):
    """BASELINE.json config 4 at its stated size as the reference's layer type: hybrid EdgeVariantGF (EdgeNet) on ER
    N = 200k, avgDeg 16, tensor GSO E = 4, K = 3, G = F = 32, B = 32, M = 1024 selected nodes — gnn_b200.SparseEdgeVariantGF
    (parameters per masked non-zero; the reference's dense weightEV would need 1.6e16 numbers).  One step = the layer's
    forward = LSI part (LSIGF with the tensor GSO) + EV part (csrc/ev.cu chains on the compact node set)."""
    import gnn_b200
    from gnn_b200 import edgevariant as evm
    import lsigf_oracle as orc
    w = WORKLOADS["cfg4"]
    dev, tdt, es = ctx.dev, ctx.tdt, ctx.es
    E, K, G, F, B, N, M = w["E"], w["K"], w["G"], w["F"], w["B"], w["N"], 1024
    gso = make_gso(w).astype(tdt)
    torch.manual_seed(4)
    layer = gnn_b200.SparseEdgeVariantGF(G, F, K, M, N, E, True).to(dev, tdt)
    layer.addGSO(gso, device=dev)
    st = layer._struct
    nnz_m = [pe["nnz"] for pe in st.per_e]
    n_diag = [int((pe["diag"] >= 0).sum()) for pe in st.per_e]
    x = torch.randn(B, G, N, generator=torch.Generator().manual_seed(1)).to(dev, tdt)
    ops_lsi = float(gso.nnz()) * (K - 1) * B * G
    ops_ev = float(sum(F * G * B * (n * (K - 1) + d) for n, d in zip(nnz_m, n_diag)))
    fwd = lambda: layer(x)                                   # noqa: E731
    with torch.no_grad(), ClockSampler(ctx.local) as clk:
        ms, launches = ctx.timed(fwd, steps, warmup)
    xA = x.index_select(2, st.A)

    def ev_only():
        for e in range(E):
            evm._chain(layer.weightEV[e], xA, st.per_e[e], st.NA, True)

    with torch.no_grad():
        ms_ev, launches_ev = ctx.timed(ev_only, steps, warmup)
    # gather-model bytes of the EV part per forward: every step reads its weights once, one B-wide state row per
    # non-zero and chain, and writes one state row per chain and node (the last step writes only Y)
    by = 0.0
    for n, d in zip(nnz_m, n_diag):
        by += F * G * d * es + F * G * d * B * es + F * G * st.NA * B * es + F * st.NA * B * es                   # k = 0 (diagonal)
        for k in range(1, K):
            by += F * G * n * es + n * 4 + F * G * n * B * es + (F * G * st.NA * B * es if k < K - 1 else 0) + 2 * F * st.NA * B * es
    out = {"workload": "hybrid EdgeVariantGF (EdgeNet) " + describe(w, ctx.args.dtype) + " M=%d" % M,
           "ms_per_step": ms, "value": (ops_lsi + ops_ev) / (ms * 1e-3), "unit": "edge-feature-op/s",
           "ops_per_step": {"lsi": ops_lsi, "edge_variant": ops_ev}, "gpu_launches": launches,
           "edge_variant_part": {"ms": ms_ev, "compact_nodes": st.NA, "masked_nnz_per_e": nnz_m,
                                 "parameters": int(sum(p.numel() for p in layer.weightEV)),
                                 "value": ops_ev / (ms_ev * 1e-3), "gpu_launches": launches_ev,
                                 "roofline": {"bound": "hbm", "kernel": "ev::step_kernel", "bytes_per_forward": by,
                                              "achieved": by / (ms_ev * 1e-3) / 1e9, "peak": ctx.peak, "unit": "GB/s",
                                              "frac": by / (ms_ev * 1e-3) / 1e9 / ctx.peak}},
           "clocks": clk.summary()}
    if not ctx.args.no_check:
        # EV part of two output features against the fp64 scipy chains, LSI part against the LSIGF oracle is cfg4's own check
        with torch.no_grad():
            yA = None
            for e in range(E):
                ye = evm._chain(layer.weightEV[e], xA, st.per_e[e], st.NA, True)
                yA = ye if yA is None else yA + ye
            errs = []
            xA_c = xA.double().cpu().numpy()
            for f in (0, F - 1):
                want = 0
                for e in range(E):
                    pe = st.per_e[e]
                    want = want + orc.evgf_sparse_chains(pe["rowptr"].cpu().numpy(), pe["col"].cpu().numpy(),
                                                         layer.weightEV[e][f].double().cpu().numpy(), xA_c, k0_identity=True)
                got = yA[:, f, :].double().cpu().numpy()
                errs.append(float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-300)))
        out["parity_max_rel"] = max(errs)
        out["parity_note"] = "EV part, output features 0 and F-1 on all %d compact nodes x %d samples vs fp64 scipy chains" % (st.NA, B)
    return out


def multi_gpu_selftest(ctx):
    """Forward AND backward of both shardings on a small graph against the fp64 oracle, over the same NCCL / NVLink ranks
    the bench uses (VERDICT r1: the partitioned backward and the fused kernels above 2 ranks had no hardware evidence)."""
    import scipy.sparse as sp
    import lsigf_oracle as orc
    from gnn_b200 import graphs
    from gnn_b200.distributed import PartitionedLSIGF
    dist, dev, world, rank = ctx.dist, ctx.dev, ctx.world, ctx.rank
    N, E, K, B = 20011, 2, 4, 2                                   # N not divisible by the world size: padded last block
    G = F = 64
    res = {}
    for dtype, tol in ((torch.float32, 1e-4), (torch.float64, 1e-10)):
        gso = graphs.er_gso(N, 12, seed=77, E=E).astype(dtype)
        gen = torch.Generator().manual_seed(5)
        h = (torch.rand(F, E, K, G, generator=gen, dtype=torch.float64) - 0.5).to(dtype)
        b = (torch.rand(F, 1, generator=gen, dtype=torch.float64) - 0.5).to(dtype)
        x_nm = torch.randn(N, B * G, generator=gen, dtype=torch.float64).to(dtype)
        dy_nm = torch.randn(N, B * F, generator=gen, dtype=torch.float64).to(dtype)
        want = None
        if rank == 0:
            S = [sp.csr_matrix((v.astype(np.float64), c, r), shape=(N, N)) for (r, c, v) in gso.csr]
            x = x_nm.double().numpy().reshape(N, B, G).transpose(1, 2, 0)
            dy = dy_nm.double().numpy().reshape(N, B, F).transpose(1, 2, 0)
            y_ref = orc.lsigf_sparse_stream(h.double().numpy(), S, x, b.double().numpy())
            dh_ref, dx_ref, db_ref = orc.lsigf_grads_sparse_stream(h.double().numpy(), S, x, dy, (F, 1))
            want = dict(y=y_ref.transpose(2, 0, 1).reshape(N, B * F), dh=dh_ref, dx=dx_ref.transpose(2, 0, 1).reshape(N, B * G), db=db_ref)
        for mode in ("nodes", "features"):
            part = PartitionedLSIGF(gso, mode=mode, device=dev)
            R = part.rows_per_rank
            pad = lambda t: torch.cat((t, torch.zeros(part.n_pad - N, t.shape[1], dtype=t.dtype)))   # noqa: E731
            if mode == "nodes":
                x_local = pad(x_nm)[part.r0:part.r1].to(dev)
            else:
                g0, g1 = part.feature_slice(G)
                x_local = x_nm.view(N, B, G)[:, :, g0:g1].reshape(N, B * (g1 - g0)).contiguous().to(dev)
            dy_rows = pad(dy_nm)[part.r0:part.r1].to(dev)
            hd, bd = h.to(dev), b.to(dev)
            with torch.no_grad():
                for _ in range(2):                               # twice: symmetric buffers are reused across calls
                    y_rows = part.forward(hd, x_local, bd, B=B)
                dh, dx, db = part.backward(hd, x_local, dy_rows, B=B, want_db=True)
            ys = [torch.empty((R, B * F), dtype=dtype, device=dev) for _ in range(world)]
            dist.all_gather(ys, y_rows.contiguous())
            if mode == "nodes":
                dxs = [torch.empty((R, B * G), dtype=dtype, device=dev) for _ in range(world)]
                dist.all_gather(dxs, dx.contiguous())
                dx_full = torch.cat(dxs)[:N]
            else:
                per = (G + world - 1) // world
                mine = torch.zeros(N, B, per, dtype=dtype, device=dev)
                g0, g1 = part.feature_slice(G)
                mine[:, :, :g1 - g0] = dx.reshape(N, B, g1 - g0)
                dxs = [torch.empty_like(mine) for _ in range(world)]
                dist.all_gather(dxs, mine)
                dx_full = torch.cat([d[:, :, :max(0, min(G, (p + 1) * per) - min(G, p * per))] for p, d in enumerate(dxs)], dim=2).reshape(N, B * G)
            if rank == 0:
                key = "%s_%s" % (mode, "f32" if dtype == torch.float32 else "f64")
                errs = {"y": max_rel(torch.cat(ys)[:N], want["y"]), "dh": max_rel(dh, want["dh"]),
                        "dx": max_rel(dx_full, want["dx"]), "db": max_rel(db, want["db"]), "tol": tol,
                        "fused": bool(part.fused)}
                if mode == "nodes" and part._arenas:
                    errs["symmetric_memory"] = next(iter(part._arenas.values())).kind
                errs["ok"] = bool(max(errs[k] for k in ("y", "dh", "dx", "db")) < tol)
                res[key] = errs
            part.close()
            del part
    return res


def multi_gpu_arm(ctx, w, out_fd):
    from gnn_b200.distributed import PartitionedLSIGF
    args, dev, tdt, es, lib, dist = ctx.args, ctx.dev, ctx.tdt, ctx.es, ctx.lib, ctx.dist
    world, rank = ctx.world, ctx.rank
    E, K, G, F, B, N = w["E"], w["K"], w["G"], w["F"], w["B"], w["N"]
    gso = make_gso(w).astype(tdt)
    nnz_e = gso.nnz() // E
    ops_per_step = float(gso.nnz()) * (K - 1) * B * G
    h_cpu, b_cpu = seeded_taps(w, tdt)
    h, b = h_cpu.to(dev), b_cpu.to(dev)
    x_nm = torch.randn(N, B * G, generator=torch.Generator().manual_seed(1)).to(tdt)     # same full x on every rank
    out = {}

    def build(mode):
        part = PartitionedLSIGF(gso, mode=mode, device=dev, fused=False if args.no_fused else None, fence=args.fence,
                                symm_backend=args.symm, multicast=args.multicast)
        if mode == "grid":
            x_local = part.grid_tile(x_nm, B, G).to(dev)        # rows of my row group x features of my column group
        elif mode == "nodes":
            xp = torch.cat((x_nm, torch.zeros(part.n_pad - N, B * G, dtype=tdt)))
            x_local = xp[part.r0:part.r1].contiguous().to(dev)
        else:
            g0, g1 = part.feature_slice(G)
            x_local = x_nm.view(N, B, G)[:, :, g0:g1].reshape(N, B * (g1 - g0)).contiguous().to(dev)
        fwd = lambda: part.forward(h, x_local, b, B=B)          # noqa: E731
        graphed = False
        if (not args.no_graph) and part.fused and args.fence == "flags":
            try:
                with torch.no_grad():
                    fwd = part.graphed(h, x_local, b, B=B)
                graphed = True
            except Exception as exc:                             # keep the eager step; say why
                out.setdefault("graph_errors", {})[mode] = repr(exc)[:200]
        return part, x_local, fwd, graphed

    modes = ["nodes", "features"] if args.mode == "auto" else [args.mode]
    vq = 8 if tdt == torch.float32 else 4
    if args.mode == "auto" and world >= 4 and world % 2 == 0 and G % (world // 2) == 0 and (G // (world // 2)) % vq == 0 \
            and B * (G // (world // 2)) >= 2 * vq and not args.no_fused:
        modes.append("grid")                                     # 2-D process grid (2 row groups x world/2 column groups)
    want = None
    if not args.no_check and rank == 0:                          # fp64 CPU oracle at full size, once, before any timing
        t0 = time.time()
        want = oracle_forward_nm(gso, h_cpu, b_cpu, x_nm, B, G)
        oracle_s = time.time() - t0
    tried = {}
    tried_fb = {}
    parity = {}
    built = {}
    for mode in modes:
        try:
            built[mode] = build(mode)
        except Exception as exc:                                 # a sharding that cannot be built here is skipped, loudly
            out.setdefault("modes_skipped", {})[mode] = repr(exc)[:200]
            ok_t = torch.tensor([0], device=dev)
        else:
            ok_t = torch.tensor([1], device=dev)
        dist.all_reduce(ok_t, op=dist.ReduceOp.MIN)
        if int(ok_t.item()) == 0:
            if mode in built:
                built.pop(mode)[0].close()
            out.setdefault("modes_skipped", {}).setdefault(mode, "failed on another rank")
            continue
        with torch.no_grad():
            ms_probe, _ = ctx.timed(built[mode][2], 5, 3)
        tried[mode] = ms_probe
        if not args.no_check:                                    # every probed sharding is checked; a wrong one is never timed
            with torch.no_grad():
                y_rows = built[mode][2]().contiguous()
            ys = [torch.empty_like(y_rows) for _ in range(world)]
            dist.all_gather(ys, y_rows)
            good = torch.tensor([1], device=dev)
            if rank == 0:
                parity[mode] = max_rel(torch.cat(ys)[:N], want)
                good[0] = 1 if parity[mode] < ctx.tol else 0
            dist.broadcast(good, 0)
            del ys
            if int(good.item()) == 0:
                tried.pop(mode)
                built.pop(mode)[0].close()
                out.setdefault("modes_skipped", {})[mode] = "parity_max_rel %.3e above tolerance" % parity.get(mode, float("nan"))
                continue
        if not args.no_bwd and mode != "grid":   # forward + the collective backward (dh, db all-reduced; dx sharded like x)
            part_m, x_m = built[mode][0], built[mode][1]
            dy_rows = torch.randn(part_m.rows_per_rank, B * F, generator=torch.Generator().manual_seed(100 + rank)).to(dev, tdt)

            def fwd_bwd(part_m=part_m, x_m=x_m, dy_rows=dy_rows):
                part_m.forward(h, x_m, b, B=B)
                part_m.backward(h, x_m, dy_rows, B=B, want_db=True)

            with torch.no_grad():
                tried_fb[mode], _ = ctx.timed(fwd_bwd, max(3, args.steps // 4), 2)
    if not tried:
        raise SystemExit("bench.py: no multi-GPU sharding passed its parity check: %r" % out.get("modes_skipped"))
    mode = min(tried, key=tried.get)
    if len(modes) > 1:
        pick = torch.tensor([modes.index(mode)], device=dev)
        dist.broadcast(pick, 0)                                  # every rank times the same sharding
        mode = modes[int(pick.item())]
    for m in list(built):
        if m != mode:
            built.pop(m)[0].close()                              # collective: every rank drops the same sharding
            torch.cuda.empty_cache()
    part, x_local, fwd, graphed = built[mode]
    hops = E * (K - 1)
    cap = hops * (args.steps + args.warmup)
    if not graphed:
        lib.b200gf_profile_hops(part.plan.handle, cap)
    with torch.no_grad(), ClockSampler(ctx.local) as clk:
        ms, launches = ctx.timed(fwd, args.steps, args.warmup)
    hop_ms = []
    if not graphed:
        hop_ms = ctypes_floats(lib, part.plan, cap)[hops * args.warmup:]
        lib.b200gf_profile_hops(part.plan.handle, 0)
    else:
        # a replayed graph launches no kernel from the host: count the graph's kernels once by running one eager step,
        # and time the hops in a separate eager pass (same kernels, same buffers)
        with torch.no_grad():
            lib.b200gf_launch_count(1)
            part.forward(h, x_local, b, B=B)
            launches = int(lib.b200gf_launch_count(1)) * args.steps
            lib.b200gf_profile_hops(part.plan.handle, hops * 8)
            for _ in range(8):
                part.forward(h, x_local, b, B=B)
            torch.cuda.synchronize()
            hop_ms = ctypes_floats(lib, part.plan, hops * 8)[hops * 3:]
            lib.b200gf_profile_hops(part.plan.handle, 0)
        dist.barrier()     # eager and replayed steps alternate the double-buffered operands independently: never overlap them
    # parity of the TIMED path at full size, after the timed region: gather every rank's rows, compare on rank 0
    if not args.no_check:
        with torch.no_grad():
            y_rows = fwd().contiguous()
        ys = [torch.empty_like(y_rows) for _ in range(world)]
        dist.all_gather(ys, y_rows)
        if rank == 0:
            out["parity_max_rel"] = max_rel(torch.cat(ys)[:N], want)
            out["parity_note"] = "all %d x %d outputs (rows gathered from %d ranks) vs the fp64 CPU oracle at full size (%.1f s on the host)" % (N, B * F, world, oracle_s)
            out["modes_parity"] = parity
        del ys
        dist.barrier()
    # e2e: every rank copies its shard in from pinned host memory and its result rows back
    xh = x_local.cpu().pin_memory()
    if graphed:
        def compute(xd):
            x_local.copy_(xd)
            return fwd().contiguous()
    else:
        compute = lambda xd: part.forward(h, xd, b, B=B).contiguous()   # noqa: E731
    pipe = E2EPipeline(dev, xh, (part.rows_per_rank, B * F), compute)
    yh = pipe.yh[0]
    with torch.no_grad():
        ms_e2e, _ = ctx.timed(pipe.step, args.steps, 3)
    del pipe
    if tried_fb:              # training step: the sharding with the faster forward + backward (may differ from the forward's)
        best = min(tried_fb, key=tried_fb.get)
        out["fwd_bwd"] = {"ms_per_step": tried_fb[best], "unit": "edge-feature-op/s",
                          "value": float(gso.nnz()) * (K - 1) * B * (G + F) / (tried_fb[best] * 1e-3),
                          "note": "partitioned forward + backward, %s sharding" % best, "modes_probed_ms": tried_fb}
    if mode == "grid":
        c_loc, nnz_loc, rows_loc = B * (G // part.Pc), part.local_nnz // E, part.rows_per_group
    elif mode == "nodes":
        c_loc, nnz_loc, rows_loc = B * G, part.local_nnz // E, part.rows_per_rank
    else:
        g0, g1 = part.feature_slice(G)
        c_loc, nnz_loc, rows_loc = B * (g1 - g0), nnz_e, N
    rf = hop_roofline(ctx, hop_ms, ms * max(1, len(hop_ms) // max(hops, 1)), nnz_loc, rows_loc, c_loc,
                      "hop kernel, rank 0 shard: %d rows x %d columns, %d nnz%s" %
                      (rows_loc, c_loc, nnz_loc, " (fused all-gather epilogue)" if mode == "nodes" and part.fused else
                       (" (all-gather + scatter epilogue)" if mode == "grid" else "")), src_rows=N)
    out["roofline"] = rf
    out["e2e"] = {"value": ops_per_step / (ms_e2e * 1e-3), "unit": "edge-feature-op/s",
                  "h2d_bytes_per_step": xh.numel() * es * world, "d2h_bytes_per_step": yh.numel() * es * world,
                  "ms_per_step": ms_e2e}
    out["clocks"] = clk.summary()
    out["modes_probed_ms"] = tried
    symm = None
    if mode in ("nodes", "grid") and part._arenas:
        symm = next(iter(part._arenas.values())).kind
    if mode == "grid":
        how = " (%d row groups x %d column groups; all-gather in the column group + scatter in the row group fused into the hop kernel: %s, peer-flag fences)" % (part.Pr, part.Pc, symm)
    elif mode == "nodes" and part.fused:
        how = " (all-gather fused into the hop kernel: %s, peer-flag fences)" % symm
    else:
        how = " (fused hop+NVLink scatter, %s fence)" % args.fence if part.fused else " (NCCL collectives)"
    parallelism = "%s-partition x%d%s%s" % (mode, world, how, ", CUDA graph" if graphed else "")
    if not args.no_selftest:
        st = multi_gpu_selftest(ctx)
        if rank == 0:
            out["selftest"] = st
    lt = torch.tensor([launches], device=dev)
    dist.all_reduce(lt)                                           # launches of all ranks inside the timed region
    if rank == 0:
        line = {
            "metric": "LSIGF edge-feature ops/s", "value": ops_per_step / (ms * 1e-3), "unit": "edge-feature-op/s",
            "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": True,
            "scaling": "strong", "vs_baseline": None, "dtype": args.dtype, "data": "synthetic",
            "config": {"workload": describe(w, args.dtype), "name": args.workload, "nnz": gso.nnz(), "parallelism": parallelism,
                       "l2": "inputs larger than L2 (x and every z_k are %d MB each; no flush needed)" % (N * B * G * es // 2 ** 20)
                       if N * B * G * es > L2_BYTES else "working set fits L2: numbers are L2-warm",
                       "ops_per_step": ops_per_step,
                       "note": "x is the node-major shard each rank owns (layout conversion is not part of the N > 1 step)"},
            "gpu_launches": int(lt.item()),
        }
        line.update(out)
        bad = []
        if "parity_max_rel" in line and not line["parity_max_rel"] < ctx.tol:
            bad.append("parity_max_rel %.3e" % line["parity_max_rel"])
        for k, v in line.get("selftest", {}).items():
            if not v.get("ok", False):
                bad.append("selftest %s" % k)
        line["parity_ok"] = not bad
        out_fd.emit(json.dumps(line))
        if bad:
            sys.stderr.write("bench.py: PARITY FAILURE: %s\n" % ", ".join(bad))
    dist.barrier()
    code = 0
    flag = torch.tensor([1 if (rank == 0 and not line["parity_ok"]) else 0], device=dev)
    dist.all_reduce(flag)
    if int(flag.item()):
        code = 3
    dist.destroy_process_group()
    if code:
        sys.exit(code)


DUMP_BYTES = 32 * 2 ** 20   # what --dump-outputs writes at most (all files together stay far below 64 MB)


def dump_outputs(dirname, y):
    """Writes the timed path's output y [B, F, N] (what LSIGF returns) to DIR/y.npy in its own float type: all of it when it
    fits DUMP_BYTES, else the columns of a fixed seeded sample of nodes, sorted, whose indices go to DIR/y_nodes.npy
    (float64, exact).  Inputs are seeded, so two builds run with the same arguments can be compared file by file."""
    os.makedirs(dirname, exist_ok=True)
    B, F, N = y.shape
    es = y.element_size()
    n = min(N, max(1, DUMP_BYTES // (B * F * es)))
    if n < N:
        nodes = np.sort(np.random.default_rng(0).choice(N, n, replace=False))
        y = y[:, :, torch.from_numpy(nodes).to(y.device)]
        np.save(os.path.join(dirname, "y_nodes.npy"), nodes.astype(np.float64))
    np.save(os.path.join(dirname, "y.npy"), y.detach().cpu().numpy())


def run_gpu_arm(args, w):
    out_fd = _JsonOnlyStdout()
    ctx = Ctx(args)
    if ctx.world > 1:
        return multi_gpu_arm(ctx, w, out_fd)
    res, gso = single_gpu_workload(ctx, args.workload, w, args.steps, args.warmup, full=True,
                                   keep_last=bool(args.dump_outputs))
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, res.pop("last_output"))
    line = {
        "metric": "LSIGF edge-feature ops/s", "value": res["value"], "unit": "edge-feature-op/s",
        "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "ms_per_step": res["ms_per_step"], "higher_is_better": True,
        "scaling": "strong", "vs_baseline": None, "dtype": args.dtype, "data": "synthetic",
        "config": {"workload": describe(w, args.dtype), "name": args.workload, "nnz": res["nnz"], "parallelism": "single",
                   "l2": res["l2"], "ops_per_step": res["ops_per_step"]},
    }
    for k in ("gpu_launches", "roofline", "e2e", "fwd_bwd", "clocks", "parity_max_rel", "parity_note"):
        if k in res:
            line[k] = res[k]
    bad = []
    if "parity_max_rel" in res and not res["parity_max_rel"] < ctx.tol:
        bad.append("%s parity_max_rel %.3e" % (args.workload, res["parity_max_rel"]))
    # the other single-GPU configurations of BASELINE.json, same run, fewer steps
    extra = [c for c in args.configs.split(",") if c and c != args.workload] if args.configs else []
    if extra:
        line["configs"] = {}
    for name in extra:
        torch.cuda.empty_cache()
        if name == "cfg4ev":
            try:
                r = edge_variant_workload(ctx, max(3, min(args.steps, 5)), 3)
                line["configs"][name] = r
                if r.get("parity_max_rel") is not None and not r["parity_max_rel"] < ctx.tol:
                    bad.append("cfg4ev parity_max_rel %.3e" % r["parity_max_rel"])
            except Exception as exc:
                line["configs"][name] = {"error": repr(exc)[:300]}
            continue
        try:
            r, _ = single_gpu_workload(ctx, name, WORKLOADS[name], max(3, min(args.steps, 10)), 3, full=False)
            rf = r.get("roofline") or {}
            line["configs"][name] = {"workload": describe(WORKLOADS[name], args.dtype), "ms_per_step": r["ms_per_step"],
                                     "value": r["value"], "unit": r["unit"], "parity_max_rel": r.get("parity_max_rel"),
                                     "hop_frac_of_hbm_peak": rf.get("frac"), "hop_ms": rf.get("ms_per_launch"),
                                     "hop_share": rf.get("kernel_share_of_step"), "gpu_launches": r["gpu_launches"],
                                     "l2": r["l2"], "clocks": r["clocks"]}
            if r.get("parity_max_rel") is not None and not r["parity_max_rel"] < ctx.tol:
                bad.append("%s parity_max_rel %.3e" % (name, r["parity_max_rel"]))
        except Exception as exc:   # an extra config must not take the headline line down with it
            line["configs"][name] = {"error": repr(exc)[:300]}
    if not args.no_cpu_baseline:
        _, _, block = cpu_baseline_block(w, reps=5)
        line["cpu_baseline"] = block
        if w["B"] * w["G"] <= 256:   # second CPU line at the FULL graph size: sparse torch restatement, not reference code
            try:
                line["cpu_sparse_baseline"] = cpu_sparse_sample(w, gso, usable_cores())
            except Exception as exc:  # never let the extra baseline break the bench line
                line["cpu_sparse_baseline"] = {"error": str(exc)[:200]}
    line["parity_ok"] = not bad
    out_fd.emit(json.dumps(line))
    if bad:
        sys.stderr.write("bench.py: PARITY FAILURE: %s\n" % ", ".join(bad))
        sys.exit(3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--workload", default="er1m", choices=sorted(WORKLOADS))
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--mode", default="auto", choices=["auto", "nodes", "features", "grid"],
                    help="multi-GPU sharding (DESIGN.md §4): node rows (north_star), feature columns, the 2-D grid of both "
                         "(4 / 8 GPUs), or probe all that apply, check each against the oracle and time the fastest (default)")
    ap.add_argument("--dtype", default="f32", choices=["f32", "f64"], help="arithmetic type (headline: f32)")
    ap.add_argument("--configs", default="cfg2,cfg3,cfg4,cfg4ev",
                    help="N = 1: other BASELINE.json configurations measured in the same run ('' = none)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the last step's output to DIR/*.npy (single GPU; a seeded sample of "
                         "nodes when it is larger than 32 MB)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-full-size-cpu", action="store_true", help="reference arm: skip the full-size sparse CPU figure")
    ap.add_argument("--no-check", action="store_true", help="skip the full-size parity check against the CPU oracle")
    ap.add_argument("--no-selftest", action="store_true", help="multi-GPU: skip the small forward+backward self-test")
    ap.add_argument("--no-bwd", action="store_true", help="multi-GPU: skip the forward + partitioned backward timing")
    ap.add_argument("--fence", default="flags", choices=["flags", "nccl"],
                    help="multi-GPU fused path: peer flags in symmetric memory (default) or a 4-byte NCCL all-reduce")
    ap.add_argument("--no-graph", action="store_true", help="multi-GPU fused path: do not replay the step as a CUDA graph")
    ap.add_argument("--no-fused", action="store_true", help="multi-GPU: NCCL collectives instead of the fused kernels")
    ap.add_argument("--multicast", action="store_true",
                    help="node sharding: write every row once with multimem.st (NVSwitch multicast) instead of P peer stores")
    ap.add_argument("--symm", default="auto", choices=["auto", "torch", "ipc"],
                    help="node sharding: symmetric memory through torch (multicast when available) or plain CUDA IPC")
    args = ap.parse_args()
    if args.dump_outputs and (args.gpus != 1 or args.impl != "b200"):
        ap.error("--dump-outputs is for the single-GPU CUDA path (--gpus 1)")
    args.warmup = max(3, args.warmup)
    w = WORKLOADS[args.workload]
    if args.impl == "reference":
        run_reference_arm(args, w)
    else:
        run_gpu_arm(args, w)


if __name__ == "__main__":
    main()
