"""Windowed hop (csrc/spmm.cu: launch_windows) over the window-major operator copies of b200gf_plan_set_hop_windows.

A plan's hop with a window copy runs one spmm_hop_multirow_v2_kernel launch per (128-byte column chunk, source window):
window 0 stores its sums (EPI_NONE), every later window adds its sums into the destination (EPI_ACCUM).  At test sizes
plan creation builds no window copy, so each row forces one with b200gf_plan_set_hop_windows, names the instantiations
it must launch, and holds both hop directions to the componentwise fp64 bound of tests/test_kernel_dispatch.py.  The same
hop with the copy dropped must agree to 1e-5 (fp32) / 1e-12 (fp64) of max |ref|: only the order of the window sums
differs.  Outputs start as SENT followed by canary rows, pad columns of the source hold NaN, and a rerun must be
bit-identical.  The fused scatter and all-gather epilogues keep the plain hop.
"""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import lsigf_oracle as orc
from dispatch_harness import F32, F64, NPD, SENT, Result, _check, _graph, _lib, _padded, _st, check_case, child_traced


def _wide(dtype):
    return "float,int,8" if dtype == F32 else "double,int,4"


def _win(dtype, mode):
    """The windowed hop's instantiation: 4 lanes x 32 bytes per row chunk, 4-lane row groups, epilogue `mode`."""
    return r"spmm_hop_multirow_v2_kernel<%s,4,4,4,256,%d,3,%d>" % (_wide(dtype), 4 if dtype == F32 else 3, mode)


def _v2(dtype, mode):
    """The plain wide-row hop of 256-byte rows: 8 lanes x 32 bytes, epilogue `mode`."""
    return r"spmm_hop_v2_kernel<%s,8,4,256,%d,3,%d," % (_wide(dtype), 4 if dtype == F32 else 3, mode)


def _plan(gnn_b200, m, dtype):
    return gnn_b200.gso.Plan.from_host_csr([(m.indptr, m.indices, m.data)], m.shape[0], dtype, torch.device("cuda"))


def _hop_case(dtype, C, ld, R, N=3000, graph="rand"):
    """b200gf_hop, both directions, with a window copy of R rows, then again without it."""
    def run():
        import gnn_b200
        cabi, lib = _lib()
        m = _graph(graph, N)
        npd = NPD[dtype]
        mr = sp.csr_matrix((m.data.astype(npd).astype(np.float64), m.indices, m.indptr), shape=m.shape)
        plan = _plan(gnn_b200, m, dtype)
        assert plan.info(8) == 0, "no window copy at test sizes"
        ops = {cabi.HOP_FWD: mr.T.tocsr(), cabi.HOP_BWD: mr}
        g = torch.Generator(device="cpu").manual_seed(C * 7 + ld + R)
        X = torch.randn(N, C, generator=g, dtype=torch.float64).to(dtype)
        src = torch.full((N, ld), float("nan"), dtype=dtype, device="cuda")
        src[:, :C] = X.cuda()
        Xd = X.double().numpy()
        res = Result()
        outs = {}
        for rows in (R, 0):
            _check(lib.b200gf_plan_set_hop_windows(plan.handle, rows))
            assert plan.info(8) == rows
            for direction, op in ops.items():
                dst = torch.full((N + 3, ld), SENT, dtype=dtype, device="cuda")
                _check(lib.b200gf_hop(plan.handle, 0, direction, src.data_ptr(), ld, dst.data_ptr(), ld, C, _st()))
                outs[rows, direction] = dst
                if rows == 0:
                    continue
                ref = op @ Xd
                lens = np.diff(op.indptr)[:, None]
                res.checks.append(("dir%d" % direction, dst[:N, :C], ref,
                                   orc.dot_bound(np.maximum(lens, 1), abs(op) @ np.abs(Xd), npd)))
                res.canaries.append(("cols>=padded", dst[:, min(ld, _padded(C, dtype)):]))
                res.canaries.append(("rows>=N", dst[N:]))
                res.outputs.append(dst[:N, :C])
                res.finite.append(("valid", dst[:N, :C]))
        tol = 1e-5 if dtype == F32 else 1e-12
        for direction in ops:
            a, b = outs[R, direction][:N, :C], outs[0, direction][:N, :C]
            scale = float(b.double().abs().max()) or 1.0
            assert float((a.double() - b.double()).abs().max()) <= tol * scale, "windows vs none: dir %d" % direction
        if graph == "sym":
            assert torch.equal(res.outputs[0], res.outputs[1]), "symmetric S: FWD and BWD must be bit-identical"
        return res
    return run


def _lsigf_case(dtype, R, N=2000, B=8, G=40, F=24, K=4, E=2, graphed=False):
    """LSIGF forward + backward through gnn_b200.LSIGF with window copies of R rows, against the fp64 dense oracle and
    against the same call without them; graphed: the windowed forward + backward also replayed from a CUDA graph, bit
    for bit."""
    def run():
        import gnn_b200
        cabi, lib = _lib()
        c = orc.random_case(5, N=N, B=B, G=G, F=F, K=K, E=E, avg_deg=8, bias="F1")
        rnd = lambda a: torch.tensor(a, dtype=dtype).double().numpy()  # noqa: E731
        gso = gnn_b200.SparseGSO.from_dense(torch.tensor(c["S"], dtype=dtype))
        plan = gso.plan("cuda")
        dy = torch.tensor(c["dy"], dtype=dtype, device="cuda")
        got = {}
        for rows in (R, 0):
            _check(lib.b200gf_plan_set_hop_windows(plan.handle, rows))
            h, x, b = (torch.tensor(c[k], dtype=dtype, device="cuda").requires_grad_(True) for k in ("h", "x", "b"))
            y = gnn_b200.LSIGF(h, gso, x, b)
            y.backward(dy)
            got[rows] = [t.detach().clone() for t in (y, h.grad, x.grad, b.grad)]
        torch.cuda.synchronize()
        res = Result()
        if graphed:
            _check(lib.b200gf_plan_set_hop_windows(plan.handle, R))
            h, x, b = (torch.tensor(c[k], dtype=dtype, device="cuda").requires_grad_(True) for k in ("h", "x", "b"))

            def step():
                h.grad = x.grad = b.grad = None
                y = gnn_b200.LSIGF(h, gso, x, b)
                y.backward(dy)
                return y

            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                step()
            torch.cuda.current_stream().wait_stream(s)
            graph = torch.cuda.CUDAGraph()
            h.grad = x.grad = b.grad = None
            with torch.cuda.graph(graph):
                y_g = gnn_b200.LSIGF(h, gso, x, b)
                y_g.backward(dy)
            graph.replay()
            torch.cuda.synchronize()
            for name, a, e in zip(("y", "dh", "dx", "db"), (y_g, h.grad, x.grad, b.grad), got[R]):
                res.same.append(("graphed %s vs eager" % name, a.detach(), e))
            _check(lib.b200gf_plan_set_hop_windows(plan.handle, 0))
        y_ref = orc.lsigf_dense(rnd(c["h"]), rnd(c["S"]), rnd(c["x"]), rnd(c["b"]))
        dh_ref, dx_ref, db_ref = orc.lsigf_grads_dense(rnd(c["h"]), rnd(c["S"]), rnd(c["x"]), rnd(c["dy"]), (F, 1))
        tol_ref, tol_off = (1e-4, 1e-5) if dtype == F32 else (1e-11, 1e-12)
        for name, out, off, ref in zip(("y", "dh", "dx", "db"), got[R], got[0], (y_ref, dh_ref, dx_ref, db_ref)):
            o = out.double().cpu().numpy().reshape(ref.shape)
            scale = float(np.abs(ref).max())
            assert float(np.abs(o - ref).max()) <= tol_ref * scale, "%s vs the fp64 oracle" % name
            assert float((out.double() - off.double()).abs().max()) <= tol_off * scale, "%s vs no windows" % name
            res.outputs.append(out)
            res.finite.append((name, out))
        return res
    return run


def _epilogue_case(dtype, kind, C=64, ld=64, N=3000, R=1100):
    """The fused scatter (one peer: a local buffer) and all-gather (one peer, no multicast) epilogues on a plan with a
    window copy: the plain hop runs, and both its outputs match the reference."""
    def run():
        import gnn_b200
        cabi, lib = _lib()
        m = _graph("rand", N)
        npd = NPD[dtype]
        mr = sp.csr_matrix((m.data.astype(npd).astype(np.float64), m.indices, m.indptr), shape=m.shape)
        plan = _plan(gnn_b200, m, dtype)
        _check(lib.b200gf_plan_set_hop_windows(plan.handle, R))
        g = torch.Generator(device="cpu").manual_seed(C)
        X = torch.randn(N, C, generator=g, dtype=torch.float64).to(dtype)
        src = torch.full((N, ld), float("nan"), dtype=dtype, device="cuda")
        src[:, :C] = X.cuda()
        op = mr.T.tocsr()
        Xd = X.double().numpy()
        ref = op @ Xd
        bound = orc.dot_bound(np.maximum(np.diff(op.indptr)[:, None], 1), abs(op) @ np.abs(Xd), npd)
        peer = torch.full((N + 3, ld), SENT, dtype=dtype, device="cuda")
        peers = cabi.ptr_array([peer.data_ptr()])
        res = Result()
        if kind == "scatter":
            dst = torch.full((N + 3, ld), SENT, dtype=dtype, device="cuda")
            _check(lib.b200gf_hop_scatter(plan.handle, 0, cabi.HOP_FWD, src.data_ptr(), ld, dst.data_ptr(), ld, C, peers, 1,
                                          N, ld, 0, C, 0, _st()))
            res.checks.append(("dst", dst[:N, :C], ref, bound))
            res.canaries.append(("dst rows>=N", dst[N:]))
            res.outputs.append(dst[:N, :C])
        else:
            _check(lib.b200gf_hop_bcast(plan.handle, 0, cabi.HOP_FWD, src.data_ptr(), ld, C, peers, 1, None, 0, ld, _st()))
        res.checks.append(("peer", peer[:N, :C], ref, bound))
        res.canaries.append(("peer rows>=N", peer[N:]))
        res.outputs.append(peer[:N, :C])
        _check(lib.b200gf_plan_set_hop_windows(plan.handle, 0))
        return res
    return run


def _rows():
    rows = []
    # (dtype, C, ld, R, extra); N = 3000 unless given: R = 1500, 1100, 600, 5000 give 2, 3, 5 and 1 windows
    table = [
        (F32, 61, 64, 1500, {}),
        (F32, 64, 64, 1100, {}),
        (F32, 100, 104, 600, {}),              # four chunks, the last one partial
        (F32, 61, 64, 5000, {}),
        (F64, 29, 32, 1100, {}),
        (F64, 50, 52, 600, {}),
        (F64, 50, 52, 1500, {}),
        (F32, 61, 64, 7000, dict(N=24000)),    # the hub graph: a 20 000-entry row and column
        (F64, 29, 32, 5000, dict(N=24000)),
        (F32, 100, 104, 1100, dict(graph="sym")),
    ]
    for dt, C, ld, R, extra in table:
        N = extra.get("N", 3000)
        tag = "win-%s-C%d-ld%d-R%d%s" % ("f32" if dt == F32 else "f64", C, ld, R,
                                         "".join("-%s%s" % (k, v) for k, v in sorted(extra.items())))
        kernels = [_win(dt, 0)] + ([_win(dt, 4)] if R < N else [])
        rows.append((tag, _hop_case(dt, C, ld, R, **extra), kernels))
    for N in (1, 3, 7):
        rows.append(("win-tinyN%d-f32" % N, _hop_case(F32, 61, 64, 2, N=N, graph="tiny"),
                     [_win(F32, 0)] + ([_win(F32, 4)] if N > 2 else [])))
    rows.append(("win-lsigf-f32", _lsigf_case(F32, 700), [_win(F32, 0), _win(F32, 4)]))
    rows.append(("win-lsigf-f64", _lsigf_case(F64, 900, G=20), [_win(F64, 0), _win(F64, 4)]))
    rows.append(("win-lsigf-graphed-f32", _lsigf_case(F32, 700, graphed=True), [_win(F32, 0), _win(F32, 4)]))
    rows.append(("win-scatter-f32", _epilogue_case(F32, "scatter"), [_v2(F32, 1)]))
    rows.append(("win-bcast-f32", _epilogue_case(F32, "bcast"), [_v2(F32, 2)]))
    return rows


CASES = _rows()


def test_set_hop_windows_rejects_bad_arguments_without_gpu():
    cabi, lib = _lib()
    assert lib.b200gf_plan_set_hop_windows(None, 0) == -1
    assert lib.b200gf_plan_set_hop_windows(None, 1000) == -1
    assert lib.b200gf_plan_set_hop_windows(None, -1) == -1


@pytest.mark.gpu
def test_set_hop_windows_on_a_plan():
    """A negative R is rejected; partitioned and device-built plans take no window copy."""
    import gnn_b200
    cabi, lib = _lib()
    N = 3000
    m = _graph("rand", N)
    plan = _plan(gnn_b200, m, F32)
    assert lib.b200gf_plan_set_hop_windows(plan.handle, -5) == -1
    assert plan.info(8) == 0
    t = m.T.tocsr()
    r0, r1 = N // 3, N // 3 + N // 2
    fwd, bwd = t[r0:r1], m[r0:r1]
    part = gnn_b200.gso.Plan.from_ops([(fwd.indptr, fwd.indices, fwd.data)], [(bwd.indptr, bwd.indices, bwd.data)],
                                      r1 - r0, N, F32, "cuda")
    assert lib.b200gf_plan_set_hop_windows(part.handle, 1000) == -2
    assert lib.b200gf_plan_set_hop_windows(part.handle, 0) == -2
    assert part.info(8) == 0
    dev = lambda a, dt: torch.as_tensor(a).to("cuda", dt)  # noqa: E731
    ops = [(dev(t.indptr, torch.int64), dev(t.indices, torch.int32), dev(t.data, F32))]
    bops = [(dev(m.indptr, torch.int64), dev(m.indices, torch.int32), dev(m.data, F32))]
    devp = gnn_b200.gso.Plan.from_device_ops(ops, bops, N, F32, "cuda")
    assert lib.b200gf_plan_set_hop_windows(devp.handle, 1000) == -2
    assert devp.info(8) == 0


traced = child_traced("test_hop_windows", "CASES")


@pytest.mark.gpu
@pytest.mark.parametrize("cid,fn,kernels", CASES, ids=[c[0] for c in CASES])
def test_window(cid, fn, kernels, traced):
    check_case(cid, fn, kernels, traced[cid])


@pytest.mark.gpu
def test_full_size_windows_on_against_off():
    """bench.py's headline graph (er1m) builds a window copy by default; its LSIGF forward and gradients agree with the
    same plan's without one.  tests/test_gpu_fullsize.py holds the default (windowed) path to the fp64 oracle."""
    import gnn_b200
    from gnn_b200 import graphs
    cabi, lib = _lib()
    N, G, F, K = 1_000_000, 64, 64, 5
    gso = graphs.er_gso(N, 32, seed=1, E=1)
    plan = gso.plan("cuda")
    assert plan.info(8) > 0, "er1m takes the windowed hop by default"
    g = torch.Generator().manual_seed(1234)
    h = (torch.rand(F, 1, K, G, generator=g) * 2 - 1) / np.sqrt(G * K)
    b = (torch.rand(F, 1, generator=g) * 2 - 1) / np.sqrt(G * K)
    x = torch.randn(1, G, N, generator=g)
    dy = torch.randn(1, F, N, generator=g).cuda()
    got = {}
    for rows in (plan.info(8), 0):
        _check(lib.b200gf_plan_set_hop_windows(plan.handle, rows))
        hd, bd, xd = (t.cuda().requires_grad_(True) for t in (h, b, x))
        y = gnn_b200.LSIGF(hd, gso, xd, bd)
        y.backward(dy)
        got[rows] = [t.detach().double() for t in (y, hd.grad, xd.grad, bd.grad)]
    on, off = got.values()
    for name, a, r in zip(("y", "dh", "dx", "db"), on, off):
        scale = float(r.abs().max()) or 1.0
        assert float((a - r).abs().max()) <= 1e-5 * scale, name


@pytest.mark.gpu
def test_rejected_rebuild_leaves_a_symmetric_plan_whole():
    """A window size whose offsets do not fit 32 bits (R = 1 at N = 50 000: W * (N + 1) > 2^31) is EUNSUPPORTED and
    leaves the plan's copies as they were; both hop directions of the symmetric plan still match the reference, bit for
    bit between them."""
    import gnn_b200
    cabi, lib = _lib()
    N, C, R = 50_000, 64, 20_000
    m = _graph("sym", N)
    plan = _plan(gnn_b200, m, F32)
    assert plan.info(6) == 1, "symmetric plan"
    _check(lib.b200gf_plan_set_hop_windows(plan.handle, R))
    assert lib.b200gf_plan_set_hop_windows(plan.handle, 1) == -2
    assert plan.info(8) == R
    mr = sp.csr_matrix((m.data.astype(np.float32).astype(np.float64), m.indices, m.indptr), shape=m.shape)
    g = torch.Generator(device="cpu").manual_seed(11)
    X = torch.randn(N, C, generator=g, dtype=torch.float64).to(F32)
    Xd = X.double().numpy()
    src = X.cuda()
    outs = []
    for direction, op in ((cabi.HOP_FWD, mr.T.tocsr()), (cabi.HOP_BWD, mr)):
        dst = torch.full((N, C), SENT, dtype=F32, device="cuda")
        _check(lib.b200gf_hop(plan.handle, 0, direction, src.data_ptr(), C, dst.data_ptr(), C, C, _st()))
        torch.cuda.synchronize()
        bound = orc.dot_bound(np.maximum(np.diff(op.indptr)[:, None], 1), abs(op) @ np.abs(Xd), np.float32)
        assert orc.bound_violation(dst.double().cpu().numpy(), op @ Xd, bound) <= 1.0, "direction %d" % direction
        outs.append(dst)
    assert torch.equal(outs[0], outs[1])
    _check(lib.b200gf_plan_set_hop_windows(plan.handle, 0))
    assert plan.info(8) == 0
