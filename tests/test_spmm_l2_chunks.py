"""L2-sized column chunks of the wide-row hop (csrc/spmm.cu: hop_chunk_lanes).

When the rows a hop gathers from do not fit the device's L2 at the row width's chunk (L = 8, 16 or 32 lanes of 32 bytes),
spmm_hop_v2_kernel runs narrower chunks (L = 16, 8 or 4).  At test sizes every source fits the L2, so each row here
forces a chunk width with b200gf_plan_set_l2_bytes (an L2 of exactly N * L * 32 bytes), names the kernel instantiation it
must launch, and holds both hop directions to the componentwise fp64 bound of tests/test_kernel_dispatch.py.  The same
hop with the sizing off (L2 = 0, the row width's chunk) must agree to 1e-5 (fp32) / 1e-12 (fp64) of max |ref|: only the
order of the chunk fold differs.  Outputs start as SENT followed by canary rows, pad columns of the source hold NaN, and
a rerun must be bit-identical.  Partitioned plans ignore the override.  When not even 4-lane chunks fit, they are still
taken for rows of at most 256 bytes of a graph whose gathers spread over the whole source if a chunk is at most 3x the
L2; a banded graph and wider rows keep the row width's chunk.
"""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import lsigf_oracle as orc
from dispatch_harness import F32, F64, NPD, SENT, Result, _check, _graph, _lib, _padded, _st, check_case, child_traced


def _band(N, half=20, seed=0):
    """Neighbours within `half` of the row: no gather lands far from the diagonal (a graph with locality)."""
    rng = np.random.default_rng(seed)
    rows = np.repeat(np.arange(N), 2 * half)
    cols = np.clip(rows + rng.integers(-half, half + 1, rows.size), 0, N - 1)
    m = sp.coo_matrix((rng.standard_normal(rows.size), (rows, cols)), shape=(N, N)).tocsr()
    m.sum_duplicates()
    m.sort_indices()
    return m


def _hop_case(dtype, C, ld, lanes, N=3000, graph="rand", plan_kind="full"):
    """b200gf_hop, both directions, with the plan's L2 set to N * lanes * 32 bytes, then again with it at 0."""
    def run():
        import gnn_b200
        cabi, lib = _lib()
        m = _band(N) if graph == "band" else _graph(graph, N)
        npd = NPD[dtype]
        mr = sp.csr_matrix((m.data.astype(npd).astype(np.float64), m.indices, m.indptr), shape=m.shape)
        if plan_kind == "full":
            plan = gnn_b200.SparseGSO.from_scipy([m], dtype=dtype).plan("cuda")
            ops = {cabi.HOP_FWD: mr.T.tocsr(), cabi.HOP_BWD: mr}
            n_rows = N
        else:   # partitioned: rows [r0, r1) of S^T and of S, global columns
            r0, r1 = N // 3, N // 3 + N // 2
            fwd, bwd = mr.T.tocsr()[r0:r1], mr[r0:r1]
            plan = gnn_b200.gso.Plan.from_ops([(fwd.indptr, fwd.indices, fwd.data)], [(bwd.indptr, bwd.indices, bwd.data)],
                                              r1 - r0, N, dtype, "cuda")
            ops = {cabi.HOP_FWD: fwd, cabi.HOP_BWD: bwd}
            n_rows = r1 - r0
        assert plan.info(7) > 0, "plan creation reads the device's L2 size"
        g = torch.Generator(device="cpu").manual_seed(C * 7 + ld)
        X = torch.randn(N, C, generator=g, dtype=torch.float64).to(dtype)
        src = torch.full((N, ld), float("nan"), dtype=dtype, device="cuda")
        src[:, :C] = X.cuda()
        Xd = X.double().numpy()
        res = Result()
        outs = {}
        for l2 in (N * lanes * 32, 0):
            _check(lib.b200gf_plan_set_l2_bytes(plan.handle, l2))
            for direction, op in ops.items():
                dst = torch.full((n_rows + 3, ld), SENT, dtype=dtype, device="cuda")
                _check(lib.b200gf_hop(plan.handle, 0, direction, src.data_ptr(), ld, dst.data_ptr(), ld, C, _st()))
                outs[l2, direction] = dst
                if l2 == 0:
                    continue
                ref = op @ Xd
                lens = np.diff(op.indptr)[:, None]
                res.checks.append(("dir%d" % direction, dst[:n_rows, :C], ref,
                                   orc.dot_bound(np.maximum(lens, 1), abs(op) @ np.abs(Xd), npd)))
                res.canaries.append(("cols>=padded", dst[:, min(ld, _padded(C, dtype)):]))
                res.canaries.append(("rows>=n_rows", dst[n_rows:]))
                res.outputs.append(dst[:n_rows, :C])
                res.finite.append(("valid", dst[:n_rows, :C]))
        _check(lib.b200gf_plan_set_l2_bytes(plan.handle, 0))
        tol = 1e-5 if dtype == F32 else 1e-12
        for direction, op in ops.items():
            a, b = outs[N * lanes * 32, direction][:n_rows, :C], outs[0, direction][:n_rows, :C]
            scale = float(b.double().abs().max()) or 1.0
            assert float((a.double() - b.double()).abs().max()) <= tol * scale, "forced chunk vs L2 = 0: dir %d" % direction
        if graph == "sym":
            assert torch.equal(res.outputs[0], res.outputs[1]), "symmetric S: FWD and BWD must be bit-identical"
        return res
    return run


def _lsigf_case(dtype, lanes, N=2000, B=8, G=40, F=24, K=4, E=2):
    """LSIGF forward + backward (b200gf_forward / b200gf_backward through gnn_b200.LSIGF) with the plan's L2 set to
    N * lanes * 32 bytes, against the fp64 dense oracle and against the same call with the sizing off."""
    def run():
        import gnn_b200
        cabi, lib = _lib()
        c = orc.random_case(5, N=N, B=B, G=G, F=F, K=K, E=E, avg_deg=8, bias="F1")
        rnd = lambda a: torch.tensor(a, dtype=dtype).double().numpy()  # noqa: E731
        gso = gnn_b200.SparseGSO.from_dense(torch.tensor(c["S"], dtype=dtype))
        plan = gso.plan("cuda")
        got = {}
        for l2 in (N * lanes * 32, 0):
            _check(lib.b200gf_plan_set_l2_bytes(plan.handle, l2))
            h, x, b = (torch.tensor(c[k], dtype=dtype, device="cuda").requires_grad_(True) for k in ("h", "x", "b"))
            y = gnn_b200.LSIGF(h, gso, x, b)
            y.backward(torch.tensor(c["dy"], dtype=dtype, device="cuda"))
            got[l2] = [t.detach().clone() for t in (y, h.grad, x.grad, b.grad)]
        torch.cuda.synchronize()
        y_ref = orc.lsigf_dense(rnd(c["h"]), rnd(c["S"]), rnd(c["x"]), rnd(c["b"]))
        dh_ref, dx_ref, db_ref = orc.lsigf_grads_dense(rnd(c["h"]), rnd(c["S"]), rnd(c["x"]), rnd(c["dy"]), (F, 1))
        tol_ref, tol_off = (1e-4, 1e-5) if dtype == F32 else (1e-11, 1e-12)
        res = Result()
        for name, out, off, ref in zip(("y", "dh", "dx", "db"), got[N * lanes * 32], got[0], (y_ref, dh_ref, dx_ref, db_ref)):
            o = out.double().cpu().numpy().reshape(ref.shape)
            scale = float(np.abs(ref).max())
            assert float(np.abs(o - ref).max()) <= tol_ref * scale, "%s vs the fp64 oracle" % name
            assert float((out.double() - off.double()).abs().max()) <= tol_off * scale, "%s vs L2 = 0" % name
            res.outputs.append(out)
            res.finite.append((name, out))
        _check(lib.b200gf_plan_set_l2_bytes(plan.handle, 0))
        return res
    return run


def _v2(dtype, L):
    return r"spmm_hop_v2_kernel<%s,int,%d,%d," % ("float" if dtype == F32 else "double", 32 // (4 if dtype == F32 else 8), L)


def _rows():
    rows = []
    # (dtype, C, ld, forced lanes, expected lanes, extra)
    table = [
        (F32, 1100, 1104, 4, 4, {}),
        (F32, 1100, 1104, 8, 8, {}),
        (F32, 1100, 1104, 16, 16, {}),
        (F32, 100, 104, 8, 8, {}),              # 13 vectors: the second chunk is partial
        (F32, 61, 64, 4, 4, {}),                # 8 vectors, tail pad in the second chunk
        (F32, 64, 64, 4, 4, {}),
        (F64, 600, 600, 4, 4, {}),
        (F64, 600, 600, 8, 8, {}),
        (F64, 29, 32, 4, 4, {}),                # 8 vectors, 3 pad columns in the last chunk
        (F64, 50, 52, 8, 8, {}),
        (F32, 1100, 1104, 4, 4, dict(N=24000)),  # the hub graph: a 20 000-entry row and column
        (F64, 50, 52, 4, 4, dict(N=24000)),
        (F32, 100, 104, 8, 8, dict(graph="sym")),
        (F32, 1100, 1104, 4, 32, dict(plan_kind="ops")),   # partitioned plans keep the row width's chunk
        (F32, 61, 64, 2, 4, {}),                # 4-lane chunks at 2x the L2: random gathers still take them
        (F64, 29, 32, 2, 4, {}),
        (F32, 61, 64, 2, 8, dict(graph="band")),  # ... gathers near the diagonal keep the row width's chunk
        (F32, 61, 64, 1, 8, {}),                # 4-lane chunks at 4x the L2: the row width's chunk stays
        (F64, 50, 52, 2, 16, {}),               # ... and so do 4-lane chunks of rows wider than 256 bytes
    ]
    for dt, C, ld, lanes, want, extra in table:
        tag = "chunk-%s-C%d-ld%d-L%d%s" % ("f32" if dt == F32 else "f64", C, ld, lanes,
                                           "".join("-%s%s" % (k, v) for k, v in sorted(extra.items())))
        rows.append((tag, _hop_case(dt, C, ld, lanes, **extra), [_v2(dt, want)]))
    for N in (1, 3, 7):
        rows.append(("chunk-tinyN%d-f32" % N, _hop_case(F32, 61, 64, 4, N=N, graph="tiny"), [_v2(F32, 4)]))
    rows.append(("chunk-lsigf-f32-L4", _lsigf_case(F32, 4), [_v2(F32, 4)]))
    rows.append(("chunk-lsigf-f64-L8", _lsigf_case(F64, 8, G=20), [_v2(F64, 8)]))
    return rows


CASES = _rows()


def test_set_l2_bytes_rejects_bad_arguments_without_gpu():
    cabi, lib = _lib()
    assert lib.b200gf_plan_set_l2_bytes(None, 0) == -1
    assert lib.b200gf_plan_info(None, 7) == -1


traced = child_traced("test_spmm_l2_chunks", "CASES")


@pytest.mark.gpu
@pytest.mark.parametrize("cid,fn,kernels", CASES, ids=[c[0] for c in CASES])
def test_chunk(cid, fn, kernels, traced):
    check_case(cid, fn, kernels, traced[cid])
