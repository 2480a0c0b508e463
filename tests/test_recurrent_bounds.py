"""The recurrent and time-varying graph layers on the GPU, held to the componentwise fp64 bounds of
oracle/recurrent_oracle.py on the kernel branches they really launch.

Each row of RECURRENT_CASES runs one layer forward and backward (GatedGRNN, the gated HiddenStates, LSIGF_DB, GRNN_DB)
at a shape that reaches the named kernels through the layer's own data movement: node-major recurrent states fed back
with ld = B*H, the [1, G, M] space-time view of LSIGF_DB, the delay-line hops of GRNN_DB on one multi-operator plan with
dst = empty_like(src).  Every output, input gradient and parameter gradient is compared with the oracle's (v, beta), and
a rerun must be bit-identical.  The oracle runs once per row, deferred to check_case (not inside the traced child run).
The _SlabOps rows call the delay-line hop directly for every operator and direction, into SENT-filled destinations
with rows past R and columns past C as canaries and NaN in the source's pad columns.  Operands follow the case builders of tests/test_recurrent_oracle.py (|S| row and column
sums <= 1, contracting hidden taps, positive-mean signals).  The table is checked on the CPU by
tests/test_dispatch_tables.py (its kernel regexes against the built library).
"""
import numpy as np
import pytest
import torch

import lsigf_oracle as orc
import recurrent_oracle as ro
from dispatch_harness import F32, F64, NPD, SENT, Result, _check, _graph, _lib, _st, check_case, child_traced
from test_recurrent_oracle import (db_gso, grnn_case, grnn_db_case, hidden_case, lsigf_db_case, oracle_grnn,
                                   oracle_grnn_db, oracle_hidden, oracle_lsigf_db, run_grnn, run_grnn_db, run_hidden,
                                   run_lsigf_db)

_CASES, _ORACLE = {}, {}


def _case(cid, build):
    """The row's inputs, built once per process."""
    if cid not in _CASES:
        _CASES[cid] = build()
    return _CASES[cid]


def _result(cid, got, oracle):
    """Result with every output the oracle bounds.  The references are deferred: check_case computes the fp64 oracle once
    per row when it checks it, never inside a traced run or a rerun."""
    def ref(k, shape):
        def get():
            if cid not in _ORACLE:
                _ORACLE[cid] = oracle()
            v, beta = _ORACLE[cid][k]
            assert v.size == int(np.prod(shape)), (k, v.shape, shape)
            return v.reshape(shape), beta.reshape(shape)
        return get
    res = Result()
    for k in sorted(got):
        if got[k] is None:
            continue
        t = got[k].detach()
        res.checks.append((k, t, ref(k, tuple(t.shape)), None))
        res.outputs.append(t.clone())
    assert len(res.checks) >= 4, sorted(got)
    return res


def _gso(c, dtype):
    import gnn_b200
    return gnn_b200.SparseGSO.from_scipy(c["S"], dtype=dtype)


def _er_graph(N):
    """graphs.er_gso(N, 8) as a scipy CSR (the builders rescale it)."""
    import scipy.sparse as sp
    from gnn_b200.graphs import er_gso
    rowptr, col, val = er_gso(N, 8, seed=7, dtype=torch.float64).csr[0]
    return sp.csr_matrix((val, col, rowptr), shape=(N, N))


def _grnn_row(dtype, graph_N, graph="rand", **kw):
    def run():
        assert not torch.backends.cuda.matmul.allow_tf32
        cid = ("grnn", dtype, graph_N, graph, tuple(sorted(kw.items())))
        gso = (lambda: _graph("rand", graph_N)) if graph == "rand" else (lambda: _er_graph(graph_N))
        c = _case(cid, lambda: grnn_case(1, graph_N, dtype=NPD[dtype], gso=gso(), **kw))
        got = run_grnn(c, dtype, "cuda", _case(cid + ("gso",), lambda: _gso(c, dtype)))
        torch.cuda.synchronize()
        return _result(cid, got, lambda: oracle_grnn(c, NPD[dtype]))
    return run


def _hidden_row(dtype, kind, N, **kw):
    def run():
        assert not torch.backends.cuda.matmul.allow_tf32
        cid = ("hidden", dtype, kind, N, tuple(sorted(kw.items())))
        c = _case(cid, lambda: hidden_case(2, kind, N, dtype=NPD[dtype], gso=_graph("rand", N), **kw))
        got = run_hidden(c, dtype, "cuda", _case(cid + ("gso",), lambda: _gso(c, dtype)))
        torch.cuda.synchronize()
        return _result(cid, got, lambda: oracle_hidden(c, NPD[dtype]))
    return run


def _lsigf_db_row(dtype, **kw):
    def run():
        cid = ("lsigf_db", dtype, tuple(sorted(kw.items())))
        c = _case(cid, lambda: lsigf_db_case(3, dtype=NPD[dtype], **kw))
        got = run_lsigf_db(c, dtype, "cuda")
        torch.cuda.synchronize()
        return _result(cid, got, lambda: oracle_lsigf_db(c, NPD[dtype]))
    return run


def _grnn_db_row(dtype, **kw):
    def run():
        assert not torch.backends.cuda.matmul.allow_tf32
        cid = ("grnn_db", dtype, tuple(sorted(kw.items())))
        c = _case(cid, lambda: grnn_db_case(4, dtype=NPD[dtype], **kw))
        got = run_grnn_db(c, dtype, "cuda")
        torch.cuda.synchronize()
        return _result(cid, got, lambda: oracle_grnn_db(c, NPD[dtype]))
    return run


def _slab_row(dtype, B, T, N, E, C, zero_t):
    """delayed._SlabOps directly: the plan of (T-1)*E delay-line operators of one GSO batch (S[:, zero_t] all zero: an
    empty operator in the middle of the plan).  Every operator o, HOP_FWD (A_o^T src) and HOP_BWD (A_o src), for
    src / dst with ld = C (the delay line's own layout: no pad column) and ld = C + pad; dst [R+2, ld] starts as SENT,
    pad columns of src hold NaN.  Each result is held to dot_bound against the scipy operators of ro.slab_ops, the
    columns past C and the two rows past R must keep SENT."""
    def run():
        import gnn_b200
        from gnn_b200 import delayed
        cabi, lib = _lib()
        cid = ("slab", dtype, B, T, N, E, C, zero_t)
        npd = NPD[dtype]

        def build():
            rng = np.random.default_rng(5)
            S = db_gso(rng, B, T, E, N, npd, zero={(b, zero_t) for b in range(B)})
            X = ro.rounded(orc.biased_uniform(rng, (B * N, C)), npd)
            return S, X, ro.slab_ops(S), delayed._SlabOps(torch.tensor(S, dtype=dtype, device="cuda"))
        S, X, A, ops = _case(cid, build)
        R = B * N
        assert len(A) == (T - 1) * E and A[(zero_t - 1) * E].nnz == 0
        q = 32 // np.dtype(npd).itemsize
        res = Result()
        for ld in (C, C + q):
            src = torch.full((R, ld), float("nan"), dtype=dtype, device="cuda")
            src[:, :C] = torch.tensor(X, dtype=dtype)
            for o in range(len(A)):
                for direction, M in ((cabi.HOP_FWD, A[o].T.tocsr()), (cabi.HOP_BWD, A[o])):
                    dst = torch.full((R + 2, ld), SENT, dtype=dtype, device="cuda")
                    _check(lib.b200gf_hop(ops.plan.handle, o, direction, src.data_ptr(), ld, dst.data_ptr(), ld, C, _st()))
                    n = np.maximum(np.diff(M.indptr), 1)[:, None]
                    name = "o%d-dir%d-ld%d" % (o, direction, ld)
                    res.checks.append((name, dst[:R, :C], M @ X, orc.dot_bound(n, abs(M) @ np.abs(X), npd)))
                    res.canaries.append((name + " rows>=R", dst[R:]))
                    if ld > C:
                        res.canaries.append((name + " cols>=C", dst[:, C:]))
                    res.finite.append((name, dst[:R, :C]))
                    res.outputs.append(dst)
        torch.cuda.synchronize()
        return res
    return run


F32C, F64C, TC32 = r"tap_contract_kernel<float>", r"tap_contract_kernel<double>", r"tc_contract_kernel<32>"
V2F8, ROWS = r"spmm_hop_v2_kernel<float,int,8,8,", r"narrow_rowptr_kernel"
# (id, row, kernels); the hop named first is the one of the recurrent state, delay line or space-time input
RECURRENT_CASES = [
    # static GSO: GatedGRNN on the 3000-node graph with every lane mapping's row lengths (dispatch_harness._graph)
    ("rec-grnn-B1-H5-tanh-f32", _grnn_row(F32, 3000, B=1, T=4, F=3, H=5, K=3),       # ld 5: scalar lanes
     [r"spmm_hop_kernel<float,1,32,", F32C]),
    ("rec-grnn-B1-H5-tanh-f64", _grnn_row(F64, 3000, B=1, T=4, F=3, H=5, K=3),
     [r"spmm_hop_kernel<double,1,32,", F64C]),
    ("rec-grnn-B3-H20-relu-f32", _grnn_row(F32, 3000, B=3, T=5, F=4, H=20, K=3, sigma="relu"),   # 240-byte rows
     [r"spmm_hop_kernel<float,4,16,", F32C]),
    ("rec-grnn-B3-H20-relu-f64", _grnn_row(F64, 3000, B=3, T=5, F=4, H=20, K=3, sigma="relu"),
     [r"spmm_hop_v2_kernel<double,int,4,16,", F64C]),
    ("rec-grnn-B4-H32-F16-f32", _grnn_row(F32, 3000, B=4, T=6, F=16, H=32, K=3),
     [r"spmm_hop_v2_kernel<float,int,8,16,", TC32, r"tap_grad_multi_kernel<3>"]),
    ("rec-grnn-B2-H48-F32-K4-f32", _grnn_row(F32, 3000, B=2, T=4, F=32, H=48, K=4),
     [r"spmm_hop_v2_kernel<float,int,8,16,", r"tc_contract_kernel<64>", r"tap_grad_multi_kernel<4>"]),
    ("rec-grnn-B2-H32-F16-f64", _grnn_row(F64, 3000, B=2, T=4, F=16, H=32, K=3),
     [r"spmm_hop_v2_kernel<double,int,4,16,", r"contract_f64_kernel<4>"]),
    ("rec-grnn-time-gates-f32", _grnn_row(F32, 3000, B=2, T=4, F=4, H=32, K=3, gates="time"), [V2F8, TC32]),
    ("rec-grnn-node-gates-f32", _grnn_row(F32, 3000, B=2, T=4, F=4, H=32, K=3, gates="node"), [V2F8, TC32]),
    # N = 300: the bound of Linear(H*N -> 1) grows with gamma_{H*N}; here it stays below a gate's change over one step
    ("rec-time-gated-f32", _hidden_row(F32, "time", 300, B=2, T=4, F=4, H=32, K=3), [V2F8, TC32]),
    ("rec-node-gated-f32", _hidden_row(F32, "node", 3000, B=2, T=4, F=4, H=32, K=3),   # GraphFilter(H -> 1): FMA
     [V2F8, TC32, F32C]),
    ("rec-node-gated-f64", _hidden_row(F64, "node", 3000, B=2, T=4, F=4, H=32, K=3),
     [r"spmm_hop_v2_kernel<double,int,4,16,", r"contract_f64_kernel<4>", F64C]),
    # the hub graph: a 20 000-entry row and column.  The GSO is scaled by the hub's |S| row sum and lsigf_envelope takes
    # the longest row for every element, so this row holds the hub's row and column to their bound; the other rows'
    # hops are checked by the 3000-node rows above, where the bound is not dominated by one long row
    ("rec-grnn-hub-N24000-f32", _grnn_row(F32, 24000, B=2, T=3, F=4, H=32, K=3), [V2F8, TC32]),
    # graphs.er_gso(100 000, degree 8): the recursion at scale against the fp64 oracle
    ("rec-grnn-er-N100000-H64-f32", _grnn_row(F32, 100_000, graph="er", B=2, T=3, F=4, H=64, K=3),
     [r"spmm_hop_v2_kernel<float,int,8,16,", r"tc_contract_kernel<64>"]),
    # time-varying GSO: LSIGF_DB on the space-time operator built on the device
    ("rec-lsigf-db-flocking-f32", _lsigf_db_row(F32, B=20, T=60, N=50, G=6, F=32, K=3),  # x ld 6, 60 000 nodes
     [r"spmm_hop_kernel<float,1,32,", ROWS]),
    ("rec-lsigf-db-G32-F64-E2-FN-f32", _lsigf_db_row(F32, B=4, T=8, N=50, G=32, F=64, K=3, E=2, bias="FN"),
     [V2F8, r"tc_contract_kernel<64>", r"tap_grad_multi_kernel<5>", ROWS]),
    ("rec-lsigf-db-G16-F32-f64", _lsigf_db_row(F64, B=4, T=8, N=50, G=16, F=32, K=3),
     [r"spmm_hop_v2_kernel<double,int,4,8,", r"contract_f64_kernel<4>", ROWS]),
    ("rec-lsigf-db-T1-f32", _lsigf_db_row(F32, B=3, T=1, N=50, G=6, F=8, K=3),            # an empty operator
     [r"spmm_hop_kernel<float,1,32,", ROWS]),
    ("rec-lsigf-db-zero-block-f32", _lsigf_db_row(F32, B=3, T=5, N=50, G=6, F=8, K=3, zero=((1, 2),)),
     [r"spmm_hop_kernel<float,1,32,", ROWS]),
    # GRNN_DB: delay-line hops on one plan of (T-1)*E operators, dst = empty_like(src), ld = C = (K-1)*H
    ("rec-grnn-db-H32-E2-f32", _grnn_db_row(F32, B=4, T=30, N=50, F=4, H=32, K=3, E=2),   # C = 64, operators 0..57
     [V2F8, ROWS]),
    ("rec-grnn-db-H5-K4-f32", _grnn_db_row(F32, B=4, T=8, N=50, F=3, H=5, K=4),           # C = ld = 15: no pad column
     [r"spmm_hop_kernel<float,1,32,", ROWS]),
    ("rec-grnn-db-H32-f64", _grnn_db_row(F64, B=4, T=8, N=50, F=4, H=32, K=3),
     [r"spmm_hop_v2_kernel<double,int,4,16,", ROWS]),
    ("rec-grnn-db-empty-op-f32", _grnn_db_row(F32, B=4, T=8, N=50, F=4, H=32, K=3, E=2,   # S[:, 3] = 0: operators
                                              zero=tuple((b, 3) for b in range(4))),     # 4 and 5 are empty
     [V2F8, ROWS]),
    ("rec-grnn-db-K1-f32", _grnn_db_row(F32, B=3, T=6, N=50, F=4, H=8, K=1),              # no delay line, no slab plan
     [F32C, r"tap_grad_multi_kernel<1>"]),
    ("rec-grnn-db-T1-f32", _grnn_db_row(F32, B=3, T=1, N=50, F=4, H=8, K=3), [F32C]),
    # delayed._SlabOps directly, every operator and both directions, canaries past C and past R
    ("rec-slab-C15-f32", _slab_row(F32, B=4, T=6, N=50, E=1, C=15, zero_t=3), [r"spmm_hop_kernel<float,1,32,"]),
    ("rec-slab-C64-E2-f32", _slab_row(F32, B=4, T=6, N=50, E=2, C=64, zero_t=3), [V2F8]),
    ("rec-slab-C64-f64", _slab_row(F64, B=4, T=6, N=50, E=1, C=64, zero_t=2), [r"spmm_hop_v2_kernel<double,int,4,16,"]),
]

traced = child_traced("test_recurrent_bounds", "RECURRENT_CASES")


@pytest.mark.gpu
@pytest.mark.parametrize("cid,fn,kernels", RECURRENT_CASES, ids=[c[0] for c in RECURRENT_CASES])
def test_recurrent_case(cid, fn, kernels, traced):
    check_case(cid, fn, kernels, traced[cid])
