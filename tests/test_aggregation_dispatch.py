"""One case per launch branch of the aggregation GNNs' graph product (aggregation.py), each held by
dispatch_harness.check_case to oracle/aggregation_oracle.py's componentwise bound.

The product launches no kernel of its own: every level of the forward (R) and backward (R^T) chains is one b200gf_hop
on a plan from b200gf_plan_create_ops, so the rows name the existing hop instantiations the row width selects, once per
level.  This table owns no kernel (test_kernel_dispatch.py owns them), so it is not one of test_dispatch_tables.py's
TABLES; its CPU tests below check that every regex names a kernel of the built library and that each case's operators
split into the levels its row expects.

Branches: float32 / float64; split depth 1, 2 and 3 in the forward, 1 and 2 in the backward; C = 1; C not a multiple of
the 16- or 32-byte vector; narrow rows (multi-row kernels) and wide rows (32-byte lanes).  Every row checks z and dx
within their bounds, NaN in the input's pad columns unread, canaries beside the input untouched, and bit-identical
reruns.
"""
import functools
import re

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import aggregation_oracle as aao
from dispatch_harness import F32, F64, NPD, SENT, Result, _padded, check_case, child_traced, library_kernels

NAME = {F32: "float", F64: "double"}

# graph name: (N, average degree, selected nodes P, maxN); the depths of the split chains of R and R^T
GRAPHS = {
    "small": (500, 3, 3, 3),        # (1, 1): no row past ROW_SPLIT
    "mid": (3000, 6, 80, 8),        # (2, 2): saturated rows of R (3000 entries), rows of R^T up to P maxN = 640
    "big": (70000, 8, 1, 10),       # (3, 1): saturated rows of 70 000 entries
}
DEPTHS = {"small": (1, 1), "mid": (2, 2), "big": (3, 1)}


@functools.lru_cache(maxsize=None)
def graph(name):
    """A random directed graph plus a ring (so that every node is reached) and the oracle's operator for the first P
    nodes of a fixed random selection."""
    N, deg, P, maxN = GRAPHS[name]
    rng = np.random.default_rng(N)
    rows = np.concatenate([np.repeat(np.arange(N), deg), np.arange(N)])
    cols = np.concatenate([rng.integers(0, N, N * deg), (np.arange(N) + 1) % N])
    A = sp.csr_matrix((rng.uniform(-1, 1, len(rows)) / deg, (rows, cols)), shape=(N, N))
    A.sum_duplicates()
    A.sort_indices()
    sel = rng.choice(N, P, replace=False)
    return A, sel, aao.operator([A], sel, maxN)


def _case(dtype, gname, B, F):
    cache = {}

    def run():
        import gnn_b200
        from gnn_b200 import aggregation
        N, _, P, maxN = GRAPHS[gname]
        A, sel, (R, Rabs, r_err) = graph(gname)
        if "op" not in cache:
            cache["op"] = aggregation.AggregationOperator(gnn_b200.SparseGSO.from_scipy([A]), sel, maxN)
        op = cache["op"]
        fwd, bwd = op.levels(torch.device("cuda"), dtype)
        assert (len(fwd), len(bwd)) == DEPTHS[gname]
        C = B * F
        pc = _padded(C, dtype)
        rng = np.random.default_rng(C + N)
        xh = rng.standard_normal((B, F, N)).astype(NPD[dtype]).astype(np.float64)
        # x: a node-major view of a buffer [N + 1, pc + 8]: NaN in its pad columns [C, pc), SENT past them and in row N
        buf = torch.full((N + 1, pc + 8), SENT, dtype=dtype, device="cuda")
        buf[:N, C:pc] = float("nan")
        buf[:N, :C] = torch.tensor(xh.reshape(C, N).T, dtype=dtype)
        buf.requires_grad_(True)
        x = buf[:N, :C].view(N, B, F).permute(1, 2, 0)
        z = aggregation._aggregate_cuda(op, x)
        dzh = rng.standard_normal(tuple(z.shape))
        z.backward(torch.tensor(dzh, dtype=dtype, device="cuda"))
        dx = buf.grad[:N, :C].view(N, B, F).permute(1, 2, 0)
        if "ref" not in cache:
            zr, zb = aao.forward(R, Rabs, r_err, xh, 1, maxN, NPD[dtype])
            dzr = torch.tensor(dzh, dtype=dtype).double().numpy()
            dxr, dxb = aao.backward(R, Rabs, r_err, dzr, 1, maxN, N, NPD[dtype])
            cache["ref"] = (zr, zb, dxr, dxb)
        zr, zb, dxr, dxb = cache["ref"]
        res = Result()
        res.checks += [("z", z, zr, zb), ("dx", dx, dxr, dxb)]
        res.canaries += [("x row N", buf.detach()[N:]), ("x cols past the pad", buf.detach()[:, pc:])]
        res.finite += [("z", z), ("dx", dx)]
        res.outputs += [z.detach(), dx.detach()]
        return res
    return run


def _rows():
    rows = []
    for dt in (F32, F64):
        n = NAME[dt]
        v4 = 4 if dt == F32 else 2        # elements per 16-byte vector
        v8 = 8 if dt == F32 else 4        # elements per 32-byte vector
        branches = [
            # (id, graph, B, F, kernel regex)
            ("C1-mid", "mid", 1, 1, r"spmm_hop_multirow_kernel<%s,%d,1,8," % (n, v4)),
            ("narrow-unaligned-small", "small", 1, 13 if dt == F32 else 7,
             r"spmm_hop_multirow_v2_kernel<%s,int,%d," % (n, v8)),
            ("narrow-mid", "mid", 1, 29 if dt == F32 else 15, r"spmm_hop_multirow_kernel<%s,%d,8,32," % (n, v4)),
            ("wide-small", "small", 4 if dt == F32 else 2, 25, r"spmm_hop_v2_kernel<%s,int,%d,16," % (n, v8)),
            ("narrow-big", "big", 2, 4 if dt == F32 else 2, r"spmm_hop_multirow_kernel<%s,%d,2,8," % (n, v4)),
            ("wide-big", "big", 4 if dt == F32 else 2, 25, r"spmm_hop_v2_kernel<%s,int,%d,16," % (n, v8)),
        ]
        for cid, g, B, F, k in branches:
            rows.append(("agg-%s-%s" % (n, cid), _case(dt, g, B, F), [k] * sum(DEPTHS[g])))
    return rows


AGGREGATION_CASES = _rows()

traced = child_traced("test_aggregation_dispatch", "AGGREGATION_CASES")


def test_every_regex_matches_a_kernel_in_the_library():
    """A typo in a row's kernel regex fails here, not on the GPU."""
    names = library_kernels()
    if names is None:
        pytest.skip("cuobjdump / cu++filt or the library not available")
    for cid, _, ks in AGGREGATION_CASES:
        for k in ks:
            assert any(re.search(k, n) for n in names), (cid, k)


@pytest.mark.parametrize("gname", sorted(GRAPHS))
def test_case_operators_split_into_the_expected_levels(gname):
    """The split depths the rows expect, from the oracle's R and R^T; `big` really saturates past 65 536 = 256^2."""
    from gnn_b200.aggregation import split_levels
    A, sel, (R, _, _) = graph(gname)
    RT = R.T.tocsr()
    depth = tuple(len(split_levels(M.indptr, M.indices.astype(np.int32), M.data, M.shape[1])) for M in (R, RT))
    assert depth == DEPTHS[gname]


@pytest.mark.gpu
@pytest.mark.parametrize("cid,fn,kernels", AGGREGATION_CASES, ids=[c[0] for c in AGGREGATION_CASES])
def test_aggregation_dispatch(cid, fn, kernels, traced):
    check_case(cid, fn, kernels, traced[cid])
