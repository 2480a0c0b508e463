"""One case per launch branch of the localized activations' entry points (b200gf_local_activation_forward / _backward,
csrc/layer.cu), each held by dispatch_harness.check_case to oracle/local_activation_oracle.py's componentwise bound.

The entry points run MaxPoolLocal's kernels, maxpool_fwd_kernel and maxpool_bwd_kernel, generalised in place: the ring
list format selects the K-hop gather-select, the selection argument the max or the lower median.  This table owns no
kernel (test_kernel_dispatch.py owns them), so it is not one of test_dispatch_tables.py's TABLES; its CPU test below
checks that every regex names a kernel of the built library.

Every row checks y within its bound, agg_k and the chosen nodes exact, canaries beside every output, and NaN input pads
unread.  Determinism exemption: the backward scatters w_k dy with atomicAdd, so the order of its additions (and its last
bits) may change from run to run; its rows check only the bounds.  Forward rows rerun bit-identically.
"""
import re

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import local_activation_oracle as lao
from dispatch_harness import (F32, F64, NPD, SENT, Result, _lib, _st, check_case, child_traced, library_kernels)

NAME = {F32: "float", F64: "double"}


def _graph(N, deg, seed, hub=0):
    """Random directed pattern with about `deg` entries per row, nodes 1 and 2 isolated (every prefix of length one),
    and node 0 a hub with `hub` out-neighbours when hub > 0."""
    rng = np.random.default_rng(seed)
    m = sp.random(N, N, density=deg / N, random_state=seed, format="lil")
    for i in (1, 2):
        m[i, :] = 0
        m[:, i] = 0
    if hub:
        m[0, rng.choice(np.arange(3, N), hub, replace=False)] = 1.0
    return sp.csr_matrix(m)


def _case(dtype, op, K, N=700, C=37, deg=3, ties=False, hub=0, backward=False, seed=0):
    """b200gf_local_activation_forward (and _backward): x [N, ld] with NaN pads, y [N+1, ld+2] and agg [K, N+1, ld] of
    SENT, arg [K, N, C]; backward: dx [N+1, ld+1] of SENT (dx = w0 dy is written, not added to)."""
    from gnn_b200.graphtools_sparse import ring_neighborhoods
    cache = {}

    def run():
        cabi, lib = _lib()
        enum = cabi.F32 if dtype == F32 else cabi.F64
        rng = np.random.default_rng(seed + 1000 * K + N + C)
        if "rings" not in cache:
            cache["rings"] = ring_neighborhoods(_graph(N, deg, seed, hub), K)
        rowptr, col, ring_end = cache["rings"]
        xh = rng.standard_normal((N, C))
        if ties:
            xh = np.round(xh * 2) / 2 + 0.0                   # coarse grid: many equal values, no -0
        xh = xh.astype(NPD[dtype]).astype(np.float64)
        wh = rng.uniform(-1, 1, K + 1).astype(NPD[dtype]).astype(np.float64)
        ld = (C + 7) // 8 * 8 + 8
        x = torch.full((N, ld), float("nan"), dtype=dtype, device="cuda")
        x[:, :C] = torch.tensor(xh, dtype=dtype)
        w = torch.tensor(wh, dtype=dtype, device="cuda")
        dev = lambda a: torch.from_numpy(a).cuda()             # noqa: E731
        rp, cl, re_ = dev(rowptr), dev(col), dev(ring_end)
        y = torch.full((N + 1, ld + 2), SENT, dtype=dtype, device="cuda")
        agg = torch.full((K, N + 1, ld), SENT, dtype=dtype, device="cuda")
        arg = torch.full((K, N, C), 0x5A, dtype=torch.int32, device="cuda")
        # agg_k lives at agg + (k-1) N ld: view the first K N rows of the buffer as [K, N, ld]
        aggv = agg.view(-1)[:K * N * ld].view(K, N, ld)
        rc = lib.b200gf_local_activation_forward(enum, op, x.data_ptr(), ld, N, C, rp.data_ptr(), cl.data_ptr(),
                                                 re_.data_ptr(), K, w.data_ptr(), y.data_ptr(), ld + 2, agg.data_ptr(),
                                                 ld, arg.data_ptr(), _st())
        assert rc == 0, lib.b200gf_strerror(rc)
        if "ref" not in cache:
            cache["ref"] = lao.forward(xh, wh, rowptr, col, ring_end, K, op, NPD[dtype])
        yr, yb, aggr, argr = cache["ref"]
        res = Result()
        res.checks.append(("y", y[:N, :C], yr, yb))
        res.same += [("agg_k is the selected value", aggv[:, :, :C].cpu(), torch.tensor(aggr, dtype=dtype)),
                     ("arg_k is the selected node", arg.cpu(), torch.tensor(argr, dtype=torch.int32))]
        res.canaries += [("y cols>=C", y[:, C:]), ("y row N", y[N:]), ("agg cols>=C", aggv[:, :, C:]),
                         ("agg tail", agg.view(-1)[K * N * ld:])]
        res.finite += [("y", y[:N, :C])]
        res.outputs += [y[:N, :C], aggv[:, :, :C], arg]
        if not backward:
            return res
        dyh = rng.standard_normal((N, C)).astype(NPD[dtype]).astype(np.float64)
        dy = torch.full((N, ld), float("nan"), dtype=dtype, device="cuda")
        dy[:, :C] = torch.tensor(dyh, dtype=dtype)
        dx = torch.full((N + 1, ld + 1), SENT, dtype=dtype, device="cuda")
        rc = lib.b200gf_local_activation_backward(enum, dy.data_ptr(), ld, arg.data_ptr(), N, C, K, w.data_ptr(),
                                                  dx.data_ptr(), ld + 1, _st())
        assert rc == 0, lib.b200gf_strerror(rc)
        if "dref" not in cache:
            cache["dref"] = lao.backward(xh, dyh, wh, aggr, argr, NPD[dtype])
        dxr, dxb, _, _ = cache["dref"]
        res.checks.append(("dx", dx[:N, :C], dxr, dxb))
        res.canaries += [("dx cols>=C", dx[:, C:]), ("dx row N", dx[N:])]
        res.outputs.append(dx[:N, :C])
        res.nondeterministic = True
        return res
    return run


def _rows():
    rows = []
    for dt in (F32, F64):
        n = NAME[dt]
        fwd = [r"maxpool_fwd_kernel<%s>" % n]
        bwd = fwd + [r"maxpool_bwd_kernel<%s>" % n] * 2
        for op, opn in ((lao.MAX, "max"), (lao.MEDIAN, "median")):
            for K in (1, 2, 3):
                rows.append(("la-%s-%s-K%d" % (opn, n, K), _case(dt, op, K), fwd))
            rows.append(("la-%s-%s-ties-K2" % (opn, n), _case(dt, op, 2, ties=True, seed=1), fwd))
            rows.append(("la-%s-%s-hub-K2" % (opn, n), _case(dt, op, 2, N=3000, C=13, deg=2, hub=1200, seed=2), fwd))
            rows.append(("la-%s-%s-C1-K1" % (opn, n), _case(dt, op, 1, C=1, seed=3), fwd))
            rows.append(("la-%s-%s-bwd-K2" % (opn, n), _case(dt, op, 2, backward=True, seed=4), bwd))
            rows.append(("la-%s-%s-bwd-ties-K3" % (opn, n), _case(dt, op, 3, C=16, ties=True, backward=True, seed=5),
                         bwd))
    return rows


LOCAL_CASES = _rows()

traced = child_traced("test_local_activation_dispatch", "LOCAL_CASES")


def test_every_regex_matches_a_kernel_in_the_library():
    """A typo in a row's kernel regex fails here, not on the GPU."""
    names = library_kernels()
    if names is None:
        pytest.skip("cuobjdump / cu++filt or the library not available")
    for cid, _, ks in LOCAL_CASES:
        for k in ks:
            assert any(re.search(k, n) for n in names), (cid, k)


def test_hub_row_is_at_least_a_thousand_long():
    from gnn_b200.graphtools_sparse import ring_neighborhoods
    rowptr, _, ring_end = ring_neighborhoods(_graph(3000, 2, 2, 1200), 2)
    assert ring_end[0, 1] > 1000 and int(np.diff(rowptr).max()) > 1000
    assert np.all(ring_end[[1, 2]] == 1)                      # isolated nodes: prefixes of length one


@pytest.mark.gpu
@pytest.mark.parametrize("cid,fn,kernels", LOCAL_CASES, ids=[c[0] for c in LOCAL_CASES])
def test_local_activation_dispatch(cid, fn, kernels, traced):
    check_case(cid, fn, kernels, traced[cid])


def test_entry_points_reject_bad_arguments_before_any_launch():
    """EINVAL / EUNSUPPORTED with null device pointers never dereferenced: no GPU is needed."""
    import ctypes
    cabi, lib = _lib()
    p = ctypes.c_void_p(16)                                   # never dereferenced: every call fails its checks first
    fwd = lambda dtype=cabi.F32, op=0, x=p, x_ld=8, N=4, C=8, K=1, y_ld=8, agg_ld=8, w=p: \
        lib.b200gf_local_activation_forward(dtype, op, x, x_ld, N, C, p, p, p, K, w, p, y_ld, p, agg_ld, p, None)  # noqa
    assert fwd(x=None) == -1 and fwd(w=None) == -1
    assert fwd(N=-1) == -1 and fwd(C=0) == -1 and fwd(K=0) == -1
    assert fwd(x_ld=7) == -1 and fwd(y_ld=7) == -1 and fwd(agg_ld=7) == -1
    assert fwd(op=2) == -2 and fwd(N=2 ** 31) == -2 and fwd(dtype=7) == -2
    bwd = lambda dy=p, dy_ld=8, N=4, C=8, K=1, dx_ld=8, w=p: \
        lib.b200gf_local_activation_backward(cabi.F32, dy, dy_ld, p, N, C, K, w, p, dx_ld, None)  # noqa: E731
    assert bwd(dy=None) == -1 and bwd(w=None) == -1 and bwd(N=-1) == -1 and bwd(K=0) == -1
    assert bwd(dy_ld=7) == -1 and bwd(dx_ld=7) == -1 and bwd(N=2 ** 31) == -2
    assert fwd(N=0) == 0 and bwd(N=0) == 0                    # nothing to do: no launch
