"""One case per launch branch of the two-score attention entry points (b200gf_attention_forward / _backward, which run
csrc/egate.cu's softmax kernels with s_src read at the column node and s_dst at the row node), each held to
oracle/attention_oracle.py's componentwise fp64 bound by tests/dispatch_harness.py's check_case.  The table owns no
kernel: it names only egate.cu's, which tests/test_egate_dispatch.py owns (tests/test_dispatch_tables.py).

Every row calls the C entry points directly with the mixer (1, 1) the layers pass and names the kernels its branch
must launch; the launches are traced with torch.profiler in a child process (dispatch_harness.child_traced).  Outputs
start as NaN followed by 4 KB of SENT, which must survive.  Every output is held to attention_envelope, and a second
run must be bit-identical.  Rows with `parity` also run the edge-gate entry point on s_src = s_dst with the same mixer
and require the same bits: the generalised kernels compute what edge gating always computed.

Inputs sit on a coarse grid (multiples of 2^-10 in [-8, 8], or of 2^-4 in [-96, 96] for the large-logit rows), so the
logit s_src[j] + s_dst[i] is exact in fp32 and fp64 and LeakyReLU' takes the same branch in the kernel and in the fp64
restatement.  The masks are the union over E edge features (E = 2 rows: S_0 and a transposed, re-weighted copy).
"""
import functools

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import attention_oracle as ao
import egate_oracle as ego
import lsigf_oracle as orc
import test_egate_dispatch as ed
import test_egate_oracle as eo
from dispatch_harness import F32, F64, NPD, Result, _bits, _check, _lib, _st, check_case, child_traced, kernel_names

GRID = ed.GRID


@functools.lru_cache(maxsize=None)
def attention_pat(kind, N, E, dtype):
    """The mask CSR (and its transpose) of E edge features: S_0 = test_egate_dispatch's egate_graph(kind) (S_ii = -1
    nodes, entries below the tolerance), S_1 = 0.5 S_0^T with the same -1 diagonal, so the union differs from S_0's
    mask.  Also returns the mask of S_0 alone (for the emulated wrong kernel that reads it)."""
    rows, cols, vals = ed.egate_graph(kind, N, dtype)
    S0 = sp.csr_matrix((vals, (rows, cols)), shape=(N, N))
    S = [S0]
    if E == 2:
        S1 = sp.csr_matrix(0.5 * S0.T)
        S1.setdiag(S0.diagonal())
        S1.eliminate_zeros()
        S.append(S1)

    def csr(m_rows, m_cols):
        rp = np.concatenate([[0], np.cumsum(np.bincount(m_rows, minlength=N))]).astype(np.int64)
        return dict(N=N, nnz=int(m_rows.size), m_rowptr=rp, m_col=m_cols.astype(np.int32),
                    mT_rowptr=np.concatenate([[0], np.cumsum(np.bincount(m_cols, minlength=N))]).astype(np.int64),
                    mT_perm=np.argsort(m_cols * N + m_rows, kind="stable").astype(np.int32))
    return csr(*ao.attention_mask_coo(S)), csr(*ao.attention_mask_coo(S[:1]))


@functools.lru_cache(maxsize=None)
def attn2_inputs(dtype, N, Bs, graph, E, s_kind):
    npd = NPD[dtype]
    pat, _ = attention_pat(graph, N, E, dtype)
    rng = np.random.default_rng(N + 17 * Bs + 5 * E + len(s_kind))
    if s_kind == "generic":
        s_src, s_dst = ((rng.standard_normal((N, Bs)) * 3).astype(npd).astype(np.float64) for _ in range(2))
    else:
        step, top = GRID["large" if s_kind == "large" else "grid"]
        s_src, s_dst = (rng.integers(-int(top / step), int(top / step) + 1, (N, Bs)) * step for _ in range(2))
        s_src[::7] = 0
        s_dst[::7] = 0
        if s_kind == "ties":
            s_src[:, 0] = 0.5
    alpha = ao.attention_forward(pat["m_rowptr"], pat["m_col"], s_src, s_dst)
    alpha_in = alpha.astype(npd).astype(np.float64)
    dalpha = rng.standard_normal(alpha.shape).astype(npd).astype(np.float64)
    dlogit, dsig1, dsig2 = ao.attention_backward(pat["m_rowptr"], pat["m_col"], s_src, s_dst, alpha_in, dalpha)
    env = ao.attention_envelope(npd, pat, s_src, s_dst, alpha=alpha_in, dalpha=dalpha)
    return dict(pat=pat, s_src=s_src, s_dst=s_dst, alpha_in=alpha_in, dalpha=dalpha,
                ref=dict(alpha=alpha, dlogit=dlogit, dsig1=dsig1, dsig2=dsig2), env=env)


def _attn2_case(dtype, N, Bs, graph="rand", E=2, s_kind="grid", backward=True, parity=False):
    def run():
        cabi, lib = _lib()
        enum = cabi.F32 if dtype == F32 else cabi.F64
        inp = attn2_inputs(dtype, N, Bs, graph, E, s_kind)
        pat, ref, env = inp["pat"], inp["ref"], inp["env"]
        nnz = pat["nnz"]
        d = ed._dev_pat(pat)
        dev = lambda a: torch.tensor(a, dtype=dtype, device="cuda")          # noqa: E731
        s_src, s_dst, ones = dev(inp["s_src"]), dev(inp["s_dst"]), dev([1.0, 1.0])
        res = Result()
        ab = ed._nan_out(nnz * Bs, dtype)
        _check(lib.b200gf_attention_forward(enum, N, nnz, Bs, d["m_rowptr"].data_ptr(), d["m_col"].data_ptr(),
                                            s_src.data_ptr(), s_dst.data_ptr(), ones.data_ptr(), ab.data_ptr(), _st()))
        alpha = ab[:nnz * Bs].view(nnz, Bs)
        res.canaries.append(("alpha tail", ab[nnz * Bs:]))
        res.checks.append(("alpha", alpha, ref["alpha"], env["alpha"]))
        res.outputs.append(alpha)
        res.finite.append(("alpha", alpha))
        if backward:
            a_in, da = dev(inp["alpha_in"]), dev(inp["dalpha"])
            dl, d1, d2 = ed._nan_out(nnz * Bs, dtype), ed._nan_out(N * Bs, dtype), ed._nan_out(N * Bs, dtype)
            _check(lib.b200gf_attention_backward(enum, N, nnz, Bs, d["m_rowptr"].data_ptr(), d["m_col"].data_ptr(),
                                                 d["mT_rowptr"].data_ptr(), d["mT_perm"].data_ptr(), s_src.data_ptr(),
                                                 s_dst.data_ptr(), ones.data_ptr(), a_in.data_ptr(), da.data_ptr(),
                                                 dl.data_ptr(), d1.data_ptr(), d2.data_ptr(), _st()))
            for name, (t, n) in dict(dlogit=(dl, nnz), dsig1=(d1, N), dsig2=(d2, N)).items():
                v = t[:n * Bs].view(n, Bs)
                res.canaries.append((name + " tail", t[n * Bs:]))
                res.checks.append((name, v, ref[name], env[name]))
                res.outputs.append(v)
                res.finite.append((name, v))
            if nnz == 0:
                assert bool((d1[:N * Bs] == 0).all() and (d2[:N * Bs] == 0).all()), "empty mask: dsig must be exactly 0"
        if parity:
            # s_src = s_dst = s: the edge-gate entry points on the same mask and mixer give the same bits
            e_ab = ed._nan_out(nnz * Bs, dtype)
            t_ab = ed._nan_out(nnz * Bs, dtype)
            _check(lib.b200gf_egate_attention_forward(enum, N, nnz, Bs, d["m_rowptr"].data_ptr(), d["m_col"].data_ptr(),
                                                      s_src.data_ptr(), ones.data_ptr(), e_ab.data_ptr(), _st()))
            _check(lib.b200gf_attention_forward(enum, N, nnz, Bs, d["m_rowptr"].data_ptr(), d["m_col"].data_ptr(),
                                                s_src.data_ptr(), s_src.data_ptr(), ones.data_ptr(), t_ab.data_ptr(),
                                                _st()))
            assert torch.equal(_bits(e_ab), _bits(t_ab)), "edge-gate and two-score entry points differ on s_src = s_dst"
        return res
    return run


_kernels = ed._attn_kernels          # the same three kernels as edge gating's attention: no new __global__ function


ATTN2_ROWS = [
    # E = 2 union masks with rows of 0, 1 and 31 .. 129 entries, S_ii = -1 nodes, entries below the tolerance
    ("attn2-f32-Bs1", dict(dtype=F32, N=3000, Bs=1), _kernels("float")),
    ("attn2-f32-Bs13-parity", dict(dtype=F32, N=3000, Bs=13, parity=True), _kernels("float")),
    ("attn2-f64-Bs6", dict(dtype=F64, N=3000, Bs=6), _kernels("double")),
    ("attn2-f64-E1-parity", dict(dtype=F64, N=3000, Bs=4, E=1, parity=True), _kernels("double")),
    ("attn2-f32-large-logits", dict(dtype=F32, N=3000, Bs=4, s_kind="large"), _kernels("float")),
    ("attn2-f64-large-logits", dict(dtype=F64, N=3000, Bs=3, s_kind="large"), _kernels("double")),
    ("attn2-f32-ties", dict(dtype=F32, N=3000, Bs=3, s_kind="ties"), _kernels("float")),
    ("attn2-f32-generic-fwd", dict(dtype=F32, N=3000, Bs=5, s_kind="generic", backward=False), _kernels("float", False)),
    # S_e = -I for both e: nnz = 0, nothing written to alpha, dsig1 = dsig2 = 0
    ("attn2-f32-empty-mask", dict(dtype=F32, N=50, Bs=3, graph="empty"), _kernels("float")),
    # the 20 000-entry mask row and column, N Bs > 132 * 16 * 256: the grid-stride loops take several passes
    ("attn2-hub-f32", dict(dtype=F32, N=24000, Bs=32), _kernels("float")),
    ("attn2-hub-f64", dict(dtype=F64, N=24000, Bs=32), _kernels("double")),
]
for _n in (1, 3, 7):
    ATTN2_ROWS.append(("attn2-tinyN%d-f32" % _n, dict(dtype=F32, N=_n, Bs=2, graph="tiny"), _kernels("float")))
    ATTN2_ROWS.append(("attn2-tinyN%d-f64" % _n, dict(dtype=F64, N=_n, Bs=3, graph="tiny"), _kernels("double")))

ATTENTION_CASES = [(cid, _attn2_case(**kw), ks) for cid, kw, ks in ATTN2_ROWS]


# ------------------------------------------------------------------------------------------------------------ CPU
def _emulate(inp, ft, rng, bug=None, pat0=None):
    """The two-score forward (and backward, when correct) computed in ft as a correct kernel may, or with `bug`:
    "swap" (s_src read at the row node, s_dst at the column node), "columns" (softmax over the mask's columns),
    "no_diagonal" (the diagonal dropped from the mask), "mask_e0" (the mask of edge feature 0 alone)."""
    pat = inp["pat"]
    s_src, s_dst = inp["s_src"].astype(ft), inp["s_dst"].astype(ft)
    N = pat["N"]
    rows = ego._rows_of(pat["m_rowptr"])
    cols = pat["m_col"].astype(np.int64)
    keep = np.ones(pat["nnz"], bool)
    if bug == "no_diagonal":
        keep = rows != cols
    if bug == "mask_e0":
        k0 = ego._rows_of(pat0["m_rowptr"]) * N + pat0["m_col"]
        keep = np.isin(rows * N + cols, k0)
    r, c = rows[keep], cols[keep]
    if bug == "columns":
        r, c = c, r                               # the row of the softmax is the column node
    order = np.argsort(r * N + c, kind="stable")
    rp = np.concatenate([[0], np.cumsum(np.bincount(r, minlength=N))]).astype(np.int64)
    src_at, dst_at = (c, r) if bug != "columns" else (r, c)
    if bug == "swap":
        x = s_dst[src_at] + s_src[dst_at]
    else:
        x = s_src[src_at] + s_dst[dst_at]
    x = x[order]
    e = np.where(x > 0, x, ft(0.2) * x)
    rr = ego._rows_of(rp)
    w = eo._exp(e - ego._segmax(rp, e).astype(ft)[rr], rng)
    tot = eo._seq(rp, w, rng)
    with np.errstate(divide="ignore"):                    # empty rows: their 1 / 0 is read by no entry
        alpha_sub = w * (ft(1) / tot)[rr]
    alpha = np.zeros((pat["nnz"], s_src.shape[1]), ft)
    alpha[np.nonzero(keep)[0][order]] = alpha_sub
    out = dict(alpha=alpha)
    if bug is None:
        a_in, da = inp["alpha_in"].astype(ft), inp["dalpha"].astype(ft)
        rpm = pat["m_rowptr"]
        dot = eo._seq(rpm, a_in, rng, b=da)
        de = a_in * (da - dot[rows])
        xm = s_src[cols] + s_dst[rows]
        dl = np.where(xm > 0, de, ft(0.2) * de)
        out.update(dlogit=dl, dsig2=eo._seq(rpm, dl, rng),
                   dsig1=eo._seq(pat["mT_rowptr"], dl, rng, perm=pat["mT_perm"]))
    return out


@pytest.mark.parametrize("dtype", [F32, F64])
def test_emulated_kernel_meets_the_bound_and_wrong_ones_miss_it(dtype):
    ft = NPD[dtype]
    rng = np.random.default_rng(11)
    for N, Bs, graph in ((3000, 3, "rand"), (7, 2, "tiny")):
        inp = attn2_inputs(dtype, N, Bs, graph, 2, "grid")
        _, pat0 = attention_pat(graph, N, 2, dtype)
        env, ref = inp["env"], inp["ref"]
        good = _emulate(inp, ft, rng)
        for name, v in good.items():
            assert orc.bound_violation(v, ref[name], env[name]) <= 1.0, (N, name)
        if N < 10:
            continue
        for bug in ("swap", "columns", "no_diagonal", "mask_e0"):
            bad = _emulate(inp, ft, rng, bug, pat0)
            viol = orc.bound_violation(bad["alpha"], ref["alpha"], env["alpha"])
            assert viol > 1e3, (bug, viol)


def test_union_mask_differs_from_edge_feature_0():
    pat, pat0 = attention_pat("rand", 3000, 2, F32)
    assert pat["nnz"] > pat0["nnz"]
    pat1, pat01 = attention_pat("rand", 3000, 1, F32)
    assert np.array_equal(pat1["m_col"], pat01["m_col"])
    ref = ego.egate_pattern(3000, *ed.egate_graph("rand", 3000, F32))
    assert np.array_equal(pat1["m_rowptr"], ref["m_rowptr"]) and np.array_equal(pat1["m_col"], ref["m_col"])


def test_every_row_names_only_egate_kernels():
    assert kernel_names(ATTENTION_CASES) == {"egate_softmax_kernel", "egate_softmax_bwd_kernel", "egate_colsum_kernel"}


# ------------------------------------------------------------------------------------------------------------ GPU
traced = child_traced("test_attention_dispatch", "ATTENTION_CASES")


@pytest.mark.gpu
@pytest.mark.parametrize("cid,fn,kernels", ATTENTION_CASES, ids=[c[0] for c in ATTENTION_CASES])
def test_attention_dispatch(cid, fn, kernels, traced):
    check_case(cid, fn, kernels, traced[cid])
