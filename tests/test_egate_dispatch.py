"""One case per launch branch of the edge-gated layer's kernels (csrc/egate.cu), each held to oracle/egate_oracle.py's
componentwise fp64 bound by tests/dispatch_harness.py's check_case.  This table owns the kernels of egate.cu
(tests/test_dispatch_tables.py).

Every row calls the C entry points directly and names the kernels its branch must launch (regexes on the demangled
name); the launches are traced with torch.profiler in a child process (dispatch_harness.child_traced).  Outputs start
as NaN and are followed by 4 KB of SENT; the pad columns [Bs*C, ld) of dst and dsrc start as SENT and must keep it,
and input pad columns hold NaN, which must reach no output.  Every output is held to egate_envelope, and a second run
must be bit-identical.

Attention inputs sit on a coarse grid (s a multiple of 2^-10 in [-8, 8], or of 2^-4 in [-96, 96] for the large-logit
rows; mixer values with 5 significant bits), so the logit a1 s_j + a2 s_i is exact in fp32 and fp64 and LeakyReLU'
takes the same branch in the kernel and in the fp64 restatement.  Some logits are exactly 0.  The backward takes the
restatement's alpha, rounded to the kernel's dtype, as its input.

The builders `attn_inputs` / `hop_inputs` and the row lists ATTN_ROWS / HOP_ROWS are shared with
tests/test_egate_oracle.py, which checks on the CPU that an emulated correct kernel meets the bound at every one of
these shapes and that emulated wrong kernels do not.
"""
import functools

import numpy as np
import pytest
import torch

import egate_oracle as ego
from dispatch_harness import F32, F64, NPD, SENT, Result, _bits, _check, _graph, _lib, _st, check_case, child_traced

MIXER = (0.6875, -1.3125)                  # 11/16, -21/16: exact products with grid values of s
GRID = {"grid": (2.0 ** -10, 8.0), "large": (2.0 ** -4, 96.0)}


@functools.lru_cache(maxsize=None)
def egate_graph(kind, N, dtype):
    """S as COO (rows, cols, vals exact in dtype).  "rand": _graph's non-symmetric pattern (rows and columns of
    0, 1, 3 .. 129 entries, and at N > 20 000 a 20 000-entry row and column), with S_ii = -1 on every node i % 5 == 2
    (its diagonal leaves the mask but stays a hop entry, pos = -1) and an entry of 1e-12, below the mask's tolerance, in
    every 9th row.  "tiny": the same on _graph's tiny pattern.  "empty": S = -I, an empty mask."""
    if kind == "empty":
        idx = np.arange(N)
        return idx, idx, -np.ones(N)
    m = _graph(kind, N).tocoo()
    rows, cols, vals = m.row.astype(np.int64), m.col.astype(np.int64), m.data.astype(NPD[dtype]).astype(np.float64)
    keep = ~((rows == cols) & (rows % 5 == 2))
    rows, cols, vals = rows[keep], cols[keep], vals[keep]
    neg = np.arange(2, N, 5)
    rows, cols, vals = np.concatenate((rows, neg)), np.concatenate((cols, neg)), np.concatenate((vals, -np.ones(neg.size)))
    first = np.unique(rows[rows != cols], return_index=True)[1]
    small = first[rows[rows != cols][first] % 9 == 0]
    vals[np.nonzero(rows != cols)[0][small]] = NPD[dtype](1e-12)
    o = np.argsort(rows * N + cols)
    return rows[o], cols[o], vals[o]


@functools.lru_cache(maxsize=None)
def egate_pat(kind, N, dtype):
    return ego.egate_pattern(N, *egate_graph(kind, N, dtype))


@functools.lru_cache(maxsize=None)
def attn_inputs(dtype, N, Bs, graph, s_kind):
    """s [N, Bs] on the grid (every 7th node 0, so that some logits are exactly 0), "ties": sample 0 constant (every
    row's logits equal), "generic": normal reals (forward only).  Returns inputs, references and bounds."""
    npd = NPD[dtype]
    pat = egate_pat(graph, N, dtype)
    rng = np.random.default_rng(N + 17 * Bs + len(s_kind))
    if s_kind == "generic":
        s = (rng.standard_normal((N, Bs)) * 3).astype(npd).astype(np.float64)
    else:
        step, top = GRID["large" if s_kind == "large" else "grid"]
        s = rng.integers(-int(top / step), int(top / step) + 1, (N, Bs)) * step
        s[::7] = 0
        if s_kind == "ties":
            s[:, 0] = 0.5
    alpha = ego.attention_forward(pat["m_rowptr"], pat["m_col"], s, MIXER)
    alpha_in = alpha.astype(npd).astype(np.float64)
    dalpha = rng.standard_normal(alpha.shape).astype(npd).astype(np.float64)
    dlogit, dsig1, dsig2 = ego.attention_backward(pat["m_rowptr"], pat["m_col"], s, MIXER, alpha_in, dalpha)
    env = ego.egate_envelope(npd, pat, s=s, mixer=MIXER, alpha=alpha_in, dalpha=dalpha)
    return dict(pat=pat, s=s, alpha_in=alpha_in, dalpha=dalpha,
                ref=dict(alpha=alpha, dlogit=dlogit, dsig1=dsig1, dsig2=dsig2), env=env)


@functools.lru_cache(maxsize=None)
def hop_inputs(dtype, N, Bs, C, graph):
    """gate [Bs, nnz] in (0, 1), src and ddst [N, Bs, C] biased-uniform, all exact in dtype."""
    npd = NPD[dtype]
    pat = egate_pat(graph, N, dtype)
    rng = np.random.default_rng(N + 7 * Bs + 31 * C)
    r = lambda shape: rng.uniform(-0.25, 1.0, shape).astype(npd).astype(np.float64)   # noqa: E731
    gate = rng.uniform(0.0, 1.0, (Bs, pat["nnz"])).astype(npd).astype(np.float64)
    src, ddst = r((N, Bs, C)), r((N, Bs, C))
    dst = ego.gated_hop_forward(pat["t_rowptr"], pat["t_col"], pat["t_val"], pat["t_pos"], gate, src)
    dsrc, dgate = ego.gated_hop_backward(pat["s_rowptr"], pat["s_col"], pat["s_val"], pat["s_pos"], pat["m_rowptr"],
                                         pat["m_col"], pat["m_sval"], gate, src, ddst)
    env = ego.egate_envelope(npd, pat, gate=gate, src=src, ddst=ddst)
    return dict(pat=pat, gate=gate, src=src, ddst=ddst, ref=dict(dst=dst, dsrc=dsrc, dgate=dgate), env=env)


def _dev_pat(pat):
    out = {}
    for k, v in pat.items():
        if isinstance(v, np.ndarray) and v.dtype.kind == "i":
            out[k] = torch.tensor(v, device="cuda")
    return out


def _nan_out(n, dtype, off=0):
    """n NaN elements at offset off of a buffer of SENT, followed by 4 KB of SENT."""
    pad = 4096 // torch.empty(0, dtype=dtype).element_size()
    t = torch.full((off + n + pad,), SENT, dtype=dtype, device="cuda")
    t[off:off + n] = float("nan")
    return t


def _attn_case(dtype, N, Bs, graph="rand", s_kind="grid", backward=True):
    """b200gf_egate_attention_forward (+ _backward) through the C ABI against attn_inputs' references."""
    def run():
        cabi, lib = _lib()
        enum = cabi.F32 if dtype == F32 else cabi.F64
        inp = attn_inputs(dtype, N, Bs, graph, s_kind)
        pat, ref, env = inp["pat"], inp["ref"], inp["env"]
        nnz = pat["nnz"]
        d = _dev_pat(pat)
        dev = lambda a: torch.tensor(a, dtype=dtype, device="cuda")          # noqa: E731
        s, mixer = dev(inp["s"]), dev(MIXER)
        res = Result()
        ab = _nan_out(nnz * Bs, dtype)
        _check(lib.b200gf_egate_attention_forward(enum, N, nnz, Bs, d["m_rowptr"].data_ptr(), d["m_col"].data_ptr(),
                                                  s.data_ptr(), mixer.data_ptr(), ab.data_ptr(), _st()))
        alpha = ab[:nnz * Bs].view(nnz, Bs)
        res.canaries.append(("alpha tail", ab[nnz * Bs:]))
        res.checks.append(("alpha", alpha, ref["alpha"], env["alpha"]))
        res.outputs.append(alpha)
        res.finite.append(("alpha", alpha))
        if backward:
            a_in, da = dev(inp["alpha_in"]), dev(inp["dalpha"])
            dl, d1, d2 = _nan_out(nnz * Bs, dtype), _nan_out(N * Bs, dtype), _nan_out(N * Bs, dtype)
            _check(lib.b200gf_egate_attention_backward(enum, N, nnz, Bs, d["m_rowptr"].data_ptr(), d["m_col"].data_ptr(),
                                                       d["mT_rowptr"].data_ptr(), d["mT_perm"].data_ptr(), s.data_ptr(),
                                                       mixer.data_ptr(), a_in.data_ptr(), da.data_ptr(), dl.data_ptr(),
                                                       d1.data_ptr(), d2.data_ptr(), _st()))
            outs = dict(dlogit=(dl, nnz), dsig1=(d1, N), dsig2=(d2, N))
            for name, (t, n) in outs.items():
                v = t[:n * Bs].view(n, Bs)
                res.canaries.append((name + " tail", t[n * Bs:]))
                res.checks.append((name, v, ref[name], env[name]))
                res.outputs.append(v)
                res.finite.append((name, v))
            if nnz == 0:
                assert bool((d1[:N * Bs] == 0).all() and (d2[:N * Bs] == 0).all()), "empty mask: dsig must be exactly 0"
        return res
    return run


def _gate_view(gate, kind, dtype):
    """The gate [Bs, nnz] laid out as the layer stores it: "bs" [Bs, nnz] (sample stride nnz, position stride 1); "slab"
    the time slab t = 1 of a [nnz, T = 3, Bs] store (sample stride 1, position stride T*Bs, offset Bs), as the hidden
    filter reads q_check[:, t].  Returns (tensor holding the storage, element pointer, sample stride, position stride)."""
    Bs, nnz = gate.shape
    esz = torch.empty(0, dtype=dtype).element_size()
    if nnz == 0:                           # nothing is read: a canary buffer stands in
        t = torch.full((64,), SENT, dtype=dtype, device="cuda")
        return t, t.data_ptr(), 0, 1
    if kind == "bs":
        t = torch.tensor(gate, dtype=dtype, device="cuda")
        return t, t.data_ptr(), nnz, 1
    T = 3
    store = torch.full((nnz, T, Bs), float("nan"), dtype=dtype, device="cuda")
    store[:, 1] = torch.tensor(gate.T, dtype=dtype, device="cuda")
    v = store[:, 1].t()
    return store, store.data_ptr() + v.storage_offset() * esz, v.stride(0), v.stride(1)


def _hop_case(dtype, N, Bs, C, ld, graph="rand", off=0, gate="bs", bwd="both", dgate_layout="nb", aligned_twin=False):
    """b200gf_gated_hop_forward and _backward through the C ABI against hop_inputs' references.  src / ddst [N, ld] with
    NaN pad columns, at element offset off of their buffers (off = 1: one element past a 16-byte boundary); dst / dsrc
    [N, ld] at the same offset, pad columns SENT.  bwd: "both", "dsrc", "dgate" or None.  dgate_layout "nb": [nnz, Bs]
    (strides (1, Bs), as the layer writes it), "bn": [Bs, nnz] (strides (nnz, 1)).  aligned_twin: run the forward and
    dsrc a second time at offset 0 and require the same bits."""
    def run():
        cabi, lib = _lib()
        enum = cabi.F32 if dtype == F32 else cabi.F64
        inp = hop_inputs(dtype, N, Bs, C, graph)
        pat, ref, env = inp["pat"], inp["ref"], inp["env"]
        nnz, BC = pat["nnz"], Bs * C
        d = _dev_pat(pat)
        dev = lambda a: torch.tensor(a, dtype=dtype, device="cuda")          # noqa: E731
        t_val, s_val, m_sval = dev(pat["t_val"]), dev(pat["s_val"]), dev(pat["m_sval"])
        g_store, g_ptr, g_sb, g_sp = _gate_view(inp["gate"], gate, dtype)
        esz = t_val.element_size()
        res = Result()

        def node_major(a, o):
            buf = torch.full((o + N * ld + 8,), float("nan"), dtype=dtype, device="cuda")
            buf[o:o + N * ld].view(N, ld)[:, :BC] = dev(a.reshape(N, BC))
            return buf

        def out_buf(o):
            buf = _nan_out(N * ld, dtype, o)
            buf[o:o + N * ld].view(N, ld)[:, BC:] = SENT
            return buf

        def fence(name, buf, o):
            v = buf[o:o + N * ld].view(N, ld)
            res.canaries += [(name + " before", buf[:o]), (name + " pad columns", v[:, BC:]),
                             (name + " tail", buf[o + N * ld:])]
            return v[:, :BC].reshape(N, Bs, C)

        def forward(o):
            src = node_major(inp["src"], o)
            dst = out_buf(o)
            _check(lib.b200gf_gated_hop_forward(enum, N, Bs, C, d["t_rowptr"].data_ptr(), d["t_col"].data_ptr(),
                                                t_val.data_ptr(), d["t_pos"].data_ptr(), g_ptr, g_sb, g_sp,
                                                src.data_ptr() + o * esz, ld, dst.data_ptr() + o * esz, ld, _st()))
            return src, dst

        def backward(o, src):
            ddst = node_major(inp["ddst"], o)
            dsrc = out_buf(o) if bwd in ("both", "dsrc") else None
            dg = _nan_out(nnz * Bs, dtype) if bwd in ("both", "dgate") else None
            d_sb, d_sp = (1, Bs) if dgate_layout == "nb" else (nnz, 1)
            _check(lib.b200gf_gated_hop_backward(
                enum, N, Bs, C, d["s_rowptr"].data_ptr(), d["s_col"].data_ptr(), s_val.data_ptr(),
                d["s_pos"].data_ptr(), d["m_rowptr"].data_ptr(), d["m_col"].data_ptr(), m_sval.data_ptr(), g_ptr, g_sb,
                g_sp, src.data_ptr() + o * esz, ld, ddst.data_ptr() + o * esz, ld,
                None if dsrc is None else dsrc.data_ptr() + o * esz, ld, None if dg is None else dg.data_ptr(), d_sb,
                d_sp, _st()))
            return dsrc, dg

        src, dst = forward(off)
        outs = [("dst", fence("dst", dst, off))]
        if bwd is not None:
            dsrc, dg = backward(off, src)
            if dsrc is not None:
                outs.append(("dsrc", fence("dsrc", dsrc, off)))
            if dg is not None:
                res.canaries.append(("dgate tail", dg[nnz * Bs:]))
                v = dg[:nnz * Bs].view(nnz, Bs).t() if dgate_layout == "nb" else dg[:nnz * Bs].view(Bs, nnz)
                outs.append(("dgate", v))
                zero = torch.tensor(pat["m_sval"] == 0, device="cuda")
                assert bool((v[:, zero] == 0).all()), "dgate must be exactly 0 where the mask has no S entry"
        for name, v in outs:
            res.checks.append((name, v, ref[name], env[name]))
            res.outputs.append(v)
            res.finite.append((name, v))
        res.keep = g_store
        if aligned_twin:
            src0, dst0 = forward(0)
            twin = [("dst", fence("aligned dst", dst0, 0))]
            if bwd in ("both", "dsrc"):
                twin.append(("dsrc", fence("aligned dsrc", backward(0, src0)[0], 0)))
            for name, v in twin:
                got = dict(outs)[name]
                assert torch.equal(_bits(got), _bits(v)), "%s: misaligned and aligned runs differ" % name
        return res
    return run


def _attn_kernels(t, backward=True):
    return [r"egate_softmax_kernel<%s>" % t] + \
        ([r"egate_softmax_bwd_kernel<%s>" % t, r"egate_colsum_kernel<%s>" % t] if backward else [])


def _hop_kernels(t, v, bwd="both", v_bwd=None):
    ks = [r"egate_hop_kernel<%s,%d>" % (t, v)]
    if bwd in ("both", "dsrc"):
        ks.append(r"egate_hop_kernel<%s,%d>" % (t, v if v_bwd is None else v_bwd))
    if bwd in ("both", "dgate"):
        ks.append(r"egate_sddmm_kernel<%s>" % t)
    return ks


# (id, keyword arguments of _attn_case, kernels)
ATTN_ROWS = [
    # mask rows of 0, 1 and 31 .. 129 entries, S_ii = -1 nodes and entries below the tolerance, exact zero logits
    ("attn-f32-Bs1", dict(dtype=F32, N=3000, Bs=1), _attn_kernels("float")),
    ("attn-f32-Bs13", dict(dtype=F32, N=3000, Bs=13), _attn_kernels("float")),
    ("attn-f64-Bs6", dict(dtype=F64, N=3000, Bs=6), _attn_kernels("double")),
    # logits spread over more than 100: the max shift keeps fp32 exp finite, the smallest alpha underflow
    ("attn-f32-large-logits", dict(dtype=F32, N=3000, Bs=4, s_kind="large"), _attn_kernels("float")),
    ("attn-f64-large-logits", dict(dtype=F64, N=3000, Bs=3, s_kind="large"), _attn_kernels("double")),
    # sample 0: every row's logits equal
    ("attn-f32-ties", dict(dtype=F32, N=3000, Bs=3, s_kind="ties"), _attn_kernels("float")),
    ("attn-f32-generic-fwd", dict(dtype=F32, N=3000, Bs=5, s_kind="generic", backward=False),
     _attn_kernels("float", False)),
    # S = -I: nnz = 0, nothing written to alpha, dsig1 = dsig2 = 0
    ("attn-f32-empty-mask", dict(dtype=F32, N=50, Bs=3, graph="empty"), _attn_kernels("float")),
    # the 20 000-entry mask row and column, N Bs > 132 * 16 * 256: the grid-stride loops take several passes
    ("attn-hub-f32", dict(dtype=F32, N=24000, Bs=32), _attn_kernels("float")),
    ("attn-hub-f64", dict(dtype=F64, N=24000, Bs=32), _attn_kernels("double")),
]
for _n in (1, 3, 7):
    ATTN_ROWS.append(("attn-tinyN%d-f32" % _n, dict(dtype=F32, N=_n, Bs=2, graph="tiny"), _attn_kernels("float")))
    ATTN_ROWS.append(("attn-tinyN%d-f64" % _n, dict(dtype=F64, N=_n, Bs=3, graph="tiny"), _attn_kernels("double")))

HOP_ROWS = [
    # 16-byte lanes, padded ld; the gate of a time slab (sample stride 1, position stride T Bs, non-zero offset)
    ("gated-hop-f32-C4-V4", dict(dtype=F32, N=3000, Bs=3, C=4, ld=16), _hop_kernels("float", 4)),
    ("gated-hop-f32-C8-V4-slab-gate", dict(dtype=F32, N=3000, Bs=5, C=8, ld=44, gate="slab"), _hop_kernels("float", 4)),
    # scalar lanes: C % 4 != 0, and ld % 4 != 0 with C % 4 == 0
    ("gated-hop-f32-C3-V1", dict(dtype=F32, N=3000, Bs=4, C=3, ld=13), _hop_kernels("float", 1)),
    ("gated-hop-f32-ld-odd-V1", dict(dtype=F32, N=3000, Bs=2, C=4, ld=10, gate="slab"), _hop_kernels("float", 1)),
    # src, dst, ddst and dsrc one element past a 16-byte boundary: scalar lanes, the same bits as the aligned run
    ("gated-hop-f32-misaligned-V1", dict(dtype=F32, N=3000, Bs=3, C=4, ld=12, off=1, aligned_twin=True),
     _hop_kernels("float", 1) + _hop_kernels("float", 4, bwd="dsrc")),
    ("gated-hop-f64-C2-V2", dict(dtype=F64, N=3000, Bs=3, C=2, ld=8, gate="slab"), _hop_kernels("double", 2)),
    ("gated-hop-f64-C3-V1", dict(dtype=F64, N=3000, Bs=2, C=3, ld=7), _hop_kernels("double", 1)),
    # backward halves alone, and dgate in the [Bs, nnz] layout (strides (nnz, 1))
    ("gated-hop-f32-dsrc-only", dict(dtype=F32, N=3000, Bs=3, C=4, ld=12, bwd="dsrc"), _hop_kernels("float", 4, "dsrc")),
    ("gated-hop-f32-dgate-only-bn", dict(dtype=F32, N=3000, Bs=3, C=5, ld=15, bwd="dgate", dgate_layout="bn"),
     _hop_kernels("float", 1, "dgate")),
    ("gated-hop-f64-both-bn", dict(dtype=F64, N=3000, Bs=4, C=2, ld=8, dgate_layout="bn", gate="slab"),
     _hop_kernels("double", 2)),
    # S = -I: every entry outside the mask (dst = dsrc = 0); there is no gate to differentiate, so, as in the layer,
    # the backward computes dsrc alone
    ("gated-hop-f32-empty-mask", dict(dtype=F32, N=50, Bs=2, C=4, ld=8, graph="empty", bwd="dsrc"),
     _hop_kernels("float", 4, "dsrc")),
    # the 20 000-entry row and column, N Bs C / V > 132 * 16 * 256
    ("gated-hop-hub-f32", dict(dtype=F32, N=24000, Bs=32, C=4, ld=128, gate="slab"), _hop_kernels("float", 4)),
    ("gated-hop-hub-f64", dict(dtype=F64, N=24000, Bs=32, C=2, ld=64), _hop_kernels("double", 2)),
]
for _n in (1, 3, 7):
    HOP_ROWS.append(("gated-hop-tinyN%d-f32" % _n, dict(dtype=F32, N=_n, Bs=2, C=4, ld=8, graph="tiny"),
                     _hop_kernels("float", 4)))
    HOP_ROWS.append(("gated-hop-tinyN%d-f64" % _n, dict(dtype=F64, N=_n, Bs=3, C=3, ld=9, graph="tiny", gate="slab"),
                     _hop_kernels("double", 1)))

EGATE_CASES = [(cid, _attn_case(**kw), ks) for cid, kw, ks in ATTN_ROWS] + \
    [(cid, _hop_case(**kw), ks) for cid, kw, ks in HOP_ROWS]


# ------------------------------------------------------------------------------------------------------------ CPU
def test_attention_rows_have_exact_zero_logits_and_underflow():
    """The grid rows contain logits that are exactly 0 (LeakyReLU'(0) = 0.2 on both sides), and the large-logit rows
    spread their logits over more than 100, enough to overflow an unshifted fp32 exp and underflow some alpha."""
    inp = attn_inputs(F32, 3000, 13, "rand", "grid")
    p = inp["pat"]
    x = ego.attention_logits(p["m_rowptr"], p["m_col"], inp["s"], MIXER)
    assert (x == 0).sum() > 10
    assert np.array_equal(x.astype(np.float32).astype(np.float64), x)
    big = attn_inputs(F32, 3000, 4, "rand", "large")
    xb = ego.attention_logits(big["pat"]["m_rowptr"], big["pat"]["m_col"], big["s"], MIXER)
    assert xb.max() - xb.min() > 100 and xb.max() > 89
    assert (big["ref"]["alpha"] < np.finfo(np.float32).tiny).any()


# ------------------------------------------------------------------------------------------------------------ GPU
traced = child_traced("test_egate_dispatch", "EGATE_CASES")


@pytest.mark.gpu
@pytest.mark.parametrize("cid,fn,kernels", EGATE_CASES, ids=[c[0] for c in EGATE_CASES])
def test_egate_dispatch(cid, fn, kernels, traced):
    check_case(cid, fn, kernels, traced[cid])
