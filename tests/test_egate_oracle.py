"""CPU tests of oracle/egate_oracle.py's restatement of the four edge-gated entry points (csrc/egate.cu) and of
egate_envelope, the componentwise bound tests/test_egate_dispatch.py holds the kernels to, and of the argument checks
of those entry points.

* The restatement is pinned to the torch restatement with autograd (egate_attention_coo / egate_hop_coo), which
  tests/test_edge_gated.py pins to the reference's fixtures; its pattern equals gnn_b200.EdgeGatePattern's.
* The envelope separates a correct kernel from subtly wrong ones.  An emulated correct kernel (arithmetic in the
  kernel's dtype, sums in a shuffled order, fused multiply-adds as an fp64 product-plus-add rounded to fp32, exp pushed
  by up to 2 ulp in fp32 and 1 ulp in fp64) meets it at every shape and dtype of the GPU table.  Emulations of wrong
  kernels miss it by more than WIDE; the margins measured here are listed beside WRONG."""
import ctypes

import numpy as np
import pytest
import torch

import egate_oracle as ego
import lsigf_oracle as orc
import test_egate_dispatch as ed
from dispatch_harness import F32, NPD

WIDE = 3.0
MIXER = ed.MIXER


def _rel(a, b):
    return np.abs(np.asarray(a) - b).max() / max(np.abs(b).max(), 1e-300)


# ------------------------------------------------------------------------------------------------ pinning
def _small_graph(seed=5, N=23):
    """Non-symmetric, with empty rows, S_ii = -1 nodes (one of them an empty mask row), entries below the tolerance."""
    rng = np.random.default_rng(seed)
    S = np.where(rng.random((N, N)) < 0.2, rng.standard_normal((N, N)), 0.0)
    S[4] = 0                                       # no entries: the mask row is the diagonal alone
    S[6] = 0
    S[6, 6] = -1.0                                 # only entry S_ii = -1: an empty mask row
    S[::5, ::5] = np.where(np.eye(N)[::5, ::5] > 0, -1.0, S[::5, ::5])
    S[7, 8], S[9, 1] = 1e-12, -1e-12
    rows, cols = np.nonzero(S)
    return N, rows, cols, S[rows, cols]


def test_pattern_matches_the_layers_pattern():
    from gnn_b200 import edgegated as eg
    N, rows, cols, vals = _small_graph()
    S = np.zeros((N, N))
    S[rows, cols] = vals
    pat = ego.egate_pattern(N, rows, cols, vals)
    lp = eg.EdgeGatePattern(torch.tensor(S).reshape(1, N, N))
    assert pat["nnz"] == lp.nnz and np.diff(pat["m_rowptr"])[6] == 0
    for name in eg.EdgeGatePattern._TENSORS:
        if name in pat:
            assert np.array_equal(pat[name], getattr(lp, name).numpy()), name


def test_attention_matches_torch_restatement_and_autograd():
    N, rows, cols, vals = _small_graph()
    pat = ego.egate_pattern(N, rows, cols, vals)
    rng = np.random.default_rng(1)
    Bs = 4
    s, dalpha = rng.standard_normal((N, Bs)) * 2, rng.standard_normal((pat["nnz"], Bs))
    mixer = np.array([0.7, -1.3])
    m_rows = torch.from_numpy(ego._rows_of(pat["m_rowptr"]))
    st, mt = torch.tensor(s.T.copy(), requires_grad=True), torch.tensor(mixer, requires_grad=True)
    at = ego.egate_attention_coo(st, mt, m_rows, torch.from_numpy(pat["m_col"].astype(np.int64)), N)
    (at * torch.tensor(dalpha.T)).sum().backward()
    alpha = ego.attention_forward(pat["m_rowptr"], pat["m_col"], s, mixer)
    assert _rel(alpha, at.detach().numpy().T) < 1e-12
    dlogit, dsig1, dsig2 = ego.attention_backward(pat["m_rowptr"], pat["m_col"], s, mixer, alpha, dalpha)
    assert _rel(mixer[0] * dsig1 + mixer[1] * dsig2, st.grad.numpy().T) < 1e-12
    assert _rel([(s * dsig1).sum(), (s * dsig2).sum()], mt.grad.numpy()) < 1e-12
    assert np.array_equal(dsig2[6], np.zeros(Bs)) and np.allclose(ego._segsum(pat["m_rowptr"], dlogit), dsig2)


def test_gated_hop_matches_torch_restatement_and_autograd():
    N, rows, cols, vals = _small_graph()
    pat = ego.egate_pattern(N, rows, cols, vals)
    rng = np.random.default_rng(2)
    Bs, C = 3, 2
    gate, src, ddst = rng.random((Bs, pat["nnz"])), rng.standard_normal((N, Bs, C)), rng.standard_normal((N, Bs, C))
    mr = torch.from_numpy(ego._rows_of(pat["m_rowptr"]))
    mc = torch.from_numpy(pat["m_col"].astype(np.int64))
    ut, gt = torch.tensor(src.transpose(1, 2, 0).copy(), requires_grad=True), torch.tensor(gate, requires_grad=True)
    out = ego.egate_hop_coo(ut, gt * torch.tensor(pat["m_sval"]), mr, mc)               # [Bs, C, N]
    (out * torch.tensor(ddst.transpose(1, 2, 0))).sum().backward()
    dst = ego.gated_hop_forward(pat["t_rowptr"], pat["t_col"], pat["t_val"], pat["t_pos"], gate, src)
    dsrc, dgate = ego.gated_hop_backward(pat["s_rowptr"], pat["s_col"], pat["s_val"], pat["s_pos"], pat["m_rowptr"],
                                         pat["m_col"], pat["m_sval"], gate, src, ddst)
    assert _rel(dst, out.detach().numpy().transpose(2, 0, 1)) < 1e-12
    assert _rel(dsrc, ut.grad.numpy().transpose(2, 0, 1)) < 1e-12
    assert _rel(dgate, gt.grad.numpy()) < 1e-12
    assert np.all(dgate[:, pat["m_sval"] == 0] == 0)


# ------------------------------------------------------------------------------------------------ emulated kernels
def _fma(a, b, c):
    """fl(a b + c) with one rounding for fp32 (the fp32 product is exact in fp64); fp64 rounds twice."""
    if a.dtype == np.float32:
        return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)
    return a * b + c


def _seq(rowptr, a, rng, b=None, perm=None, order=True):
    """Per CSR row, acc = acc + a (or fma(a, b, acc)) over the row's entries in a random order, in a's dtype.
    perm: entry it of the CSR reads element perm[it] of a and b (the transposed mask)."""
    rowptr = np.asarray(rowptr, np.int64)
    n, nnz = len(rowptr) - 1, int(rowptr[-1])
    rows = ego._rows_of(rowptr)
    idx = np.arange(nnz) if perm is None else np.asarray(perm, np.int64)
    shuffled = np.argsort(rows + (rng.random(nnz) if order else 0), kind="stable")
    rank = np.empty(nnz, np.int64)
    rank[shuffled] = np.arange(nnz) - rowptr[rows[shuffled]]
    by = np.argsort(rank, kind="stable")
    acc = np.zeros((n,) + a.shape[1:], a.dtype)
    start = 0
    for c in np.bincount(rank):
        sel = by[start:start + c]
        start += c
        r, e = rows[sel], idx[sel]
        acc[r] = acc[r] + a[e] if b is None else _fma(a[e], b[e], acc[r])
    return acc


def _exp(d, rng):
    """exp in d's dtype, pushed by up to 2 ulp (fp32) or 1 ulp (fp64) at random."""
    with np.errstate(over="ignore"):
        w = np.exp(d.astype(np.float64)).astype(d.dtype)
    k = rng.integers(-2 if d.dtype == np.float32 else -1, 3 if d.dtype == np.float32 else 2, w.shape)
    for step in (1, 2):
        w = np.where(k >= step, np.nextafter(w, np.inf), w)
        w = np.where(k <= -step, np.nextafter(w, -np.inf), w)
    return w


def _logit(pat, s, ft, bug=None):
    a1, a2 = (ft(v) for v in (MIXER[::-1] if bug == "mixer_swap" else MIXER))
    rows = ego._rows_of(pat["m_rowptr"])
    x = _fma(np.full(pat["nnz"], a1, ft)[:, None], s[pat["m_col"]], a2 * s[rows])
    return x, np.where(x > 0, x, ft(0.2) * x), rows


def emu_attention(pat, s, alpha_in, dalpha, ft, rng, bug=None):
    """The two attention kernels computed in ft as a correct kernel may, or with `bug`."""
    s, alpha_in, dalpha = s.astype(ft), alpha_in.astype(ft), dalpha.astype(ft)
    rp = pat["m_rowptr"]
    x, e, rows = _logit(pat, s, ft, bug)
    m = ego._segmax(rp, e).astype(ft)
    d = e if bug == "no_max_shift" else e - m[rows]
    w = _exp(d, rng)
    if bug == "sum_drops_last":                   # the normaliser misses the last entry of every row
        last = np.zeros(len(w), bool)
        last[rp[1:][np.diff(rp) > 0] - 1] = True
        tot = _seq(rp, np.where(last[:, None], ft(0), w), rng)
    else:
        tot = _seq(rp, w, rng)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        alpha = w * (ft(1) / tot)[rows]
    dot = _seq(rp, alpha_in, rng, b=dalpha)
    de = alpha_in * (dalpha - dot[rows])
    branch = (e - m[rows]) if bug == "slope_from_shifted" else x
    dl = np.where(branch > 0, de, ft(0.01 if bug == "slope_001" else 0.2) * de)
    dsig2 = _seq(rp, dl, rng)
    dsig1 = dsig2 if bug == "dsig1_over_row" else _seq(pat["mT_rowptr"], dl, rng, perm=pat["mT_perm"])
    return dict(alpha=alpha, dlogit=dl, dsig1=dsig1, dsig2=dsig2)


def _gate_store(gate, rng, T=3, t=1):
    """The gate as the time slab t of a [nnz, T, Bs] store, the other slabs other gate values: (flat, off, sb, sp)."""
    Bs, nnz = gate.shape
    store = rng.random((nnz, T, Bs)).astype(gate.dtype)
    store[:, t] = gate.T
    return store.ravel(), t * Bs, 1, T * Bs


def emu_hop(rowptr, col, val, pos, gate, src, ft, rng, bug=None):
    """The hop kernel in ft (w = fl(gate val), fused multiply-adds in a shuffled order), or with `bug`."""
    Bs, nnz = gate.shape
    src, val = src.astype(ft), np.asarray(val).astype(ft)
    pos = np.asarray(pos, np.int64)
    flat, off, sb, sp = _gate_store(gate.astype(ft), rng)
    if bug == "gate_strides_swapped":
        sb, sp = sp, sb
    b = np.arange(Bs)[None, :]
    g = flat[np.clip(off + b * sb + np.maximum(pos, 0)[:, None] * sp, 0, flat.size - 1)] if nnz else \
        np.zeros((len(pos), Bs), ft)
    g = np.where(pos[:, None] >= 0, g, ft(1) if bug == "pos_minus1_as_gate1" else ft(0))
    w = g * val[:, None]                                                   # [nnz_S, Bs]
    C = src.shape[2]
    a = np.broadcast_to(w[:, :, None], (len(pos), Bs, C))
    out = _seq(rowptr, np.ascontiguousarray(a), rng, b=src[np.asarray(col, np.int64)])
    if bug == "lane_swap":                      # lanes 1 and 2 of every 4-vector of a row
        flat_out = out.reshape(len(out), -1)
        flat_out[:, 1::4], flat_out[:, 2::4] = flat_out[:, 2::4].copy(), flat_out[:, 1::4].copy()
    return out


def emu_dgate(pat, src, ddst, ft, rng, bug=None):
    src, ddst = src.astype(ft), ddst.astype(ft)
    rows, col = ego._rows_of(pat["m_rowptr"]), np.asarray(pat["m_col"], np.int64)
    C = src.shape[2]
    acc = np.zeros((pat["nnz"], src.shape[1]), ft)
    for c in rng.permutation(C):
        acc = _fma(src[rows, :, c], ddst[col, :, c], acc)
    out = (pat["m_sval"].astype(ft)[:, None] * acc).T
    if bug == "dgate_transposed":            # the value of q = (i, j) stored at (j, i); entries without a twin get 0
        N = pat["N"]
        key = rows * N + col
        tw = np.searchsorted(key, col * N + rows)
        ok = tw < len(key)
        ok[ok] = key[tw[ok]] == (col * N + rows)[ok]
        moved = np.zeros_like(out)
        moved[:, tw[ok]] = out[:, ok]
        out = moved
    return out


def emu_hop_all(inp, ft, rng, bug=None):
    p = inp["pat"]
    dst = emu_hop(p["t_rowptr"], p["t_col"], p["t_val"], p["t_pos"], inp["gate"], inp["src"], ft, rng, bug)
    dsrc = emu_hop(p["s_rowptr"], p["s_col"], p["s_val"], p["s_pos"], inp["gate"], inp["ddst"], ft, rng, bug)
    return dict(dst=dst, dsrc=dsrc, dgate=emu_dgate(p, inp["src"], inp["ddst"], ft, rng, bug))


def _attn_shapes():
    return sorted({(kw["dtype"] == F32, kw["N"], kw["Bs"], kw.get("graph", "rand"), kw.get("s_kind", "grid"))
                   for _, kw, _ in ed.ATTN_ROWS})


def _hop_shapes():
    return sorted({(kw["dtype"] == F32, kw["N"], kw["Bs"], kw["C"], kw.get("graph", "rand")) for _, kw, _ in ed.HOP_ROWS})


@pytest.mark.parametrize("shape", _attn_shapes(), ids=["%s-N%d-Bs%d-%s-%s" % ((("f32" if a[0] else "f64"),) + a[1:])
                                                        for a in _attn_shapes()])
def test_envelope_accepts_correct_attention_kernel(shape):
    f32, N, Bs, graph, s_kind = shape
    dtype = F32 if f32 else torch.float64
    inp = ed.attn_inputs(dtype, N, Bs, graph, s_kind)
    out = emu_attention(inp["pat"], inp["s"], inp["alpha_in"], inp["dalpha"], NPD[dtype], np.random.default_rng(N))
    worst = {name: orc.bound_violation(out[name], inp["ref"][name], inp["env"][name])
             for name in ("alpha", "dlogit", "dsig1", "dsig2")}
    print(shape, {k: "%.3g" % v for k, v in worst.items()})
    assert max(worst.values()) <= 1.0, worst


@pytest.mark.parametrize("shape", _hop_shapes(), ids=["%s-N%d-Bs%d-C%d-%s" % ((("f32" if a[0] else "f64"),) + a[1:])
                                                       for a in _hop_shapes()])
def test_envelope_accepts_correct_hop_kernels(shape):
    f32, N, Bs, C, graph = shape
    dtype = F32 if f32 else torch.float64
    inp = ed.hop_inputs(dtype, N, Bs, C, graph)
    out = emu_hop_all(inp, NPD[dtype], np.random.default_rng(N + C))
    worst = {name: orc.bound_violation(out[name], inp["ref"][name], inp["env"][name]) for name in ("dst", "dsrc", "dgate")}
    print(shape, {k: "%.3g" % v for k, v in worst.items()})
    assert max(worst.values()) <= 1.0, worst


# (bug, output it shows in, case); error / bound measured on the CPU with these seeds at the end of each line
WRONG = [
    ("mixer_swap", "alpha", "grid"),              # a1 applied to the row node, a2 to the column node: 2.4e10
    # the normaliser misses the last entry of each row: inf (a row of one entry divides by 0)
    ("sum_drops_last", "alpha", "grid"),
    ("no_max_shift", "alpha", "large"),           # exp(e) without the max shift overflows fp32: inf (NaN)
    ("slope_from_shifted", "dlogit", "grid"),     # LeakyReLU' read from e - m (<= 0 everywhere): 2.2e6
    ("slope_001", "dlogit", "grid"),              # negative slope 0.01 instead of 0.2: 2.3e6
    # dsig1 summed over the mask row instead of the column: 3.4e36 (a column without entries)
    ("dsig1_over_row", "dsig1", "grid"),
    # an S entry outside the mask (S_ii = -1) gated by 1: 7.1e36 (a row whose only entry is S_ii = -1)
    ("pos_minus1_as_gate1", "dst", None),
    # the gate read with its sample and position strides exchanged: 1.8e9
    ("gate_strides_swapped", "dst", None),
    ("lane_swap", "dst", None),                   # lanes 1 and 2 of each 4-vector exchanged: 2.3e10
    ("dgate_transposed", "dgate", None),          # dgate of (i, j) written at the mask entry (j, i): 3.1e7
]


@pytest.mark.parametrize("bug,out,s_kind", WRONG, ids=[w[0] for w in WRONG])
def test_envelope_rejects_wrong_kernel(bug, out, s_kind):
    rng = np.random.default_rng(3)
    if s_kind is not None:
        inp = ed.attn_inputs(F32, 3000, 13 if s_kind == "grid" else 4, "rand", s_kind)
        got = emu_attention(inp["pat"], inp["s"], inp["alpha_in"], inp["dalpha"], np.float32, rng, bug)
    else:
        inp = ed.hop_inputs(F32, 3000, 5, 8, "rand")
        got = emu_hop_all(inp, np.float32, rng, bug)
    v = orc.bound_violation(got[out], inp["ref"][out], inp["env"][out])
    print("%s: %s error / bound %.3g" % (bug, out, v))
    assert v > WIDE, (bug, v)


# ------------------------------------------------------------------------------------------------ C ABI checks
def test_egate_abi_rejects_bad_arguments_without_gpu():
    """Every call below returns before any CUDA call (the fake pointers are never dereferenced)."""
    import gnn_b200
    cabi = gnn_b200._cabi
    lib = cabi.load()
    EINVAL, EUNSUP = -1, -2
    p = ctypes.c_void_p(256)
    base = dict(dtype=cabi.F32, N=10, nnz=20, Bs=4, C=3, rowptr=p, col=p, rowptrT=p, permT=p, s=p, mixer=p, alpha=p,
                dalpha=p, dlogit=p, dsig1=p, dsig2=p, val=p, pos=p, m_rowptr=p, m_col=p, m_sval=p, gate=p, g_sb=1,
                g_sp=4, src=p, src_ld=12, dst=p, dst_ld=12, ddst=p, ddst_ld=12, dsrc=p, dsrc_ld=12, dgate=p, d_sb=1,
                d_sp=4)

    def af(**kw):
        a = dict(base, **kw)
        return lib.b200gf_egate_attention_forward(a["dtype"], a["N"], a["nnz"], a["Bs"], a["rowptr"], a["col"], a["s"],
                                                  a["mixer"], a["alpha"], None)

    def ab(**kw):
        a = dict(base, **kw)
        return lib.b200gf_egate_attention_backward(a["dtype"], a["N"], a["nnz"], a["Bs"], a["rowptr"], a["col"],
                                                   a["rowptrT"], a["permT"], a["s"], a["mixer"], a["alpha"], a["dalpha"],
                                                   a["dlogit"], a["dsig1"], a["dsig2"], None)

    def hf(**kw):
        a = dict(base, **kw)
        return lib.b200gf_gated_hop_forward(a["dtype"], a["N"], a["Bs"], a["C"], a["rowptrT"], a["col"], a["val"],
                                            a["pos"], a["gate"], a["g_sb"], a["g_sp"], a["src"], a["src_ld"], a["dst"],
                                            a["dst_ld"], None)

    def hb(**kw):
        a = dict(base, **kw)
        return lib.b200gf_gated_hop_backward(a["dtype"], a["N"], a["Bs"], a["C"], a["rowptr"], a["col"], a["val"],
                                             a["pos"], a["m_rowptr"], a["m_col"], a["m_sval"], a["gate"], a["g_sb"],
                                             a["g_sp"], a["src"], a["src_ld"], a["ddst"], a["ddst_ld"], a["dsrc"],
                                             a["dsrc_ld"], a["dgate"], a["d_sb"], a["d_sp"], None)

    for call in (af, ab, hf, hb):
        for v in (0, -1):
            assert call(Bs=v) == EINVAL, (call.__name__, v)
        assert call(N=-1) == EINVAL, call.__name__
        assert call(dtype=7) == EUNSUP, call.__name__
        assert call(N=2 ** 31) == EUNSUP, call.__name__
    for call in (af, ab):
        assert call(nnz=-1) == EINVAL and call(nnz=2 ** 31) == EUNSUP
    for call in (hf, hb):
        for v in (0, -1):
            assert call(C=v) == EINVAL, (call.__name__, v)
    for name in ("rowptr", "s", "mixer", "col", "alpha"):
        assert af(**{name: None}) == EINVAL, name
    for name in ("rowptr", "rowptrT", "s", "mixer", "dsig1", "dsig2", "col", "permT", "alpha", "dalpha", "dlogit"):
        assert ab(**{name: None}) == EINVAL, name
    for name in ("rowptrT", "col", "val", "pos", "gate", "src", "dst"):
        assert hf(**{name: None}) == EINVAL, name
    assert hf(src_ld=11) == EINVAL and hf(dst_ld=11) == EINVAL
    assert hb(dsrc=None, dgate=None) == EINVAL
    assert hb(ddst=None) == EINVAL
    for name in ("rowptr", "col", "val", "pos", "gate"):       # needed by dsrc
        assert hb(**{name: None}) == EINVAL, name
    for name in ("m_rowptr", "m_col", "m_sval", "src"):         # needed by dgate
        assert hb(**{name: None}) == EINVAL, name
    assert hb(src_ld=11) == EINVAL and hb(ddst_ld=11) == EINVAL and hb(dsrc_ld=11) == EINVAL
    # nothing to do: OK and no launch
    n0 = lib.b200gf_launch_count(0)
    assert af(N=0) == 0 and ab(N=0) == 0 and hf(N=0) == 0 and hb(N=0) == 0
    assert lib.b200gf_launch_count(0) == n0
