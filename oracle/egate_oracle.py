"""fp64 restatement of the edge-gated recurrent layer.  TEST INFRASTRUCTURE — NOT PRODUCT CODE.

EdgeGatedHiddenState (alegnn/utils/graphML.py:4033-4209): two ungated gate GRNNs, sparse learnAttentionGSO
(:640-737) on their trajectories, and GatedGRNN's edge path (:1410-1451, :1474-1514), written with per-non-zero index
arithmetic in torch so that autograd gives every gradient and the restatement runs at sizes where the reference's dense
B*T x N x N gates cannot be allocated.  Pinned against the reference's own results in tests/golden/grnn_edge_cases.npz
(oracle/make_golden_edge.py) by tests/test_edge_gated.py; the at-scale GPU test trusts it from there.

Conventions as in the reference: x [B, T, F, N], z0 [B, H, N], z [B, T, H, N]; the shift is the row-vector product
(u S)[j] = sum_i u[i] S[i, j].  Device-agnostic (the tensors' device is used).

The second half restates the four C entry points of csrc/egate.cu in numpy / scipy fp64, on the operands and layouts
of include/b200gf.h, with `egate_envelope`, the componentwise bound tests/test_egate_dispatch.py holds the kernels to.
tests/test_egate_oracle.py pins them to the torch restatement above and tests the bound on emulated kernels.
"""
import numpy as np
import scipy.sparse as sp

from lsigf_oracle import unit_roundoff

# edge-gated recurrent layer: EdgeGatedHiddenState (graphML.py:4033-4209) with per-non-zero index arithmetic
# --------------------------------------------------------------------------------------------
def egate_mask_coo(N, rows, cols, vals, tol=1e-9):
    """Mask of |S + I| > tol (graphML.py:692, :726-728) from S's COO (numpy; no duplicates).  Returns (m_rows, m_cols,
    m_sval) in row-major order, m_sval = S_ij on the mask (0 where S has no entry)."""
    rows, cols, vals = np.asarray(rows, np.int64), np.asarray(cols, np.int64), np.asarray(vals)
    S = sp.csr_matrix((vals, (rows, cols)), shape=(N, N))
    A = (S + sp.identity(N, dtype=vals.dtype, format="csr")).tocoo()
    keep = np.abs(A.data) > tol
    m_rows, m_cols = A.row[keep].astype(np.int64), A.col[keep].astype(np.int64)
    order = np.argsort(m_rows * N + m_cols)
    m_rows, m_cols = m_rows[order], m_cols[order]
    m_sval = np.asarray(S[m_rows, m_cols]).ravel() if m_rows.size else np.zeros(0, vals.dtype)
    return m_rows, m_cols, m_sval


def egate_attention_coo(s, mixer, m_rows, m_cols, N):
    """Sparse learnAttentionGSO (graphML.py:640-737, P = E = F = 1): s [Bs, N] (= W z per node), mixer [2] ->
    alpha [Bs, nnz_mask], softmax over the mask row i of LeakyReLU_0.2(mixer[0] s_j + mixer[1] s_i)."""
    import torch
    Bs = s.shape[0]
    e = torch.nn.functional.leaky_relu(mixer[0] * s[:, m_cols] + mixer[1] * s[:, m_rows], 0.2)
    mx = torch.full((Bs, N), -float("inf"), dtype=s.dtype, device=s.device)
    mx = mx.scatter_reduce(1, m_rows.expand(Bs, -1), e.detach(), "amax")
    w = torch.exp(e - mx[:, m_rows])
    den = torch.zeros((Bs, N), dtype=s.dtype, device=s.device).index_add(1, m_rows, w)
    return w / den[:, m_rows]


def _egate_hop(u, w, rows, cols):
    g = (w if w.dim() == 2 else w.unsqueeze(0))[:, None, :] * u[:, :, rows]
    return u.new_zeros(u.shape).index_add(2, cols, g)


def egate_hop_coo(u, w, rows, cols):
    """(u S~)[b, c, j] = sum over the entries (i, j) of w[b, q] u[b, c, i]; u [Bs, C, N], w [Bs, nnz] or [nnz]
    (w = gate * S_ij on the mask, or S_ij alone for an ungated hop).  Checkpointed: autograd keeps u and w, not the
    [Bs, C, nnz] gathered operand, so the oracle runs at N = 50 000 in fp64."""
    import torch
    from torch.utils.checkpoint import checkpoint
    if torch.is_grad_enabled() and (u.requires_grad or w.requires_grad):
        return checkpoint(_egate_hop, u, w, rows, cols, use_reentrant=False)
    return _egate_hop(u, w, rows, cols)


def _grnn_coo(a, b, x, z0, sigma, xb, zb, hop_x, hop_z):
    """GatedGRNN (graphML.py:1292-1527) without output gates; hop_x(u) shifts [B*T, F, N], hop_z(u, t) [B, H, N]."""
    import torch
    H, _, K, F = a.shape
    B, T, _, N = x.shape

    def filt(taps, u, hop):
        us = [u]
        for _ in range(1, K):
            u = hop(u)
            us.append(u)
        y = torch.einsum("bkcn,hkc->bhn", torch.stack(us, 1), taps[:, 0])
        return y
    Ax = filt(a, x.reshape(B * T, F, N), hop_x)
    if xb is not None:
        Ax = Ax + xb.reshape(1, H, 1)
    Ax = Ax.reshape(B, T, H, N)
    zt, out = z0, []
    for t in range(T):
        Bz = filt(b, zt, lambda u: hop_z(u, t))
        if zb is not None:
            Bz = Bz + zb.reshape(1, H, 1)
        zt = sigma(Ax[:, t] + Bz)
        out.append(zt)
    return torch.stack(out, 1)


def edge_gated_hidden_state_coo(p, N, rows, cols, vals, x, z0, sigma, tol=1e-9):
    """EdgeGatedHiddenState.forward (graphML.py:4133-4178) on S's COO (rows, cols, vals numpy), in torch with autograd.
    p: the layer's state_dict as torch tensors (reference key names; xBias / zBias absent without bias).  Returns
    (z [B, T, H, N], qHat, qCheck [B, T, nnz_mask], (m_rows, m_cols))."""
    import torch
    dev, dt = x.device, x.dtype
    B, T, _, _ = x.shape
    H = p["aWeights"].shape[0]
    m_rows, m_cols, m_sval = egate_mask_coo(N, rows, cols, vals, tol)
    r = torch.as_tensor(np.asarray(rows, np.int64), device=dev)
    c = torch.as_tensor(np.asarray(cols, np.int64), device=dev)
    v = torch.as_tensor(np.asarray(vals), device=dev).to(dt)
    mr, mc = torch.as_tensor(m_rows, device=dev), torch.as_tensor(m_cols, device=dev)
    ms = torch.as_tensor(m_sval, device=dev).to(dt)
    plain = lambda u: egate_hop_coo(u, v, r, c)                                   # noqa: E731

    def gate_grnn(pre):
        return _grnn_coo(p[pre + "aWeights"], p[pre + "bWeights"], x, z0, torch.tanh, p.get(pre + "xBias"),
                         p.get(pre + "zBias"), plain, lambda u, t: plain(u))

    def attention(zg, pre):
        s = torch.einsum("btHn,H->btn", zg, p[pre + "weight"].reshape(H)).reshape(B * T, N)
        return egate_attention_coo(s, p[pre + "mixer"].reshape(2), mr, mc, N).reshape(B, T, -1)
    qHat = attention(gate_grnn("inputGateGRNN."), "inputGateGAT.")
    qCheck = attention(gate_grnn("forgetGateGRNN."), "forgetGateGAT.")
    qh = qHat.reshape(B * T, -1)
    z = _grnn_coo(p["aWeights"], p["bWeights"], x, z0, sigma, p.get("xBias"), p.get("zBias"),
                  lambda u: egate_hop_coo(u, qh * ms, mr, mc), lambda u, t: egate_hop_coo(u, qCheck[:, t] * ms, mr, mc))
    return z, qHat, qCheck, (m_rows, m_cols)


# the four C entry points of csrc/egate.cu (include/b200gf.h), restated in numpy / scipy fp64
# --------------------------------------------------------------------------------------------
def egate_pattern(N, rows, cols, vals, tol=1e-9):
    """The CSRs the entry points read, built from S's COO (numpy, no duplicates), with the member names of
    gnn_b200.EdgeGatePattern: mask CSR m_rowptr / m_col and its transpose mT_rowptr / mT_perm, m_sval (S in mask
    order), the CSR of S^T (t_rowptr, t_col = i, t_val, t_pos) and of S (s_rowptr, s_col = j, s_val, s_pos), where
    *_pos is the entry's position in the mask or -1.  Offsets int64, indices int32."""
    rows, cols, vals = np.asarray(rows, np.int64), np.asarray(cols, np.int64), np.asarray(vals, np.float64)
    m_rows, m_cols, m_sval = egate_mask_coo(N, rows, cols, vals, tol)
    m_key = m_rows * N + m_cols
    key = rows * N + cols
    pos = np.searchsorted(m_key, key)
    hit = pos < m_key.size
    hit[hit] = m_key[pos[hit]] == key[hit]
    pos = np.where(hit, pos, -1)

    def rowptr(r):
        return np.concatenate([[0], np.cumsum(np.bincount(r, minlength=N))]).astype(np.int64)
    o, oT = np.argsort(key, kind="stable"), np.argsort(cols * N + rows, kind="stable")
    return dict(N=N, nnz=int(m_key.size), m_rowptr=rowptr(m_rows), m_col=m_cols.astype(np.int32),
                mT_rowptr=rowptr(m_cols), mT_perm=np.argsort(m_cols * N + m_rows, kind="stable").astype(np.int32),
                m_sval=np.asarray(m_sval, np.float64),
                s_rowptr=rowptr(rows[o]), s_col=cols[o].astype(np.int32), s_val=vals[o], s_pos=pos[o].astype(np.int32),
                t_rowptr=rowptr(cols[oT]), t_col=rows[oT].astype(np.int32), t_val=vals[oT],
                t_pos=pos[oT].astype(np.int32))


def _rows_of(rowptr):
    rowptr = np.asarray(rowptr, np.int64)
    return np.repeat(np.arange(len(rowptr) - 1), np.diff(rowptr))


def _segsum(rowptr, v):
    """Per-row sums of v [nnz, ...] over the CSR segments (0 for an empty row)."""
    rowptr = np.asarray(rowptr, np.int64)
    n, nnz = len(rowptr) - 1, int(rowptr[-1])
    R = sp.csr_matrix((np.ones(nnz), np.arange(nnz), rowptr), shape=(n, nnz))
    return np.asarray(R @ v.reshape(nnz, int(np.prod(v.shape[1:])))).reshape((n,) + v.shape[1:])


def _colsum(col, v, N):
    """Per-column sums of v [nnz, ...] over the entries of each column."""
    nnz = len(col)
    Ct = sp.csr_matrix((np.ones(nnz), (np.asarray(col, np.int64), np.arange(nnz))), shape=(N, nnz))
    return np.asarray(Ct @ v.reshape(nnz, int(np.prod(v.shape[1:])))).reshape((N,) + v.shape[1:])


def _segmax(rowptr, v):
    """Per-row maxima of v [nnz, Bs] (-inf for an empty row)."""
    rowptr = np.asarray(rowptr, np.int64)
    out = np.full((len(rowptr) - 1,) + v.shape[1:], -np.inf)
    live = np.diff(rowptr) > 0
    if live.any():
        out[live] = np.maximum.reduceat(v, rowptr[:-1][live], axis=0)
    return out


def attention_logits(rowptr, col, s, mixer):
    """x[q, b] = a1 s[j, b] + a2 s[i, b] (before the LeakyReLU), q = (i, j) in the mask CSR; s [N, Bs]."""
    s = np.asarray(s, np.float64)
    a1, a2 = (float(v) for v in np.asarray(mixer, np.float64).reshape(2))
    return a1 * s[np.asarray(col, np.int64)] + a2 * s[_rows_of(rowptr)]


def attention_forward(rowptr, col, s, mixer):
    """b200gf_egate_attention_forward: alpha [nnz, Bs] = softmax over each mask row of LeakyReLU_0.2(a1 s_j + a2 s_i)."""
    x = attention_logits(rowptr, col, s, mixer)
    e = np.where(x > 0, x, 0.2 * x)
    rows = _rows_of(rowptr)
    w = np.exp(e - _segmax(rowptr, e)[rows])
    return w / _segsum(rowptr, w)[rows]


def attention_backward(rowptr, col, s, mixer, alpha, dalpha):
    """b200gf_egate_attention_backward with alpha and dalpha [nnz, Bs] taken as given:
    dlogit = alpha (dalpha - sum_row alpha dalpha) LeakyReLU'(x) (LeakyReLU'(0) = 0.2, as torch and the kernel),
    dsig2 [N, Bs] = sum over each mask row of dlogit, dsig1 [N, Bs] = sum over each mask column."""
    alpha, dalpha = np.asarray(alpha, np.float64), np.asarray(dalpha, np.float64)
    rows = _rows_of(rowptr)
    N = len(rowptr) - 1
    dot = _segsum(rowptr, alpha * dalpha)
    slope = np.where(attention_logits(rowptr, col, s, mixer) > 0, 1.0, 0.2)
    dlogit = slope * alpha * (dalpha - dot[rows])
    return dlogit, _colsum(col, dlogit, N), _segsum(rowptr, dlogit)


def _hop(rowptr, col, val, pos, gate, src):
    """dst[r, b, :] = sum over row r's entries it (pos >= 0) of val[it] gate[b, pos[it]] src[col[it], b, :]."""
    gate = np.asarray(gate, np.float64)
    src = np.asarray(src, np.float64)
    n = len(rowptr) - 1
    pos = np.asarray(pos, np.int64)
    live = pos >= 0
    w = np.zeros((src.shape[1], len(pos)))
    w[:, live] = gate[:, pos[live]] * np.asarray(val, np.float64)[None, live]
    out = np.zeros((n,) + src.shape[1:])
    for b in range(src.shape[1]):
        out[:, b] = sp.csr_matrix((w[b], np.asarray(col, np.int64), np.asarray(rowptr, np.int64)),
                                  shape=(n, src.shape[0])) @ src[:, b]
    return out


def gated_hop_forward(rowptrT, colT, valT, posT, gate, src):
    """b200gf_gated_hop_forward: dst [N, Bs, C] = src S~ per sample, over the CSR of S^T; gate [Bs, nnz], src [N, Bs, C]."""
    return _hop(rowptrT, colT, valT, posT, gate, src)


def gated_hop_backward(rowptr, col, val, pos, m_rowptr, m_col, m_sval, gate, src, ddst):
    """b200gf_gated_hop_backward: dsrc [N, Bs, C] = the same hop over the CSR of S applied to ddst, and
    dgate [Bs, nnz] = m_sval[q] sum_c src[i, b, c] ddst[j, b, c] for every mask entry q = (i, j)."""
    src, ddst = np.asarray(src, np.float64), np.asarray(ddst, np.float64)
    dgate = np.einsum("qbc,qbc->bq", src[_rows_of(m_rowptr)], ddst[np.asarray(m_col, np.int64)])
    return _hop(rowptr, col, val, pos, gate, ddst), dgate * np.asarray(m_sval, np.float64)[None, :]


def egate_envelope(dtype, pat, s=None, mixer=None, alpha=None, dalpha=None, gate=None, src=None, ddst=None):
    """Componentwise first-order bounds on the outputs of the four entry points computed in `dtype` (every input
    already rounded to it).  pat: egate_pattern's dict.  Returns dict name -> bound for the outputs the given inputs
    determine: alpha (s, mixer), dlogit / dsig1 / dsig2 (s, mixer, alpha, dalpha), dst (gate, src), dsrc (gate, ddst),
    dgate (src, ddst).  u = lsigf_oracle.unit_roundoff (doubled for fp64 to cover this restatement's own rounding),
    and every bound carries the floor tiny = 4 * finfo.tiny * (n + 2) for underflow, n the length of the sum.

    Gated hops.  Each entry multiplies fl(gate * val) (one rounding) into a fused multiply-add (one more), so an output
    over a row of n entries has |err| <= (n + 2) u M, M = the same hop run on |S|, |gate| and |src|, with n the length
    of that row of S^T (dst) or of S (dsrc).  dgate = m_sval * (C fused multiply-adds): (C + 2) u |m_sval| sum_c |src ddst|.

    Attention backward (alpha, dalpha, s and the mixer exact).  With the coarse-grid inputs the dispatch cases use, the
    logit a1 s_j + a2 s_i is exact in fp32 and fp64, so the slope of LeakyReLU' is the same on both sides.  The row
    dot product takes n fused multiply-adds, dalpha - dot one rounding, alpha * (.) one more and the slope one more
    (plus one for fp32 0.2f != 0.2 on the negative branch):
        |d dlogit| <= (n + 4 [+ 1]) u slope alpha (|dalpha| + sum_row alpha |dalpha|).
    dsig2 / dsig1 sum those over a row / column of n entries: the sum of their bounds + n u sum |dlogit|.

    Attention forward.  The error of alpha is relative to alpha.  The kernel computes d_q = e_q - m with m the row max;
    the error of the computed d_q (in units of u) is at most
        kappa_q = |a1 s_j| + |a2 s_i| + |x_q| + 2 |e_q| + |d_q|
    (two products and a sum for x, LeakyReLU is 1-Lipschitz so a sign flip of x costs no more than x's error, the 0.2
    product and its constant, the subtraction).  An error common to every d of a row (the computed max) cancels in
    the ratio, so alpha_q's relative error is at most u (kappa_q + max_row kappa + n + c0): its own d, the weighted
    mean of the others', n - 1 sums, and c0 = 10 for exp (<= 2 ulp = 4u in fp32 without fast math, twice: alpha_q's own
    and the sum's) + 1/sum + the final product.  Entries whose exp underflows lose at most the floor."""
    u = unit_roundoff(dtype)
    fl = 4.0 * np.finfo(np.dtype(dtype)).tiny
    out = {}
    m_rowptr, m_col, N = pat["m_rowptr"], pat["m_col"], pat["N"]
    R = np.diff(m_rowptr).astype(np.float64)                  # mask row lengths
    RT = np.bincount(np.asarray(m_col, np.int64), minlength=N).astype(np.float64)
    rows = _rows_of(m_rowptr)
    if s is not None:
        s = np.asarray(s, np.float64)
        a1, a2 = (float(v) for v in np.asarray(mixer, np.float64).reshape(2))
        x = attention_logits(m_rowptr, m_col, s, mixer)
        e = np.where(x > 0, x, 0.2 * x)
        d = e - _segmax(m_rowptr, e)[rows]
        kappa = np.abs(a1 * s[np.asarray(m_col, np.int64)]) + np.abs(a2 * s[rows]) + np.abs(x) + 2 * np.abs(e) + np.abs(d)
        kmax = _segmax(m_rowptr, kappa)[rows]
        al = attention_forward(m_rowptr, m_col, s, mixer)
        out["alpha"] = al * u * (kappa + kmax + R[rows][:, None] + 10) + fl * (R[rows][:, None] + 2)
        if alpha is not None:
            alpha, dalpha = np.asarray(alpha, np.float64), np.asarray(dalpha, np.float64)
            neg = x <= 0
            slope = np.where(neg, 0.2, 1.0)
            Mdot = _segsum(m_rowptr, alpha * np.abs(dalpha))
            c = R[rows][:, None] + 4 + neg
            bl = c * u * slope * alpha * (np.abs(dalpha) + Mdot[rows]) + fl * (R[rows][:, None] + 2)
            dlogit, _, _ = attention_backward(m_rowptr, m_col, s, mixer, alpha, dalpha)
            adl = np.abs(dlogit)
            out["dlogit"] = bl
            out["dsig2"] = _segsum(m_rowptr, bl + R[rows][:, None] * u * adl) + fl * (R[:, None] + 2)
            out["dsig1"] = _colsum(m_col, bl + RT[np.asarray(m_col, np.int64)][:, None] * u * adl, N) \
                + fl * (RT[:, None] + 2)
    ag = None if gate is None else np.abs(np.asarray(gate, np.float64))
    if gate is not None and src is not None:
        n = np.diff(pat["t_rowptr"]).astype(np.float64)[:, None, None]
        M = _hop(pat["t_rowptr"], pat["t_col"], np.abs(pat["t_val"]), pat["t_pos"], ag, np.abs(src))
        out["dst"] = (n + 2) * u * M + fl * (n + 2)
    if gate is not None and ddst is not None:
        n = np.diff(pat["s_rowptr"]).astype(np.float64)[:, None, None]
        M = _hop(pat["s_rowptr"], pat["s_col"], np.abs(pat["s_val"]), pat["s_pos"], ag, np.abs(ddst))
        out["dsrc"] = (n + 2) * u * M + fl * (n + 2)
    if src is not None and ddst is not None:
        C = np.shape(src)[2]
        _, Mg = gated_hop_backward(pat["s_rowptr"], pat["s_col"], pat["s_val"], pat["s_pos"], m_rowptr, m_col,
                                   np.abs(pat["m_sval"]), np.zeros((np.shape(src)[1], pat["nnz"])), np.abs(src),
                                   np.abs(ddst))
        out["dgate"] = (C + 2) * u * Mg + fl * (C + 2)
    return out
