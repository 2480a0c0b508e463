"""fp64 restatement of the graph attention layers.  TEST INFRASTRUCTURE — NOT PRODUCT CODE.

graphAttention, graphAttentionLSIGF, graphAttentionEVGF (alegnn/utils/graphML.py:739-969) on the COO of the mask of
S + I, in torch with autograd (device-agnostic), built on egate_oracle's per-non-zero index arithmetic
(`egate_hop_coo`) with the attention generalised to two score arrays: the column node j is scored by s_src = a1^T W x,
the row node i by s_dst = a2^T W x.  Pinned against the reference's own results in tests/golden/attention_cases.npz
(oracle/make_golden_attention.py) by tests/test_attention.py; the at-scale GPU test trusts it from there.

The second half restates the two-score C entry points (b200gf_attention_forward / _backward) in numpy fp64 with
`attention_envelope`, the componentwise bound tests/test_attention_dispatch.py holds them to: egate_oracle's
`egate_envelope` with a1 s_j, a2 s_i replaced by s_src[j], s_dst[i] (egate_envelope itself is unchanged).
"""
import numpy as np
import scipy.sparse as sp

import egate_oracle as ego
from lsigf_oracle import unit_roundoff


def attention_mask_coo(S, tol=1e-9):
    """Mask of the reference (graphML.py:692, :726-728) from a list of E scipy matrices S_e: off the diagonal
    sum_e |S_e,ij| > tol, on it sum_e |S_e,ii + 1| > tol.  Returns (m_rows, m_cols) in row-major order."""
    N = S[0].shape[0]
    A = sum(abs(sp.csr_matrix(s) + sp.identity(N, format="csr")) for s in S).tocoo()
    keep = A.data > tol
    r, c = A.row[keep].astype(np.int64), A.col[keep].astype(np.int64)
    o = np.argsort(r * N + c)
    return r[o], c[o]


def attention_coo(s_src, s_dst, m_rows, m_cols, N):
    """alpha [Bs, nnz] = softmax over the mask row i of LeakyReLU_0.2(s_src[:, j] + s_dst[:, i]); s_* [Bs, N]."""
    import torch
    Bs = s_src.shape[0]
    e = torch.nn.functional.leaky_relu(s_src[:, m_cols] + s_dst[:, m_rows], 0.2)
    mx = torch.full((Bs, N), -float("inf"), dtype=e.dtype, device=e.device)
    mx = mx.scatter_reduce(1, m_rows.expand(Bs, -1), e.detach(), "amax")
    w = torch.exp(e - mx[:, m_rows])
    den = torch.zeros((Bs, N), dtype=e.dtype, device=e.device).index_add(1, m_rows, w)
    return w / den[:, m_rows]


class CooGSO:
    """The mask and each S_e on the mask, as torch index tensors on `device`."""

    def __init__(self, S, device, dtype, tol=1e-9):
        import torch
        self.N = S[0].shape[0]
        mr, mc = attention_mask_coo(S, tol)
        self.mr = torch.as_tensor(mr, device=device)
        self.mc = torch.as_tensor(mc, device=device)
        # S_e restricted to the mask, in mask order (entries outside it are gated to zero)
        self.sval = [torch.as_tensor(np.asarray(sp.csr_matrix(s)[mr, mc]).ravel(), device=device).to(dtype)
                     for s in S]

    def attention(self, Wx, a):
        """Wx [B, P, F, N], a [P, 2F] (one edge feature) -> alpha [B*P, nnz]."""
        B, P, F, N = Wx.shape
        import torch
        s_src = torch.einsum("bpfn,pf->bpn", Wx, a[:, :F]).reshape(B * P, N)
        s_dst = torch.einsum("bpfn,pf->bpn", Wx, a[:, F:]).reshape(B * P, N)
        return attention_coo(s_src, s_dst, self.mr, self.mc, N)

    def hop(self, u, w):
        """u [Bs, C, N] (row vector per (b, c)), w [Bs, nnz] on the mask -> u (w on the mask)."""
        return ego.egate_hop_coo(u, w, self.mr, self.mc)


def graph_attention(g, x, a, W):
    """graphAttention: x [B, G, N], a [P, E, 2F], W [P, E, F, G] -> [B, P, F, N]."""
    import torch
    B, G, N = x.shape
    P, E, F, _ = W.shape
    y = 0
    for e in range(E):
        Wx = torch.einsum("pfg,bgn->bpfn", W[:, e], x)
        al = g.attention(Wx, a[:, e])
        y = y + g.hop(Wx.reshape(B * P, F, N), al * g.sval[e]).reshape(B, P, F, N)
    return y


def graph_attention_lsigf(g, h, x, a, W, b=None):
    """graphAttentionLSIGF: h [E, K], x [B, G, N], a [P, E, 2F], W [P, E, F, G] -> [B, P, F, N]."""
    import torch
    E, K = h.shape
    B, G, N = x.shape
    P, _, F, _ = W.shape
    taps = h.reshape(1, 1, E, K, 1) * W.permute(0, 3, 1, 2).reshape(P, F, E, 1, G)
    y = 0
    for e in range(E):
        al = g.attention(torch.einsum("pfg,bgn->bpfn", W[:, e], x), a[:, e])
        u = x.unsqueeze(1).expand(B, P, G, N).reshape(B * P, G, N)
        for k in range(K):
            if k > 0:
                u = g.hop(u, al)
            y = y + torch.einsum("bpgn,pfg->bpfn", u.reshape(B, P, G, N), taps[:, :, e, k])
    return y if b is None else y + b


def graph_attention_evgf(g, x, a, W, b=None):
    """graphAttentionEVGF: x [B, G, N], a [P, K, E, 2F], W [P, K, E, F, G] -> [B, P, F, N]."""
    import torch
    B, G, N = x.shape
    P, K, E, F, _ = W.shape
    y = 0
    for e in range(E):
        u = torch.einsum("pfg,bgn->bpfn", W[:, 0, e], x).reshape(B * P, F, N)
        for k in range(K):
            al = g.attention(torch.einsum("pfg,bgn->bpfn", W[:, k, e], x), a[:, k, e])
            u = g.hop(u, al * g.sval[e])
            y = y + u.reshape(B, P, F, N)
    return y if b is None else y + b


# the two-score C entry points (include/b200gf.h), restated in numpy fp64
# --------------------------------------------------------------------------------------------
def attention_logits(rowptr, col, s_src, s_dst):
    """x[q, b] = s_src[j, b] + s_dst[i, b], q = (i, j) in the mask CSR; s_* [N, Bs]."""
    return np.asarray(s_src, np.float64)[np.asarray(col, np.int64)] + np.asarray(s_dst, np.float64)[ego._rows_of(rowptr)]


def attention_forward(rowptr, col, s_src, s_dst):
    """b200gf_attention_forward (mixer (1, 1)): alpha [nnz, Bs]."""
    x = attention_logits(rowptr, col, s_src, s_dst)
    e = np.where(x > 0, x, 0.2 * x)
    rows = ego._rows_of(rowptr)
    w = np.exp(e - ego._segmax(rowptr, e)[rows])
    return w / ego._segsum(rowptr, w)[rows]


def attention_backward(rowptr, col, s_src, s_dst, alpha, dalpha):
    """b200gf_attention_backward (mixer (1, 1)): (dlogit, dsig1 = column sums = d/ds_src, dsig2 = row sums = d/ds_dst)."""
    alpha, dalpha = np.asarray(alpha, np.float64), np.asarray(dalpha, np.float64)
    rows = ego._rows_of(rowptr)
    N = len(rowptr) - 1
    dot = ego._segsum(rowptr, alpha * dalpha)
    slope = np.where(attention_logits(rowptr, col, s_src, s_dst) > 0, 1.0, 0.2)
    dlogit = slope * alpha * (dalpha - dot[rows])
    return dlogit, ego._colsum(col, dlogit, N), ego._segsum(rowptr, dlogit)


def attention_envelope(dtype, pat, s_src, s_dst, alpha=None, dalpha=None):
    """Componentwise first-order bounds on alpha (and dlogit, dsig1, dsig2 given alpha and dalpha) of the two-score
    entry points computed in `dtype`: egate_envelope's attention bounds (see there for the derivation) with the two
    products a1 s_j, a2 s_i replaced by s_src[j], s_dst[i] (the mixer (1, 1) multiplies exactly)."""
    u = unit_roundoff(dtype)
    fl = 4.0 * np.finfo(np.dtype(dtype)).tiny
    out = {}
    m_rowptr, m_col, N = pat["m_rowptr"], pat["m_col"], pat["N"]
    R = np.diff(m_rowptr).astype(np.float64)
    RT = np.bincount(np.asarray(m_col, np.int64), minlength=N).astype(np.float64)
    rows = ego._rows_of(m_rowptr)
    s_src, s_dst = np.asarray(s_src, np.float64), np.asarray(s_dst, np.float64)
    x = attention_logits(m_rowptr, m_col, s_src, s_dst)
    e = np.where(x > 0, x, 0.2 * x)
    d = e - ego._segmax(m_rowptr, e)[rows]
    kappa = np.abs(s_src[np.asarray(m_col, np.int64)]) + np.abs(s_dst[rows]) + np.abs(x) + 2 * np.abs(e) + np.abs(d)
    kmax = ego._segmax(m_rowptr, kappa)[rows]
    al = attention_forward(m_rowptr, m_col, s_src, s_dst)
    out["alpha"] = al * u * (kappa + kmax + R[rows][:, None] + 10) + fl * (R[rows][:, None] + 2)
    if alpha is not None:
        alpha, dalpha = np.asarray(alpha, np.float64), np.asarray(dalpha, np.float64)
        neg = x <= 0
        slope = np.where(neg, 0.2, 1.0)
        Mdot = ego._segsum(m_rowptr, alpha * np.abs(dalpha))
        c = R[rows][:, None] + 4 + neg
        bl = c * u * slope * alpha * (np.abs(dalpha) + Mdot[rows]) + fl * (R[rows][:, None] + 2)
        dlogit, _, _ = attention_backward(m_rowptr, m_col, s_src, s_dst, alpha, dalpha)
        adl = np.abs(dlogit)
        out["dlogit"] = bl
        out["dsig2"] = ego._segsum(m_rowptr, bl + R[rows][:, None] * u * adl) + fl * (R[:, None] + 2)
        out["dsig1"] = ego._colsum(m_col, bl + RT[np.asarray(m_col, np.int64)][:, None] * u * adl, N) \
            + fl * (RT[:, None] + 2)
    return out
