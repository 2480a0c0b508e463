"""fp64 restatement of the edge-gated recurrent layer.  TEST INFRASTRUCTURE — NOT PRODUCT CODE.

EdgeGatedHiddenState (alegnn/utils/graphML.py:4033-4209): two ungated gate GRNNs, sparse learnAttentionGSO
(:640-737) on their trajectories, and GatedGRNN's edge path (:1410-1451, :1474-1514), written with per-non-zero index
arithmetic in torch so that autograd gives every gradient and the restatement runs at sizes where the reference's dense
B*T x N x N gates cannot be allocated.  Pinned against the reference's own results in tests/golden/grnn_edge_cases.npz
(oracle/make_golden_edge.py) by tests/test_edge_gated.py; the at-scale GPU test trusts it from there.

Conventions as in the reference: x [B, T, F, N], z0 [B, H, N], z [B, T, H, N]; the shift is the row-vector product
(u S)[j] = sum_i u[i] S[i, j].  Device-agnostic (the tensors' device is used).
"""
import numpy as np
import scipy.sparse as sp

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
