"""fp64 restatement of the edge-variant filter's C ABI (b200gf_ev_forward / b200gf_ev_backward, include/b200gf.h) and
componentwise error envelopes for it.  TEST INFRASTRUCTURE — NOT PRODUCT CODE (same rules as lsigf_oracle.py).

Operands are the header's, batch innermost: pattern CSR (rowptr [NA+1], col [nnz]) shared by every (f, k, g);
w [F, K, G, nnz]; xT [G, NA, B]; Y, dY [F, NA, B]; chain states u_k [F*G, NA, B].  Column convention u_k = Phi_k u_{k-1},
u_{-1} = x_g (alegnn graphML.py:464,475), Y_f = sum_g sum_k u_k.  diag (int [NA] or None): position of row i's diagonal
entry in the pattern, -1 if it is not live.  When given, Phi_0 is diagonal: u_0[i] = w_0[diag[i]] x[i] (0 where
diag[i] = -1), whatever the other k = 0 slots hold, and only the diagonal slots of dw_0 are live (the rest are 0).
"""
import numpy as np
import scipy.sparse as sp

from lsigf_oracle import unit_roundoff


def _phi(rowptr, col, diag, w_fkg, k, NA):
    """Phi_k of one (f, g) chain as a scipy CSR matrix (at k = 0 with diag: the diagonal matrix of the diag slots)."""
    if k == 0 and diag is not None:
        d = np.asarray(diag, dtype=np.int64)
        coef = np.zeros(NA)
        on = d >= 0
        coef[on] = w_fkg[d[on]]
        return sp.diags(coef, format="csr")
    return sp.csr_matrix((w_fkg, np.asarray(col, dtype=np.int64), np.asarray(rowptr, dtype=np.int64)), shape=(NA, NA))


def ev_forward(rowptr, col, diag, w, xT):
    """-> (Y [F, NA, B], U [K-1, F*G, NA, B]) with U[k] = u_k, the states b200gf_ev_forward keeps for the backward."""
    w = np.asarray(w, dtype=np.float64)
    xT = np.asarray(xT, dtype=np.float64)
    F, K, G, nnz = w.shape
    _, NA, B = xT.shape
    Y = np.zeros((F, NA, B))
    U = np.zeros((max(K - 1, 0), F * G, NA, B))
    for f in range(F):
        for g in range(G):
            u = xT[g]
            for k in range(K):
                u = _phi(rowptr, col, diag, w[f, k, g], k, NA) @ u
                Y[f] += u
                if k < K - 1:
                    U[k, f * G + g] = u
    return Y, U


def ev_backward(rowptr, col, diag, w, xT, dY):
    """-> (dw [F, K, G, nnz], dxT [G, NA, B], lam [K, F*G, NA, B]) for upstream dY [F, NA, B]:
        lam_{K-1} = dY,   lam_{k-1} = dY + Phi_k^T lam_k,
        dw_k[(f, g), q = (i, j)] = sum_b lam_k[i, b] prev[j, b]     (prev = u_{k-1}, x_g at k = 0),
        dxT_g = sum_f Phi_0(f, g)^T lam_0.
    With diag, dw_0 has only the slots diag[i] >= 0, at (i, i)."""
    w = np.asarray(w, dtype=np.float64)
    xT = np.asarray(xT, dtype=np.float64)
    dY = np.asarray(dY, dtype=np.float64)
    F, K, G, nnz = w.shape
    _, NA, B = xT.shape
    _, U = ev_forward(rowptr, col, diag, w, xT)
    rows = np.repeat(np.arange(NA), np.diff(np.asarray(rowptr, dtype=np.int64)))
    cols = np.asarray(col, dtype=np.int64)
    if diag is not None:
        d = np.asarray(diag, dtype=np.int64)
        slots0, i0 = d[d >= 0], np.nonzero(d >= 0)[0]
    dw = np.zeros((F, K, G, nnz))
    dxT = np.zeros((G, NA, B))
    lam = np.zeros((K, F * G, NA, B))
    for f in range(F):
        for g in range(G):
            fg = f * G + g
            lk = dY[f]
            for k in range(K - 1, -1, -1):
                lam[k, fg] = lk
                prev = U[k - 1, fg] if k > 0 else xT[g]
                if k == 0 and diag is not None:
                    dw[f, 0, g, slots0] = np.einsum("nb,nb->n", lk[i0], prev[i0])
                else:
                    dw[f, k, g] = np.einsum("nb,nb->n", lk[rows], prev[cols])
                phi = _phi(rowptr, col, diag, w[f, k, g], k, NA)
                if k == 0:
                    dxT[g] += phi.T @ lk
                else:
                    lk = dY[f] + phi.T @ lk
    return dw, dxT, lam


def ev_depths(rowptr, col, K, G, F, B):
    """Accumulation depths c of each output (|error| <= c u M to first order, M the run on absolute values).
    R / RT: longest pattern row / column.  Y: K chained row products, G + K sums.  lam: K-1 chained column products
    that each start from dY.  dw: B products of lam and u, each carrying its own error.  dxT: F column products of lam_0."""
    R = int(np.diff(np.asarray(rowptr, dtype=np.int64)).max(initial=0))
    NA = len(rowptr) - 1
    RT = int(np.bincount(np.asarray(col, dtype=np.int64), minlength=NA).max(initial=0))
    c_u = (K - 1) * R                     # u_{K-2}, the deepest state dw reads
    c_lam = (K - 1) * RT + K
    return dict(Y=K * R + G + K + 2, dw=B + c_lam + c_u + 2, dxT=F * RT + c_lam + 2)


def ev_envelope(rowptr, col, diag, w, xT, dY, dtype):
    """Componentwise bounds on Y, dw, dxT of a kernel computing in `dtype` (inputs already rounded to it):
    c u M + tiny, M = ev_forward / ev_backward on |w|, |x|, |dY|, c = ev_depths.  Returns dict name -> bound array."""
    aw, ax, ady = (np.abs(np.asarray(a, dtype=np.float64)) for a in (w, xT, dY))
    F, K, G, _ = aw.shape
    B = ax.shape[2]
    MY, _ = ev_forward(rowptr, col, diag, aw, ax)
    Mdw, Mdx, _ = ev_backward(rowptr, col, diag, aw, ax, ady)
    c = ev_depths(rowptr, col, K, G, F, B)
    u = unit_roundoff(dtype)
    tiny = 4.0 * np.finfo(np.dtype(dtype)).tiny * (sum(c.values()) + 1)
    return dict(Y=c["Y"] * u * MY + tiny, dw=c["dw"] * u * Mdw + tiny, dxT=c["dxT"] * u * Mdx + tiny)
