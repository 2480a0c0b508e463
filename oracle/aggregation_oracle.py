"""float64 restatement of the aggregation GNNs' graph product (AggregationGNN, alegnn/modules/architectures.py:2920-3228)
with the componentwise error bounds the CUDA path is held to.

TEST INFRASTRUCTURE.  R[(p*E + e)*maxN + q, m] = (S_e^q)[m, sel[p]] from scipy sparse powers in float64; it is the
reference's SN [nNodes, E, N, maxN] (on the GSO reordered so that sel comes first) without its zeros.  The Conv1d operand
is z[b*P + p, e*F + f, q] = sum_m x[b, f, m] R[(p, e, q), m], and the input gradient dx = R^T dz.

Bounds.  The CUDA path forms R by maxN - 1 sparse products in float64, casts it to the layer's dtype and sums each row
in a fixed tree of at most n entries, so per element
    |z - z_ref| <= (gamma_{n+2}(dtype) + gamma_{(maxN-1) d}(fp64)) (|R| |x|)(element),
with n the longest row of R (of R^T for dx), d the longest row of S and |R| the same powers of |S|.  An element no
selected node reaches has the bound 0: it must come out exactly 0 (the bound is held at the smallest normal double so
that the ratio error / bound stays defined).
"""
import numpy as np
import scipy.sparse as sp
import torch

import lsigf_oracle as orc


def gso_mats(S):
    """A dense [N, N] / [E, N, N] array or a list of sparse matrices as a list of float64 CSR matrices."""
    if isinstance(S, (list, tuple)):
        return [sp.csr_matrix(m, dtype=np.float64) for m in S]
    S = np.asarray(S, dtype=np.float64)
    return [sp.csr_matrix(m) for m in (S[None] if S.ndim == 2 else S)]


def operator(S, sel, maxN):
    """(R, |R| envelope, relative error of R's float64 powers) as CSR [P*E*maxN, N]."""
    mats = gso_mats(S)
    E, N, P = len(mats), mats[0].shape[0], len(sel)
    blocks, ablocks = [], []
    for A in mats:
        D = sp.csr_matrix((np.ones(P), (np.asarray(sel), np.arange(P))), shape=(N, P))
        Dabs = D.copy()
        per_q, abs_q = [], []
        for q in range(maxN):
            per_q.append(D.T.tocsr())
            abs_q.append(Dabs.T.tocsr())
            D, Dabs = (A @ D).tocsr(), (abs(A) @ Dabs).tocsr()
        blocks.append(per_q)
        ablocks.append(abs_q)
    # row (p*E + e)*maxN + q is row p of blocks[e][q], stacked at (e*maxN + q)*P + p
    perm = np.arange(P * E * maxN).reshape(E, maxN, P).transpose(2, 0, 1).reshape(-1)
    stack = lambda b: sp.vstack([m for per_q in b for m in per_q]).tocsr()[perm]   # noqa: E731
    d = max(int(np.diff(A.indptr).max()) if A.nnz else 0 for A in mats)
    R, Rabs = stack(blocks), stack(ablocks)
    R.sort_indices()
    Rabs.sort_indices()
    return R, Rabs, orc.gamma(max(1, (maxN - 1) * d), np.float64)


def to_conv(zn, P, E, maxN, B, F):
    """node-major rows (p, e, q) x columns (b, f) -> the Conv1d operand [(B*P), E*F, maxN]."""
    return zn.reshape(P, E, maxN, B, F).transpose(3, 0, 1, 4, 2).reshape(B * P, E * F, maxN)


def from_conv(z, P, E, maxN, B, F):
    return z.reshape(B, P, E, F, maxN).transpose(1, 2, 4, 0, 3).reshape(P * E * maxN, B * F)


def _longest(M):
    return int(np.diff(M.indptr).max()) if M.shape[0] else 0


def forward(R, Rabs, r_err, x, E, maxN, dtype):
    """(z, bound) for x [B, F, N] (float64 values of the layer's input)."""
    B, F, N = x.shape
    P = R.shape[0] // (E * maxN)
    xn = x.reshape(B * F, N).T
    zn, zabs = R @ xn, Rabs @ np.abs(xn)
    bound = np.maximum((orc.gamma(_longest(R) + 2, dtype) + r_err) * zabs, np.finfo(np.float64).tiny)
    return to_conv(zn, P, E, maxN, B, F), to_conv(bound, P, E, maxN, B, F)


def backward(R, Rabs, r_err, dz, E, maxN, N, dtype):
    """(dx [B, F, N], bound) for dz [(B*P), E*F, maxN]."""
    P = R.shape[0] // (E * maxN)
    B, F = dz.shape[0] // P, dz.shape[1] // E
    dzn = from_conv(dz, P, E, maxN, B, F)
    RT, RTabs = R.T.tocsr(), Rabs.T.tocsr()
    dxn, dxabs = RT @ dzn, RTabs @ np.abs(dzn)
    bound = np.maximum((orc.gamma(_longest(RT) + 2, dtype) + r_err) * dxabs, np.finfo(np.float64).tiny)
    return dxn.T.reshape(B, F, N), bound.T.reshape(B, F, N)


def aggregate_torch(R, E, maxN, x):
    """The product as differentiable torch ops on x's device and dtype (small operators: R densified), for running the
    layers' host code without the CUDA path."""
    B, F, N = x.shape
    P = R.shape[0] // (E * maxN)
    Rt = torch.tensor(R.toarray(), dtype=x.dtype, device=x.device)
    zn = Rt @ x.reshape(B * F, N).T
    return zn.reshape(P, E, maxN, B, F).permute(3, 0, 1, 4, 2).reshape(B * P, E * F, maxN)

