"""fp64 restatement of the node-variant filter's C ABI (b200gf_nv_forward / b200gf_nv_backward, include/b200gf.h) with
scipy CSR, componentwise error envelopes for it, and NodeVariantGF's copyNodes search.  TEST INFRASTRUCTURE — NOT
PRODUCT CODE (same rules as lsigf_oracle.py).

Operands are the reference's: h [F, E, K, G, M] (tap m of node n is copy[n]), S_list = E scipy matrices [N, N],
x [B, G, N], b None / [F, 1] / [F, N], dy [B, F, N].  Row-vector shift (x S)[., j] = sum_i x[., i] S[i, j], so the
node-major shifted signal is Z_{e,k} = (S_e^T)^k X with X [N, B*G].
"""
import numpy as np
import scipy.sparse as sp

from lsigf_oracle import unit_roundoff

zeroTolerance = 1e-9


def _shifts(S_list, x, K):
    """Z [E, K, N, B, G]: Z[e, k] = x S_e^k, node-major."""
    B, G, N = x.shape
    X = np.ascontiguousarray(np.transpose(x, (2, 0, 1)).reshape(N, B * G))
    E = len(S_list)
    Z = np.zeros((E, K, N, B * G))
    for e, S in enumerate(S_list):
        St = sp.csr_matrix(S).T.tocsr()
        z = X
        for k in range(K):
            Z[e, k] = z
            z = St @ z
    return Z.reshape(E, K, N, B, G)


def nv_forward(h, copy, S_list, x, b=None):
    """y [B, F, N] = sum_{e,k,g} h[f, e, k, g, copy[n]] (x_g S_e^k)[n] + b."""
    h = np.asarray(h, dtype=np.float64)
    x = np.asarray(x, dtype=np.float64)
    K = h.shape[2]
    Ht = h[..., np.asarray(copy, dtype=np.int64)]                          # [F, E, K, G, N]
    Z = _shifts(S_list, x, K)
    y = np.einsum("fekgn,eknbg->bfn", Ht, Z)
    if b is not None:
        y = y + np.asarray(b, dtype=np.float64)
    return y


def nv_backward(h, copy, S_list, x, dy, bias_shape=None):
    """-> (dx [B, G, N], dh [F, E, K, G, M], db or None) of y = nv_forward(...) for upstream dy [B, F, N].
        dz_{e,k}[n, b, g] = sum_f h[f, e, k, g, copy[n]] dy[b, f, n],   dx = sum_{e,k} S_e^k dz_{e,k} (node-major)
        dh[f, e, k, g, m] = sum_{n: copy[n] = m} sum_b (x_g S_e^k)[b, n] dy[b, f, n]."""
    h = np.asarray(h, dtype=np.float64)
    x = np.asarray(x, dtype=np.float64)
    dy = np.asarray(dy, dtype=np.float64)
    F, E, K, G, M = h.shape
    B, _, N = x.shape
    copy = np.asarray(copy, dtype=np.int64)
    Ht = h[..., copy]
    Z = _shifts(S_list, x, K)
    dz = np.einsum("fekgn,bfn->eknbg", Ht, dy)
    dxn = np.zeros((N, B * G))
    for e, S in enumerate(S_list):
        S = sp.csr_matrix(S)
        acc = np.zeros((N, B * G))
        for k in range(K - 1, -1, -1):                                     # Horner: S (dz_{k} + S (dz_{k+1} + ...))
            acc = dz[e, k].reshape(N, B * G) + (S @ acc if k < K - 1 else 0.0)
        dxn += acc
    dx = np.transpose(dxn.reshape(N, B, G), (1, 2, 0))
    dHt = np.einsum("eknbg,bfn->fekgn", Z, dy)
    dh = np.zeros((F, E, K, G, M))
    np.add.at(np.moveaxis(dh, 4, 0), copy, np.moveaxis(dHt, 4, 0))
    db = None
    if bias_shape is not None:
        db = dy.sum(axis=(0, 2))[:, None] if bias_shape[1] == 1 else dy.sum(axis=0)
    return dx, dh, db


def nv_depths(S_list, K, E, G, F, B, counts):
    """Accumulation depths c (|error| <= c u M to first order, M the run on absolute values).  R: longest row or column of
    any S_e.  y: K-1 chained hops, then T G products.  dx: a Horner chain of K-1 hops and adds per e, the F products of
    each dz, the E chains summed.  dh: K-1 hops to make Z, then cnt_m B products for tap m (counts [M])."""
    R = max(max(np.diff(sp.csr_matrix(S).indptr).max(initial=0), np.diff(sp.csc_matrix(S).indptr).max(initial=0))
            for S in S_list)
    hop = (K - 1) * int(R)
    T = 1 + E * (K - 1)
    return dict(y=hop + T * G + 2, dx=hop + (K - 1) + F + E + 2, dh=hop + np.asarray(counts) * B + 2)


def nv_envelope(h, copy, S_list, x, b, dy, dtype):
    """Componentwise bounds on y, dx, dh (, db) of a kernel computing in `dtype` (inputs already rounded to it):
    c u M + tiny, M = nv_forward / nv_backward on |h|, |S|, |x|, |b|, |dy|, c = nv_depths.  Returns dict name -> array."""
    h = np.asarray(h, dtype=np.float64)
    F, E, K, G, M = h.shape
    B, _, N = np.shape(x)
    copy = np.asarray(copy, dtype=np.int64)
    S_abs = [abs(sp.csr_matrix(S)).astype(np.float64) for S in S_list]
    babs = None if b is None else np.abs(np.asarray(b, dtype=np.float64))
    My = nv_forward(np.abs(h), copy, S_abs, np.abs(x), babs)
    Mdx, Mdh, Mdb = nv_backward(np.abs(h), copy, S_abs, np.abs(x), np.abs(np.asarray(dy, dtype=np.float64)),
                                None if b is None else np.shape(b))
    counts = np.bincount(copy, minlength=M)
    c = nv_depths(S_list, K, E, G, F, B, counts)
    u = unit_roundoff(dtype)
    tiny = 4.0 * np.finfo(np.dtype(dtype)).tiny * (c["y"] + c["dx"] + N * B + 2)
    out = dict(y=c["y"] * u * My + tiny, dx=c["dx"] * u * Mdx + tiny, dh=c["dh"] * u * Mdh + tiny)
    if Mdb is not None:
        out["db"] = ((N * B if np.shape(b)[1] == 1 else B) + 2) * u * Mdb + tiny
    return out


def copy_nodes_search(S_list, M):
    """copyNodes by a breadth-first search FROM every node n >= M along its out-edges (S[i, j] != 0: i -> j) until the
    first level that holds nodes below M; the smallest of them.  Nodes below M map to themselves, M >= N gives
    arange(N).  Returns None for a node that reaches no independent node."""
    N = sp.csr_matrix(S_list[0]).shape[0]
    if M >= N:
        return np.arange(N)
    A = None
    for S in S_list:
        a = abs(sp.csr_matrix(S)).astype(np.float64)
        A = a if A is None else A + a
    A = (A > zeroTolerance).tocsr()
    out = list(range(M))
    for n in range(M, N):
        seen = {n}
        level = [n]
        hit = None
        while level and hit is None:
            nxt = set()
            for i in level:
                for j in A.indices[A.indptr[i]:A.indptr[i + 1]]:
                    if j not in seen:
                        seen.add(int(j))
                        nxt.add(int(j))
            found = [j for j in nxt if j < M]
            hit = min(found) if found else None
            level = list(nxt)
        out.append(hit)
    return np.array(out, dtype=object if any(v is None for v in out) else np.int64)
