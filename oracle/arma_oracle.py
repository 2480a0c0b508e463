"""fp64 restatement of the ARMA graph filter by Jacobi iterations (jARMA, alegnn/utils/graphML.py:490-638) and of its
gradients, with scipy CSR, and componentwise error envelopes for it.  TEST INFRASTRUCTURE — NOT PRODUCT CODE (same rules
as lsigf_oracle.py).

Operands are the reference's: psi, varphi [F, E, P, G], phi [F, E, K, G], S_list = E scipy matrices [N, N],
x [B, G, N], b None / [F, 1] / [F, N], dU [B, F, N].  With S~_e = S_e - diag(S_e), d_e = diag(S_e) and, per column
(f, e, p, g), r = 1 / (d_e - psi[f,e,p,g]) (a vector over the nodes), the chains are in the COLUMN convention S~ v:

    z_0 = r . x_g,  z_t = r . (S~ z_{t-1})  (t <= tMax);     y_0 = x_g,  y_t = r . (S~ y_{t-1})  (t <= tMax + 1)
    u[b,f] = sum_{e,p,g} ( varphi sum_t (-1)^t z_t + (-1)^(tMax+1) y_{tMax+1} ) + LSIGF(phi, S, x) + b

Every column runs its own chain here (vectorised over the columns, but with its own r); the kernels' constant-diagonal
reformulation is checked against this form, not used by it.  Gradients by adjoints:
    lambda_tMax = (-1)^tMax varphi dU,   lambda_t = (-1)^t varphi dU + S~^T (r . lambda_{t+1})
    mu_{tMax+1} = (-1)^(tMax+1) dU,      mu_t = S~^T (r . mu_{t+1})
    dx_g = sum_{e,f,p} r . lambda_0 + sum_e S~^T sum_{f,p} (r . mu_1)   (+ the LSIGF part)
    dpsi = sum_{n,b} ( sum_t lambda_t r z_t + sum_{t>=1} mu_t r y_t ),   dvarphi = sum_{n,b} dU sum_t (-1)^t z_t
"""
import numpy as np
import scipy.sparse as sp

from lsigf_oracle import lsigf_grads_sparse, lsigf_sparse, unit_roundoff


def split_gso(S_list):
    """-> (St_list, d_list): the off-diagonal parts S~_e (CSR) and the diagonals d_e (dense, implicit zeros included)."""
    St, d = [], []
    for S in S_list:
        S = sp.csr_matrix(S, dtype=np.float64)
        de = S.diagonal().copy()
        off = sp.csr_matrix(S - sp.diags(de))
        off.eliminate_zeros()
        St.append(off)
        d.append(de)
    return St, d


def _chains(psi, varphi, St_list, d_list, x, tMax, dtype, absolute):
    """Per edge feature: r [N, F, P, G], zs[t] = z_t and ys[t] = y_{t+1} as [N, B, F, P, G] (t = 0..tMax), computed in
    `dtype`.  absolute: r, S~ and x replaced by their absolute values (for the envelopes)."""
    F, E, P, G = psi.shape
    B, _, N = x.shape
    X = np.ascontiguousarray(np.transpose(np.asarray(x, dtype=dtype), (2, 0, 1)))           # [N, B, G]
    Xb = np.broadcast_to(X[:, :, None, None, :], (N, B, F, P, G)).astype(dtype)
    out = []
    for e in range(E):
        St = St_list[e].astype(dtype)
        r = (np.asarray(1.0, dtype) / (np.asarray(d_list[e], dtype)[:, None, None, None] - psi[None, :, e].astype(dtype)))
        if absolute:
            St, r, Xb = abs(St), np.abs(r), np.abs(Xb)
        rb = r[:, None]

        def hop(v):
            return (St @ v.reshape(N, -1)).reshape(v.shape).astype(dtype)
        zs = [rb * Xb]
        for _ in range(tMax):
            zs.append(rb * hop(zs[-1]))
        ys, y = [], Xb
        for _ in range(tMax + 1):
            y = rb * hop(y)
            ys.append(y)
        out.append((St, r, zs, ys))
    return out


def arma_chain_terms(psi, varphi, St_list, d_list, x, tMax, dtype=np.float64, absolute=False, h2_sign=None,
                     h2_varphi=False):
    """sum_{e,p,g} (varphi sum_t (-1)^t z_t + h2 y_{tMax+1}) as [B, F, N], for given operators St_list (next = St @ v)
    and diagonals d_list.  h2 defaults to (-1)^(tMax+1); h2_varphi multiplies the H2 term by varphi (both only for
    emulating wrong kernels).  absolute: every sign dropped and every operand taken by absolute value."""
    psi = np.asarray(psi, dtype=np.float64)
    varphi = np.asarray(varphi, dtype=np.float64)
    F, E, P, G = psi.shape
    B, _, N = np.shape(x)
    h2 = (-1.0) ** (tMax + 1) if h2_sign is None else h2_sign
    u = np.zeros((N, B, F), dtype=dtype)
    for e, (St, r, zs, ys) in enumerate(_chains(psi, varphi, St_list, d_list, x, tMax, dtype, absolute)):
        vp = varphi[:, e].astype(dtype)
        if absolute:
            vp = np.abs(vp)
        zsum = np.zeros_like(zs[0])
        for t, z in enumerate(zs):
            zsum = zsum + (z if absolute or t % 2 == 0 else -z)
        u = u + np.einsum("nbfpg,fpg->nbf", zsum, vp).astype(dtype)
        last = ys[-1] * vp[None, None] if h2_varphi else ys[-1]
        u = u + (np.abs(h2) if absolute else h2) * last.sum(axis=(3, 4)).astype(dtype)
    return np.transpose(u, (1, 2, 0))


def arma_forward(psi, varphi, phi, S_list, x, b=None, tMax=5, dtype=np.float64):
    """u [B, F, N] = jARMA(psi, varphi, phi, S, x, b, tMax), computed in `dtype` (fp64 for the oracle)."""
    St, d = split_gso(S_list)
    u = arma_chain_terms(psi, varphi, St, d, x, tMax, dtype)
    u = u + lsigf_sparse(np.asarray(phi, dtype), [sp.csr_matrix(S).astype(dtype) for S in S_list], np.asarray(x, dtype))
    if b is not None:
        u = u + np.asarray(b, dtype)
    return u


def _adjoints(psi, varphi, St_list, d_list, x, dU, tMax, absolute=False):
    """(dx [B, G, N], dpsi, dvarphi [F, E, P, G]) of the chain terms, fp64.  absolute: the same on absolute values."""
    psi = np.asarray(psi, dtype=np.float64)
    varphi = np.asarray(varphi, dtype=np.float64)
    F, E, P, G = psi.shape
    B, _, N = np.shape(x)
    DU = np.ascontiguousarray(np.transpose(np.asarray(dU, dtype=np.float64), (2, 0, 1)))[..., None, None]   # [N,B,F,1,1]
    if absolute:
        DU = np.abs(DU)
    sg = (lambda t: 1.0) if absolute else (lambda t: (-1.0) ** t)
    h2 = 1.0 if absolute else (-1.0) ** (tMax + 1)
    dxn = np.zeros((N, B, G))
    dpsi, dvarphi = np.zeros((F, E, P, G)), np.zeros((F, E, P, G))
    for e, (St, r, zs, ys) in enumerate(_chains(psi, varphi, St_list, d_list, x, tMax, np.float64, absolute)):
        StT = St.T.tocsr()
        vp = np.abs(varphi[:, e]) if absolute else varphi[:, e]
        rb = r[:, None]

        def hopT(v):
            return (StT @ v.reshape(N, -1)).reshape(v.shape)
        lam = sg(tMax) * vp[None, None] * DU
        mu = np.broadcast_to(h2 * DU, lam.shape)
        gp = lam * rb * zs[tMax] + mu * rb * ys[tMax]
        gv = sg(tMax) * DU * zs[tMax]
        for t in range(tMax - 1, -1, -1):
            lam = sg(t) * vp[None, None] * DU + hopT(rb * lam)
            mu = hopT(rb * mu)
            gp = gp + lam * rb * zs[t] + mu * rb * ys[t]
            gv = gv + sg(t) * DU * zs[t]
        dxn += (rb * lam).sum(axis=(2, 3)) + (StT @ (rb * mu).sum(axis=(2, 3)).reshape(N, -1)).reshape(N, B, G)
        dpsi[:, e] = gp.sum(axis=(0, 1))
        dvarphi[:, e] = gv.sum(axis=(0, 1))
    return np.transpose(dxn, (1, 2, 0)), dpsi, dvarphi


def arma_backward(psi, varphi, phi, S_list, x, dU, tMax=5, bias_shape=None):
    """Gradients of u = arma_forward(...) for upstream dU: dict dx, dpsi, dvarphi, dphi (and db when bias_shape)."""
    St, d = split_gso(S_list)
    dx, dpsi, dvarphi = _adjoints(psi, varphi, St, d, x, dU, tMax)
    dphi, dx3, db = lsigf_grads_sparse(np.asarray(phi, np.float64), S_list, np.asarray(x, np.float64),
                                       np.asarray(dU, np.float64), bias_shape)
    out = dict(dx=dx + dx3, dpsi=dpsi, dvarphi=dvarphi, dphi=dphi)
    if bias_shape is not None:
        out["db"] = db
    return out


def constant_taps(psi, varphi, c, tMax):
    """h' [F, E, tMax + 2, G] of the constant-diagonal reformulation (diagonal c_e in edge feature e): with
    rho = 1 / (c_e - psi), h'[:, :, k] = sum_p varphi (-1)^k rho^(k+1) (k <= tMax), h'[:, :, tMax+1] =
    (-1)^(tMax+1) sum_p rho^(tMax+1); the chain terms are then LSIGF(h', [S~_e^T], x)."""
    rho = 1.0 / (np.asarray(c, np.float64).reshape(1, -1, 1, 1) - np.asarray(psi, np.float64))
    taps = [((-1.0) ** k * np.asarray(varphi, np.float64) * rho ** (k + 1)).sum(axis=2) for k in range(tMax + 1)]
    taps.append((-1.0) ** (tMax + 1) * (rho ** (tMax + 1)).sum(axis=2))
    return np.stack(taps, axis=2)


def arma_depths(psi, S_list, tMax, K, B, N, G, F):
    """Accumulation depths c (|error| <= c u M to first order, M the computation on absolute values).
    R: the longest row or column of any S~_e; R3: of any S_e (the LSIGF residue).  kappa bounds the relative error of
    r = 1 / (d - psi) in units of u: (|d| + |psi|) / |d - psi| + 1.  A chain step is a hop (R), a scaling by r
    (kappa + 1) and the fma into it; the output adds E P G (tMax + 2) chain terms, the residue's (K - 1) R3 + T G and the
    bias; gradients add the adjoint chain, the fold over F P, the narrow hop, and N B rows in the column sums."""
    St, d = split_gso(S_list)
    psi = np.asarray(psi, np.float64)
    F_, E, P, G_ = psi.shape
    R = max(max(np.diff(m.indptr).max(initial=0), np.diff(m.tocsc().indptr).max(initial=0)) for m in St)
    R3 = max(max(np.diff(sp.csr_matrix(S).indptr).max(initial=0), np.diff(sp.csc_matrix(S).indptr).max(initial=0))
             for S in S_list)
    kappa = max(float(((np.abs(d[e])[:, None] + np.abs(psi[:, e].reshape(1, -1)))
                       / np.abs(d[e][:, None] - psi[:, e].reshape(1, -1))).max(initial=1.0)) for e in range(E))
    step = int(R) + kappa + 3
    chain = (tMax + 1) * step
    T = 1 + E * (K - 1)
    lsigf_y = (K - 1) * int(R3) + T * G + 2
    lsigf_dx = (K - 1) * int(R3) + T * F + 2
    return dict(y=chain + E * P * G * (tMax + 2) + lsigf_y + 4,
                dx=2 * chain + (tMax + 1) * 3 + F * P + int(R) + E + lsigf_dx + 4,
                dpsi=2 * chain + (tMax + 1) * 5 + N * B + 4,
                dvarphi=chain + (tMax + 1) * 2 + N * B + 4,
                dphi=(K - 1) * int(R3) + N * B + 2,
                db=N * B + 2)


def arma_envelope(psi, varphi, phi, S_list, x, b, dU, tMax, dtype):
    """Componentwise bounds on u, dx, dpsi, dvarphi, dphi (, db) of a kernel computing in `dtype` (inputs already rounded
    to it): c u M + tiny, M = the forward / backward on absolute values, c = arma_depths.  Returns dict name -> array."""
    psi = np.asarray(psi, np.float64)
    phi = np.asarray(phi, np.float64)
    F, E, P, G = psi.shape
    K = phi.shape[2]
    B, _, N = np.shape(x)
    St, d = split_gso(S_list)
    S_abs = [abs(sp.csr_matrix(S)).astype(np.float64) for S in S_list]
    xa, dUa = np.abs(np.asarray(x, np.float64)), np.abs(np.asarray(dU, np.float64))
    My = arma_chain_terms(psi, varphi, St, d, x, tMax, np.float64, absolute=True) + lsigf_sparse(np.abs(phi), S_abs, xa)
    if b is not None:
        My = My + np.abs(np.asarray(b, np.float64))
    dx_a, dpsi_a, dvar_a = _adjoints(psi, varphi, St, d, x, dU, tMax, absolute=True)
    dphi_a, dx3_a, db_a = lsigf_grads_sparse(np.abs(phi), S_abs, xa, dUa, None if b is None else np.shape(b))
    c = arma_depths(psi, S_list, tMax, K, B, N, G, F)
    u = unit_roundoff(dtype)
    tiny = 4.0 * np.finfo(np.dtype(dtype)).tiny * (c["y"] + c["dx"] + c["dpsi"] + 2)
    out = dict(y=c["y"] * u * My + tiny, dx=c["dx"] * u * (dx_a + dx3_a) + tiny, dpsi=c["dpsi"] * u * dpsi_a + tiny,
               dvarphi=c["dvarphi"] * u * dvar_a + tiny, dphi=c["dphi"] * u * dphi_a + tiny)
    if b is not None:
        out["db"] = ((N * B if np.shape(b)[1] == 1 else B) + 2) * u * db_a + tiny
    return out
