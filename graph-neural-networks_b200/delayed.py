"""Batch- and time-varying graph filter on the CUDA LSIGF path (SURVEY.md §8f rank 4).

    LSIGF_DB(h, S, x, b=None)                   <- alegnn/utils/graphML.py:977-1094
    GraphFilter_DB(G, F, K, E=1, bias=True)     <- graphML.py:3278-3393
    GRNN_DB(a, b, S, x, z0, sigma, xBias, zBias) <- graphML.py:1096-1290   (recursion over the same GSO batch, below)
    HiddenState_DB(F, H, K, sigma, E, bias)     <- graphML.py:3395-3538

    y_f(b, t) = sum_e sum_k sum_g h[f,e,k,g]  x_g(b, t-k) S_e(b, t-k+1) ... S_e(b, t)  +  bias_f
    (row-vector convention, signals before t = 0 are zero: graphML.py:1060-1075)

The reference runs B*T small dense N x N products per tap (N = 50 agents in the flocking examples).  Here the whole
batch is ONE sparse graph filter: stack the B*T copies of the node set into M = B*T*N "space-time" nodes and put
S_e(b, t) on the block that links copy (b, t-1) to copy (b, t):

        S_big_e[(b, t-1, i), (b, t, j)] = S_e(b, t)[i, j]          (zero elsewhere; nothing enters t = 0)

Then (x S_big^k)[(b,t,:)] = x(b, t-k) S(b, t-k+1) ... S(b, t) is exactly the delayed shift, the unit delay and the
zero history included, and LSIGF_DB(h, S, x, b) = LSIGF(h, S_big, x_big, b_big) with a single "sample" of M nodes.
One plan per GSO batch, K-1 launches of the same CSR hop kernel over all B*T graphs at once, one contraction — the
same CUDA path (and C ABI) as the static filter, instead of (K-1) batched GEMM launches plus permute copies.
"""
import math
import weakref

import torch
import torch.nn as nn

from . import _cabi
from . import graphML as _gml
from .gso import Plan

_CACHE = {}
_CACHE_MAX = 4


def block_delay_csr(S):
    """S [B, T, E, N, N] (pattern = S != 0) -> ([(rowptr int64 [M+1], col int32 [nnz], val [nnz]) for e], M = B*T*N):
    CSR (row i lists S_big_e[i, j], columns ascending) of the space-time operator described in the module docstring."""
    assert S.dim() == 5 and S.shape[3] == S.shape[4]
    B, T, E, N, _ = S.shape
    M = B * T * N
    assert M < 2 ** 31, "b200gf: B*T*N must fit the int32 column index"
    out = []
    for e in range(E):
        rowptr = torch.zeros(M + 1, dtype=torch.int64, device=S.device)
        if T > 1:
            Se = S[:, 1:, e]                                       # S(b, t) for t = 1 .. T-1  [B, T-1, N, N]
            nz = (Se != 0).nonzero(as_tuple=False)                 # (b, t-1, i, j), row-major = sorted by (row, col)
            bb, tt, ii, jj = nz.unbind(1)
            rows = (bb * T + tt) * N + ii                          # source copy (b, t-1)
            cols = (bb * T + tt + 1) * N + jj                      # destination copy (b, t)
            vals = Se[bb, tt, ii, jj].contiguous()
            rowptr[1:] = torch.cumsum(torch.bincount(rows, minlength=M), 0)
        else:
            cols = torch.zeros(0, dtype=torch.int64, device=S.device)
            vals = torch.zeros(0, dtype=S.dtype, device=S.device)
        out.append((rowptr, cols.to(torch.int32).contiguous(), vals))
    return out, M


def transpose_csr_device(csr, M):
    """CSR (rowptr, col, val) of an M x M operator -> CSR of its transpose, on the same device: one stable sort by column
    (entries of an output row keep ascending source-row order, like the host builder's counting sort)."""
    rowptr, col, val = csr
    rows = torch.repeat_interleave(torch.arange(M, device=rowptr.device), rowptr[1:] - rowptr[:-1])
    order = torch.sort(col.to(torch.int64), stable=True)[1]
    t_rowptr = torch.zeros(M + 1, dtype=torch.int64, device=rowptr.device)
    t_rowptr[1:] = torch.cumsum(torch.bincount(col.to(torch.int64), minlength=M), 0)
    return t_rowptr, rows[order].to(torch.int32).contiguous(), val[order].contiguous()


def _plan_for_batch(S):
    """Plan of the space-time operator, cached per (storage, version): GraphFilter_DB.addGSO is called once per batch
    (architecturesTime.py) and every layer of the network shares that GSO tensor."""
    if S.requires_grad:
        raise NotImplementedError("b200gf: gradients w.r.t. the GSO are not part of the LSIGF path")
    if S.device.type != "cuda":
        raise RuntimeError("b200gf: LSIGF_DB needs CUDA tensors (there is no CPU fallback); got GSO on %s" % S.device)
    key = (S.data_ptr(), S._version, tuple(S.shape), tuple(S.stride()), S.dtype, str(S.device))
    for k in [k for k, h in _CACHE.items() if h[0]() is None]:     # GSO batch already collected: free its plan now
        del _CACHE[k]
    hit = _CACHE.get(key)
    if hit is not None and hit[0]() is S:
        return hit[1]
    csr, M = block_delay_csr(S)
    # both operators are built on the device (one sort for the transpose) and adopted device to device: no host round trip
    plan = Plan.from_device_ops([transpose_csr_device(c, M) for c in csr], csr, M, S.dtype, S.device)
    if len(_CACHE) >= _CACHE_MAX:
        _CACHE.pop(next(iter(_CACHE)))
    _CACHE[key] = (weakref.ref(S), plan)
    return plan


def _filter_on_space_time_graph(h, S, x_big, b_big):
    """LSIGF over the M-node operator of `S`; x_big [1, G, M] (node-major view), b_big None / [F, 1] / [F, M]."""
    _gml.check_operands("LSIGF_DB", x_big, (h, b_big), S)
    if S.device != x_big.device:
        raise RuntimeError("b200gf: GSO on %s but x on %s" % (S.device, x_big.device))
    return _gml._LSIGFFunction.apply(h, x_big, b_big, _plan_for_batch(S))


# tests swap this for the CPU oracle applied to block_delay_csr(S) to check the host logic without a GPU
_apply = _filter_on_space_time_graph


def LSIGF_DB(h, S, x, b=None):
    """LSIGF_DB(filter_taps, GSO, input, bias=None)   (graphML.py:977-1094)

    h [F, E, K, G]; S [B, T, E, N, N]; x [B, T, G, N]; b [F, 1] or [F, N] or None  ->  y [B, T, F, N]."""
    assert len(h.shape) == 4
    F = h.shape[0]
    E = h.shape[1]
    G = h.shape[3]
    assert len(S.shape) == 5
    B = S.shape[0]
    T = S.shape[1]
    assert S.shape[2] == E
    N = S.shape[3]
    assert S.shape[4] == N
    assert len(x.shape) == 4
    assert x.shape[0] == B
    assert x.shape[1] == T
    assert x.shape[2] == G
    assert x.shape[3] == N
    M = B * T * N
    # space-time node-major input [M, G] (node index (b, t, n)), handed to the filter as a [1, G, M] view of it
    x_big = x.permute(0, 1, 3, 2).reshape(M, G).t().unsqueeze(0)
    b_big = b
    if b is not None:
        assert b.dim() == 2 and b.shape[0] == F and b.shape[1] in (1, N)
        if b.shape[1] == N and M != N:
            b_big = b.repeat(1, B * T)                              # per-node bias, the same for every (b, t)
    y_big = _apply(h, S, x_big, b_big)                              # [1, F, M]
    return y_big[0].reshape(F, B, T, N).permute(1, 2, 0, 3)         # [B, T, F, N], still a view of the node-major buffer


class GraphFilter_DB(nn.Module):
    """GraphFilter_DB(in_features, out_features, filter_taps, edge_features=1, bias=True)

    Same surface as graphML.py:3278-3393: parameters `weight` [F, E, K, G], `bias` [F, 1] or None;
    addGSO(S [B, T, E, N, N]); forward(x [B, T, G, N]) -> [B, T, F, N]."""

    def __init__(self, G, F, K, E=1, bias=True):
        super().__init__()
        self.G = G
        self.F = F
        self.K = K
        self.E = E
        self.S = None
        self.weight = nn.parameter.Parameter(torch.Tensor(F, E, K, G))
        if bias:
            self.bias = nn.parameter.Parameter(torch.Tensor(F, 1))
        else:
            self.register_parameter("bias", None)
        self.reset_parameters()

    def reset_parameters(self):
        stdv = 1. / math.sqrt(self.G * self.K)      # graphML.py:3353-3358
        self.weight.data.uniform_(-stdv, stdv)
        if self.bias is not None:
            self.bias.data.uniform_(-stdv, stdv)

    def addGSO(self, S):
        assert len(S.shape) == 5                    # graphML.py:3362
        assert S.shape[2] == self.E
        self.N = S.shape[3]
        assert S.shape[4] == self.N
        self.S = S

    def forward(self, x):
        assert len(x.shape) == 4
        B = x.shape[0]
        assert self.S.shape[0] == B
        T = x.shape[1]
        assert self.S.shape[1] == T
        assert x.shape[3] == self.N
        return LSIGF_DB(self.weight, self.S, x, self.bias)

    def extra_repr(self):
        reprString = "in_features=%d, out_features=%d, " % (self.G, self.F) + "filter_taps=%d, " % (self.K) + \
                     "edge_features=%d, " % (self.E) + "bias=%s, " % (self.bias is not None)
        if self.S is not None:
            reprString += "GSO stored"
        else:
            reprString += "no GSO stored"
        return reprString


# ---------------------------------------------------------------------------------------------------
# GRNN_DB: z_t = sigma(A(S) x_t + B(S) z_{t-1}) on a batch- and time-varying GSO (graphML.py:1096-1290)
# ---------------------------------------------------------------------------------------------------
def slab_csr(S):
    """S [B, T, E, N, N] -> (fwd, bwd, R = B*N): for every operator index o = (t-1)*E + e, t = 1 .. T-1, the block-diagonal
    (over the batch) shift of time step t on R = B*N rows ordered (b, n):   A_o[(b, i), (b, j)] = S[b, t, e, i, j].
    bwd[o] = CSR of A_o (row (b, i) lists j ascending), fwd[o] = CSR of its transpose (the gather form of the row-vector
    shift z <- z S_t): lists of (rowptr int64 [R+1], col int32, val) tensors on S's device.  One nonzero(), one stable
    sort; the per-operator arrays are slices of the batch-wide ones."""
    assert S.dim() == 5 and S.shape[3] == S.shape[4]
    B, T, E, N, _ = S.shape
    R = B * N
    n_ops = max(T - 1, 0) * E
    assert R < 2 ** 31, "b200gf: B*N must fit the int32 column index"
    if n_ops == 0:
        return [], [], R
    Sp = S[:, 1:].permute(1, 2, 0, 3, 4)                       # [T-1, E, B, N, N]: nonzero() comes out sorted by (o, row, col)
    nz = (Sp != 0).nonzero(as_tuple=False)
    tt, ee, bb, ii, jj = nz.unbind(1)
    vals = Sp[tt, ee, bb, ii, jj].contiguous()
    op = tt * E + ee
    rows = bb * N + ii
    cols = bb * N + jj

    def split(ops_sorted, major, minor, v):
        """entries sorted by (operator, major): per-operator CSR with `major` as the row and `minor` as the column."""
        cum = torch.zeros(n_ops * R + 1, dtype=torch.int64, device=S.device)
        cum[1:] = torch.cumsum(torch.bincount(ops_sorted * R + major, minlength=n_ops * R), 0)
        starts = cum[::R].tolist()                              # n_ops + 1 segment boundaries (one host read)
        out = []
        for o in range(n_ops):
            lo, hi = starts[o], starts[o + 1]
            out.append((cum[o * R:(o + 1) * R + 1] - lo, minor[lo:hi].to(torch.int32).contiguous(), v[lo:hi].contiguous()))
        return out

    bwd = split(op, rows, cols, vals)
    order = torch.sort(op * R + cols, stable=True)[1]          # by (operator, col), rows stay ascending inside a column
    fwd = split(op[order], cols[order], rows[order], vals[order])
    return fwd, bwd, R


class _HopFunction(torch.autograd.Function):
    """dst = A_o src for one operator of a plan (b200gf_hop, HOP_FWD); the gradient is the other operator (HOP_BWD)."""

    @staticmethod
    def forward(ctx, src, plan, o):
        if src.device.type != "cuda":
            raise RuntimeError("b200gf: GRNN_DB needs CUDA tensors (there is no CPU fallback); got the state on %s" % src.device)
        lib = _cabi.load()
        src = src.contiguous()
        dst = torch.empty_like(src)
        _cabi.check(lib.b200gf_hop(plan.handle, o, _cabi.HOP_FWD, src.data_ptr(), src.stride(0), dst.data_ptr(), dst.stride(0),
                                   src.shape[1], _cabi.stream()))
        ctx.plan, ctx.o = plan, o
        return dst

    @staticmethod
    def backward(ctx, g):
        lib = _cabi.load()
        g = g.contiguous()
        out = torch.empty_like(g)
        _cabi.check(lib.b200gf_hop(ctx.plan.handle, ctx.o, _cabi.HOP_BWD, g.data_ptr(), g.stride(0), out.data_ptr(), out.stride(0),
                                   g.shape[1], _cabi.stream()))
        return out, None, None


class _SlabOps:
    """The (T-1)*E per-time-step operators of one GSO batch as ONE device plan (b200gf_plan_create_device with
    (T-1)*E operators on B*N rows); hop(o, src) runs the library's CSR hop kernel with operator o."""

    def __init__(self, S):
        if S.requires_grad:
            raise NotImplementedError("b200gf: gradients w.r.t. the GSO are not part of the LSIGF path")
        if S.device.type != "cuda":
            raise RuntimeError("b200gf: GRNN_DB needs CUDA tensors (there is no CPU fallback); got GSO on %s" % S.device)
        if S.dtype not in (torch.float32, torch.float64):
            raise RuntimeError("b200gf: GRNN_DB supports float32 and float64, got %s" % S.dtype)
        fwd, bwd, R = slab_csr(S)
        self.plan = Plan.from_device_ops(fwd, bwd, R, S.dtype, S.device) if fwd else None

    def hop(self, o, src):
        return _HopFunction.apply(src, self.plan, o)


_SLAB_CACHE = {}


def _slab_ops_cuda(S):
    """_SlabOps of a GSO batch, cached per (storage, version) like the space-time plan of LSIGF_DB."""
    key = (S.data_ptr(), S._version, tuple(S.shape), tuple(S.stride()), S.dtype, str(S.device))
    for k in [k for k, h in _SLAB_CACHE.items() if h[0]() is None]:
        del _SLAB_CACHE[k]
    hit = _SLAB_CACHE.get(key)
    if hit is not None and hit[0]() is S:
        return hit[1]
    ops = _SlabOps(S)
    if len(_SLAB_CACHE) >= _CACHE_MAX:
        _SLAB_CACHE.pop(next(iter(_SLAB_CACHE)))
    _SLAB_CACHE[key] = (weakref.ref(S), ops)
    return ops


# tests swap this for a torch.sparse implementation over slab_csr(S) to check the recursion without a GPU
_slab_ops = _slab_ops_cuda


def GRNN_DB(a, b, S, x, z0, sigma, xBias=None, zBias=None):
    """GRNN_DB(signal_to_hidden_taps, hidden_to_hidden_taps, GSO, input, initial_hidden, nonlinearity,
               signal_bias, hidden_bias)                                             (graphML.py:1096-1290)

    a [H, E, K, F]; b [H, E, K, H]; S [B, T, E, N, N]; x [B, T, F, N]; z0 [B, H, N]; biases: H elements or None.
    Returns the hidden-state trajectory z [B, T, H, N],
        z_t = sigma( sum_{e,k} a_{e,k} x_{t-k} S_{t-k+1..t}  +  sum_{e,k} b_{e,k} z_{t-1-k} S_{t-k+1..t} ),   z_{-1} = z0.

    A(S)x for all time steps is one LSIGF_DB call (graphML.py:1164).  The hidden-to-hidden term keeps, per edge feature,
    the delay line D_k(t) = z_{t-1-k} S_{t-k+1} ... S_t  (k = 1 .. K-1) node-major as [B*N, (K-1)*H]: one CSR hop per
    time step and edge feature advances all K-1 delays at once (D_k(t) = D_{k-1}(t-1) S_t, the reference's
    `torch.matmul(Sz, St)` at :1224 / :1257 on dense N x N blocks), and the taps are applied row-locally."""
    H = a.shape[0]
    E = a.shape[1]
    K = a.shape[2]
    F = a.shape[3]
    assert b.shape[0] == H
    assert b.shape[1] == E
    assert b.shape[2] == K
    assert b.shape[3] == H
    B = S.shape[0]
    T = S.shape[1]
    assert S.shape[2] == E
    N = S.shape[3]
    assert S.shape[4] == N
    assert x.shape[0] == B
    assert x.shape[1] == T
    assert x.shape[2] == F
    assert x.shape[3] == N
    assert z0.shape[0] == B
    assert z0.shape[1] == H
    assert z0.shape[2] == N
    if xBias is not None:
        xBias = xBias.reshape(H, 1)
    Ax = LSIGF_DB(a, S, x, xBias)                                    # [B, T, H, N], a view of the node-major result
    Ax_t = Ax.permute(1, 0, 3, 2).unbind(0)                           # T x [B, N, H]
    ops = _slab_ops(S) if (K > 1 and T > 1) else None
    R = B * N
    W0 = b[:, :, 0, :].sum(1).t()                                     # [H', H]: the k = 0 tap sees z_{t-1} for every e
    We = [b[:, e, 1:, :].permute(1, 2, 0).reshape((K - 1) * H, H) for e in range(E)] if K > 1 else []
    zb = None if zBias is None else zBias.reshape(1, 1, H)
    zprev2 = None
    zprev = z0.permute(0, 2, 1).reshape(R, H)                         # z_{-1}, rows (b, n)
    D = [None] * E                                                    # delay lines [R, (K-1)*H]; None = still all zero
    states = []
    for t in range(T):
        Bz = zprev @ W0
        if t >= 1 and K > 1:
            for e in range(E):
                if D[e] is None:
                    src = torch.cat((zprev2, zprev2.new_zeros(R, (K - 2) * H)), dim=1) if K > 2 else zprev2
                else:
                    src = torch.cat((zprev2, D[e][:, :(K - 2) * H]), dim=1) if K > 2 else zprev2
                D[e] = ops.hop((t - 1) * E + e, src)                  # [D_1(t) .. D_{K-1}(t)]
                Bz = Bz + D[e] @ We[e]
        pre = Ax_t[t] + Bz.view(B, N, H)
        if zb is not None:
            pre = pre + zb
        zt = sigma(pre.permute(0, 2, 1))                              # the nonlinearity sees the reference's [B, H, N]
        states.append(zt)
        zprev2 = zprev
        zprev = zt.permute(0, 2, 1).reshape(R, H)
    return torch.stack(states, dim=1)                                 # [B, T, H, N]


class HiddenState_DB(nn.Module):
    """HiddenState_DB(signal_features, hidden_features, filter_taps, nonlinearity=torch.tanh, edge_features=1, bias=True)

    Same surface as graphML.py:3395-3538: parameters aWeights [H,E,K,F], bWeights [H,E,K,H], xBias / zBias [H,1];
    addGSO(S [B,T,E,N,N]); forward(x [B,T,F,N], z0 [B,H,N]) -> (z [B,T,H,N], z_T [B,1,1,H,N])."""

    def __init__(self, F, H, K, nonlinearity=torch.tanh, E=1, bias=True):
        super().__init__()
        self.F = F
        self.H = H
        self.K = K
        self.E = E
        self.S = None
        self.bias = bias
        self.sigma = nonlinearity
        self.aWeights = nn.parameter.Parameter(torch.Tensor(H, E, K, F))
        self.bWeights = nn.parameter.Parameter(torch.Tensor(H, E, K, H))
        if self.bias:
            self.xBias = nn.parameter.Parameter(torch.Tensor(H, 1))
            self.zBias = nn.parameter.Parameter(torch.Tensor(H, 1))
        else:
            self.register_parameter("xBias", None)
            self.register_parameter("zBias", None)
        self.reset_parameters()

    def reset_parameters(self):
        stdv = 1. / math.sqrt(self.F * self.K)      # graphML.py:3475-3482
        self.aWeights.data.uniform_(-stdv, stdv)
        self.bWeights.data.uniform_(-stdv, stdv)
        if self.bias:
            self.xBias.data.uniform_(-stdv, stdv)
            self.zBias.data.uniform_(-stdv, stdv)

    def addGSO(self, S):
        assert len(S.shape) == 5                    # graphML.py:3517
        assert S.shape[2] == self.E
        self.N = S.shape[3]
        assert S.shape[4] == self.N
        self.S = S

    def forward(self, x, z0):
        assert self.S is not None
        assert len(x.shape) == 4
        B = x.shape[0]
        assert self.S.shape[0] == B
        T = x.shape[1]
        assert self.S.shape[1] == T
        assert x.shape[2] == self.F
        N = x.shape[3]
        assert len(z0.shape) == 3
        assert z0.shape[0] == B
        assert z0.shape[1] == self.H
        assert z0.shape[2] == N
        z = GRNN_DB(self.aWeights, self.bWeights, self.S, x, z0, self.sigma, xBias=self.xBias, zBias=self.zBias)
        return z, z[:, T - 1:T].unsqueeze(1)

    def extra_repr(self):
        reprString = "in_features=%d, hidden_features=%d, " % (self.F, self.H) + "filter_taps=%d, " % (self.K) + \
                     "edge_features=%d, " % (self.E) + "bias=%s, " % (self.bias) + "nonlinearity=%s" % (self.sigma)
        if self.S is not None:
            reprString += "GSO stored"
        else:
            reprString += "no GSO stored"
        return reprString
