"""ARMA graph filters by Jacobi iterations on sparse CUDA kernels (csrc/arma/arma.cu).

    jARMA(psi, varphi, phi, S, x, b=None, tMax=5)        <- alegnn/utils/graphML.py:490-638
    GraphFilterARMA(G, F, P, K, E=1, bias=True, tMax=5)   <- graphML.py:2714-2847  (same attributes, parameter names
                                                             and shapes, same initialisation order)

With S~_e = S_e - diag(S_e), d_e = diag(S_e) and, for every column (f, e, p, g), r = 1 / (d_e - psi[f,e,p,g]) (a vector
over the nodes), the reference computes, in the column convention S~ v,

    z_0 = r . x_g,  z_t = r . (S~ z_{t-1});   y_0 = x_g,  y_t = r . (S~ y_{t-1})
    u[b,f] = sum_{e,p,g} ( varphi sum_{t=0}^{tMax} (-1)^t z_t + (-1)^(tMax+1) y_{tMax+1} ) + LSIGF(phi, S, x) + b

by building Sbar^-1 S~ as [F, E, P, G, N, N] dense tensors (205 GB each at F = G = 16, P = 2, N = 10 000).  Here:

  * constant diagonal (every d_e[i] equal, bitwise, implicit zeros included; every zero-diagonal adjacency and every
    normalised Laplacian of a graph without isolated nodes): r is a scalar rho = 1 / (c_e - psi), all columns share the
    chain S~^k x, and edge feature e is an LSIGF over the operator S~_e^T with tMax + 2 taps
        h'[f,e,k,g] = sum_p varphi (-1)^k rho^(k+1)  (k <= tMax),   h'[f,e,tMax+1,g] = (-1)^(tMax+1) sum_p rho^(tMax+1)
    built in torch (autograd differentiates it), so a hop reads B G columns instead of B F P G;
  * any other diagonal (a combinatorial Laplacian, weighted self-loops): the per-column chains of all (f, p, g) run side
    by side, both chains in one wide node-major state per edge feature, advanced by the plan's hop kernel and scaled /
    accumulated by arma.cu's element-wise kernels (b200gf_arma_forward / _backward).

The choice is made per edge feature from the GSO (`ArmaOperator`), and both paths sum into one output.  The residue term
and the bias are the LSIGF forward and backward on the plan of S.  CPU tensors raise; there is no dense fallback.
"""
import math
import weakref

import numpy as np
import scipy.sparse as sp
import torch
import torch.nn as nn

from . import _cabi
from .graphML import (LSIGF, _as_bcn_view, _bias_2d, _grad_in_input_layout, _lsigf_backward_nm, _lsigf_forward_nm,
                      _workspace, check_operands, node_major_ld, plan_on, to_node_major)
from .gso import Plan, SparseGSO, _dense_key, dense_to_csr, plan_for


# ---------------------------------------------------------------------------------------------------------------
# the operator: S~^T plans, diagonals, constant-diagonal flags
# ---------------------------------------------------------------------------------------------------------------
class ArmaOperator:
    """What the ARMA paths need of a GSO, built once: per edge feature e the CSR of S~_e^T (so a plan's FWD hop computes
    S~_e v and its BWD hop S~_e^T v), the diagonal d_e, and whether d_e is constant (bitwise equal across all N entries).
    `plan(es, device)` / `diag(es, device)` return the plan and the [len(es), N] diagonals of the edge features `es`
    (cached per subset and device).  S: dense tensor [E, N, N] (any device) or SparseGSO."""

    def __init__(self, S):
        if isinstance(S, Plan):
            raise TypeError("b200gf: jARMA needs the GSO's diagonal: pass a dense tensor or a SparseGSO, not a device Plan")
        if isinstance(S, torch.Tensor) and S.layout != torch.strided:
            S = SparseGSO.from_torch_sparse(S)
        self.E, self.N = int(S.shape[0]), int(S.shape[1])
        self.dtype = S.dtype
        self._csr, diags = [], []
        if isinstance(S, SparseGSO):
            for (r, c, v) in S.csr:
                m = sp.csr_matrix((v, c, r), shape=(self.N, self.N))
                d = m.diagonal().copy()
                off = sp.csr_matrix(m - sp.diags(d, format="csr"))
                off.eliminate_zeros()
                t = off.T.tocsr()
                t.sort_indices()
                self._csr.append((t.indptr.astype(np.int64), t.indices.astype(np.int32), t.data))
                diags.append(torch.from_numpy(d))
        else:
            St = S.detach()
            for e in range(self.E):
                d = torch.diagonal(St[e]).clone()
                self._csr.append(dense_to_csr((St[e] - torch.diag(d)).t().contiguous()))
                diags.append(d)
        self._d = torch.stack(diags) if diags else torch.zeros((0, self.N), dtype=self.dtype)
        bits = self._d.view(torch.int32 if self._d.element_size() == 4 else torch.int64)
        self.constant = [bool(self.N == 0 or (bits[e] == bits[e, 0]).all()) for e in range(self.E)]
        self.const_value = [float(self._d[e, 0]) if self.N else 0.0 for e in range(self.E)]
        self._plans, self._diags = {}, {}

    @staticmethod
    def _key(es, device):
        device = torch.device(device)
        return tuple(es), (device.type, device.index if device.index is not None else torch.cuda.current_device())

    def plan(self, es, device):
        key = self._key(es, device)
        p = self._plans.get(key)
        if p is None:
            p = self._plans[key] = Plan.from_host_csr([self._csr[e] for e in es], self.N, self.dtype, device)
        return p

    def diag(self, es, device):
        key = self._key(es, device)
        d = self._diags.get(key)
        if d is None:
            d = self._diags[key] = self._d[list(es)].to(device=device).contiguous()
        return d

    def index(self, es, device):
        """int64 tensor of `es` on the device (cached: a per-call host copy would break CUDA-graph capture)."""
        key = ("index",) + self._key(es, device)
        t = self._diags.get(key)
        if t is None:
            t = self._diags[key] = torch.tensor(list(es), dtype=torch.int64, device=device)
        return t

    def constants(self, es, dtype, device):
        """[1, len(es), 1, 1] tensor of the constant diagonal values c_e of `es` (cached, as `index`)."""
        key = ("const", dtype) + self._key(es, device)
        t = self._diags.get(key)
        if t is None:
            t = self._diags[key] = torch.tensor([self.const_value[e] for e in es], dtype=dtype,
                                                device=device).reshape(1, -1, 1, 1)
        return t


_OP_CACHE = {}
_OP_CACHE_MAX = 16


def arma_operator(S):
    """The ArmaOperator of a GSO, cached per (tensor, version, device) for dense tensors (as plan_for caches plans, so
    the reference's GraphFilterARMA, whose addGSO keeps a dense S, is served after install) and per object otherwise."""
    for k in [k for k, hit in _OP_CACHE.items() if hit[0]() is None]:
        del _OP_CACHE[k]
    if isinstance(S, torch.Tensor) and S.layout == torch.strided:
        if S.requires_grad:
            raise NotImplementedError("b200gf: gradients w.r.t. the GSO are not part of the jARMA path "
                                      "(the reference keeps S as a plain attribute, graphML.py:2812)")
        key = ("dense",) + _dense_key(S)
    else:
        key = ("obj", id(S), getattr(S, "_version", 0))
    hit = _OP_CACHE.get(key)
    if hit is None or hit[0]() is not S:
        if len(_OP_CACHE) >= _OP_CACHE_MAX:
            _OP_CACHE.pop(next(iter(_OP_CACHE)))
        hit = _OP_CACHE[key] = (weakref.ref(S), ArmaOperator(S))
    return hit[1]


# ---------------------------------------------------------------------------------------------------------------
# general path: autograd over the C ABI
# ---------------------------------------------------------------------------------------------------------------
class _ARMAFunction(torch.autograd.Function):
    """u = LSIGF(phi, S, x) + b + the ARMA chains of the edge features of `aplan` (psi, varphi: [F, E', P, G] for those
    edge features, d: their diagonals [E', N]).  The H3 term and the bias are written by the LSIGF forward, the chains
    are added in place by b200gf_arma_forward; the backward mirrors it."""

    @staticmethod
    def forward(ctx, psi, varphi, phi, x, b, hplan, aplan, d, tMax, keep):
        lib = _cabi.load()
        F_, _, P, G = psi.shape
        K = phi.shape[2]
        B, _, N = x.shape
        psic, varc, phic = psi.contiguous(), varphi.contiguous(), phi.contiguous()
        ctx.x_node_major = node_major_ld(x) is not None
        xn, x_ld = to_node_major(x)
        ybuf, ldf, bias_per_node = _lsigf_forward_nm(hplan, phic, xn, x_ld, b, B, G, F_, K, _cabi.ACT_NONE)
        states = None
        if keep:
            st_bytes = lib.b200gf_arma_workspace_bytes(aplan.handle, B, G, F_, P, tMax, 3)
            states = _workspace(max(st_bytes, 1), x.device)
        aws_bytes = lib.b200gf_arma_workspace_bytes(aplan.handle, B, G, F_, P, tMax, 1 if keep else 0)
        aws = _workspace(aws_bytes, x.device)
        _cabi.check(lib.b200gf_arma_forward(aplan.handle, d.data_ptr(), psic.data_ptr(), varc.data_ptr(), tMax, B, G,
                                            F_, P, xn.data_ptr(), x_ld, ybuf.data_ptr(), ldf,
                                            None if states is None else states.data_ptr(), aws.data_ptr(), aws_bytes,
                                            _cabi.stream()))
        ctx.hplan, ctx.aplan, ctx.x_ld, ctx.tMax = hplan, aplan, x_ld, tMax
        ctx.bias_per_node = bias_per_node
        ctx.bias_shape = None if b is None else tuple(b.shape)
        ctx.dims = (B, G, F_, K, P, N)
        if keep:
            ctx.save_for_backward(psic, varc, phic, xn, d, states)
        return _as_bcn_view(ybuf, B, F_, N)

    @staticmethod
    def backward(ctx, du):
        lib = _cabi.load()
        psic, varc, phic, xn, d, states = ctx.saved_tensors
        B, G, F_, K, P, N = ctx.dims
        dun, du_ld = to_node_major(du)
        need_dx, need_db = ctx.needs_input_grad[3], ctx.needs_input_grad[4]
        dxbuf, ldc, dphi, db = _lsigf_backward_nm(ctx.hplan, dun, du_ld, xn, ctx.x_ld, phic, need_dx, need_db,
                                                  ctx.bias_shape, ctx.bias_per_node, B, G, F_, K)
        dpsi, dvarphi = torch.empty_like(psic), torch.empty_like(varc)
        aws_bytes = lib.b200gf_arma_workspace_bytes(ctx.aplan.handle, B, G, F_, P, ctx.tMax, 2)
        aws = _workspace(aws_bytes, du.device)
        _cabi.check(lib.b200gf_arma_backward(ctx.aplan.handle, d.data_ptr(), psic.data_ptr(), varc.data_ptr(), ctx.tMax,
                                             B, G, F_, P, dun.data_ptr(), du_ld, states.data_ptr(),
                                             None if dxbuf is None else dxbuf.data_ptr(), ldc, dpsi.data_ptr(),
                                             dvarphi.data_ptr(), aws.data_ptr(), aws_bytes, _cabi.stream()))
        dx = _grad_in_input_layout(dxbuf, ldc, B, G, N, ctx.x_node_major) if need_dx else None
        return dpsi, dvarphi, dphi, dx, db, None, None, None, None, None


# ---------------------------------------------------------------------------------------------------------------
# constant-diagonal path: taps of an LSIGF over S~^T
# ---------------------------------------------------------------------------------------------------------------
def constant_taps(psi, varphi, c, tMax):
    """h' [F, E, tMax + 2, G] of the constant-diagonal form for diagonals c ([1, E, 1, 1] tensor): rho = 1 / (c_e - psi),
    h'[:, :, k] = sum_p varphi (-1)^k rho^(k+1) for k <= tMax and h'[:, :, tMax+1] = (-1)^(tMax+1) sum_p rho^(tMax+1)."""
    rho = 1.0 / (c - psi)
    taps, pw = [], rho
    for k in range(tMax + 1):
        taps.append((varphi * pw).sum(dim=2) * (-1.0) ** k)
        if k < tMax:
            pw = pw * rho
    taps.append(pw.sum(dim=2) * (-1.0) ** (tMax + 1))
    return torch.stack(taps, dim=2)


# ---------------------------------------------------------------------------------------------------------------
# dispatch
# ---------------------------------------------------------------------------------------------------------------
def _dispatch_cuda(psi, varphi, phi, S, x, b, tMax, path=None):
    """Device part of jARMA: loud checks (there is no CPU path), the operator lookup, and per edge feature the
    constant-diagonal or the general path, summed into one output.  path = None chooses from the GSO; "general" runs
    every edge feature on the general path and "constant" every one on the constant path (each must be constant).
    `_dispatch` is the hook the CPU tests replace with the oracle to exercise the host logic around it."""
    check_operands("jARMA", x, (psi, varphi, phi, b), S)
    op = arma_operator(S)
    E = op.E
    if path is None:
        ce = [e for e in range(E) if op.constant[e]]
    elif path == "general":
        ce = []
    elif path == "constant":
        if not all(op.constant):
            raise ValueError("b200gf: the constant-diagonal path needs a constant diagonal in every edge feature")
        ce = list(range(E))
    else:
        raise ValueError("b200gf: path must be None, 'general' or 'constant', got %r" % (path,))
    ge = [e for e in range(E) if e not in ce]
    hplan = plan_on(S, x.device)
    if ge:
        idx = op.index(ge, x.device)
        keep = torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (psi, varphi, phi, x, b))
        u = _ARMAFunction.apply(psi.index_select(1, idx), varphi.index_select(1, idx), phi, x, b, hplan,
                                op.plan(ge, x.device), op.diag(ge, x.device), int(tMax), keep)
    else:
        u = LSIGF(phi, hplan, x, b)
    if ce:
        idx = op.index(ce, x.device)
        h = constant_taps(psi.index_select(1, idx), varphi.index_select(1, idx), op.constants(ce, x.dtype, x.device),
                          tMax)
        u = u + LSIGF(h, op.plan(ce, x.device), x)
    return u


_dispatch = _dispatch_cuda


def jARMA(psi, varphi, phi, S, x, b=None, tMax=5):
    """jARMA(inverse_taps, direct_taps, filter_taps, GSO, input, bias=None, tMax=5): ARMA graph filter by tMax Jacobi
    iterations.

    Same contract as the reference (alegnn/utils/graphML.py:490-638):
        psi, varphi [F, E, P, G]; phi [F, E, K, G]; S [E, N, N] (dense tensor or SparseGSO); x [B, G, N];
        b None, or any bias form LSIGF accepts ([F, 1], [F, N], [1, F, 1], [1, F, N]); returns u [B, F, N]
    """
    F_ = psi.shape[0]
    E = psi.shape[1]
    P = psi.shape[2]
    G = psi.shape[3]
    assert varphi.shape[0] == F_                 # graphML.py:549-552
    assert varphi.shape[1] == E
    assert varphi.shape[2] == P
    assert varphi.shape[3] == G
    assert phi.shape[0] == F_                    # graphML.py:553-555
    assert phi.shape[1] == E
    assert phi.shape[3] == G
    assert x.shape[1] == G                       # graphML.py:557
    N = x.shape[2]
    assert S.shape[0] == E                       # graphML.py:559-560
    assert S.shape[1] == S.shape[2] == N
    tMax = int(tMax)
    if tMax < 0:
        raise ValueError("b200gf: jARMA needs tMax >= 0, got %d" % tMax)
    return _dispatch(psi, varphi, phi, S, x, _bias_2d(b, F_, N, "jARMA"), tMax)


class GraphFilterARMA(nn.Module):
    """GraphFilterARMA(in_features, out_features, denominator_taps, residue_taps, edge_features=1, bias=True, tMax=5)

    Same surface as the reference layer (alegnn/utils/graphML.py:2714-2847): attributes G, F, P, K, E, tMax, S, N;
    parameters `inverseWeight`, `directWeight` [F, E, P, G], `filterWeight` [F, E, K, G] and `bias` [F, 1] (or None),
    initialised in the same order from the same ranges; `addGSO(S)`, `forward(x)`, `extra_repr()`.  `addGSO` also
    accepts a SparseGSO and builds the ARMA operator and the residue plan once."""

    def __init__(self, G, F, P, K, E=1, bias=True, tMax=5):
        super().__init__()
        self.G = G
        self.F = F
        self.P = P
        self.K = K
        self.E = E
        self.tMax = tMax
        self.S = None
        self.inverseWeight = nn.parameter.Parameter(torch.Tensor(F, E, P, G))
        self.directWeight = nn.parameter.Parameter(torch.Tensor(F, E, P, G))
        self.filterWeight = nn.parameter.Parameter(torch.Tensor(F, E, K, G))
        if bias:
            self.bias = nn.parameter.Parameter(torch.Tensor(F, 1))
        else:
            self.register_parameter("bias", None)
        self.reset_parameters()

    def reset_parameters(self):
        stdv = 1. / math.sqrt(self.G * self.P)      # graphML.py:2798-2803
        self.inverseWeight.data.uniform_(1. + 1. / stdv, 1. + 2. / stdv)
        self.directWeight.data.uniform_(-stdv, stdv)
        self.filterWeight.data.uniform_(-stdv, stdv)
        if self.bias is not None:
            self.bias.data.uniform_(-stdv, stdv)

    def addGSO(self, S):
        assert len(S.shape) == 3                    # graphML.py:2807
        assert S.shape[0] == self.E                 # graphML.py:2809
        self.N = S.shape[1]
        assert S.shape[2] == self.N                 # graphML.py:2811
        self.S = S
        if torch.cuda.is_available() and (isinstance(S, SparseGSO) or
                                          (isinstance(S, torch.Tensor) and S.device.type == "cuda")):
            arma_operator(S)
            plan_for(S)

    def forward(self, x):
        B = x.shape[0]
        F = x.shape[1]
        Nin = x.shape[2]
        if Nin < self.N:                            # zero-pad the node axis, graphML.py:2820-2824
            x = torch.cat((x, torch.zeros(B, F, self.N - Nin, dtype=x.dtype, device=x.device)), dim=2)
        u = jARMA(self.inverseWeight, self.directWeight, self.filterWeight, self.S, x, b=self.bias, tMax=self.tMax)
        if Nin < self.N:                            # keep the first Nin nodes, graphML.py:2832-2833
            u = u[:, :, :Nin]
        return u

    def extra_repr(self):
        reprString = "in_features=%d, " % self.G
        reprString += "out_features=%d, " % self.F
        reprString += "denominator_taps=%d, " % self.P
        reprString += "residue_taps=%d, " % self.K
        reprString += "edge_features=%d, " % self.E
        reprString += "bias=%s, " % (self.bias is not None)
        if self.S is not None:
            reprString += "GSO stored"
        else:
            reprString += "no GSO stored"
        return reprString
