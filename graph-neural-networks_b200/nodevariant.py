"""Node-variant graph filters on sparse CUDA kernels (csrc/nv/nv.cu).

    NVGF(h, S, x, b=None)                       <- alegnn/utils/graphML.py:293-387
    NodeVariantGF(G, F, K, M, E=1, bias=True)   <- graphML.py:2317-2509   (same attributes, parameter names and shapes)

    y_f = sum_e sum_k sum_g diag(h_k^{efg}) S_e^k x_g + b_f

Every node has its own taps, or (NodeVariantGF with M < N) copies the taps of a nearby "independent" node.  The reference
shifts with dense matmuls against an N x N S and materialises z * h as B*F*E*K*G*N elements; here the E(K-1) shifts are
the LSIGF path's sparse hops and the per-node tap contraction reads each node's tap block through a node -> tap map
(`TapMap`), so the [F,E,K,G,N] index_select of the reference is never built.

`NodeVariantGF.addGSO` finds the tap of every node without a dense matrix: a level-synchronous breadth-first search from
the M independent nodes over the reversed edges of the pattern sum_e |S_e| > 1e-9, carrying the smallest source index
(`copy_nodes`).  Where the reference's search never ends (a node that cannot reach any of the first M nodes), this raises
ValueError naming those nodes.

Host code is PyTorch; the arithmetic runs in libb200gf.so through the C ABI of include/b200gf.h.  CPU tensors raise.
"""
import math

import numpy as np
import scipy.sparse as sp
import torch
import torch.nn as nn

from . import _cabi
from .graphML import (_as_bcn_view, _bias_arg, _grad_in_input_layout, _workspace, check_operands, node_major_ld,
                      padded_ld, plan_on, to_node_major)
from .gso import Plan, SparseGSO, plan_for

zeroTolerance = 1e-9   # graphTools.py:45


# ---------------------------------------------------------------------------------------------------------------
# node -> tap map
# ---------------------------------------------------------------------------------------------------------------
class TapMap:
    """Which tap block every node reads: node_tap [N] (int32, the layer's copyNodes), and its inverse, the nodes of every
    tap in ascending order as CSR: tap_rowptr [M+1] (int64), tap_nodes [N] (int32).  Built once on the host;
    `on(device)` returns (node_tap, tap_rowptr, tap_nodes) on a device (cached)."""

    def __init__(self, copy_nodes, M):
        copy = np.asarray(copy_nodes, dtype=np.int64).reshape(-1)
        self.N, self.M = int(copy.size), int(M)
        if self.N and (copy.min() < 0 or copy.max() >= self.M):
            raise ValueError("b200gf: node taps must lie in [0, %d)" % self.M)
        rowptr = np.zeros(self.M + 1, dtype=np.int64)
        rowptr[1:] = np.cumsum(np.bincount(copy, minlength=self.M))
        self.node_tap = torch.from_numpy(copy.astype(np.int32))
        self.tap_rowptr = torch.from_numpy(rowptr)
        self.tap_nodes = torch.from_numpy(np.argsort(copy, kind="stable").astype(np.int32))
        self._devices = {}

    def on(self, device):
        device = torch.device(device)
        if device.type == "cuda" and device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        hit = self._devices.get(str(device))
        if hit is None:
            hit = tuple(t.to(device) for t in (self.node_tap, self.tap_rowptr, self.tap_nodes))
            self._devices[str(device)] = hit
        return hit


_IDENTITY = {}


def _identity_taps(N):
    """NVGF's map: node n reads tap n (M = N)."""
    hit = _IDENTITY.get(N)
    if hit is None:
        if len(_IDENTITY) >= 16:
            _IDENTITY.pop(next(iter(_IDENTITY)))
        hit = _IDENTITY[N] = TapMap(np.arange(N), N)
    return hit


# ---------------------------------------------------------------------------------------------------------------
# copyNodes without a dense matrix
# ---------------------------------------------------------------------------------------------------------------
def gso_pattern(S):
    """scipy CSR (bool) of sum_e |S_e| > 1e-9, row i listing its neighbours j (graphTools.py:424-434).  S: dense tensor
    or array [E, N, N] (any device), torch sparse tensor, or SparseGSO."""
    if isinstance(S, Plan):
        raise TypeError("b200gf: NodeVariantGF.addGSO needs the GSO's pattern: pass a dense tensor or a SparseGSO, "
                        "not a device Plan")
    if isinstance(S, torch.Tensor) and S.layout != torch.strided:
        S = SparseGSO.from_torch_sparse(S)
    if isinstance(S, SparseGSO):
        N = S.N
        acc = sp.csr_matrix((N, N), dtype=np.float64)
        for (r, c, v) in S.csr:
            acc = acc + sp.csr_matrix((np.abs(v).astype(np.float64), c, r), shape=(N, N))
        A = (acc > zeroTolerance).tocsr()
    else:
        St = torch.as_tensor(S).detach()
        N = St.shape[1]
        nz = (St.abs().sum(0) > zeroTolerance).nonzero(as_tuple=False).cpu().numpy()
        A = sp.csr_matrix((np.ones(len(nz), dtype=bool), (nz[:, 0], nz[:, 1])), shape=(N, N))
    A.sort_indices()
    return A


def copy_nodes(S, M):
    """copyNodes of NodeVariantGF.addGSO (graphML.py:2413-2468) as an int64 array [N].

    Nodes below M keep their own tap; M >= N gives arange(N).  Every other node n copies the smallest independent node
    (index < M) among those at the smallest hop distance from n along the edges i -> j of S[i, j] != 0, which is what the
    reference's repeated computeNeighborhood(S, K, nb=M) followed by min(...) yields.  Raises ValueError for nodes that
    cannot reach any independent node (the reference's loop never ends there)."""
    N = int(S.shape[1])
    if M >= N:
        return np.arange(N, dtype=np.int64)
    AT = gso_pattern(S).T.tocsr()                    # row j: the nodes i with an edge i -> j
    indptr, indices = AT.indptr.astype(np.int64), AT.indices.astype(np.int64)
    label = np.full(N, -1, dtype=np.int64)
    label[:M] = np.arange(M)
    frontier = np.arange(M, dtype=np.int64)
    while frontier.size:
        starts = indptr[frontier]
        cnt = indptr[frontier + 1] - starts
        tot = int(cnt.sum())
        if tot == 0:
            break
        offs = np.repeat(starts - np.cumsum(cnt) + cnt, cnt) + np.arange(tot)
        cand = indices[offs]
        src = np.repeat(label[frontier], cnt)
        keep = label[cand] < 0
        cand, src = cand[keep], src[keep]
        if cand.size == 0:
            break
        order = np.lexsort((src, cand))              # by node, then by source label: the first of a node is its minimum
        cand, src = cand[order], src[order]
        first = np.ones(cand.size, dtype=bool)
        first[1:] = cand[1:] != cand[:-1]
        frontier = cand[first]
        label[frontier] = src[first]
    missing = np.nonzero(label < 0)[0]
    if missing.size:
        shown = ", ".join(str(int(n)) for n in missing[:20]) + (", ..." if missing.size > 20 else "")
        raise ValueError("b200gf: NodeVariantGF.addGSO: %d node(s) cannot reach any of the first M = %d nodes along the "
                         "GSO's edges, so no node tap can be copied to them (the reference's search never ends here): "
                         "%s" % (missing.size, M, shown))
    return label


# ---------------------------------------------------------------------------------------------------------------
# autograd over the C ABI
# ---------------------------------------------------------------------------------------------------------------
class _NVGFFunction(torch.autograd.Function):
    """y = NVGF(h[..., node_tap], S, x, b) with S inside `plan` and the node -> tap map `taps`."""

    @staticmethod
    def forward(ctx, h, x, b, plan, taps):
        lib = _cabi.load()
        F_, E, K, G, M = h.shape
        B, _, N = x.shape
        dt = x.dtype
        hc = h.contiguous()
        ctx.x_node_major = node_major_ld(x) is not None
        xn, x_ld = to_node_major(x)
        node_tap, tap_rowptr, tap_nodes = taps.on(x.device)
        T = 1 + E * (K - 1)
        W = torch.empty((M, T, G, F_), dtype=dt, device=x.device)
        _cabi.check(lib.b200gf_nv_pack_taps(_cabi.DTYPE[dt], hc.data_ptr(), W.data_ptr(), F_, E, K, G, M, _cabi.stream()))
        bc, bias_per_node = _bias_arg(b)
        ldf = padded_ld(B * F_, dt)
        ybuf = torch.empty((N, ldf), dtype=dt, device=x.device)
        ws_bytes = lib.b200gf_nv_workspace_bytes(plan.handle, B, G, F_, K, M, 0)
        ws = _workspace(ws_bytes, x.device)
        _cabi.check(lib.b200gf_nv_forward(plan.handle, xn.data_ptr(), x_ld, W.data_ptr(), node_tap.data_ptr(), M,
                                          None if bc is None else bc.data_ptr(), bias_per_node, ybuf.data_ptr(), ldf,
                                          ws.data_ptr(), ws_bytes, B, G, F_, K, _cabi.stream()))
        ctx.plan, ctx.taps, ctx.x_ld = plan, taps, x_ld
        ctx.bias_per_node = bias_per_node
        ctx.bias_shape = None if b is None else tuple(b.shape)
        ctx.dims = (B, G, F_, K, E, N, M)
        ctx.save_for_backward(W, xn)
        return _as_bcn_view(ybuf, B, F_, N)

    @staticmethod
    def backward(ctx, dy):
        lib = _cabi.load()
        W, xn = ctx.saved_tensors
        B, G, F_, K, E, N, M = ctx.dims
        dt = W.dtype
        dyn, dy_ld = to_node_major(dy)
        node_tap, tap_rowptr, tap_nodes = ctx.taps.on(dy.device)
        need_dh, need_dx, need_db = ctx.needs_input_grad[0], ctx.needs_input_grad[1], ctx.needs_input_grad[2]
        dh = torch.empty((F_, E, K, G, M), dtype=dt, device=dy.device)
        ldc = padded_ld(B * G, dt)
        dxbuf = torch.empty((N, ldc), dtype=dt, device=dy.device) if need_dx else None
        db = torch.empty(ctx.bias_shape, dtype=dt, device=dy.device) if (ctx.bias_shape and need_db) else None
        ws_bytes = lib.b200gf_nv_workspace_bytes(ctx.plan.handle, B, G, F_, K, M, 1)
        ws = _workspace(ws_bytes, dy.device)
        _cabi.check(lib.b200gf_nv_backward(ctx.plan.handle, dyn.data_ptr(), dy_ld, xn.data_ptr(), ctx.x_ld, W.data_ptr(),
                                           node_tap.data_ptr(), M, tap_rowptr.data_ptr(), tap_nodes.data_ptr(),
                                           None if dxbuf is None else dxbuf.data_ptr(), ldc, dh.data_ptr(),
                                           None if db is None else db.data_ptr(), ctx.bias_per_node, ws.data_ptr(),
                                           ws_bytes, B, G, F_, K, _cabi.stream()))
        dx = _grad_in_input_layout(dxbuf, ldc, B, G, N, ctx.x_node_major) if need_dx else None
        return (dh if need_dh else None), dx, db, None, None


def _check_bias(b, F_, N):
    """The reference adds b by broadcasting (graphML.py:385-386): [F, 1] (NodeVariantGF's bias) or [F, N]."""
    if b is None:
        return None
    if b.dim() == 1 and b.shape[0] == F_ and N == 1:
        b = b.reshape(F_, 1)
    if not (b.dim() == 2 and b.shape[0] == F_ and b.shape[1] in (1, N)):
        raise RuntimeError("b200gf: NVGF bias must be [F, 1] or [F, N] = [%d, 1] or [%d, %d]; got %s"
                           % (F_, F_, N, tuple(b.shape)))
    return b


def _dispatch_cuda(h, S, x, b, taps):
    """Device part of NVGF: loud checks (there is no CPU path), plan lookup, the autograd function over the C ABI.
    `_dispatch` is the hook the CPU tests replace with the oracle to exercise the host logic around it."""
    check_operands("NVGF", x, (h, b), S)
    return _NVGFFunction.apply(h, x, b, plan_on(S, x.device), taps)


_dispatch = _dispatch_cuda


def NVGF(h, S, x, b=None):
    """NVGF(filter_taps, GSO, input, bias=None): node-variant graph filter, then bias.

    Same contract as the reference (alegnn/utils/graphML.py:293-387):
        h [F, E, K, G, N]; S [E, N, N] (dense tensor, or SparseGSO / Plan); x [B, G, N]; b [F, 1], [F, N] or None
        returns y [B, F, N],  y_f = sum_e sum_k sum_g diag(h_k^{efg}) S_e^k x_g + b_f
    """
    F_, E, K, G, N = h.shape
    assert S.shape[0] == E                       # graphML.py:344
    assert S.shape[1] == S.shape[2] == N         # graphML.py:345
    assert x.shape[1] == G                       # graphML.py:347
    assert x.shape[2] == N                       # graphML.py:348
    return _dispatch(h, S, x, _check_bias(b, F_, N), _identity_taps(N))


class NodeVariantGF(nn.Module):
    """NodeVariantGF(in_features, out_features, shift_taps, node_taps, edge_features=1, bias=True)

    Same surface as the reference layer (alegnn/utils/graphML.py:2317-2509): attributes G, F, K, M, E, S, N, copyNodes;
    parameters `weight` [F, E, K, G, M] and `bias` [F, 1] (or None), initialised in the same order; `addGSO(S)`,
    `forward(x)`, `extra_repr()`.  `addGSO` also accepts a SparseGSO, computes copyNodes without a dense matrix
    (`copy_nodes`) and builds the node -> tap map once per GSO."""

    def __init__(self, G, F, K, M, E=1, bias=True):
        super().__init__()
        self.G = G
        self.F = F
        self.K = K
        self.M = M
        self.E = E
        self.S = None
        self.weight = nn.parameter.Parameter(torch.Tensor(F, E, K, G, M))
        if bias:
            self.bias = nn.parameter.Parameter(torch.Tensor(F, 1))
        else:
            self.register_parameter("bias", None)
        self.reset_parameters()

    def reset_parameters(self):
        stdv = 1. / math.sqrt(self.G * self.K * self.M)   # graphML.py:2395-2400
        self.weight.data.uniform_(-stdv, stdv)
        if self.bias is not None:
            self.bias.data.uniform_(-stdv, stdv)

    def addGSO(self, S):
        assert len(S.shape) == 3                    # graphML.py:2404
        assert S.shape[0] == self.E                 # graphML.py:2406
        self.N = S.shape[1]
        assert S.shape[2] == self.N                 # graphML.py:2408
        copy = copy_nodes(S, self.M)
        self.S = S
        device = S.device if isinstance(S, torch.Tensor) else torch.device("cpu")
        self.copyNodes = torch.from_numpy(copy).to(device)
        self.taps = TapMap(copy, self.M)
        if torch.cuda.is_available() and (isinstance(S, SparseGSO) or
                                          (isinstance(S, torch.Tensor) and S.device.type == "cuda")):
            plan_for(S)

    def forward(self, x):
        B = x.shape[0]
        F = x.shape[1]
        Nin = x.shape[2]
        if Nin < self.N:                            # zero-pad the node axis, graphML.py:2487-2489
            x = torch.cat((x, torch.zeros(B, F, self.N - Nin, dtype=x.dtype, device=x.device)), dim=2)
        u = _dispatch(self.weight, self.S, x, self.bias, self.taps)
        if Nin < self.N:                            # keep the first Nin nodes, graphML.py:2496-2497
            u = u[:, :, :Nin]
        return u

    def extra_repr(self):
        reprString = "in_features=%d, out_features=%d, " % (self.G, self.F) + \
                     "shift_taps=%d, node_taps=%d, " % (self.K, self.M) + \
                     "edge_features=%d, " % (self.E) + "bias=%s, " % (self.bias is not None)
        if self.S is not None:
            reprString += "GSO stored"
        else:
            reprString += "no GSO stored"
        return reprString
