"""Localized activation functions on K-hop neighbourhoods (SURVEY.md §2.1 row 6, a "next" candidate of §8f).

    MaxLocalActivation(K)        <- alegnn/utils/graphML.py:1535-1660
    MedianLocalActivation(K)     <- alegnn/utils/graphML.py:1662-1810

Same surface (parameter `weight [1, K+1]`, `addGSO`, `forward`, `reset_parameters`) and the same results as the reference
layers: out = sum_{k=0..K} w_k * agg_k(x), agg_0 = x, agg_k = max / lower median over the k-hop neighbourhood of each
node.  `addGSO` takes a dense GSO or a `SparseGSO` and builds one ring-ordered list per node
(`graphtools_sparse.ring_neighborhoods`: the node, then its 1-hop ring, ..., its K-hop ring), which serves every k.

CUDA tensors run in libb200gf.so (b200gf_local_activation_forward / _backward, csrc/layer.cu): one gather-select per
(node, column) over the node's list gives every agg_k and the fused combine, on the node-major layout a GraphFilter
produces, which is consumed in place; the result is the same kind of view.  Nothing of size [B, F, N, M_k] is formed.
Ties: the max goes to the smallest node index holding the maximum (the reference's first maximum in an index-sorted
list), the median to the smallest node index holding the median value.  NaN inputs give an unspecified result.  The
input gradient is scattered with atomics (its last bits may change between runs); the weight gradient, sum x dy and
sum agg_k dy, is a deterministic torch reduction.

CPU tensors take the torch path (index matrices padded to the widest neighbourhood M_k, built from the ring lists on
first CPU use).  Both paths read a one-edge-feature GSO with the reference's rule, |S[i, j]| > 1e-9, as they read
several (sum_e |S_e[i, j]| > 1e-9); the torch path used to drop negative entries of a one-feature GSO.
"""
import math

import numpy as np
import scipy.sparse as sp
import torch
import torch.nn as nn

from . import _cabi
from .graphtools_sparse import ring_neighborhoods
from .gso import SparseGSO

_SELECT = {"MaxLocalActivation": 0, "MedianLocalActivation": 1}     # B200GF_LOCAL_MAX, B200GF_LOCAL_MEDIAN


def _scipy_mats(S):
    if isinstance(S, SparseGSO):
        return [sp.csr_matrix((v, c, r), shape=(S.N, S.N)) for (r, c, v) in S.csr]
    Sc = S.detach().cpu()
    mats = []
    for e in range(Sc.shape[0]):
        nz = Sc[e].nonzero(as_tuple=False).numpy()
        vals = Sc[e][nz[:, 0], nz[:, 1]].numpy().astype(np.float64)
        mats.append(sp.csr_matrix((vals, (nz[:, 0], nz[:, 1])), shape=(Sc.shape[1], Sc.shape[1])))
    return mats


def _padded_prefix(rowptr, col, ring_end, k):
    """Row i's k-hop neighbourhood (its ring list's prefix) sorted ascending and padded with i to the widest: [N, M_k]
    int64, graphTools.computeNeighborhood's 'matrix' form; and the lengths [N]."""
    n = len(rowptr) - 1
    lens = ring_end[:, k].astype(np.int64)
    width = int(lens.max()) if n else 0
    rows = np.repeat(np.arange(n), lens)
    pos = np.arange(int(lens.sum())) - np.repeat(np.cumsum(lens) - lens, lens)
    vals = col[np.repeat(rowptr[:-1], lens) + pos].astype(np.int64)
    vals = vals[np.lexsort((vals, rows))]
    out = np.repeat(np.arange(n, dtype=np.int64)[:, None], width, axis=1)
    out[rows, pos] = vals
    return torch.from_numpy(out), torch.from_numpy(lens)


class _LocalActivationFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, rings, K, select, name):
        from . import graphML as g
        g.check_operands(name, x, (weight,))
        rowptr, col, ring_end = rings
        lib = _cabi.load()
        B, F, N = x.shape
        C = B * F
        ctx.x_node_major = g.node_major_ld(x) is not None
        xn, x_ld = g.to_node_major(x)
        ld = g.padded_ld(C, x.dtype)
        w = weight.detach().reshape(-1).contiguous()
        y = torch.empty((N, ld), dtype=x.dtype, device=x.device)
        agg = torch.empty((K, N, ld), dtype=x.dtype, device=x.device)
        arg = torch.empty((K, N, C), dtype=torch.int32, device=x.device)
        _cabi.check(lib.b200gf_local_activation_forward(
            _cabi.DTYPE[x.dtype], select, xn.data_ptr(), x_ld, N, C, rowptr.data_ptr(), col.data_ptr(),
            ring_end.data_ptr(), K, w.data_ptr(), y.data_ptr(), ld, agg.data_ptr(), ld, arg.data_ptr(), _cabi.stream()))
        ctx.save_for_backward(xn, agg, arg, w)
        ctx.dims = (B, F, N, K, x_ld, ld)
        return g._as_bcn_view(y, B, F, N)

    @staticmethod
    def backward(ctx, dy):
        from . import graphML as g
        lib = _cabi.load()
        xn, agg, arg, w = ctx.saved_tensors
        B, F, N, K, x_ld, ld = ctx.dims
        C = B * F
        dyn, dy_ld = g.to_node_major(dy)
        dx = None
        if ctx.needs_input_grad[0]:
            dxb = torch.empty((N, ld), dtype=dy.dtype, device=dy.device)
            _cabi.check(lib.b200gf_local_activation_backward(_cabi.DTYPE[dy.dtype], dyn.data_ptr(), dy_ld, arg.data_ptr(),
                                                             N, C, K, w.data_ptr(), dxb.data_ptr(), ld, _cabi.stream()))
            dx = g._grad_in_input_layout(dxb, ld, B, F, N, ctx.x_node_major)
        dw = None
        if ctx.needs_input_grad[1]:
            dyv = dyn.as_strided((N, C), (dy_ld, 1))
            dw0 = (xn.as_strided((N, C), (x_ld, 1)) * dyv).sum().reshape(1)
            dwk = (agg[:, :, :C] * dyv.unsqueeze(0)).sum(dim=(1, 2))
            dw = torch.cat([dw0, dwk]).reshape(1, K + 1)
        return dx, dw, None, None, None, None


class _LocalActivation(nn.Module):
    def __init__(self, K):
        super().__init__()
        assert K > 0                                   # graphML.py:1582
        self.K = K
        self.S = None
        self.N = None
        self._rings = None                             # host (rowptr, col, ring_end) of ring_neighborhoods
        self._rings_dev = {}                           # the same on each CUDA device that ran the layer
        self._padded = None                            # the torch path's index matrices, built on first CPU use
        self.weight = nn.parameter.Parameter(torch.Tensor(1, self.K + 1))
        self.reset_parameters()

    def reset_parameters(self):
        stdv = 1. / math.sqrt(self.K)                  # graphML.py:1651
        self.weight.data.uniform_(-stdv, stdv)

    def addGSO(self, S):
        assert len(S.shape) == 3                       # graphML.py:1594
        self.N = S.shape[1]
        assert S.shape[2] == self.N
        self.S = S
        # always the list form: an edge is sum_e |S_e[i, j]| > 1e-9 for E = 1 too, as the reference's
        # computeNeighborhood reads the E x N x N array it is given (graphTools.py:424-432)
        self._rings = ring_neighborhoods(_scipy_mats(S), self.K)
        self._rings_dev = {}
        self._padded = None
        self.maxNeighborhoodSizes = [int(self._rings[2][:, k].max()) if self.N else 0 for k in range(1, self.K + 1)]

    @property
    def neighborhood(self):
        """Per hop k = 1..K: (index matrix [N, M_k] padded with the node itself, lengths [N]); 'None' before addGSO."""
        if self._rings is None:
            return "None"
        if self._padded is None:
            self._padded = [_padded_prefix(*self._rings, k) for k in range(1, self.K + 1)]
        return self._padded

    def _device_rings(self, device):
        if device not in self._rings_dev:
            self._rings_dev[device] = tuple(torch.from_numpy(a).to(device) for a in self._rings)
        return self._rings_dev[device]

    def forward(self, x):
        B, F, N = x.shape
        assert N == self.N                             # graphML.py:1617, 1768
        if x.device.type != "cuda":
            return self._forward_torch(x)
        return _LocalActivationFunction.apply(x, self.weight, self._device_rings(x.device), self.K,
                                              _SELECT[type(self).__name__], type(self).__name__)

    def _combine(self, aggs):
        xK = torch.stack(aggs, dim=3)                                   # [B, F, N, K+1]
        out = torch.matmul(xK, self.weight.unsqueeze(2))                # graphML.py:1644
        return out.reshape(xK.shape[0], xK.shape[1], self.N)

    def extra_repr(self):
        # the reference tests `self.neighborhood is not None`, and its placeholder before addGSO is the string 'None'
        return "neighborhood stored" if self.neighborhood is not None else "NO neighborhood stored"


class MaxLocalActivation(_LocalActivation):
    def _forward_torch(self, x):
        B, F, N = x.shape
        aggs = [x]
        for (idx, _) in self.neighborhood:
            idx = idx.to(x.device)
            v, _ = torch.max(x.index_select(2, idx.reshape(-1)).reshape(B, F, N, idx.shape[1]), dim=3)
            aggs.append(v)
        return self._combine(aggs)


class MedianLocalActivation(_LocalActivation):
    def _forward_torch(self, x):
        B, F, N = x.shape
        aggs = [x]
        for (idx, lens) in self.neighborhood:
            idx, lens = idx.to(x.device), lens.to(x.device)
            M = idx.shape[1]
            xn = x.index_select(2, idx.reshape(-1)).reshape(B, F, N, M)
            pad = torch.arange(M, device=x.device).unsqueeze(0) >= lens.unsqueeze(1)          # [N, M] padded slots
            xs, _ = torch.sort(xn.masked_fill(pad.reshape(1, 1, N, M), float("inf")), dim=3)
            pick = ((lens - 1) // 2).reshape(1, 1, N, 1).expand(B, F, N, 1)                  # torch.median: lower median
            aggs.append(torch.gather(xs, 3, pick).squeeze(3))
        return self._combine(aggs)


class NoActivation(nn.Module):
    """graphML.py:1812-1848"""

    def forward(self, x):
        return x

    def extra_repr(self):
        return "No Activation Function"
