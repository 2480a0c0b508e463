"""Local max-pooling over K-hop neighbourhoods for graphs the reference cannot handle (SURVEY.md §8f-1, host-side part).

    MaxPoolLocal(in_dim, out_dim, number_hops)          <- alegnn/utils/graphML.py:1850-2028

Same surface and results as the reference layer.  Differences are internal: `addGSO` also accepts a `SparseGSO`, the
neighbourhoods come from the CSR routine (`graphtools_sparse.compute_neighborhood`) instead of a pure-python search over a
dense N x N matrix (graphML.py:1953-1957 -> graphTools.py:459-500, O(N deg^K) python), and `forward` gathers only the
neighbours (`index_select`) instead of first repeating the whole signal `maxNeighborhoodSize` times (graphML.py:1990-1996).
The gather itself is a CUDA kernel of libb200gf.so on the node-major layout (b200gf_maxpool_forward / _backward,
csrc/layer.cu): it consumes the permuted view a GraphFilter returns without a transpose and returns the same kind of
view; the arg-max per output element is kept for the backward scatter.  No CPU path (CPU tensors raise), like LSIGF.
"""
import numpy as np
import scipy.sparse as sp
import torch
import torch.nn as nn

from . import _cabi
from .graphtools_sparse import compute_neighborhood
from .gso import SparseGSO


def _gather_max_cuda(x, nb32, n_out, max_nb):
    return _MaxPoolFunction.apply(x, nb32, n_out, max_nb)


_gather_max = _gather_max_cuda      # the one hook CPU tests replace (a torch gather) to exercise the layer logic


class _MaxPoolFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, nb32, n_out, max_nb):
        from . import graphML as g
        g.check_operands("MaxPoolLocal", x, ())
        lib = _cabi.load()
        B, F, Nin = x.shape
        ctx.x_node_major = g.node_major_ld(x) is not None
        xn, x_ld = g.to_node_major(x)
        C = B * F
        ld = g.padded_ld(C, x.dtype)
        out = torch.empty((n_out, ld), dtype=x.dtype, device=x.device)
        arg = torch.empty((n_out, C), dtype=torch.int32, device=x.device)
        _cabi.check(lib.b200gf_maxpool_forward(_cabi.DTYPE[x.dtype], xn.data_ptr(), x_ld, Nin, C, nb32.data_ptr(), n_out,
                                               max_nb, out.data_ptr(), ld, arg.data_ptr(), _cabi.stream()))
        ctx.save_for_backward(arg)
        ctx.dims = (B, F, Nin, n_out, ld)
        return g._as_bcn_view(out, B, F, n_out)

    @staticmethod
    def backward(ctx, dy):
        from . import graphML as g
        lib = _cabi.load()
        (arg,) = ctx.saved_tensors
        B, F, Nin, n_out, ld = ctx.dims
        dyn, dy_ld = g.to_node_major(dy)
        C = B * F
        dx = torch.empty((Nin, ld), dtype=dy.dtype, device=dy.device)
        _cabi.check(lib.b200gf_maxpool_backward(_cabi.DTYPE[dy.dtype], dyn.data_ptr(), dy_ld, arg.data_ptr(), n_out, C,
                                                dx.data_ptr(), ld, Nin, _cabi.stream()))
        return g._as_bcn_view(dx, B, F, Nin), None, None, None


class MaxPoolLocal(nn.Module):
    def __init__(self, nInputNodes, nOutputNodes, nHops):
        super().__init__()
        self.nInputNodes = nInputNodes
        self.nOutputNodes = nOutputNodes
        self.nHops = nHops
        self.neighborhood = None
        self._nb32 = None

    def addGSO(self, S):
        assert len(S.shape) == 3                     # graphML.py:1944
        self.N = S.shape[1]
        assert S.shape[2] == self.N
        if isinstance(S, SparseGSO):
            device = torch.device("cpu")
            mats = [sp.csr_matrix((v, c, r), shape=(S.N, S.N)) for (r, c, v) in S.csr]
        else:
            device = S.device
            Sc = S.detach().cpu()
            mats = []
            for e in range(Sc.shape[0]):
                nz = Sc[e].nonzero(as_tuple=False).numpy()
                vals = Sc[e][nz[:, 0], nz[:, 1]].numpy().astype(np.float64)
                mats.append(sp.csr_matrix((vals, (nz[:, 0], nz[:, 1])), shape=(self.N, self.N)))
        nb = compute_neighborhood(mats if len(mats) > 1 else mats[0], self.nHops, self.nOutputNodes,
                                  self.nInputNodes, "matrix")
        self._set_neighborhood(torch.tensor(nb, dtype=torch.int64, device=device))

    def _set_neighborhood(self, neighborhood):
        assert neighborhood.shape[0] == self.nOutputNodes
        assert neighborhood.numel() == 0 or neighborhood.max() <= self.nInputNodes
        self.maxNeighborhoodSize = neighborhood.shape[1]
        self.neighborhood = neighborhood             # same attribute (and values) as the reference layer
        self._nb32 = None

    @classmethod
    def from_reference(cls, ref):
        """Takes over an already configured reference MaxPoolLocal (its neighbourhood matrix is reused as is)."""
        m = cls(ref.nInputNodes, ref.nOutputNodes, ref.nHops)
        if getattr(ref, "neighborhood", None) is not None:
            m.N = getattr(ref, "N", ref.nInputNodes)
            m._set_neighborhood(ref.neighborhood.to(torch.int64))
        return m

    def forward(self, x):
        B, F, Nin = x.shape
        assert Nin == self.nInputNodes               # graphML.py:1977
        assert Nin >= self.nOutputNodes
        if self._nb32 is None or self._nb32.device != x.device:
            self._nb32 = self.neighborhood.to(device=x.device, dtype=torch.int32).contiguous()
        return _gather_max(x, self._nb32, self.nOutputNodes, self.maxNeighborhoodSize)

    def extra_repr(self):
        s = "in_dim=%d, out_dim=%d, number_hops = %d, " % (self.nInputNodes, self.nOutputNodes, self.nHops)
        return s + ("neighborhood stored" if self.neighborhood is not None else "NO neighborhood stored")
