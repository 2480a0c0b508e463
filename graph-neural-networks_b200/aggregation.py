"""Aggregation GNNs on a sparse aggregation operator and the library's hop kernel.

    AggregationGNN(...)              <- alegnn/modules/architectures.py:2920-3228
    MultiNodeAggregationGNN(...)     <- alegnn/modules/architectures.py:3230-3573

Same constructor signatures, attributes, module trees (`ConvLayers`, `MLP`, `AggMLP`; `aggGNNmodules[r][p]`, `MLP`) and
parameter initialisation order as the reference, so the same torch seed gives the same state_dict and reference
checkpoints load.  Everything after the aggregation (Conv1d, activation, pooling, MLPs) is the reference's torch.nn.

The reference forms S_e^q e_p for every selected node p and every q < maxN with dense numpy products and keeps them as a
dense SN [nNodes, E, N, maxN] tensor, so it needs the dense N x N GSO and nNodes E N maxN values.  Here the selected
nodes stay in the original numbering (sel = order[:nNodes]; (x_perm S_perm^q)[p] = (x S^q)[order[p]]) and the Conv1d
operand is one sparse product

    z[b*nNodes + p, e*F + f, q] = sum_m x[b, f, m] R[(p*E + e)*maxN + q, m],     R[(p, e, q), m] = (S_e^q)[m, sel[p]],

R being SN without its zeros.  R is built once per device (AggregationOperator): the powers D_{e,q} = S_e D_{e,q-1} from
the indicator columns of sel, in float64, by b200gf_hop on the GSO's plan, a bounded block of selected columns at a
time, compacted on the device.  Its rows can be as long as N, and the hop kernels give one warp or lane group to a row,
so every row longer than ROW_SPLIT entries is split into pieces (split_levels): the product runs as a chain of at most
a few b200gf_hop calls per direction, the first over the pieces, the next summing each row's pieces.  The backward is
the same on R^T.  There is no CPU path: CPU tensors raise.
"""
import numpy as np
import scipy.sparse as sp
import torch
import torch.nn as nn

from . import _cabi
from .graphML import _grad_in_input_layout, check_operands, node_major_ld, padded_ld, to_node_major
from .graphtools_sparse import perm_degree
from .gso import Plan, SparseGSO

# Longest operator row one hop handles whole.  The hop kernels give a warp (or a lane group) to a row and walk its
# entries in order, four gathers in flight per lane, so a row of n entries costs n / 4 dependent gather rounds on one
# warp while an H100 holds 132 x 48 resident warps.  256 entries are 64 rounds; the 16 saturated 630k-entry rows of an
# ER graph of 1M nodes (maxN = 5) become about 40k pieces, six waves of resident warps, where 1024-entry pieces would
# make under two and leave the last wave's warps idle.  Rows up to 256^3 = 2^24 entries need at most 3 levels.
ROW_SPLIT = 256
NNZ_MAX = 2 ** 31 - 1            # the hop kernels' 32-bit row offsets
BUILD_BLOCK_BYTES = 1 << 28      # float64 bytes of one [N, columns] block of the powers, for each of its two buffers


def as_sparse_gso(S):
    """The GSO forms the other layers accept (numpy or torch dense [N, N] / [E, N, N], SparseGSO, torch sparse [N, N] /
    [E, N, N]) as a SparseGSO, the host CSR the operator is built from.  A sparse GSO is never densified."""
    if isinstance(S, SparseGSO):
        return S
    if isinstance(S, torch.Tensor) and S.layout != torch.strided:
        return SparseGSO.from_torch_sparse([S] if S.dim() == 2 else S)
    if isinstance(S, (torch.Tensor, np.ndarray)):
        S = torch.as_tensor(S).detach()
        if S.dim() == 2:
            S = S.unsqueeze(0)
        if not (S.dim() == 3 and S.shape[1] == S.shape[2]):
            raise ValueError("b200gf: a GSO is [N, N] or [E, N, N], got %s" % (tuple(S.shape),))
        return SparseGSO.from_dense(S.cpu())
    raise TypeError("b200gf: GSO must be a numpy array, a torch tensor (dense or sparse) or a SparseGSO, got %r"
                    % type(S))


def node_order(gso, order):
    """The reference's node ordering as a list: order=None is the identity, order='Degree' graphTools.permDegree
    (graphtools_sparse.perm_degree).  The other orderings need dense eigendecompositions and are not supported."""
    if order is None:
        return list(range(gso.N))
    if order == "Degree":
        return perm_degree([sp.csr_matrix((v, c, r), shape=(gso.N, gso.N)) for (r, c, v) in gso.csr])[1]
    raise NotImplementedError("b200gf: order=%r is not supported by the sparse aggregation GNNs: only None and "
                              "'Degree' (the 'EDS' and 'SpectralProxies' orders need dense eigendecompositions)" % (order,))


def split_levels(rowptr, col, val, n_cols, L=ROW_SPLIT):
    """A host CSR operator [n_rows, n_cols] as a chain of operators none of whose rows exceeds L entries.

    Returns [(rowptr, col, val, n_rows, n_cols), ...], applied first to last: the product of the chain is the operator.
    When no row is longer than L the chain is the operator itself.  Otherwise the first level has one row per piece of
    at most L consecutive entries of a row (an empty row has no piece), and the rest of the chain is split_levels of the
    [n_rows, n_pieces] operator of ones that adds up each row's pieces.  The pieces and sums are fixed by the input, so
    the summation order is too."""
    rowptr = np.asarray(rowptr, dtype=np.int64)
    n_rows = len(rowptr) - 1
    lens = np.diff(rowptr)
    if n_rows == 0 or int(lens.max()) <= L:
        return [(rowptr, col, val, n_rows, int(n_cols))]
    pieces = (lens + L - 1) // L
    n_pieces = int(pieces.sum())
    first = np.cumsum(pieces) - pieces                           # index of each row's first piece
    starts = np.repeat(rowptr[:-1], pieces) + (np.arange(n_pieces) - np.repeat(first, pieces)) * L
    level = (np.append(starts, rowptr[-1]), col, val, n_pieces, int(n_cols))
    sum_rowptr = np.zeros(n_rows + 1, dtype=np.int64)
    np.cumsum(pieces, out=sum_rowptr[1:])
    ones = np.ones(n_pieces, dtype=np.float64)
    return [level] + split_levels(sum_rowptr, np.arange(n_pieces, dtype=np.int32), ones, n_pieces, L)


class AggregationOperator:
    """R for one (GSO, selection, maxN): row (p*E + e)*maxN + q holds column sel[p] of S_e^q.

    `host(device)` builds R and R^T once per device and keeps them as host CSR; `levels(device, dtype)` their
    split_levels chains as device plans, one set per dtype a call uses (R is formed in float64 and cast once)."""

    def __init__(self, S, sel, maxN):
        self.gso = as_sparse_gso(S)
        self.sel = np.asarray(sel, dtype=np.int64).reshape(-1)
        self.N, self.E, self.maxN = self.gso.N, self.gso.E, int(maxN)
        self.P = len(self.sel)
        if not (self.P >= 1 and self.maxN >= 1 and self.sel.min() >= 0 and self.sel.max() < self.N):
            raise ValueError("b200gf: an aggregation needs 1 <= nNodes <= N selected nodes and maxN >= 1")
        self.n_rows = self.P * self.E * self.maxN
        self._host = {}
        self._levels = {}
        self._sel = {}

    def sel_on(self, device):
        """The selected nodes as an int64 tensor on `device`, copied there once (so that a captured forward copies
        nothing from the host)."""
        device = torch.device(device)
        if device not in self._sel:
            self._sel[device] = torch.from_numpy(self.sel).to(device)
        return self._sel[device]

    @staticmethod
    def _key(device):
        device = torch.device(device)
        return device.index if device.index is not None else torch.cuda.current_device()

    def host(self, device):
        """(R, R^T) as host CSR triples (rowptr int64, col int32, val float64), built on `device`."""
        key = self._key(device)
        if key not in self._host:
            self._host[key] = self._build(torch.device("cuda", key))
        return self._host[key]

    def _powers(self, plan, e, sel, device):
        """Yields (p0, q, D) for every block of selected columns [p0, p0 + w) and q < maxN: D [N, w] holds
        S_e^q e_{sel[p0 + j]} in column j < w.  D is overwritten by the next step."""
        lib = _cabi.load()
        N = self.N
        width = max(1, min(self.P, BUILD_BLOCK_BYTES // (8 * N)))
        ld = padded_ld(width, torch.float64)
        for p0 in range(0, self.P, width):
            w = min(width, self.P - p0)
            cur = torch.zeros((N, ld), dtype=torch.float64, device=device)
            cur[sel[p0:p0 + w], torch.arange(w, device=device)] = 1.0
            nxt = torch.empty_like(cur)
            yield p0, 0, cur[:, :w]
            for q in range(1, self.maxN):
                _cabi.check(lib.b200gf_hop(plan.handle, e, _cabi.HOP_BWD, cur.data_ptr(), ld, nxt.data_ptr(), ld, w,
                                           _cabi.stream()))
                cur, nxt = nxt, cur
                yield p0, q, cur[:, :w]

    def _build(self, device):
        gso64 = self.gso.astype(torch.float64)
        plan = gso64.plan(device)
        sel = self.sel_on(device)
        # first pass: count, so that an operator past the 32-bit offsets raises before anything of its size exists
        nnz = 0
        for e in range(self.E):
            for _, _, D in self._powers(plan, e, sel, device):
                nnz += int(torch.count_nonzero(D))
        if nnz > NNZ_MAX:
            raise ValueError("b200gf: the aggregation operator of %d selected nodes, E = %d and maxN = %d on N = %d "
                             "nodes holds %d entries, more than the 2^31 - 1 that the hop's 32-bit offsets address"
                             % (self.P, self.E, self.maxN, self.N, nnz))
        rows, cols, vals = [], [], []
        for e in range(self.E):
            for p0, q, D in self._powers(plan, e, sel, device):
                m, j = D.nonzero(as_tuple=True)
                rows.append(((p0 + j) * self.E + e) * self.maxN + q)
                cols.append(m)
                vals.append(D[m, j])
        rows, cols, vals = torch.cat(rows), torch.cat(cols), torch.cat(vals)
        by_col = torch.sort(cols, stable=True)[1]
        order = by_col[torch.sort(rows[by_col], stable=True)[1]]           # by (row, column)
        t_order = order[torch.sort(cols[order], stable=True)[1]]           # by (column, row)

        def csr(r, c, v, n):
            r, c, v = r.cpu().numpy(), c.to(torch.int32).cpu().numpy(), v.cpu().numpy()
            rowptr = np.zeros(n + 1, dtype=np.int64)
            np.cumsum(np.bincount(r, minlength=n), out=rowptr[1:])
            return rowptr, c, v

        return (csr(rows[order], cols[order], vals[order], self.n_rows),
                csr(cols[t_order], rows[t_order], vals[t_order], self.N))

    def levels(self, device, dtype):
        """(forward chain, backward chain) of device plans in `dtype`: R's split_levels and R^T's."""
        key = (self._key(device), dtype)
        if key not in self._levels:
            dev = torch.device("cuda", key[0])
            (r_rowptr, r_col, r_val), (t_rowptr, t_col, t_val) = self.host(dev)
            self._levels[key] = tuple([Plan.from_ops([(rp, c, v)], None, n, nc, dtype, dev)
                                       for (rp, c, v, n, nc) in split_levels(*op)]
                                      for op in ((r_rowptr, r_col, r_val, self.N), (t_rowptr, t_col, t_val, self.n_rows)))
        return self._levels[key]


def _chain(plans, src, src_ld, C):
    """src [n_cols, src_ld] node-major through the chain: one b200gf_hop (the plan's forward operator) per level.
    Returns the last level's output [n_rows, ld] and ld."""
    lib = _cabi.load()
    ld = padded_ld(C, src.dtype)
    for plan in plans:
        dst = torch.empty((plan.n_rows, ld), dtype=src.dtype, device=src.device)
        _cabi.check(lib.b200gf_hop(plan.handle, 0, _cabi.HOP_FWD, src.data_ptr(), src_ld, dst.data_ptr(), ld, C,
                                   _cabi.stream()))
        src, src_ld = dst, ld
    return src, src_ld


class _AggregationFunction(torch.autograd.Function):
    """z = the Conv1d operand of x [B, F, N] (module docstring); dx = R^T dz."""

    @staticmethod
    def forward(ctx, x, fwd, bwd, dims):
        P, E, maxN = dims
        B, F_, N = x.shape
        C = B * F_
        ctx.x_node_major = node_major_ld(x) is not None
        xn, x_ld = to_node_major(x)
        out, _ = _chain(fwd, xn, x_ld, C)
        ctx.bwd, ctx.dims = bwd, (B, F_, N, P, E, maxN)
        return out[:, :C].view(P, E, maxN, B, F_).permute(3, 0, 1, 4, 2).reshape(B * P, E * F_, maxN)

    @staticmethod
    def backward(ctx, dz):
        if not ctx.needs_input_grad[0]:
            return None, None, None, None
        B, F_, N, P, E, maxN = ctx.dims
        C = B * F_
        ld = padded_ld(C, dz.dtype)
        dzn = torch.empty((P * E * maxN, ld), dtype=dz.dtype, device=dz.device)
        dzn[:, :C].view(P, E, maxN, B, F_).copy_(dz.reshape(B, P, E, F_, maxN).permute(1, 2, 4, 0, 3))
        dxn, dx_ld = _chain(ctx.bwd, dzn, ld, C)
        return _grad_in_input_layout(dxn, dx_ld, B, F_, N, ctx.x_node_major), None, None, None


def _aggregate_cuda(op, x):
    """The Conv1d operand [(B*nNodes), E*F, maxN] of x [B, F, N] on the CUDA path.  `_aggregate` is the hook the CPU
    tests replace with the oracle to exercise the layers' host code."""
    check_operands("AggregationGNN", x, ())
    fwd, bwd = op.levels(x.device, x.dtype)
    return _AggregationFunction.apply(x, fwd, bwd, (op.P, op.E, op.maxN))


_aggregate = _aggregate_cuda


class AggregationGNN(nn.Module):
    """AggregationGNN(dimFeatures, nFilterTaps, bias, nonlinearity, poolingFunction, poolingSize, dimLayersMLP, GSO,
    order=None, maxN=None, nNodes=1, dimLayersAggMLP=[])  (alegnn/modules/architectures.py:2920-3228)

    GSO: numpy or torch dense [N, N] / [E, N, N], SparseGSO or torch sparse.  order: None or 'Degree'.  The selected
    nodes are order[:nNodes].  Runs on CUDA tensors in float64 (as the reference) or float32; a CPU input raises.
    `.to(device)` returns the module (the reference's returns None).  `S` is the GSO as a SparseGSO and `order` the
    node ordering; there is no dense `SN`: `operator` is its sparse form."""

    def __init__(self, dimFeatures, nFilterTaps, bias, nonlinearity, poolingFunction, poolingSize, dimLayersMLP, GSO,
                 order=None, maxN=None, nNodes=1, dimLayersAggMLP=[]):
        super().__init__()
        gso = as_sparse_gso(GSO)
        N = gso.N
        if not 1 <= nNodes <= N:
            raise ValueError("b200gf: AggregationGNN selects 1 <= nNodes <= N = %d nodes, got %d" % (N, nNodes))
        self._init_layers(dimFeatures, nFilterTaps, bias, nonlinearity, poolingFunction, poolingSize, dimLayersMLP,
                          gso.E, N if maxN is None or maxN >= N else maxN, nNodes, dimLayersAggMLP)
        self.S = gso
        self.order = node_order(gso, order)
        self.operator = AggregationOperator(gso, self.order[:nNodes], self.maxN)

    def _init_layers(self, dimFeatures, nFilterTaps, bias, nonlinearity, poolingFunction, poolingSize, dimLayersMLP, E,
                     maxN, nNodes, dimLayersAggMLP):
        """Attributes and the torch.nn modules after the aggregation, built in the reference's order."""
        assert len(dimFeatures) == len(nFilterTaps) + 1
        assert len(poolingSize) == len(nFilterTaps)
        self.L = len(nFilterTaps)
        self.F = dimFeatures
        self.K = nFilterTaps
        self.E = E
        self.bias = bias
        self.sigma = nonlinearity
        self.rho = poolingFunction
        self.alpha = poolingSize
        self.dimLayersMLP = dimLayersMLP
        self.dimLayersAggMLP = dimLayersAggMLP
        self.nNodes = nNodes
        self.maxN = maxN
        self.N = [self.maxN]                                   # conv output lengths (architectures.py:3070-3077)
        for l in range(self.L):
            outConvN = self.N[l] - (self.K[l] - 1)
            self.N += [int((outConvN - (self.alpha[l] - 1) - 1) / self.alpha[l] + 1)]
        convl = []
        for l in range(self.L):
            convl.append(nn.Conv1d(self.F[l] * self.E, self.F[l + 1] * self.E, self.K[l], bias=self.bias))
            convl.append(self.sigma())
            convl.append(self.rho(self.alpha[l]))
        self.ConvLayers = nn.Sequential(*convl)
        fc = []
        if len(self.dimLayersMLP) > 0:
            fc.append(nn.Linear(self.N[-1] * self.F[-1] * self.E, dimLayersMLP[0], bias=self.bias))
            for l in range(len(dimLayersMLP) - 1):
                fc.append(self.sigma())
                fc.append(nn.Linear(dimLayersMLP[l], dimLayersMLP[l + 1], bias=self.bias))
        self.MLP = nn.Sequential(*fc)
        aggfc = []
        if len(self.dimLayersAggMLP) > 0:
            dimInputAggMLP = dimLayersMLP[-1] if len(dimLayersMLP) > 0 else self.N[-1] * self.F[-1] * self.E
            aggfc.append(nn.Linear(dimInputAggMLP * nNodes, dimLayersAggMLP[0], bias=self.bias))
            for l in range(len(dimLayersAggMLP) - 1):
                aggfc.append(self.sigma())
                aggfc.append(nn.Linear(dimLayersAggMLP[l], dimLayersAggMLP[l + 1], bias=self.bias))
        self.AggMLP = nn.Sequential(*aggfc)

    @classmethod
    def _inner(cls, *layer_args):
        """An inner module of MultiNodeAggregationGNN: the layers alone; its outer module owns the shared operator."""
        m = cls.__new__(cls)
        nn.Module.__init__(m)
        m._init_layers(*layer_args)
        m.S, m.order, m.operator = None, None, None
        return m

    def forward(self, x):
        assert len(x.shape) == 3
        assert x.shape[1] == self.F[0]
        assert x.shape[2] == self.operator.N
        return self._readout(_aggregate(self.operator, x), x.shape[0])

    def _readout(self, z, B):
        """architectures.py:3195-3221 from the Conv1d operand z [(B*nNodes), E*F, maxN] on."""
        y = self.ConvLayers(z)
        y = y.reshape([B * self.nNodes, self.F[-1] * self.N[-1] * self.E])
        y = self.MLP(y)
        y = y.permute(1, 0).reshape([y.shape[1], B, self.nNodes]).permute(1, 0, 2)
        if self.nNodes == 1 or len(self.dimLayersAggMLP) > 0:
            y = y.reshape([B, y.shape[1] * self.nNodes])
        return self.AggMLP(y)


class MultiNodeAggregationGNN(nn.Module):
    """MultiNodeAggregationGNN(nSelectedNodes, nShifts, dimFeatures, nFilterTaps, bias, nonlinearity, poolingFunction,
    poolingSize, dimLayersMLP, GSO, order=None)  (alegnn/modules/architectures.py:3230-3573)

    Outer layer r aggregates at the nodes order[:P[r]] over Q[r] shifts with one operator and one product shared by its
    P[r] inner modules; inner module p runs its ConvLayers and MLP on node order[p]'s slice.  Between outer layers the
    outputs are placed at nodes order[:P[r]] of a zero signal.  No per-node copy of the GSO is made.  Unlike the
    reference, the caller's nSelectedNodes and dimFeatures lists are not modified."""

    def __init__(self, nSelectedNodes, nShifts, dimFeatures, nFilterTaps, bias, nonlinearity, poolingFunction,
                 poolingSize, dimLayersMLP, GSO, order=None):
        super().__init__()
        gso = as_sparse_gso(GSO)
        self.N = gso.N
        self.R = len(nSelectedNodes)
        self.P = [min(p, self.N) for p in nSelectedNodes]
        assert len(nShifts) == self.R
        self.Q = nShifts
        assert len(dimFeatures) == len(nFilterTaps) == self.R
        assert len(poolingSize) == self.R
        self.F = list(dimFeatures) + [[dimFeatures[-1][-1]]]
        self.K = nFilterTaps
        self.bias = bias
        self.sigma = nonlinearity
        self.rho = poolingFunction
        self.alpha = poolingSize
        self.dimLayersMLP = dimLayersMLP
        self.S = gso
        self.order = node_order(gso, order)
        self.aggGNNmodules = nn.ModuleList()
        for r in range(self.R):
            self.aggGNNmodules.append(nn.ModuleList())
            maxN = min(self.Q[r], self.N)
            for p in range(self.P[r]):
                self.aggGNNmodules[r].append(AggregationGNN._inner(
                    self.F[r], self.K[r], self.bias, self.sigma, self.rho, self.alpha[r], [self.F[r + 1][0]], gso.E,
                    maxN, 1, []))
        fc = []
        if len(self.dimLayersMLP) > 0:
            fc.append(nn.Linear(self.P[-1] * self.F[-1][0], dimLayersMLP[0], bias=self.bias))
            for l in range(len(dimLayersMLP) - 1):
                fc.append(self.sigma())
                fc.append(nn.Linear(dimLayersMLP[l], dimLayersMLP[l + 1], bias=self.bias))
        self.MLP = nn.Sequential(*fc)
        self.operators = [AggregationOperator(gso, self.order[:self.P[r]], min(self.Q[r], self.N))
                          for r in range(self.R)]

    def forward(self, x):
        assert len(x.shape) == 3
        B = x.shape[0]
        assert x.shape[1] == self.F[0][0]
        assert x.shape[2] == self.N
        for r in range(self.R):
            P, op = self.P[r], self.operators[r]
            z = _aggregate(op, x).reshape(B, P, op.E * self.F[r][0], op.maxN)
            y = torch.stack([self.aggGNNmodules[r][p]._readout(z[:, p], B) for p in range(P)], dim=2)   # [B, F, P]
            if r < self.R - 1:
                x = y.new_zeros((B, y.shape[1], self.N)).index_copy(2, op.sel_on(y.device), y)
        return self.MLP(y.reshape(B, self.F[-1][-1] * self.P[-1]))
