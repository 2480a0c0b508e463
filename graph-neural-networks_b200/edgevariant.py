"""Edge-variant graph filter (the variant row of the path, SURVEY.md §8 a-7), executed sparsely on the GPU.

    EVGF(S, x, b=None)                                   <- alegnn/utils/graphML.py:389-488
    EdgeVariantGF(G, F, K, M, N, E=1, bias=True)         <- alegnn/utils/graphML.py:2511-2712

The reference multiplies dense N x N filter matrices Phi^(k)_{f e g}; only the entries on the masked sparsity pattern
of |S_e| + I are ever non-zero (`sparsityPatternFull`, graphML.py:2620-2663).  Here those entries are gathered once per
call into per-non-zero weights on a compact node set and the K-step chains run in `b200gf_ev_forward/backward`
(csrc/ev.cu).  Parameter names and shapes (`weightEV [F,E,K,G,N,N]`, `weightLSI [F,E,K,G]`, `bias [F,1]`) are the
reference's, so its checkpoints load; the hybrid layer's LSI part goes through this package's LSIGF.
Reference quirks kept on purpose: the hybrid layer adds the bias twice (once in EVGF :2682, once in LSIGF :2686).
"""
import math

import torch
import torch.nn as nn

from . import _cabi
from .graphML import LSIGF, check_operands

zeroTolerance = 1e-9  # graphML.py:72


class EVStructure:
    """Compact CSR patterns (one per edge feature) for a masked sparsity pattern.

    `EVStructure(pattern)`: dense bool [E, N, N] (the reference-sized layer).  `EVStructure.from_coo(N, [(rows, cols)..])`:
    the same from per-e coordinate lists, for graphs whose N x N pattern cannot be materialised (SparseEdgeVariantGF)."""

    def __init__(self, pattern=None):
        if pattern is None:
            return
        assert pattern.dim() == 3 and pattern.shape[1] == pattern.shape[2]
        nz = [pattern[e].nonzero(as_tuple=False) for e in range(pattern.shape[0])]   # row-major order
        self._build(pattern.shape[1], [(z[:, 0], z[:, 1]) for z in nz], pattern.device)

    @classmethod
    def from_coo(cls, N, coords, device):
        """coords: per e a pair (rows, cols) of int64 tensors, sorted row-major, no duplicates."""
        self = cls()
        self._build(N, [(r.to(device), c.to(device)) for (r, c) in coords], torch.device(device))
        return self

    def _build(self, N, coords, dev):
        E = len(coords)
        self.E, self.N = E, N
        touched = torch.zeros(N, dtype=torch.bool, device=dev)
        for (r, c) in coords:
            touched[r] = True
            touched[c] = True
        self.A = touched.nonzero(as_tuple=False).flatten()                     # compact set, ascending global ids
        self.NA = int(self.A.numel())
        inv = torch.full((N,), -1, dtype=torch.int64, device=dev)
        inv[self.A] = torch.arange(self.NA, device=dev)
        self.per_e = []
        for (r, c) in coords:
            ci, cj = inv[r], inv[c]
            nnz = int(ci.numel())
            rowptr = torch.zeros(self.NA + 1, dtype=torch.int64, device=dev)
            rowptr[1:] = torch.cumsum(torch.bincount(ci, minlength=self.NA), 0)
            permT = torch.argsort(cj * max(self.NA, 1) + ci)                   # entries ordered by (column, row)
            rowptrT = torch.zeros(self.NA + 1, dtype=torch.int64, device=dev)
            rowptrT[1:] = torch.cumsum(torch.bincount(cj, minlength=self.NA), 0)
            diag = torch.full((self.NA,), -1, dtype=torch.int32, device=dev)    # position of (i, i) in the pattern
            on = (ci == cj).nonzero(as_tuple=False).flatten()
            diag[ci[on]] = on.to(torch.int32)
            self.per_e.append(dict(
                nnz=nnz, rowptr=rowptr, col=cj.to(torch.int32).contiguous(), rowidx=ci.to(torch.int32).contiguous(),
                rowptrT=rowptrT, colT=ci[permT].to(torch.int32).contiguous(), perm=permT.contiguous(), diag=diag,
                rows_global=r, cols_global=c,
                lin=(r * N + c).contiguous() if N * N < 2 ** 62 else None))     # flat index into a dense [N, N] matrix


class _EVChain(torch.autograd.Function):
    """y_e[b, f, i in A] = sum_g sum_k (Phi^(k) ... Phi^(0) x_g)[i] for one edge feature (csrc/ev.cu, batch innermost).
    k0_identity: step 0 is the layer's identity mask on the selected nodes (only the diagonal weights of k = 0 are live)."""

    @staticmethod
    def forward(ctx, w, xA, pe, NA, k0_identity):
        lib = _cabi.load()
        F_, K, G, nnz = w.shape
        B = xA.shape[0]
        w = w.contiguous()
        xT = xA.permute(1, 2, 0).contiguous()                                   # [G, NA, B]
        train = ctx.needs_input_grad[0] or ctx.needs_input_grad[1]
        n_states = max(K - 1, 1) if train else min(max(K - 1, 1), 2)
        states = torch.empty((n_states, F_ * G, NA, B), dtype=w.dtype, device=w.device)
        Y = torch.empty((F_, NA, B), dtype=w.dtype, device=w.device)
        diag = pe["diag"].data_ptr() if k0_identity else None
        _cabi.check(lib.b200gf_ev_forward(_cabi.DTYPE[w.dtype], NA, B, G, F_, K, pe["rowptr"].data_ptr(),
                                          pe["col"].data_ptr(), diag, nnz, w.data_ptr(), xT.data_ptr(), states.data_ptr(),
                                          n_states, Y.data_ptr(), _cabi.stream()))
        ctx.pe, ctx.NA, ctx.k0 = pe, NA, k0_identity
        ctx.save_for_backward(w, xT, states)
        return Y.permute(2, 0, 1)                                               # [B, F, NA] view

    @staticmethod
    def backward(ctx, dy):
        lib = _cabi.load()
        w, xT, states = ctx.saved_tensors
        pe, NA = ctx.pe, ctx.NA
        F_, K, G, nnz = w.shape
        B = xT.shape[2]
        assert states.shape[0] >= K - 1, "forward ran without gradients enabled"
        dY = dy.permute(1, 2, 0).contiguous()                                   # [F, NA, B]
        lam = torch.empty((2, F_ * G, NA, B), dtype=w.dtype, device=w.device)
        dw = torch.zeros_like(w)
        dxT = torch.empty_like(xT)
        diag = pe["diag"].data_ptr() if ctx.k0 else None
        _cabi.check(lib.b200gf_ev_backward(_cabi.DTYPE[w.dtype], NA, B, G, F_, K, pe["rowptr"].data_ptr(),
                                           pe["col"].data_ptr(), pe["rowptrT"].data_ptr(), pe["colT"].data_ptr(),
                                           pe["perm"].data_ptr(), diag, nnz, w.data_ptr(), xT.data_ptr(),
                                           states.data_ptr(), dY.data_ptr(), lam.data_ptr(), dw.data_ptr(),
                                           dxT.data_ptr(), _cabi.stream()))
        return dw, dxT.permute(2, 0, 1), None, None, None


def _require_cuda(x):
    check_operands("EdgeVariantGF", x, ())


def _run_chain(w, xA, pe, NA, k0_identity=False):
    return _EVChain.apply(w, xA, pe, NA, k0_identity)


_chain = _run_chain      # the one hook the CPU tests replace (a dense torch chain) to exercise the layer logic


def _evgf_sparse(Phi, struct, x, b, k0_identity=False):
    F_, E, K, G, N, _ = Phi.shape
    B = x.shape[0]
    check_operands("EVGF", x, (Phi,))
    y = torch.zeros((B, F_, N), dtype=x.dtype, device=x.device)
    if struct.NA > 0:
        xA = x.index_select(2, struct.A)
        yA = None
        for e in range(E):
            pe = struct.per_e[e]
            if pe["nnz"] == 0:
                continue
            w = Phi[:, e].reshape(F_, K, G, N * N).index_select(3, pe["lin"])   # [F, K, G, nnz], differentiable gather
            ye = _chain(w, xA, pe, struct.NA, k0_identity)
            yA = ye if yA is None else yA + ye
        if yA is not None:
            y = y.index_add(2, struct.A, yA)
    if b is not None:
        y = y + b
    return y


def EVGF(S, x, b=None):
    """EVGF(filter_matrices, input, bias=None): same contract as alegnn/utils/graphML.py:389-488.
    S [F, E, K, G, N, N] dense filter matrices (zeros off the pattern), x [B, G, N], b [F, 1] / [F, N] / None."""
    F_, E, K, G, N = S.shape[0], S.shape[1], S.shape[2], S.shape[3], S.shape[4]
    assert S.shape[5] == N                       # graphML.py:441
    assert x.shape[1] == G                       # graphML.py:443
    assert x.shape[2] == N                       # graphML.py:444
    pattern = (S.detach() != 0).any(dim=0).any(dim=1).any(dim=1)                # [E, N, N]
    return _evgf_sparse(S, EVStructure(pattern), x, b)


class EdgeVariantGF(nn.Module):
    """EdgeVariantGF(in_features, out_features, shift_taps, selected_nodes, number_nodes, edge_features=1, bias=True)
    — same surface as the reference layer (graphML.py:2511-2712)."""

    def __init__(self, G, F, K, M, N, E=1, bias=True):
        super().__init__()
        self.G, self.F, self.K, self.E, self.M, self.N = G, F, K, E, M, N
        self.S = None
        self.weightEV = nn.parameter.Parameter(torch.Tensor(F, E, K, G, N, N))
        if self.M < self.N:
            self.weightLSI = nn.parameter.Parameter(torch.Tensor(F, E, K, G))
        else:
            self.register_parameter("weightLSI", None)
        if bias:
            self.bias = nn.parameter.Parameter(torch.Tensor(F, 1))
        else:
            self.register_parameter("bias", None)
        self.reset_parameters()

    def reset_parameters(self):
        stdv = 1. / math.sqrt(self.G * self.K * self.N)      # graphML.py:2601
        self.weightEV.data.uniform_(-stdv, stdv)
        if self.weightLSI is not None:
            self.weightLSI.data.uniform_(-stdv, stdv)
        if self.bias is not None:
            self.bias.data.uniform_(-stdv, stdv)

    def addGSO(self, S):
        assert len(S.shape) == 3
        assert S.shape[0] == self.E
        self.N = S.shape[1]
        assert S.shape[2] == self.N
        self.S = S
        N, M, E, K = self.N, self.M, self.E, self.K
        eye = torch.eye(N, device=S.device, dtype=S.dtype).reshape(1, N, N).repeat(E, 1, 1)
        pattern = (torch.abs(S) + eye) > zeroTolerance                          # graphML.py:2620
        idx = torch.arange(N, device=S.device)
        hybrid = (idx[:, None] < M) | (idx[None, :] < M) if M < N else torch.ones(N, N, dtype=torch.bool, device=S.device)
        pattern = pattern & hybrid[None]                                        # graphML.py:2624-2644
        self.sparsityPattern = pattern.to(S.dtype)
        ident = (eye > 0) & hybrid[None]
        if K > 1:                                                               # graphML.py:2653-2663: k = 0 is the identity
            full = torch.cat([ident.reshape(1, E, 1, 1, N, N),
                              pattern.reshape(1, E, 1, 1, N, N).repeat(1, 1, K - 1, 1, 1, 1)], dim=2)
        else:
            full = ident.reshape(1, E, 1, 1, N, N)
        self.sparsityPatternFull = full.to(S.dtype)
        self._struct = EVStructure(pattern | ident)

    def forward(self, x):
        B, Fin, Nin = x.shape
        self.Phi = self.weightEV * self.sparsityPatternFull                     # graphML.py:2676
        if Nin < self.N:
            x = torch.cat((x, torch.zeros(B, Fin, self.N - Nin, dtype=x.dtype, device=x.device)), dim=2)
        uEV = _evgf_sparse(self.Phi, self._struct, x, self.bias, k0_identity=True)   # k = 0 mask is the identity (:2653-2663)
        if self.M < self.N:
            uLSI = LSIGF(self.weightLSI, self.S, x, self.bias)                  # bias again, as the reference does (:2686)
        else:
            uLSI = torch.tensor(0., dtype=uEV.dtype, device=uEV.device)
        u = uEV + uLSI
        if Nin < self.N:
            u = u[:, :, :Nin]
        return u

    def extra_repr(self):
        s = "in_features=%d, out_features=%d, " % (self.G, self.F) + "shift_taps=%d, " % (self.K) + \
            "selected_nodes=%d, " % (self.M) + "number_nodes=%d, " % (self.N) + "edge_features=%d, " % (self.E) + \
            "bias=%s, " % (self.bias is not None)
        return s + ("GSO stored" if self.S is not None else "no GSO stored")


class SparseEdgeVariantGF(nn.Module):
    """EdgeVariantGF for graphs where the reference layer cannot exist (BASELINE.json config 4: N = 200k, E = 4).

    The reference allocates `weightEV [F, E, K, G, N, N]` (graphML.py:2586) — 32*4*3*32*4e10 numbers at N = 200k — and
    multiplies it by a 0/1 mask (:2620-2663, :2676).  Only the masked entries are parameters in any meaningful sense, so
    this layer stores exactly those: per edge feature e one tensor `weightEV.<e>` of shape [F, K, G, nnz_e] on the masked
    pattern of |S_e| + I restricted to entries touching the M selected nodes (i < M or j < M), in row-major pattern
    order.  The k = 0 taps live on the diagonal entries only (identity mask); their off-diagonal slots are kept at zero
    (zero-initialised, zero gradient).  Same forward as the reference layer — including its double bias in the hybrid case
    (:2682, :2686) — through the same kernels as gnn_b200.EdgeVariantGF; `load_dense_state(...)` imports a reference /
    dense checkpoint, `dense_weightEV()` exports one (small N only).

    addGSO accepts a SparseGSO or a dense [E, N, N] tensor and must be called before parameters exist (they depend on
    the pattern), i.e. before the optimiser is built — like the reference, where addGSO is part of construction."""

    def __init__(self, G, F, K, M, N, E=1, bias=True):
        super().__init__()
        self.G, self.F, self.K, self.E, self.M, self.N = G, F, K, E, M, N
        self.S = None
        self.weightEV = None
        if self.M < self.N:
            self.weightLSI = nn.parameter.Parameter(torch.Tensor(F, E, K, G))
        else:
            self.register_parameter("weightLSI", None)
        if bias:
            self.bias = nn.parameter.Parameter(torch.Tensor(F, 1))
        else:
            self.register_parameter("bias", None)
        self._struct = None

    def _masked_coords(self, S):
        """per e: (rows, cols) of the masked pattern (|S_e| + I > tol) & (i < M or j < M), row-major, as int64 tensors."""
        from .gso import SparseGSO
        import numpy as np
        M, N = self.M, self.N
        out = []
        if isinstance(S, SparseGSO):
            for (rowptr, col, val) in S.csr:
                rows = np.repeat(np.arange(N, dtype=np.int64), np.diff(rowptr))
                cols = col.astype(np.int64)
                keep = np.abs(val) > zeroTolerance
                rows, cols = rows[keep], cols[keep]
                d = np.arange(N, dtype=np.int64)                                   # + I
                rows, cols = np.concatenate((rows, d)), np.concatenate((cols, d))
                if M < N:
                    keep = (rows < M) | (cols < M)
                    rows, cols = rows[keep], cols[keep]
                lin = np.unique(rows * N + cols)                                   # sorted row-major, duplicates (diag) merged
                out.append((torch.from_numpy(lin // N), torch.from_numpy(lin % N)))
        else:
            eye = torch.eye(N, device=S.device, dtype=S.dtype)
            idx = torch.arange(N, device=S.device)
            hybrid = (idx[:, None] < M) | (idx[None, :] < M) if M < N else torch.ones(N, N, dtype=torch.bool, device=S.device)
            for e in range(S.shape[0]):
                z = (((torch.abs(S[e]) + eye) > zeroTolerance) & hybrid).nonzero(as_tuple=False)
                out.append((z[:, 0].cpu(), z[:, 1].cpu()))
        return out

    def addGSO(self, S, device=None):
        assert len(S.shape) == 3
        assert S.shape[0] == self.E
        self.N = S.shape[1]
        assert S.shape[2] == self.N
        self.S = S
        if device is None:
            device = S.device if isinstance(S, torch.Tensor) and S.device.type == "cuda" else \
                (self.bias.device if self.bias is not None else torch.device("cpu"))
        self._struct = EVStructure.from_coo(self.N, self._masked_coords(S), device)
        fresh = self.weightEV is None
        if fresh:
            dt = self.bias.dtype if self.bias is not None else torch.get_default_dtype()
            self.weightEV = nn.ParameterList([nn.parameter.Parameter(torch.zeros(self.F, self.K, self.G, pe["nnz"], dtype=dt,
                                                                                 device=device))
                                              for pe in self._struct.per_e])
            self.reset_parameters()
        else:
            for p, pe in zip(self.weightEV, self._struct.per_e):
                assert p.shape[3] == pe["nnz"], "the new GSO has a different masked pattern than the stored parameters"

    def _k0_mask(self, pe, like):
        m = torch.zeros(pe["nnz"], dtype=like.dtype, device=like.device)
        d = pe["diag"].to(like.device)
        m[d[d >= 0].long()] = 1
        return m

    def reset_parameters(self):
        stdv = 1. / math.sqrt(self.G * self.K * self.N)      # graphML.py:2601
        if self.weightEV is not None:
            for p, pe in zip(self.weightEV, self._struct.per_e):
                p.data.uniform_(-stdv, stdv)
                p.data[:, 0] *= self._k0_mask(pe, p.data)     # k = 0: identity mask, off-diagonal slots stay zero
        if self.weightLSI is not None:
            self.weightLSI.data.uniform_(-stdv, stdv)
        if self.bias is not None:
            self.bias.data.uniform_(-stdv, stdv)

    def load_dense_state(self, weightEV=None, weightLSI=None, bias=None):
        """Import a reference checkpoint (`weightEV [F, E, K, G, N, N]`, graphML.py:2586): keeps the masked entries."""
        with torch.no_grad():
            if weightEV is not None:
                F_, E, K, G, N, _ = weightEV.shape
                assert (F_, E, K, G, N) == (self.F, self.E, self.K, self.G, self.N)
                for e, (p, pe) in enumerate(zip(self.weightEV, self._struct.per_e)):
                    v = weightEV[:, e].reshape(F_, K, G, N * N).index_select(3, pe["lin"].to(weightEV.device)).to(p.device, p.dtype)
                    v[:, 0] *= self._k0_mask(pe, v)
                    p.copy_(v)
            if weightLSI is not None and self.weightLSI is not None:
                self.weightLSI.copy_(weightLSI)
            if bias is not None and self.bias is not None:
                self.bias.copy_(bias)

    def dense_weightEV(self):
        """Export to the reference's dense parameter shape (small N only)."""
        N = self.N
        out = torch.zeros(self.F, self.E, self.K, self.G, N * N, dtype=self.weightEV[0].dtype, device=self.weightEV[0].device)
        for e, (p, pe) in enumerate(zip(self.weightEV, self._struct.per_e)):
            out[:, e].index_copy_(3, pe["lin"].to(out.device), p.detach())
        return out.reshape(self.F, self.E, self.K, self.G, N, N)

    def forward(self, x):
        B, Fin, Nin = x.shape
        st = self._struct
        if Nin < self.N:
            x = torch.cat((x, torch.zeros(B, Fin, self.N - Nin, dtype=x.dtype, device=x.device)), dim=2)
        _require_cuda(x)
        if st.A.device != x.device:
            raise RuntimeError("b200gf: call addGSO(S, device=...) with the device the layer runs on")
        yA = None
        if st.NA > 0:
            xA = x.index_select(2, st.A)
            for e in range(self.E):
                pe = st.per_e[e]
                if pe["nnz"] == 0:
                    continue
                ye = _chain(self.weightEV[e], xA, pe, st.NA, True)
                yA = ye if yA is None else yA + ye
        if self.M < self.N:
            u = LSIGF(self.weightLSI, self.S, x, self.bias)                     # bias here ...
            if self.bias is not None:
                u = u + self.bias                                               # ... and in EVGF: the reference adds it twice
            if yA is not None:                                                  # add the EV part on the rows of A (node-major)
                unb = u.permute(2, 0, 1).index_add(0, st.A, yA.permute(2, 0, 1))
                u = unb.permute(1, 2, 0)
        else:
            u = torch.zeros((B, self.F, self.N), dtype=x.dtype, device=x.device)
            if yA is not None:
                u = u.index_add(2, st.A, yA)
            if self.bias is not None:
                u = u + self.bias
        if Nin < self.N:
            u = u[:, :, :Nin]
        return u

    def extra_repr(self):
        s = "in_features=%d, out_features=%d, " % (self.G, self.F) + "shift_taps=%d, " % (self.K) + \
            "selected_nodes=%d, " % (self.M) + "number_nodes=%d, " % (self.N) + "edge_features=%d, " % (self.E) + \
            "bias=%s, " % (self.bias is not None)
        return s + ("GSO stored, %d masked parameters per (f, k, g)" % sum(pe["nnz"] for pe in self._struct.per_e)
                    if self.S is not None else "no GSO stored")
