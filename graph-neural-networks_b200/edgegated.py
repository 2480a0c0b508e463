"""Edge-gated graph recurrent layer on sparse CUDA kernels (csrc/egate.cu).

    EdgeGatedGRNN(a, b, pattern, x, z0, sigma, q_hat, q_check, xBias, zBias)   <- GatedGRNN's edge path,
                                                         alegnn/utils/graphML.py:1410-1451 (input filter), :1474-1514
    EdgeGatedHiddenState(F, H, K, nonlinearity, E, bias)                       <- graphML.py:4033-4209

    z_t = sigma( A(S~hat_t) x_t + B(S~check_t) z_{t-1} ),   S~ = q (.) S,   t = 1..T

The reference's gates are dense attention GSOs, `learnAttentionGSO` (graphML.py:640-737) of [B*T, N, N], and every
gated hop multiplies the whole batch against every sample's GSO before keeping the diagonal (graphML.py:1425-1431,
:1492-1498): compute and memory quadratic in B*T and N.  Here a gate is one value per (sample, non-zero of the mask
|S + I| > 1e-9) and a hop reads each sample's own gate values (B*T*nnz_mask gate values, B*T*nnz*C multiply-adds per
hop):

  * `EdgeGatePattern` (built once in addGSO, on the device for a CUDA dense S, from the CSR for a SparseGSO) holds the
    mask CSR of S + I and its transpose, the CSRs of S^T (forward hop) and S (backward hop) with each entry's position
    in the mask (-1 outside it), and S's values in mask order (the gate gradient);
  * `_attention` / `_gated_hop` are the two differentiable kernels; the projection s = W z, the tap contraction and the
    element-wise recursion stay in torch, node-major as in recurrent.GatedGRNN;
  * gate storage keeps the sample index innermost: q_hat is [nnz, B, T] (the input filter reads all B*T samples with
    sample stride 1), q_check is [nnz, T, B] (step t reads the slab of its B samples with sample stride 1).  The
    functional takes both as [B, T, nnz] views of any strides.

Unlike time and node gating, no gate multiplies the filter outputs (graphML.py:1447, :1514).  Only E = 1 is reachable,
as in the reference (GraphAttentional.addGSO takes one edge feature, the gate is [B, T, 1, N, N]).
"""
import math

import numpy as np
import torch
import torch.nn as nn

from . import _cabi
from . import recurrent as _rec
from .graphML import check_operands
from .gso import SparseGSO

zeroTolerance = 1e-9   # graphML.py:72


def _rowptr(rows, N):
    rp = torch.zeros(N + 1, dtype=torch.int64, device=rows.device)
    rp[1:] = torch.cumsum(torch.bincount(rows, minlength=N), 0)
    return rp


class EdgeGatePattern:
    """Sparse structure of a GSO S [E, N, N] for the edge-gated layer (E = 1) and the graph attention layers (E >= 1).

    `EdgeGatePattern(S)`: S a dense [E, N, N] tensor (built on S's device) or a SparseGSO (built from its CSR on the
    host; never densified).  `on(device)` returns the pattern on another device (cached).  Members (int64 offsets,
    int32 indices):
      mask CSR, one for all edge features (graphML.py:692, :726-728): off the diagonal sum_e |S_e,ij| > 1e-9, on it
        sum_e |S_e,ii + 1| > 1e-9:  m_rowptr, m_col (ascending), m_row; nnz = its size
      its transpose:  mT_rowptr, mT_perm (position in the mask of the k-th entry of column j)
      CSR of S^T:     t_rowptr, t_col (= i), t_val (= S_ij), t_pos (= p(i, j) in the mask, -1 outside it)
      CSR of S:       s_rowptr, s_col (= j), s_val, s_pos
      m_sval:         S_ij in mask order (0 where S has no entry, e.g. the diagonal added by + I).
    The t_*, s_* and m_sval members are those of edge feature 0; `edges[e]` is a pattern holding edge feature e's (it
    shares the mask members; edges[0] is the pattern itself).  `unit()` is the mask itself with unit values (the hop by
    alpha alone of GraphFilterAttentional)."""

    def __init__(self, S=None):
        self._devices = {}
        self._vals = {}
        self._unit = None
        if S is None:
            return
        assert len(S.shape) == 3
        E, N = int(S.shape[0]), int(S.shape[1])
        entries = []
        for e in range(E):
            if isinstance(S, SparseGSO):
                rowptr, col, val = S.csr[e]
                rows = torch.from_numpy(np.repeat(np.arange(N, dtype=np.int64), np.diff(rowptr)))
                cols = torch.from_numpy(col.astype(np.int64))
                vals = torch.from_numpy(np.ascontiguousarray(val))
                keep = vals != 0
                rows, cols, vals = rows[keep], cols[keep], vals[keep]
            else:
                nz = (S[e] != 0).nonzero(as_tuple=False)            # row-major
                rows, cols = nz[:, 0], nz[:, 1]
                vals = S[e][rows, cols]
            entries.append((rows, cols, vals.detach()))
        self._build(N, entries)

    def _build(self, N, entries):
        rows, cols, vals = entries[0]
        dev = rows.device
        E = len(entries)
        self.N = N
        self.E = E
        self.dtype = vals.dtype
        # mask: off-diagonal entries with sum_e |S_e,ij| > tol, the diagonal where sum_e |S_e,ii + 1| > tol (so S_ii = -1
        # drops out when E = 1).  The sums run over a dense [E, .] stack in e order, as the reference's sum over dim 0.
        idx = torch.arange(N, device=dev)
        diag = torch.zeros((E, N), dtype=vals.dtype, device=dev)
        off_keys = []
        for e, (r, c, v) in enumerate(entries):
            on = r == c
            diag[e, r[on]] = v[on]
            off_keys.append(r[~on] * N + c[~on])
        uk, inv = torch.unique(torch.cat(off_keys), sorted=True, return_inverse=True)
        absum = torch.zeros((E, uk.numel()), dtype=vals.dtype, device=dev)
        o = 0
        for e, (r, c, v) in enumerate(entries):
            off = r != c
            n = int(off.sum())
            absum[e, inv[o:o + n]] = v[off].abs()
            o += n
        okeep = absum.sum(0) > zeroTolerance
        dkeep = (diag + 1).abs().sum(0) > zeroTolerance
        m_key, _ = torch.sort(torch.cat((uk[okeep], idx[dkeep] * (N + 1))))
        m_row, m_col = m_key // N, m_key % N
        nnz = int(m_key.numel())
        self.nnz = nnz
        self.m_rowptr = _rowptr(m_row, N)
        self.m_col = m_col.to(torch.int32)
        self.m_row = m_row
        permT = torch.argsort(m_col * N + m_row)
        self.mT_rowptr = _rowptr(m_col, N)
        self.mT_perm = permT.to(torch.int32)
        self.edges = [self]
        for e, (r, c, v) in enumerate(entries):
            (self if e == 0 else self._child())._set_edge(N, m_key, r, c, v)
        self.device = torch.device(dev)
        self._devices[str(self.device)] = self

    def _set_edge(self, N, m_key, rows, cols, vals):
        """The members of one edge feature: each S_e entry's position in the mask, the CSRs of S_e and S_e^T."""
        dev, nnz = rows.device, self.nnz
        key = rows * N + cols
        if nnz > 0:
            pos = torch.searchsorted(m_key, key)
            hit = m_key[pos.clamp(max=nnz - 1)] == key
            pos = torch.where(hit, pos, torch.full_like(pos, -1))
        else:
            hit = torch.zeros_like(key, dtype=torch.bool)
            pos = torch.full_like(key, -1)
        m_sval = torch.zeros(nnz, dtype=vals.dtype, device=dev)
        m_sval[pos[hit]] = vals[hit]
        self.m_sval = m_sval
        o = torch.argsort(key)
        self.s_rowptr = _rowptr(rows[o], N)
        self.s_col = cols[o].to(torch.int32)
        self.s_val = vals[o]
        self.s_pos = pos[o].to(torch.int32)
        oT = torch.argsort(cols * N + rows)
        self.t_rowptr = _rowptr(cols[oT], N)
        self.t_col = rows[oT].to(torch.int32)
        self.t_val = vals[oT]
        self.t_pos = pos[oT].to(torch.int32)

    @property
    def shape(self):
        """(E, N, N), as the GSO's: the attention functionals take a pattern where the reference takes S."""
        return (self.E, self.N, self.N)

    _MASK = ("m_rowptr", "m_col", "m_row", "mT_rowptr", "mT_perm")
    _TENSORS = ("m_rowptr", "m_col", "m_row", "mT_rowptr", "mT_perm", "m_sval", "s_rowptr", "s_col", "s_val", "s_pos",
                "t_rowptr", "t_col", "t_val", "t_pos")

    def _child(self):
        """An empty pattern sharing this one's mask (to receive another edge feature's members)."""
        c = EdgeGatePattern()
        c.N, c.E, c.nnz, c.dtype = self.N, 1, self.nnz, self.dtype
        c.device = getattr(self, "device", None)
        for name in self._MASK:
            setattr(c, name, getattr(self, name))
        c.edges = [c]
        self.edges.append(c)
        return c

    def on(self, device):
        device = torch.device(device)
        if device.type == "cuda" and device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        hit = self._devices.get(str(device))
        if hit is None:
            hit = EdgeGatePattern()
            hit.N, hit.E, hit.nnz, hit.dtype, hit.device = self.N, self.E, self.nnz, self.dtype, device
            for name in self._TENSORS:
                setattr(hit, name, getattr(self, name).to(device))
            hit.edges = [hit]
            for src in self.edges[1:]:
                c = hit._child()
                for name in self._TENSORS[len(self._MASK):]:
                    setattr(c, name, getattr(src, name).to(device))
            hit._devices = self._devices
            self._devices[str(device)] = hit
        return hit

    def unit(self):
        """The mask as a hop operator with unit values (cached): the CSR of its transpose for the forward hop, the mask
        CSR for the backward one, every entry at its own mask position."""
        if self._unit is None:
            u = EdgeGatePattern()
            u.N, u.E, u.nnz, u.dtype, u.device = self.N, 1, self.nnz, self.dtype, self.device
            for name in self._MASK:
                setattr(u, name, getattr(self, name))
            ones = torch.ones(self.nnz, dtype=self.dtype, device=self.m_col.device)
            u.m_sval = ones
            u.s_rowptr, u.s_col, u.s_val = self.m_rowptr, self.m_col, ones
            u.s_pos = torch.arange(self.nnz, dtype=torch.int32, device=self.m_col.device)
            u.t_rowptr, u.t_col, u.t_val = self.mT_rowptr, self.m_row[self.mT_perm.long()].to(torch.int32), ones
            u.t_pos = self.mT_perm
            u.edges = [u]
            self._unit = u
        return self._unit

    def values(self, dtype):
        """(t_val, s_val, m_sval) in the compute dtype (cached)."""
        hit = self._vals.get(dtype)
        if hit is None:
            hit = tuple(v.to(dtype) for v in (self.t_val, self.s_val, self.m_sval))
            self._vals[dtype] = hit
        return hit


class _Attention(torch.autograd.Function):
    """alpha [nnz, Bs] = sparse learnAttentionGSO (graphML.py:640-737, P = E = F = 1) of s [N, Bs] (node-major)."""

    @staticmethod
    def forward(ctx, s, mixer, pat):
        check_operands("the edge-gate attention", s, ())
        lib = _cabi.load()
        s = s.contiguous()
        mixer = mixer.reshape(2).to(s.dtype).contiguous()
        N, Bs = s.shape
        alpha = torch.empty((pat.nnz, Bs), dtype=s.dtype, device=s.device)
        _cabi.check(lib.b200gf_egate_attention_forward(_cabi.DTYPE[s.dtype], N, pat.nnz, Bs, pat.m_rowptr.data_ptr(),
                                                       pat.m_col.data_ptr(), s.data_ptr(), mixer.data_ptr(),
                                                       alpha.data_ptr(), _cabi.stream()))
        ctx.pat = pat
        ctx.save_for_backward(s, mixer, alpha)
        return alpha

    @staticmethod
    def backward(ctx, dalpha):
        lib = _cabi.load()
        s, mixer, alpha = ctx.saved_tensors
        pat = ctx.pat
        N, Bs = s.shape
        dalpha = dalpha.contiguous()
        dlogit = torch.empty_like(alpha)
        dsig1 = torch.empty_like(s)
        dsig2 = torch.empty_like(s)
        _cabi.check(lib.b200gf_egate_attention_backward(_cabi.DTYPE[s.dtype], N, pat.nnz, Bs, pat.m_rowptr.data_ptr(),
                                                        pat.m_col.data_ptr(), pat.mT_rowptr.data_ptr(),
                                                        pat.mT_perm.data_ptr(), s.data_ptr(), mixer.data_ptr(),
                                                        alpha.data_ptr(), dalpha.data_ptr(), dlogit.data_ptr(),
                                                        dsig1.data_ptr(), dsig2.data_ptr(), _cabi.stream()))
        ds = mixer[0] * dsig1 + mixer[1] * dsig2
        dmixer = torch.stack(((s * dsig1).sum(), (s * dsig2).sum()))
        return ds, dmixer, None


def _row_ld(u):
    """Leading dimension of node-major u [N, Bs, C].  With N = 1 torch may report any row stride (a permuted [B, H, 1]
    tensor is already "contiguous" with stride 1); only row 0 is read, so Bs*C is as good as any and the entry points
    require ld >= Bs*C."""
    return u.stride(0) if u.shape[0] > 1 else u.shape[1] * u.shape[2]


def _gate_ptr(gate, u, pat):
    """The gate's address.  With an empty mask every S entry lies outside it (pos = -1), so the kernels read no gate,
    but the empty gate tensor has a null address, which the entry points reject: hand them u's instead."""
    return gate.data_ptr() if pat.nnz > 0 else u.data_ptr()


class _GatedHop(torch.autograd.Function):
    """u [N, Bs, C] (node-major) -> (u S~_b) per sample b, S~_b = gate[b] (.) S;  gate [Bs, nnz] of any strides."""

    @staticmethod
    def forward(ctx, u, gate, pat):
        check_operands("the edge-gated hop", u, ())
        lib = _cabi.load()
        N, Bs, C = u.shape
        if u.stride(2) != 1 or u.stride(1) != C:
            u = u.contiguous()
        out = torch.empty((N, Bs, C), dtype=u.dtype, device=u.device)
        t_val, _, _ = pat.values(u.dtype)
        _cabi.check(lib.b200gf_gated_hop_forward(_cabi.DTYPE[u.dtype], N, Bs, C, pat.t_rowptr.data_ptr(),
                                                 pat.t_col.data_ptr(), t_val.data_ptr(), pat.t_pos.data_ptr(),
                                                 _gate_ptr(gate, u, pat), gate.stride(0), gate.stride(1), u.data_ptr(),
                                                 _row_ld(u), out.data_ptr(), Bs * C, _cabi.stream()))
        ctx.pat = pat
        ctx.save_for_backward(u, gate)
        return out

    @staticmethod
    def backward(ctx, dout):
        lib = _cabi.load()
        u, gate = ctx.saved_tensors
        pat = ctx.pat
        N, Bs, C = u.shape
        dout = dout.contiguous()
        du = torch.empty_like(dout) if ctx.needs_input_grad[0] else None
        dg = torch.empty((pat.nnz, Bs), dtype=u.dtype, device=u.device) if ctx.needs_input_grad[1] else None
        if du is None and (dg is None or pat.nnz == 0):          # nothing to write (an empty mask has no gate)
            return None, None if dg is None else dg.t(), None
        _, s_val, m_sval = pat.values(u.dtype)
        _cabi.check(lib.b200gf_gated_hop_backward(
            _cabi.DTYPE[u.dtype], N, Bs, C, pat.s_rowptr.data_ptr(), pat.s_col.data_ptr(), s_val.data_ptr(),
            pat.s_pos.data_ptr(), pat.m_rowptr.data_ptr(), pat.m_col.data_ptr(), m_sval.data_ptr(),
            _gate_ptr(gate, u, pat), gate.stride(0), gate.stride(1), u.data_ptr(), _row_ld(u), dout.data_ptr(), Bs * C,
            None if du is None else du.data_ptr(), Bs * C, None if dg is None or pat.nnz == 0 else dg.data_ptr(), 1, Bs,
            _cabi.stream()))
        return du, None if dg is None else dg.t(), None


def _run_attention(s, mixer, pat):
    return _Attention.apply(s, mixer, pat)


def _run_gated_hop(u, gate, pat):
    return _GatedHop.apply(u, gate, pat)


# the two hooks the CPU tests replace with torch restatements to check the host logic without a GPU
_attention = _run_attention
_gated_hop = _run_gated_hop


def _filter(taps, u, gate, pat, bias):
    """sum_k taps[:, 0, k, :] applied to u S~^k (k = 0 unshifted), node-major: u [N, Bs, C] -> [N, Bs, H]."""
    H, _, K, C = taps.shape
    us = [u]
    for _ in range(1, K):
        u = _gated_hop(u, gate, pat)
        us.append(u)
    N, Bs = u.shape[0], u.shape[1]
    # contraction order (e, k, c) of graphML.py:1442-1443 / :1509-1510, E = 1
    y = torch.matmul(torch.stack(us, dim=2).reshape(N, Bs, K * C), taps.reshape(H, K * C).t())
    if bias is not None:
        y = y + bias.reshape(H)
    return y


def EdgeGatedGRNN(a, b, pattern, x, z0, sigma, q_hat, q_check, xBias=None, zBias=None):
    """Edge path of GatedGRNN (graphML.py:1292-1527 with 5-D gates) on per-non-zero gates.

    a [H, 1, K, F]; b [H, 1, K, H]; pattern: EdgeGatePattern of S; x [B, T, F, N]; z0 [B, H, N];
    q_hat, q_check [B, T, nnz] (any strides; pattern.nnz = size of the mask of S + I, in its CSR order): the reference's
    dense gates restricted to the mask, q_hat[b, t] gates the input filter of (b, t), q_check[:, t] the hidden filter
    that produces z_{t+1}.  xBias, zBias: H elements or None.  Returns z [B, T, H, N]."""
    H, E, K, F = a.shape
    assert E == 1, "edge gating runs on one edge feature (graphML.py:4190-4197)"
    assert tuple(b.shape) == (H, E, K, H)
    B, T = x.shape[0], x.shape[1]
    N = x.shape[3]
    assert x.shape[2] == F and N == pattern.N
    assert tuple(z0.shape) == (B, H, N)
    nnz = pattern.nnz
    assert tuple(q_hat.shape) == (B, T, nnz) and tuple(q_check.shape) == (B, T, nnz)
    pat = pattern.on(x.device)

    # A(S~hat) x for all B*T samples at once (graphML.py:1410-1451), node-major [N, B*T, F] -> [N, B, T, H]
    qh = q_hat.reshape(B * T, nnz)
    u = x.permute(3, 0, 1, 2).reshape(N, B * T, F)
    Ax = _filter(a, u, qh, pat, xBias).reshape(N, B, T, H)
    Ax_t = Ax.unbind(2)
    qc = q_check.unbind(1)                                              # T x [B, nnz]
    zt = z0.permute(2, 0, 1)                                            # [N, B, H]
    states = []
    for t in range(T):
        Bz = _filter(b, zt, qc[t], pat, zBias)                         # B(S~check_t) z_{t-1} (graphML.py:1474-1514)
        zt = sigma(Ax_t[t] + Bz).contiguous()                           # no gate multiplies the filter outputs
        states.append(zt)
    z = torch.stack(states, dim=2)                                      # [N, B, T, H]
    return z.permute(1, 2, 3, 0)


class GraphAttentionalGate(nn.Module):
    """The parameters of the reference's gate attention, GraphAttentional(H, 1, 1) (graphML.py:2898-2933): mixer
    [1, 1, 2], weight [1, 1, 1, H], initialised in the same order (weight, then mixer).  Only learnAttentionGSO
    (graphML.py:640-737) reads them; the attention itself runs in EdgeGatedHiddenState."""

    def __init__(self, G, F=1, K=1, E=1):
        super().__init__()
        assert F == 1 and K == 1 and E == 1
        self.G, self.F, self.K, self.E = G, F, K, E
        self.S = None
        self.mixer = nn.parameter.Parameter(torch.Tensor(K, E, 2 * F))
        self.weight = nn.parameter.Parameter(torch.Tensor(K, E, F, G))
        self.reset_parameters()

    def reset_parameters(self):
        stdv = 1. / math.sqrt(self.G * self.K)      # graphML.py:2920-2924
        self.weight.data.uniform_(-stdv, stdv)
        self.mixer.data.uniform_(-stdv, stdv)

    def addGSO(self, S):
        assert len(S.shape) == 3
        assert S.shape[0] == self.E
        self.N = S.shape[1]
        assert S.shape[2] == self.N
        self.S = S


class EdgeGatedHiddenState(_rec._GatedHiddenState):
    """EdgeGatedHiddenState(signal_features, hidden_features, filter_taps, nonlinearity=torch.tanh, edge_features=1,
    bias=True) — same surface, parameters and state_dict keys as graphML.py:4033-4209: aWeights [H,E,K,F],
    bWeights [H,E,K,H], xBias/zBias [H,1], inputGateGRNN / forgetGateGRNN (HiddenState, tanh), and the gate attentions
    inputGateGAT / forgetGateGAT created afresh in every addGSO (mixer [1,1,2], weight [1,1,1,H]).
    forward(x [B,T,F,N], z0 [B,H,N]) -> (z [B,T,H,N], z_T [B,1,1,H,N])."""

    def _make_gate_maps(self):
        dev = self.aWeights.device
        self.inputGateGAT = GraphAttentionalGate(self.H, 1, 1).to(dev)      # graphML.py:4190-4191
        self.forgetGateGAT = GraphAttentionalGate(self.H, 1, 1).to(dev)
        self.inputGateGAT.addGSO(self.S)
        self.forgetGateGAT.addGSO(self.S)
        self.pattern = EdgeGatePattern(self.S)

    def _gate(self, zg, gat, order):
        """Sparse learnAttentionGSO of the gate trajectory zg [B, T, H, N]: gate storage [nnz, B, T] ("bt") or
        [nnz, T, B] ("tb"), returned as a [B, T, nnz] view."""
        B, T, H, N = zg.shape
        w = gat.weight.reshape(H)
        if order == "bt":
            s = torch.matmul(zg.permute(3, 0, 1, 2), w).reshape(N, B * T)
            return _attention(s, gat.mixer.reshape(2), self._pat).view(-1, B, T).permute(1, 2, 0)
        s = torch.matmul(zg.permute(3, 1, 0, 2), w).reshape(N, T * B)
        return _attention(s, gat.mixer.reshape(2), self._pat).view(-1, T, B).permute(2, 1, 0)

    def forward(self, x, z0):
        assert self.S is not None
        assert len(x.shape) == 4
        B = x.shape[0]
        T = x.shape[1]
        assert x.shape[2] == self.F
        N = x.shape[3]
        assert len(z0.shape) == 3
        assert z0.shape[0] == B
        assert z0.shape[1] == self.H
        assert z0.shape[2] == N
        self._pat = self.pattern.on(x.device)
        zHat, _ = self.inputGateGRNN(x, z0)                                 # graphML.py:4157-4161
        qHat = self._gate(zHat, self.inputGateGAT, "bt")
        zCheck, _ = self.forgetGateGRNN(x, z0)                              # graphML.py:4164-4168
        qCheck = self._gate(zCheck, self.forgetGateGAT, "tb")
        z = EdgeGatedGRNN(self.aWeights, self.bWeights, self._pat, x, z0, self.sigma, qHat, qCheck,
                          xBias=self.xBias, zBias=self.zBias)
        zT = z[:, T - 1:T]
        return z, zT.unsqueeze(1)
