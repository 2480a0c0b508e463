"""Graph attention layers on sparse CUDA kernels (csrc/egate.cu).

    graphAttention(x, a, W, S)                       <- alegnn/utils/graphML.py:739-809
    graphAttentionLSIGF(h, x, a, W, S, b)            <- graphML.py:811-895
    graphAttentionEVGF(x, a, W, S, b)                <- graphML.py:897-969
    GraphAttentional(G, F, K, E, nonlinearity, concatenate)                 <- graphML.py:2849-2977
    GraphFilterAttentional(G, F, K, P, E, bias, nonlinearity, concatenate)  <- graphML.py:2979-3124
    EdgeVariantAttentional(G, F, K, P, E, bias, nonlinearity, concatenate)  <- graphML.py:3126-3270

The reference builds every attention as a dense B x P x E x N x N tensor (learnAttentionGSO, graphML.py:640-737) and
hops with dense N x N matmuls.  Everything it needs lives on the mask of S + I (one mask for all edge features,
sum_e |S_e + I| > 1e-9), so here an attention is one value per (sample, mask entry) and a hop touches the non-zeros:

  * `EdgeGatePattern` (edgegated.py, built once in addGSO) holds the mask CSR, and per edge feature e the CSRs of S_e
    and S_e^T positioned in the mask; `unit()` is the mask with unit values, the operator of GraphFilterAttentional's
    hops by alpha alone;
  * `_attention(s_src, s_dst, pat)`: alpha [nnz, Bs] = softmax over the mask row i of LeakyReLU_0.2(s_src[j] + s_dst[i]),
    s_src = a1^T W x (the column node j), s_dst = a2^T W x (the row node i), the egate softmax kernels with two score
    arrays; every (edge feature, batch, head[, tap]) sample goes through one launch;
  * `_gated_hop(u, gate, pat)`: u [N, Bs, C] -> u (S (.) alpha) per sample, edgegated's gated hop;
  * projections W x, the scores (a^T W) x and the tap contractions stay in torch.

Signals are node-major with the sample index innermost.  W x is computed as [E, N, B, P, F] (one matmul), so each edge
feature's slab [N, B*P, F] is a contiguous hop operand.  There is no CPU fallback: the kernels take CUDA tensors in
float32 / float64 and raise on anything else.  No host synchronisation and no data-dependent allocation happens in the
forward or backward, so both can be captured in a CUDA graph (graphed.py).
"""
import math
import weakref

import torch
import torch.nn as nn

from . import _cabi
from . import edgegated as _eg
from .edgegated import EdgeGatePattern
from .graphML import check_operands
from .gso import SparseGSO, _dense_key


class _Attention(torch.autograd.Function):
    """alpha [nnz, Bs] = sparse learnAttentionGSO (graphML.py:640-737) of the two score arrays s_src, s_dst [N, Bs]."""

    @staticmethod
    def forward(ctx, s_src, s_dst, pat):
        check_operands("the graph attention", s_src, ())
        lib = _cabi.load()
        s_src, s_dst = s_src.contiguous(), s_dst.contiguous()
        N, Bs = s_src.shape
        mixer = _unit_mixer(s_src.device, s_src.dtype)
        alpha = torch.empty((pat.nnz, Bs), dtype=s_src.dtype, device=s_src.device)
        _cabi.check(lib.b200gf_attention_forward(_cabi.DTYPE[s_src.dtype], N, pat.nnz, Bs, pat.m_rowptr.data_ptr(),
                                                 pat.m_col.data_ptr(), s_src.data_ptr(), s_dst.data_ptr(),
                                                 mixer.data_ptr(), alpha.data_ptr(), _cabi.stream()))
        ctx.pat = pat
        ctx.save_for_backward(s_src, s_dst, alpha)
        return alpha

    @staticmethod
    def backward(ctx, dalpha):
        lib = _cabi.load()
        s_src, s_dst, alpha = ctx.saved_tensors
        pat = ctx.pat
        N, Bs = s_src.shape
        dalpha = dalpha.contiguous()
        dlogit = torch.empty_like(alpha)
        dsig1 = torch.empty_like(s_src)
        dsig2 = torch.empty_like(s_src)
        mixer = _unit_mixer(s_src.device, s_src.dtype)
        _cabi.check(lib.b200gf_attention_backward(_cabi.DTYPE[s_src.dtype], N, pat.nnz, Bs, pat.m_rowptr.data_ptr(),
                                                  pat.m_col.data_ptr(), pat.mT_rowptr.data_ptr(),
                                                  pat.mT_perm.data_ptr(), s_src.data_ptr(), s_dst.data_ptr(),
                                                  mixer.data_ptr(), alpha.data_ptr(), dalpha.data_ptr(),
                                                  dlogit.data_ptr(), dsig1.data_ptr(), dsig2.data_ptr(), _cabi.stream()))
        return dsig1, dsig2, None


_MIXERS = {}


def _unit_mixer(device, dtype):
    """The device mixer (1, 1): the logit is s_src[j] + s_dst[i], as the reference's a1Wx + a2Wx^T (graphML.py:712).
    Cached, so that a captured graph allocates nothing for it."""
    key = (str(device), dtype)
    hit = _MIXERS.get(key)
    if hit is None:
        hit = torch.ones(2, dtype=dtype, device=device)
        _MIXERS[key] = hit
    return hit


def _run_attention(s_src, s_dst, pat):
    return _Attention.apply(s_src, s_dst, pat)


# the two hooks the CPU tests replace with torch restatements to check the host logic without a GPU
_attention = _run_attention
_gated_hop = _eg._run_gated_hop


# ---------------------------------------------------------------------------------------------------
# the GSO's sparse structure, built once per GSO
# ---------------------------------------------------------------------------------------------------
_PATTERNS = {}
_PATTERNS_MAX = 16


def pattern_for(S, device):
    """The EdgeGatePattern of S (dense [E, N, N] tensor, SparseGSO or EdgeGatePattern) on `device`.  Cached per dense
    tensor and version (as gso.plan_for caches plans) or on the SparseGSO object."""
    if isinstance(S, EdgeGatePattern):
        return S.on(device)
    if isinstance(S, SparseGSO):
        hit = getattr(S, "_attention_pattern", None)
        if hit is None:
            hit = EdgeGatePattern(S)
            S._attention_pattern = hit
        return hit.on(device)
    if not isinstance(S, torch.Tensor):
        raise TypeError("b200gf: GSO must be a torch.Tensor [E,N,N], SparseGSO or EdgeGatePattern, got %r" % type(S))
    for k in [k for k, v in _PATTERNS.items() if v[0]() is None]:
        del _PATTERNS[k]
    key = _dense_key(S)
    hit = _PATTERNS.get(key)
    if hit is None or hit[0]() is not S:
        if len(_PATTERNS) >= _PATTERNS_MAX:
            _PATTERNS.pop(next(iter(_PATTERNS)))
        hit = (weakref.ref(S), EdgeGatePattern(S.detach()))
        _PATTERNS[key] = hit
    return hit[1].on(device)


def _check_slope(negative_slope):
    if negative_slope != 0.2:
        raise NotImplementedError("b200gf: the attention kernels use the reference's LeakyReLU slope 0.2, got %r"
                                  % (negative_slope,))


def _project(x, W):
    """W x for every (edge feature, head): x [B, G, N], W [P, E, F, G] -> [E, N, B, P, F] (contiguous, one matmul)."""
    B, G, N = x.shape
    P, E, F, _ = W.shape
    xn = x.permute(2, 0, 1).reshape(1, N * B, G)                          # node-major [N, B, G]
    Wt = W.permute(1, 3, 0, 2).reshape(E, G, P * F)
    return torch.matmul(xn, Wt).view(E, N, B, P, F)


def _scores(x, W, a):
    """(s_src, s_dst) [N, E*B*P] (sample index (e, b, p) innermost) of x [B, G, N], W [P, E, F, G], a [P, E, 2F]:
    s_src = a1^T W x, s_dst = a2^T W x (graphML.py:706-709), computed as (a^T W) x: one [N*B, G] x [G, 2*E*P] matmul
    instead of a reduction over W x."""
    B, G, N = x.shape
    P, E, F, _ = W.shape
    V = torch.einsum("pejf,pefg->gejp", a.reshape(P, E, 2, F), W).reshape(G, E * 2 * P)
    s = torch.matmul(x.permute(2, 0, 1).reshape(N * B, G), V).view(N, B, E, 2, P)
    s = s.permute(3, 0, 2, 1, 4).reshape(2, N, E * B * P)
    return s[0], s[1]


def _gate(alpha, k, n):
    """Samples [k*n, (k+1)*n) of alpha [nnz, Bs] as a [n, nnz] gate view (sample stride 1)."""
    return alpha[:, k * n:(k + 1) * n].t()


def _add_bias(y, b):
    return y if b is None else y + b


def graphAttention(x, a, W, S, negative_slope=0.2):
    """graphAttention(x, a, W, S) (graphML.py:739-809): x [B, G, N], a [P, E, 2F], W [P, E, F, G], S [E, N, N] (dense
    tensor, SparseGSO or EdgeGatePattern) -> y [B, P, F, N],  y[b, p] = sum_e (W_pe x)(S_e (.) alpha_bpe)."""
    B, G, N = x.shape
    P, E = a.shape[0], a.shape[1]
    assert W.shape[0] == P and W.shape[1] == E
    F = W.shape[2]
    assert a.shape[2] == int(2 * F)
    assert W.shape[3] == G
    assert S.shape[0] == E and S.shape[1] == S.shape[2] == N
    _check_slope(negative_slope)
    pat = pattern_for(S, x.device)
    Wx = _project(x, W)
    alpha = _attention(*_scores(x, W, a), pat)                            # [nnz, E*B*P]
    BP = B * P
    y = None
    for e in range(E):
        ye = _gated_hop(Wx[e].view(N, BP, F), _gate(alpha, e, BP), pat.edges[e])
        y = ye if y is None else y + ye
    return y.view(N, B, P, F).permute(1, 2, 3, 0)


def graphAttentionLSIGF(h, x, a, W, S, b=None, negative_slope=0.2):
    """graphAttentionLSIGF(h, x, a, W, S, b) (graphML.py:811-895): h [E, K], x [B, G, N], a [P, E, 2F],
    W [P, E, F, G], S [E, N, N] -> y [B, P, F, N]: an LSIGF whose k-th hop is by alpha_bpe alone (the mask with unit
    values, diagonal included), taps h[e, k] * W permuted as the reference does, then b."""
    E, K = h.shape
    B, G, N = x.shape
    P = a.shape[0]
    assert a.shape[1] == E and W.shape[0] == P and W.shape[1] == E
    F = W.shape[2]
    assert W.shape[3] == G and a.shape[2] == int(2 * F)
    assert S.shape[0] == E and S.shape[1] == S.shape[2] == N
    _check_slope(negative_slope)
    pat = pattern_for(S, x.device)
    alpha = _attention(*_scores(x, W, a), pat)                            # [nnz, E*B*P]
    # the taps exactly as graphML.py:861-864: a reshape of the permuted W, not its transpose
    taps = h.reshape([1, 1, E, K, 1]) * W.permute(0, 3, 1, 2).reshape([P, F, E, 1, G])   # [P, F, E, K, G]
    EBP = E * B * P
    u = x.permute(2, 0, 1).reshape(N, 1, B, 1, G).expand(N, E, B, P, G).reshape(N, EBP, G)
    us = [u]
    unit = pat.unit()
    for _ in range(1, K):
        u = _gated_hop(u, alpha.t(), unit)
        us.append(u)
    z = torch.stack(us, 0).view(K, N, E, B, P, G)
    y = torch.einsum("knebpg,pfekg->nbpf", z, taps)                       # contraction over (e, k, g) per head
    return _add_bias(y.permute(1, 2, 3, 0), b)


def graphAttentionEVGF(x, a, W, S, b=None, negative_slope=0.2):
    """graphAttentionEVGF(x, a, W, S, b) (graphML.py:897-969): x [B, G, N], a [P, K, E, 2F], W [P, K, E, F, G],
    S [E, N, N] -> y [B, P, F, N] = sum_e sum_{k=1..K} W_0 x (S_e (.) alpha_1) ... (S_e (.) alpha_k) + b, alpha_k scored
    with (W[:, k], a[:, k])."""
    B, G, N = x.shape
    P, K, E = a.shape[0], a.shape[1], a.shape[2]
    assert W.shape[0] == P and W.shape[1] == K and W.shape[2] == E
    F = W.shape[3]
    assert W.shape[4] == G and a.shape[3] == int(2 * F)
    assert S.shape[0] == E and S.shape[1] == S.shape[2] == N
    _check_slope(negative_slope)
    pat = pattern_for(S, x.device)
    # tap k's scores from its own (W[:, k], a[:, k]); only tap 0's projection is hopped
    Wx = _project(x, W[:, 0])                                             # [E, N, B, P, F]
    s_src, s_dst = _scores(x, W.reshape(P, K * E, F, G), a.reshape(P, K * E, 2 * F))
    alpha = _attention(s_src, s_dst, pat)                                 # [nnz, K*E*B*P], sample (k, e, b, p)
    BP = B * P
    y = None
    for e in range(E):
        u = Wx[e].view(N, BP, F)
        for k in range(K):
            u = _gated_hop(u, _gate(alpha, k * E + e, BP), pat.edges[e])
            y = u if y is None else y + u
    return _add_bias(y.view(N, B, P, F).permute(1, 2, 3, 0), b)


# ---------------------------------------------------------------------------------------------------
# layers: the reference's surface, parameters, initialisation order and state_dict keys
# ---------------------------------------------------------------------------------------------------
class _AttentionLayer(nn.Module):
    heads = "K"                                   # the attribute holding the number of heads

    def addGSO(self, S):
        """S [E, N, N]: a dense tensor or a SparseGSO.  The sparse structure is built here once (on S's device for a
        CUDA tensor, from the CSR for a SparseGSO); a dense S still on the CPU gets it on first use."""
        assert len(S.shape) == 3
        assert S.shape[0] == self.E
        self.N = S.shape[1]
        assert S.shape[2] == self.N
        self.S = S
        self.pattern = None
        if isinstance(S, SparseGSO) or (isinstance(S, torch.Tensor) and S.device.type == "cuda"):
            self.pattern = pattern_for(S, S.device if isinstance(S, torch.Tensor) else torch.device("cpu"))

    def _gso(self, device):
        if self.pattern is None:
            self.pattern = pattern_for(self.S, device)
        return self.pattern.on(device)

    def forward(self, x):
        B = x.shape[0]
        F = x.shape[1]
        Nin = x.shape[2]
        if Nin < self.N:                                                   # zero padding, graphML.py:2941-2945
            x = torch.cat((x, torch.zeros(B, F, self.N - Nin, dtype=x.dtype, device=x.device)), dim=2)
        y = self._filter(x, self._gso(x.device))                           # [B, heads, F, N]
        if self.concatenate:
            y = self.nonlinearity(y)
            H = getattr(self, self.heads)
            y = y.permute(0, 3, 1, 2).reshape([B, self.N, H * self.F]).permute(0, 2, 1)
        else:
            y = torch.mean(y, dim=1)
            y = self.nonlinearity(y)
        if Nin < self.N:
            y = torch.index_select(y, 2, torch.arange(Nin).to(y.device))
        return y


class GraphAttentional(_AttentionLayer):
    """GraphAttentional(in_features, out_features, attention_heads, edge_features=1, nonlinearity=relu,
    concatenate=True) — same surface, parameters (mixer [K, E, 2F], weight [K, E, F, G]) and initialisation as
    graphML.py:2849-2977; addGSO also takes a SparseGSO."""

    def __init__(self, G, F, K, E=1, nonlinearity=nn.functional.relu, concatenate=True):
        super().__init__()
        self.G = G
        self.F = F
        self.K = K
        self.E = E
        self.S = None
        self.pattern = None
        self.nonlinearity = nonlinearity
        self.concatenate = concatenate
        self.mixer = nn.parameter.Parameter(torch.Tensor(K, E, 2 * F))
        self.weight = nn.parameter.Parameter(torch.Tensor(K, E, F, G))
        self.reset_parameters()

    def reset_parameters(self):
        stdv = 1. / math.sqrt(self.G * self.K)                             # graphML.py:2920-2924
        self.weight.data.uniform_(-stdv, stdv)
        self.mixer.data.uniform_(-stdv, stdv)

    def _filter(self, x, pat):
        return graphAttention(x, self.mixer, self.weight, pat)

    def extra_repr(self):
        reprString = "in_features=%d, out_features=%d, " % (
            self.G, self.F) + "attention_heads=%d, " % (
            self.K) + "edge_features=%d, " % (self.E)
        if self.S is not None:
            reprString += "GSO stored: number_nodes=%d" % (self.N)
        else:
            reprString += "no GSO stored"
        return reprString


class GraphFilterAttentional(_AttentionLayer):
    """GraphFilterAttentional(in_features, out_features, filter_taps, attention_heads, edge_features=1, bias=True,
    nonlinearity=relu, concatenate=True) — graphML.py:2979-3124: mixer [P, E, 2F], weight [P, E, F, G],
    filterWeight [E, K], bias [F, 1]."""
    heads = "P"

    def __init__(self, G, F, K, P, E=1, bias=True, nonlinearity=nn.functional.relu, concatenate=True):
        super().__init__()
        self.G = G
        self.F = F
        self.K = K
        self.P = P
        self.E = E
        self.S = None
        self.pattern = None
        self.nonlinearity = nonlinearity
        self.concatenate = concatenate
        self.mixer = nn.parameter.Parameter(torch.Tensor(P, E, 2 * F))
        self.weight = nn.parameter.Parameter(torch.Tensor(P, E, F, G))
        self.filterWeight = nn.parameter.Parameter(torch.Tensor(E, K))
        if bias:
            self.bias = nn.parameter.Parameter(torch.Tensor(F, 1))
        else:
            self.register_parameter("bias", None)
        self.reset_parameters()

    def reset_parameters(self):
        stdv = 1. / math.sqrt(self.G * self.P)                             # graphML.py:3060-3067
        self.weight.data.uniform_(-stdv, stdv)
        self.mixer.data.uniform_(-stdv, stdv)
        self.filterWeight.data.uniform_(-stdv, stdv)
        if self.bias is not None:
            self.bias.data.uniform_(-stdv, stdv)

    def _filter(self, x, pat):
        return graphAttentionLSIGF(self.filterWeight, x, self.mixer, self.weight, pat, b=self.bias)

    def extra_repr(self):
        reprString = "in_features=%d, " % self.G
        reprString += "out_features=%d, " % self.F
        reprString += "filter_taps=%d, " % self.K
        reprString += "attention_heads=%d, " % self.P
        reprString += "edge_features=%d, " % self.E
        reprString += "bias=%s, " % (self.bias is not None)
        if self.S is not None:
            reprString += "GSO stored: number_nodes=%d" % (self.N)
        else:
            reprString += "no GSO stored"
        return reprString


class EdgeVariantAttentional(GraphFilterAttentional):
    """EdgeVariantAttentional(in_features, out_features, filter_taps, attention_heads, edge_features=1, bias=True,
    nonlinearity=relu, concatenate=True) — graphML.py:3126-3270: mixer [P, K, E, 2F], weight [P, K, E, F, G],
    bias [F, 1].  Concatenating reshapes the P heads to K*F features, as graphML.py:3246-3248 does."""
    heads = "K"

    def __init__(self, G, F, K, P, E=1, bias=True, nonlinearity=nn.functional.relu, concatenate=True):
        nn.Module.__init__(self)
        self.G = G
        self.F = F
        self.K = K
        self.P = P
        self.E = E
        self.S = None
        self.pattern = None
        self.nonlinearity = nonlinearity
        self.concatenate = concatenate
        self.mixer = nn.parameter.Parameter(torch.Tensor(P, K, E, 2 * F))
        self.weight = nn.parameter.Parameter(torch.Tensor(P, K, E, F, G))
        if bias:
            self.bias = nn.parameter.Parameter(torch.Tensor(F, 1))
        else:
            self.register_parameter("bias", None)
        self.reset_parameters()

    def reset_parameters(self):
        stdv = 1. / math.sqrt(self.G * self.K)                             # graphML.py:3208-3214
        self.weight.data.uniform_(-stdv, stdv)
        self.mixer.data.uniform_(-stdv, stdv)
        if self.bias is not None:
            self.bias.data.uniform_(-stdv, stdv)

    def _filter(self, x, pat):
        return graphAttentionEVGF(x, self.mixer, self.weight, pat, b=self.bias)
