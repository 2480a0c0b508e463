"""Drop-in replacements for the LSIGF path of `alegnn.utils.graphML` (reference alegnn/utils/graphML.py).

    LSIGF(h, S, x, b=None)                     <- graphML.py:83-176
    GraphFilter(G, F, K, E=1, bias=True)       <- graphML.py:2036-2155   (same attributes, parameter names and
                                                  shapes, so reference checkpoints `GFL.<i>.weight/bias` round-trip)
    install() / uninstall()                    retarget `alegnn.utils.graphML.LSIGF` / `.GraphFilter` in place
                                                  (SURVEY.md §8b): no reference file is edited.

Host code is PyTorch (tensors, autograd plumbing, streams); the arithmetic runs in libb200gf.so through the
C ABI of include/b200gf.h.  There is no CPU or eager fallback: CPU tensors raise.

Layout.  The reference keeps activations [B, G, N] with the node axis contiguous and returns y as a permuted view
of a [B, N, F] buffer (graphML.py:170-171).  Here y is a permuted view of a node-major [N, B*F(+pad)] buffer (same
logical shape [B, F, N]); when such a view comes back in as the next layer's x — directly, or through an
element-wise op such as nn.ReLU, which preserves strides — it is consumed in place with no transpose.
"""
import math

import torch
import torch.nn as nn

from . import _cabi
from .gso import Plan, SparseGSO, plan_for

_ELEMS_PER_SECTOR = {torch.float32: 8, torch.float64: 4}


def padded_ld(C, dtype):
    q = _ELEMS_PER_SECTOR[dtype]
    return (C + q - 1) // q * q


def node_major_ld(t):
    """If `t` ([B, C, N] logical) is a view of a node-major [N, ld] buffer with columns (b, c), returns ld, else None."""
    if t.dim() != 3:
        return None
    B, C, N = t.shape
    sb, sc, sn = t.stride()
    if N == 0 or B * C == 0:
        return None
    if C > 1 and sc != 1:
        return None
    if B > 1 and sb != C:
        return None
    if N > 1 and sn < B * C:
        return None
    if N == 1:
        sn = B * C
    return sn


def to_node_major(x):
    """[B, C, N] tensor -> (node-major buffer [N, ld], ld).  No copy when x already is such a view."""
    B, C, N = x.shape
    ld = node_major_ld(x)
    if ld is not None:
        return x, ld
    lib = _cabi.load()
    xc = x.contiguous()
    ld = padded_ld(B * C, x.dtype)
    buf = torch.empty((N, ld), dtype=x.dtype, device=x.device)
    _cabi.check(lib.b200gf_to_node_major(_cabi.DTYPE[x.dtype], xc.data_ptr(), buf.data_ptr(), ld, N, B * C,
                                         _cabi.stream()))
    return buf, ld


def to_feature_major(y):
    """[B, C, N] result (typically the permuted node-major view LSIGF returns) -> contiguous reference layout, with one
    coalesced tiled transpose (b200gf_to_feature_major) instead of an element-wise strided copy."""
    ld = node_major_ld(y)
    if ld is None or y.device.type != "cuda" or y.dtype not in _cabi.DTYPE:
        return y.contiguous()
    B, C, N = y.shape
    out = torch.empty((B, C, N), dtype=y.dtype, device=y.device)
    _cabi.check(_cabi.load().b200gf_to_feature_major(_cabi.DTYPE[y.dtype], y.data_ptr(), ld, out.data_ptr(), N, B * C,
                                                     _cabi.stream()))
    return out


def _as_bcn_view(buf, B, C, N):
    """node-major [N, ld] buffer -> logical [B, C, N] strided view."""
    return buf[:, :B * C].view(N, B, C).permute(1, 2, 0)


# ---------------------------------------------------------------------------------------------------
# host code shared by the layer modules: operand checks and the node-major filter frame
# ---------------------------------------------------------------------------------------------------
def check_operands(name, x, tensors, S=None):
    """Raises before any launch unless x is a CUDA tensor in a kernel dtype and every other operand the kernels read
    (`tensors`, None entries skipped) has x's dtype and device; the GSO S (dense tensor, SparseGSO or Plan) needs only
    x's dtype.  There is no CPU path, and a host tensor would reach a kernel as a host pointer."""
    if x.device.type != "cuda":
        raise RuntimeError("b200gf: %s needs CUDA tensors (there is no CPU fallback); got x on %s" % (name, x.device))
    if x.dtype not in _cabi.DTYPE:
        raise RuntimeError("b200gf: %s supports float32 and float64, got x in %s" % (name, x.dtype))
    for t in (*tensors, S):
        if t is not None and t.dtype != x.dtype:
            # torch.matmul in the reference raises on mixed dtypes too ("expected scalar type ...")
            raise RuntimeError("b200gf: %s expects its operands of one dtype, got %s and x in %s" % (name, t.dtype, x.dtype))
    for t in tensors:
        if t is not None and t.device != x.device:
            raise RuntimeError("b200gf: %s expects its operands on one device, got %s and x on %s"
                               % (name, t.device, x.device))


def plan_on(S, device):
    """plan_for(S, device), which must live on `device`."""
    plan = plan_for(S, device)
    if plan.device != device and not (plan.device.index == (device.index or 0)):
        raise RuntimeError("b200gf: GSO plan lives on %s but x is on %s" % (plan.device, device))
    return plan


def _bias_arg(b):
    """A [F, 1] or [F, N] bias as the entry points take it: (contiguous bias or None, bias_per_node)."""
    if b is None:
        return None, 0
    return b.contiguous(), 0 if b.shape[1] == 1 else 1


def _workspace(nbytes, device):
    return torch.empty((nbytes,), dtype=torch.uint8, device=device)


def _grad_in_input_layout(dxbuf, ldc, B, G, N, x_node_major):
    """The input gradient [B, G, N] from its node-major buffer: a view of it when x was one (the producer of x reads it
    through the same strides), else a contiguous tensor by one coalesced tiled transpose instead of a strided view
    that autograd would re-copy element-wise."""
    if x_node_major:
        return _as_bcn_view(dxbuf, B, G, N)
    dx = torch.empty((B, G, N), dtype=dxbuf.dtype, device=dxbuf.device)
    _cabi.check(_cabi.load().b200gf_to_feature_major(_cabi.DTYPE[dx.dtype], dxbuf.data_ptr(), ldc, dx.data_ptr(), N,
                                                     B * G, _cabi.stream()))
    return dx


def _lsigf_forward_nm(plan, hc, xn, x_ld, b, B, G, F_, K, act):
    """One b200gf_forward_act on node-major x: returns the node-major output buffer [N, ldf], ldf and bias_per_node."""
    lib = _cabi.load()
    bc, bias_per_node = _bias_arg(b)
    ldf = padded_ld(B * F_, xn.dtype)
    ybuf = torch.empty((plan.n_rows, ldf), dtype=xn.dtype, device=xn.device)
    ws_bytes = lib.b200gf_workspace_bytes(plan.handle, B, G, F_, K, _cabi.NODE_MAJOR, 0)
    ws = _workspace(ws_bytes, xn.device)
    _cabi.check(lib.b200gf_forward_act(plan.handle, xn.data_ptr(), _cabi.NODE_MAJOR, x_ld, hc.data_ptr(),
                                       None if bc is None else bc.data_ptr(), bias_per_node,
                                       ybuf.data_ptr(), _cabi.NODE_MAJOR, ldf, ws.data_ptr(), ws_bytes,
                                       B, G, F_, K, int(act), _cabi.stream()))
    return ybuf, ldf, bias_per_node


def _lsigf_backward_nm(plan, dyn, dy_ld, xn, x_ld, hc, need_dx, need_db, bias_shape, bias_per_node, B, G, F_, K):
    """One b200gf_backward on node-major dy and x: returns the node-major dx buffer (None unless need_dx), its ldc, the
    tap gradient and the bias gradient (None without a bias or unless need_db)."""
    lib = _cabi.load()
    dt, dev = hc.dtype, dyn.device
    dh = torch.empty_like(hc)
    ldc = padded_ld(B * G, dt)
    dxbuf = torch.empty((plan.n_rows, ldc), dtype=dt, device=dev) if need_dx else None
    db = torch.empty(bias_shape, dtype=dt, device=dev) if (bias_shape is not None and need_db) else None
    ws_bytes = lib.b200gf_workspace_bytes(plan.handle, B, G, F_, K, _cabi.NODE_MAJOR, 1)
    ws = _workspace(ws_bytes, dev)
    _cabi.check(lib.b200gf_backward(plan.handle, dyn.data_ptr(), _cabi.NODE_MAJOR, dy_ld,
                                    xn.data_ptr(), _cabi.NODE_MAJOR, x_ld, hc.data_ptr(),
                                    None if dxbuf is None else dxbuf.data_ptr(), _cabi.NODE_MAJOR, ldc,
                                    dh.data_ptr(), None if db is None else db.data_ptr(), bias_per_node,
                                    ws.data_ptr(), ws_bytes, B, G, F_, K, _cabi.stream()))
    return dxbuf, ldc, dh, db


class _LSIGFFunction(torch.autograd.Function):
    """y = LSIGF(h, S, x, b) with S fixed inside `plan` (graphML.py:83-176)."""

    @staticmethod
    def forward(ctx, h, x, b, plan, act=0):
        F_, E, K, G = h.shape
        B, _, N = x.shape
        hc = h.contiguous()
        ctx.x_node_major = node_major_ld(x) is not None
        xn, x_ld = to_node_major(x)
        ybuf, ldf, bias_per_node = _lsigf_forward_nm(plan, hc, xn, x_ld, b, B, G, F_, K, act)
        ctx.act = int(act)
        ctx.ldf = ldf
        ctx.plan = plan
        ctx.x_ld = x_ld
        ctx.bias_per_node = bias_per_node
        ctx.bias_shape = None if b is None else tuple(b.shape)
        ctx.dims = (B, G, F_, K, E, N)
        if act:
            ctx.save_for_backward(hc, xn, ybuf)      # the fused ReLU's backward needs only the layer output (y > 0)
        else:
            ctx.save_for_backward(hc, xn)
        return _as_bcn_view(ybuf, B, F_, N)

    @staticmethod
    def backward(ctx, dy):
        if ctx.act:
            hc, xn, ybuf = ctx.saved_tensors
        else:
            hc, xn = ctx.saved_tensors
        B, G, F_, K, E, N = ctx.dims
        dyn, dy_ld = to_node_major(dy)
        if ctx.act:                                   # dy_pre = dy * (y > 0), one pass, node-major
            masked = torch.empty((N, ctx.ldf), dtype=hc.dtype, device=dy.device)
            _cabi.check(_cabi.load().b200gf_relu_backward(_cabi.DTYPE[hc.dtype], ybuf.data_ptr(), ctx.ldf, dyn.data_ptr(),
                                                          dy_ld, masked.data_ptr(), ctx.ldf, N, B * F_, _cabi.stream()))
            dyn, dy_ld = masked, ctx.ldf
        need_dh, need_dx, need_db = ctx.needs_input_grad[0], ctx.needs_input_grad[1], ctx.needs_input_grad[2]
        dxbuf, ldc, dh, db = _lsigf_backward_nm(ctx.plan, dyn, dy_ld, xn, ctx.x_ld, hc, need_dx, need_db, ctx.bias_shape,
                                                ctx.bias_per_node, B, G, F_, K)
        dx = _grad_in_input_layout(dxbuf, ldc, B, G, N, ctx.x_node_major) if need_dx else None
        return (dh if need_dh else None), dx, db, None, None


def LSIGF(h, S, x, b=None, activation=None):
    """LSIGF(filter_taps, GSO, input, bias=None): linear shift-invariant graph filter, then bias.
    `activation="relu"` (extension, SURVEY.md §8 f-1) fuses the layer's ReLU into the contraction epilogue.

    Same contract as the reference (alegnn/utils/graphML.py:83-176):
        h [F, E, K, G]; S [E, N, N] (dense tensor, or SparseGSO / Plan); x [B, G, N]; b [F, 1] or [F, N] or None
        returns y [B, F, N],  y_f = sum_e sum_k sum_g h[f,e,k,g] (x_g S_e^k) + b_f
    """
    F_ = h.shape[0]
    E = h.shape[1]
    K = h.shape[2]
    G = h.shape[3]
    assert S.shape[0] == E                       # graphML.py:135
    N = S.shape[1]
    assert S.shape[2] == N                       # graphML.py:137
    B = x.shape[0]
    assert x.shape[1] == G                       # graphML.py:139
    assert x.shape[2] == N                       # graphML.py:140
    b = _bias_2d(b, F_, N, "LSIGF")
    if activation is None:
        return _dispatch(h, S, x, b)
    if activation != "relu":
        raise ValueError("b200gf: fused activation must be None or 'relu', got %r" % (activation,))
    return _dispatch(h, S, x, b, 1)


def _bias_2d(b, F_, N, name):
    """The bias forms LSIGF accepts, as [F, 1] or [F, N] (None stays None)."""
    if b is None:
        return None
    # the reference adds b by broadcasting (graphML.py:174-175): GraphFilter passes [F, 1], and the reference's own
    # GatedGRNN reshapes its biases to (1, F, 1) before calling LSIGF (graphML.py:1394-1404, :1461)
    if b.dim() == 3 and b.shape[0] == 1:
        b = b[0]
    elif b.dim() == 1 and N == 1:
        b = b.reshape(-1, 1)
    if not (b.dim() == 2 and b.shape[0] in (1, F_) and b.shape[1] in (1, N)):
        raise RuntimeError("b200gf: %s bias must broadcast against [B, F, N] as [F, 1], [F, N], [1, F, 1] or "
                           "[1, F, N]; got %s" % (name, tuple(b.shape)))
    if b.shape[0] == 1 and F_ > 1:
        b = b.expand(F_, b.shape[1])
    return b


def _dispatch_cuda(h, S, x, b, act=0):
    """Device part of LSIGF: loud checks (there is no CPU path), plan lookup, the autograd function over the C ABI.
    `_dispatch` is the single hook the CPU tests replace with the oracle to exercise the argument handling above."""
    check_operands("LSIGF", x, (h, b), S)
    return _LSIGFFunction.apply(h, x, b, plan_on(S, x.device), act)


_dispatch = _dispatch_cuda


class GraphFilter(nn.Module):
    """GraphFilter(in_features, out_features, filter_taps, edge_features=1, bias=True)

    Same surface as the reference layer (alegnn/utils/graphML.py:2036-2155): attributes G, F, K, E, S, N;
    parameters `weight` [F, E, K, G] and `bias` [F, 1] (or None); `addGSO(S)`, `forward(x)`, `extra_repr()`.
    `addGSO` additionally accepts a SparseGSO and builds the device plan once (cached per device).
    """

    def __init__(self, G, F, K, E=1, bias=True):
        super().__init__()
        self.G = G
        self.F = F
        self.K = K
        self.E = E
        self.S = None
        self.fused_activation = None                 # "relu" after fuse_layers(): the next module became nn.Identity
        self.weight = nn.parameter.Parameter(torch.Tensor(F, E, K, G))
        if bias:
            self.bias = nn.parameter.Parameter(torch.Tensor(F, 1))
        else:
            self.register_parameter("bias", None)
        self.reset_parameters()

    def reset_parameters(self):
        stdv = 1. / math.sqrt(self.G * self.K)      # graphML.py:2109-2114
        self.weight.data.uniform_(-stdv, stdv)
        if self.bias is not None:
            self.bias.data.uniform_(-stdv, stdv)

    def addGSO(self, S):
        assert len(S.shape) == 3                    # graphML.py:2118
        assert S.shape[0] == self.E                 # graphML.py:2120
        self.N = S.shape[1]
        assert S.shape[2] == self.N                 # graphML.py:2122
        self.S = S
        # Build (or fetch from the cache) the device CSR plan now.  A dense GSO still on the CPU gets its plan
        # when the architecture's .to(device) re-attaches it (architectures.py:463-479) or on first use.
        if torch.cuda.is_available() and (isinstance(S, (SparseGSO, Plan)) or
                                          (isinstance(S, torch.Tensor) and S.device.type == "cuda")):
            plan_for(S)

    def forward(self, x):
        B = x.shape[0]
        F = x.shape[1]
        Nin = x.shape[2]
        if Nin < self.N:                            # zero-pad the node axis, graphML.py:2131-2135
            x = torch.cat((x, torch.zeros(B, F, self.N - Nin, dtype=x.dtype, device=x.device)), dim=2)
        if self.fused_activation is None:           # the reference's call, argument for argument (graphML.py:2137)
            u = LSIGF(self.weight, self.S, x, self.bias)  # plan lookup is cached per (tensor, version, device)
        else:
            u = LSIGF(self.weight, self.S, x, self.bias, activation=self.fused_activation)
        if Nin < self.N:                            # keep the first Nin nodes, graphML.py:2142-2143
            u = u[:, :, :Nin]
        return u

    def extra_repr(self):
        reprString = "in_features=%d, out_features=%d, " % (self.G, self.F) + "filter_taps=%d, " % (self.K) + \
                     "edge_features=%d, " % (self.E) + "bias=%s, " % (self.bias is not None)
        if self.S is not None:
            reprString += "GSO stored"
        else:
            reprString += "no GSO stored"
        return reprString


def fuse_layers(model):
    """Fuse `GraphFilter -> nn.ReLU -> (NoPool | MaxPoolLocal)` triples inside every nn.Sequential of `model` (the
    reference builds its graph-filtering layers exactly like that, alegnn/modules/architectures.py:274-296):
    the ReLU moves into the filter's contraction epilogue (the nn.ReLU module is replaced by nn.Identity, so the
    Sequential keeps its indices and the checkpoint keys `GFL.<3l>.weight/bias` are unchanged) and a reference
    MaxPoolLocal is swapped for this package's CUDA gather on the node-major output.  NoPool is an identity already.
    Returns the number of fused layers."""
    from . import pooling
    fused = 0
    for seq in [m for m in model.modules() if isinstance(m, nn.Sequential)]:
        mods = list(seq._modules.items())
        for i, (name, m) in enumerate(mods):
            if isinstance(m, GraphFilter) and i + 1 < len(mods) and type(mods[i + 1][1]) is nn.ReLU:
                m.fused_activation = "relu"
                seq._modules[mods[i + 1][0]] = nn.Identity()
                fused += 1
                if i + 2 < len(mods):
                    pname, pm = mods[i + 2]
                    if type(pm).__name__ == "MaxPoolLocal" and not isinstance(pm, pooling.MaxPoolLocal):
                        seq._modules[pname] = pooling.MaxPoolLocal.from_reference(pm)
    return fused


# ---------------------------------------------------------------------------------------------------
# retargeting the reference (SURVEY.md §8b)
# ---------------------------------------------------------------------------------------------------
_SAVED = {}


def install(gml=None, edge_gating=False, node_variant=False, arma=False, attention=False, aggregation=False, archit=None):
    """Point `alegnn.utils.graphML.LSIGF`, `.GraphFilter`, `.EVGF`, `.EdgeVariantGF`, the local pooling / activation
    layers and the static-GSO recurrent layers at this package.  `edge_gating=True` also points
    `.EdgeGatedHiddenState` at the sparse edge-gated layer (edgegated.py); by default it stays the reference's.
    `node_variant=True` also points `.NVGF` and `.NodeVariantGF` at the sparse node-variant filter (nodevariant.py);
    by default they stay the reference's.  `arma=True` also points `.jARMA` and `.GraphFilterARMA` at the sparse ARMA
    filter (arma.py); by default they stay the reference's (whose residue term still runs on this package's LSIGF).
    `attention=True` also points `.GraphAttentional`, `.GraphFilterAttentional`, `.EdgeVariantAttentional` and the
    functionals `.graphAttention`, `.graphAttentionLSIGF`, `.graphAttentionEVGF` at the sparse attention layers
    (attention.py); by default they stay the reference's.  `.learnAttentionGSO`, which returns a dense tensor, is always
    the reference's.
    `aggregation=True` also points `alegnn.modules.architectures.AggregationGNN` and `.MultiNodeAggregationGNN` (or those
    of `archit`, when given) at the sparse aggregation GNNs (aggregation.py).  Both are retargeted: the reference's
    MultiNodeAggregationGNN looks AggregationGNN up as a module global and would still build a dense GSO copy per node.

    `GraphFilter.forward` in the reference looks `LSIGF` up as a module global at call time (graphML.py:2137), so
    this also accelerates its hybrid EdgeVariantGF (:2686), jARMA (:592) and GatedGRNN (:1403,:1461) call sites.
    Architectures built AFTER install() get this package's layers (plan cached in addGSO).
    """
    from . import activations, arma as arma_mod, attention as attention_mod, delayed, edgegated, edgevariant, nodevariant, pooling, recurrent
    if gml is None:
        import alegnn.utils.graphML as gml
    if id(gml) not in _SAVED:
        _SAVED[id(gml)] = (gml, {n: getattr(gml, n) for n in ("LSIGF", "GraphFilter", "EVGF", "EdgeVariantGF",
                                                             "MaxPoolLocal", "MaxLocalActivation",
                                                             "MedianLocalActivation", "HiddenState",
                                                             "TimeGatedHiddenState", "NodeGatedHiddenState",
                                                             "LSIGF_DB", "GraphFilter_DB", "GRNN_DB",
                                                             "HiddenState_DB")})
    if edge_gating:
        _SAVED[id(gml)][1].setdefault("EdgeGatedHiddenState", getattr(gml, "EdgeGatedHiddenState"))
        # per-non-zero attention gates and the per-sample gated hop (edgegated.py); gml.GatedGRNN stays the reference's
        gml.EdgeGatedHiddenState = edgegated.EdgeGatedHiddenState
    if node_variant:
        for name in ("NVGF", "NodeVariantGF"):
            _SAVED[id(gml)][1].setdefault(name, getattr(gml, name))
        # per-node tap contraction on the LSIGF hops; copyNodes by a sparse breadth-first search (nodevariant.py)
        gml.NVGF = nodevariant.NVGF
        gml.NodeVariantGF = nodevariant.NodeVariantGF
    if arma:
        for name in ("jARMA", "GraphFilterARMA"):
            _SAVED[id(gml)][1].setdefault(name, getattr(gml, name))
        # sparse Jacobi chains on the S~ plan instead of [F,E,P,G,N,N] dense operators (arma.py)
        gml.jARMA = arma_mod.jARMA
        gml.GraphFilterARMA = arma_mod.GraphFilterARMA
    if aggregation:
        from . import aggregation as aggregation_mod
        if archit is None:
            import alegnn.modules.architectures as archit
        for name in ("AggregationGNN", "MultiNodeAggregationGNN"):
            _SAVED[id(gml)][1].setdefault((archit, name), getattr(archit, name))
            setattr(archit, name, getattr(aggregation_mod, name))
    if attention:
        names = ("graphAttention", "graphAttentionLSIGF", "graphAttentionEVGF", "GraphAttentional",
                 "GraphFilterAttentional", "EdgeVariantAttentional")
        for name in names:
            _SAVED[id(gml)][1].setdefault(name, getattr(gml, name))
        # attention per non-zero of the mask of S + I and gated sparse hops instead of B x P x E x N x N tensors
        for name in names:
            setattr(gml, name, getattr(attention_mod, name))
    gml.LSIGF = LSIGF
    gml.GraphFilter = GraphFilter
    gml.EVGF = edgevariant.EVGF
    gml.EdgeVariantGF = edgevariant.EdgeVariantGF
    gml.MaxPoolLocal = pooling.MaxPoolLocal      # same layer, neighbourhoods from the CSR routine (scales past dense N x N)
    gml.MaxLocalActivation = activations.MaxLocalActivation
    gml.MedianLocalActivation = activations.MedianLocalActivation
    # static-GSO recurrent layers: node-major recursion (recurrent.py).  gml.GatedGRNN itself is left alone so that the
    # reference's EdgeGatedHiddenState (dense per-sample gated GSOs, not on this path) keeps working.
    gml.HiddenState = recurrent.HiddenState
    gml.TimeGatedHiddenState = recurrent.TimeGatedHiddenState
    gml.NodeGatedHiddenState = recurrent.NodeGatedHiddenState
    # batch-/time-varying GSOs: one space-time sparse operator per batch (delayed.py)
    gml.LSIGF_DB = delayed.LSIGF_DB
    gml.GraphFilter_DB = delayed.GraphFilter_DB
    # the recursion over the same GSO batch: the delay line advanced by one CSR hop per time step (delayed.GRNN_DB)
    gml.GRNN_DB = delayed.GRNN_DB
    gml.HiddenState_DB = delayed.HiddenState_DB
    return gml


def uninstall(gml=None):
    for key, (mod, saved) in list(_SAVED.items()):
        if gml is None or mod is gml:
            for name, obj in saved.items():
                target, attr = name if isinstance(name, tuple) else (mod, name)   # (module, name): another module
                setattr(target, attr, obj)
            del _SAVED[key]
