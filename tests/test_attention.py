"""Graph attention layers (gnn_b200.attention, csrc/egate.cu) against fixtures produced by the unmodified reference
(tests/golden/attention_cases.npz <- oracle/make_golden_attention.py: graphAttention, graphAttentionLSIGF,
graphAttentionEVGF, GraphAttentional, GraphFilterAttentional, EdgeVariantAttentional, alegnn/utils/graphML.py:739-969,
:2849-3270, and the three attention architectures).

CPU tests check the host logic (pattern over E edge features, projections, sample layouts, taps, heads, padding,
autograd wiring) with torch restatements standing in for the two kernels (`_attention`, `_gated_hop`), and the fp64
restatement oracle/attention_oracle.py against the fixtures; GPU tests run the real kernels against the fixtures, in a
CUDA graph, and at N = 200 000 against the restatement.  Each launch branch of the two-score entry points has a
componentwise-bounded row in tests/test_attention_dispatch.py."""
import os
import types

import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.nn as nn

import attention_oracle as ao
import egate_oracle as ego

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "attention_cases.npz"))
GA_TAGS = ["e1p1", "e2p3", "e1p3", "n1"]
GL_TAGS = ["k1", "k3e2", "k3p1", "k2p3", "n1"]
GE_TAGS = ["k1", "k3e2", "k3p1", "k2e2", "n1"]
LAYERS = [("ga", "cat"), ("ga", "mean"), ("gl", "cat"), ("gl", "mean"), ("ge", "cat"), ("ge", "mean"), ("ge", "n1")]
NETS = ["gat", "gcat", "eva"]
SIGMA = {0: nn.functional.relu, 1: torch.tanh}


def _rel(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


# ------------------------------------------------------------------------------------ torch restatements of the kernels
def _attention_torch(s_src, s_dst, pat):
    """s_src, s_dst [N, Bs] -> alpha [nnz, Bs], through the fp64 restatement's per-non-zero index arithmetic."""
    return ao.attention_coo(s_src.t(), s_dst.t(), pat.m_row, pat.m_col.long(), pat.N).t()


def _gated_hop_torch(u, gate, pat):
    """u [N, Bs, C], gate [Bs, nnz] -> u S~ per sample, over the pattern's CSR of S^T and its mask positions."""
    j = torch.repeat_interleave(torch.arange(pat.N, device=u.device), pat.t_rowptr.diff())
    i = pat.t_col.long()
    pos = pat.t_pos.long()
    w = torch.where(pos >= 0, gate[:, pos.clamp(min=0)] * pat.t_val.to(u.dtype), torch.zeros((), dtype=u.dtype))
    return ego.egate_hop_coo(u.permute(1, 2, 0), w, i, j).permute(2, 0, 1)


@pytest.fixture
def torch_kernels(monkeypatch):
    from gnn_b200 import attention as at
    monkeypatch.setattr(at, "_attention", _attention_torch)
    monkeypatch.setattr(at, "_gated_hop", _gated_hop_torch)


# ------------------------------------------------------------------------------------------------------- case runners
def _functional_case(kind, tag, dtype, device, sparse=False):
    import gnn_b200
    p = "%s_%s_" % (kind, tag)
    S = torch.tensor(GOLD[p + "S"], dtype=dtype, device=device)
    if sparse:
        S = gnn_b200.SparseGSO.from_dense(S.cpu())
    names = {"ga": ("x", "a", "W"), "gl": ("h", "x", "a", "W", "b"), "ge": ("x", "a", "W", "b")}[kind]
    ts = {k: torch.tensor(GOLD[p + k], dtype=dtype, device=device, requires_grad=True) for k in names
          if p + k in GOLD.files}
    if kind == "ga":
        y = gnn_b200.graphAttention(ts["x"], ts["a"], ts["W"], S)
    elif kind == "gl":
        y = gnn_b200.graphAttentionLSIGF(ts["h"], ts["x"], ts["a"], ts["W"], S, b=ts.get("b"))
    else:
        y = gnn_b200.graphAttentionEVGF(ts["x"], ts["a"], ts["W"], S, b=ts.get("b"))
    assert tuple(y.shape) == GOLD[p + "y"].shape
    y.backward(torch.tensor(GOLD[p + "dy"], dtype=dtype, device=device))
    out = {"y": (y, GOLD[p + "y"])}
    for k, t in ts.items():                                          # K = 1 in graphAttentionLSIGF: a gets no gradient
        out["d" + k] = (t.grad if t.grad is not None else torch.zeros_like(t), GOLD[p + "d" + k])
    return {k: (v.detach().cpu().numpy(), ref) for k, (v, ref) in out.items()}


def _layer_meta(kind, tag):
    seed, N, B, G, F, K, P, E, bias, cat, Nin, sg = (int(v) for v in GOLD["l%s_%s_meta" % (kind, tag)])
    return seed, N, B, G, F, K, P, E, bool(bias), bool(cat), Nin, SIGMA[sg]


def _make_layer(mod, kind, G, F, K, P, E, bias, cat, sigma):
    if kind == "ga":
        return mod.GraphAttentional(G, F, K, E, sigma, cat)
    if kind == "gl":
        return mod.GraphFilterAttentional(G, F, K, P, E, bias, sigma, cat)
    return mod.EdgeVariantAttentional(G, F, K, P, E, bias, sigma, cat)


def _layer_case(kind, tag, dtype, device, sparse=False):
    import gnn_b200
    p = "l%s_%s_" % (kind, tag)
    seed, N, B, G, F, K, P, E, bias, cat, Nin, sigma = _layer_meta(kind, tag)
    layer = _make_layer(gnn_b200, kind, G, F, K, P, E, bias, cat, sigma)
    sd = {k[len(p) + 2:]: torch.tensor(GOLD[k]) for k in GOLD.files if k.startswith(p + "p_")}
    assert list(sd) == list(layer.state_dict())                     # the reference's names, in the reference's order
    layer = layer.to(device=device, dtype=dtype)
    layer.load_state_dict(sd)
    S = torch.tensor(GOLD[p + "S"], dtype=dtype, device=device)
    layer.addGSO(gnn_b200.SparseGSO.from_dense(S.cpu()) if sparse else S)
    x = torch.tensor(GOLD[p + "x"], dtype=dtype, device=device, requires_grad=True)
    y = layer(x)
    assert tuple(y.shape) == GOLD[p + "y"].shape
    y.backward(torch.tensor(GOLD[p + "dy"], dtype=dtype, device=device))
    out = dict(y=(y, GOLD[p + "y"]), dx=(x.grad, GOLD[p + "dx"]))
    for name, prm in layer.named_parameters():
        out[name] = (prm.grad if prm.grad is not None else torch.zeros_like(prm), GOLD[p + "g_" + name])
    return {k: (v.detach().cpu().numpy(), ref) for k, (v, ref) in out.items()}


def _standin():
    gml = types.ModuleType("graphML_standin")
    for n in ("LSIGF", "GraphFilter", "EVGF", "EdgeVariantGF", "MaxPoolLocal", "MaxLocalActivation",
              "MedianLocalActivation", "HiddenState", "TimeGatedHiddenState", "NodeGatedHiddenState", "LSIGF_DB",
              "GraphFilter_DB", "GRNN_DB", "HiddenState_DB", "EdgeGatedHiddenState", "NVGF", "NodeVariantGF", "jARMA",
              "GraphFilterARMA", "graphAttention", "graphAttentionLSIGF", "graphAttentionEVGF", "GraphAttentional",
              "GraphFilterAttentional", "EdgeVariantAttentional", "learnAttentionGSO"):
        setattr(gml, n, type(n, (), {}))
    return gml


def _net_case(arch, dtype, device):
    """The fixture's two-layer network (GraphAttentionNetwork([2, 4, 3], [2, 2], relu, [N, N], NoPool, [1, 1], [5],
    True, S), or the filter networks with taps [2, 3] / [2, 2] and heads [2, 2]) rebuilt, as the reference's
    architectures.py builds it, from the layers install(attention=True) puts into a stand-in module; NoPool (an
    identity without parameters) is nn.Identity."""
    import gnn_b200
    gml = gnn_b200.install(_standin(), attention=True)
    try:
        p = "net_%s_" % arch
        seed, N, B, E = (int(v) for v in GOLD[p + "meta"])
        S = torch.tensor(GOLD[p + "S"], dtype=dtype, device=device)
        relu = nn.functional.relu
        if arch == "gat":
            layers = [gml.GraphAttentional(2, 4, 2, E, relu, True), gml.GraphAttentional(8, 3, 2, E, relu, False)]
            name = "GAT"
        elif arch == "gcat":
            layers = [gml.GraphFilterAttentional(2, 4, 2, 2, E, True, relu, True),
                      gml.GraphFilterAttentional(8, 3, 3, 2, E, True, relu, False)]
            name = "GCAT"
        else:
            layers = [gml.EdgeVariantAttentional(2, 4, 2, 2, E, True, relu, True),
                      gml.EdgeVariantAttentional(8, 3, 2, 2, E, True, relu, False)]
            name = "EVGAT"
        assert isinstance(layers[0], nn.Module) and type(layers[0]).__module__.endswith("attention")
        net = nn.Module()
        setattr(net, name, nn.Sequential(layers[0], nn.Identity(), layers[1], nn.Identity()))
        net.MLP = nn.Sequential(nn.Linear(N * 3, 5, bias=True))
        sd = {k[len(p) + 2:]: torch.tensor(GOLD[k]) for k in GOLD.files if k.startswith(p + "p_")}
        assert sorted(sd) == sorted(net.state_dict())
        net = net.to(device=device, dtype=dtype)       # before loading: the fixture's fp64 values are not fp32-exact
        net.load_state_dict(sd)
        for layer in layers:
            layer.addGSO(S)
        x = torch.tensor(GOLD[p + "x"], dtype=dtype, device=device, requires_grad=True)
        y = net.MLP(getattr(net, name)(x).reshape(B, 3 * N))
        y.backward(torch.tensor(GOLD[p + "dy"], dtype=dtype, device=device))
    finally:
        gnn_b200.uninstall(gml)
    out = dict(y=(y.detach(), GOLD[p + "y"]), dx=(x.grad, GOLD[p + "dx"]))
    for n, prm in net.named_parameters():
        out[n] = (prm.grad, GOLD[p + "g_" + n])
    return {k: (v.detach().cpu().numpy(), ref) for k, (v, ref) in out.items()}


FUNCTIONAL_CASES = [("ga", t) for t in GA_TAGS] + [("gl", t) for t in GL_TAGS] + [("ge", t) for t in GE_TAGS]


# ------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("kind,tag", FUNCTIONAL_CASES)
def test_functional_host_logic_matches_reference(kind, tag, torch_kernels):
    for sparse in (False, True):
        for name, (got, ref) in _functional_case(kind, tag, torch.float64, "cpu", sparse).items():
            assert _rel(got, ref) < 1e-12, (sparse, name)


@pytest.mark.parametrize("kind,tag", LAYERS)
def test_layer_host_logic_matches_reference(kind, tag, torch_kernels):
    for sparse in (False, True):
        for name, (got, ref) in _layer_case(kind, tag, torch.float64, "cpu", sparse).items():
            assert _rel(got, ref) < 1e-12, (sparse, name)


@pytest.mark.parametrize("arch", NETS)
def test_network_host_logic_matches_reference(arch, torch_kernels):
    for name, (got, ref) in _net_case(arch, torch.float64, "cpu").items():
        assert _rel(got, ref) < 1e-12, name


@pytest.mark.parametrize("kind,tag", FUNCTIONAL_CASES)
def test_oracle_matches_reference_fixtures(kind, tag):
    """The fp64 restatement the at-scale GPU test trusts (attention_oracle) equals the reference."""
    p = "%s_%s_" % (kind, tag)
    g = ao.CooGSO([sp.csr_matrix(s) for s in GOLD[p + "S"]], "cpu", torch.float64)
    names = {"ga": ("x", "a", "W"), "gl": ("h", "x", "a", "W", "b"), "ge": ("x", "a", "W", "b")}[kind]
    ts = {k: torch.tensor(GOLD[p + k], requires_grad=True) for k in names if p + k in GOLD.files}
    if kind == "ga":
        y = ao.graph_attention(g, ts["x"], ts["a"], ts["W"])
    elif kind == "gl":
        y = ao.graph_attention_lsigf(g, ts["h"], ts["x"], ts["a"], ts["W"], ts.get("b"))
    else:
        y = ao.graph_attention_evgf(g, ts["x"], ts["a"], ts["W"], ts.get("b"))
    y.backward(torch.tensor(GOLD[p + "dy"]))
    assert _rel(y.detach().numpy(), GOLD[p + "y"]) < 1e-12
    for k, t in ts.items():
        ref = GOLD[p + "d" + k]
        got = np.zeros(ref.shape) if t.grad is None else t.grad.numpy()
        assert (not np.any(got)) if not np.any(ref) else _rel(got, ref) < 1e-12, k


def test_fixtures_cover_the_mask_rules():
    """The E = 2 GSOs put the sub-tolerance pair (0, 2) into the mask and E = 1 leaves it out; node 1 has an empty mask
    row; S_44 = -1 is a hop entry outside the mask."""
    import gnn_b200
    for p, in_mask in (("ga_e2p3_", True), ("ga_e1p1_", False)):
        S = GOLD[p + "S"]
        pat = gnn_b200.EdgeGatePattern(torch.tensor(S))
        M = np.zeros((pat.N, pat.N), bool)
        M[pat.m_row.numpy(), pat.m_col.numpy()] = True
        assert M[0, 2] == in_mask and np.all(S[:, 0, 2] == 6e-10)
        assert not M[1].any() and not M[4, 4] and M[4, 5]
        assert (M == (np.abs(S + np.eye(pat.N)).sum(0) > 1e-9)).all()
        for e in range(S.shape[0]):
            ed = pat.edges[e]
            j = np.repeat(np.arange(pat.N), np.diff(ed.t_rowptr.numpy()))
            i = ed.t_col.numpy()
            assert sorted(zip(i, j)) == sorted(zip(*np.nonzero(S[e])))
            hop = dict(((a, b), q) for a, b, q in zip(i, j, ed.t_pos.numpy()))
            assert hop[(4, 4)] == -1 and hop[(1, 1)] == -1
            np.testing.assert_array_equal(ed.m_sval.numpy(), S[e][pat.m_row.numpy(), pat.m_col.numpy()])


def test_pattern_for_one_edge_feature_is_the_edge_gate_pattern():
    """E = 1: the pattern equals, member for member, the one edge gating has always used (oracle/egate_oracle.py's
    egate_pattern, which tests/test_egate_oracle.py pins to it), for a dense tensor and a SparseGSO."""
    import gnn_b200
    S = GOLD["ga_e1p1_S"]
    r, c = np.nonzero(S[0])
    ref = ego.egate_pattern(S.shape[1], r, c, S[0][r, c])
    for src in (torch.tensor(S), gnn_b200.SparseGSO.from_dense(torch.tensor(S))):
        pat = gnn_b200.EdgeGatePattern(src)
        assert pat.E == 1 and pat.edges == [pat] and pat.nnz == ref["nnz"]
        for name in gnn_b200.EdgeGatePattern._TENSORS:
            if name == "m_row":
                continue
            got = getattr(pat, name).numpy()
            assert got.dtype == ref[name].dtype and np.array_equal(got, ref[name]), name
        assert np.array_equal(pat.m_row.numpy(), ego._rows_of(ref["m_rowptr"]))


def test_unit_pattern_hops_by_alpha_alone():
    import gnn_b200
    S = GOLD["gl_k3e2_S"]
    pat = gnn_b200.EdgeGatePattern(torch.tensor(S))
    u = pat.unit()
    assert u.nnz == pat.nnz and bool((u.t_val == 1).all()) and bool((u.m_sval == 1).all())
    j = np.repeat(np.arange(pat.N), np.diff(u.t_rowptr.numpy()))
    mr, mc = pat.m_row.numpy(), pat.m_col.numpy()
    assert np.array_equal(mr[u.t_pos.numpy()], u.t_col.numpy()) and np.array_equal(mc[u.t_pos.numpy()], j)
    assert np.array_equal(u.s_pos.numpy(), np.arange(pat.nnz))


def test_state_dict_keys_and_seeded_parameters_match_the_reference():
    import gnn_b200
    for kind, tag in LAYERS:
        p = "l%s_%s_" % (kind, tag)
        seed, N, B, G, F, K, P, E, bias, cat, Nin, sigma = _layer_meta(kind, tag)
        torch.manual_seed(seed)
        layer = _make_layer(gnn_b200, kind, G, F, K, P, E, bias, cat, sigma).double()
        sd = layer.state_dict()
        ref = {k[len(p) + 2:]: GOLD[k] for k in GOLD.files if k.startswith(p + "p_")}
        assert list(sd) == list(ref)
        for k in ref:
            assert np.array_equal(sd[k].numpy(), ref[k]), (kind, tag, k)
    assert repr(gnn_b200.GraphFilterAttentional(3, 2, 3, 2, 1, False)).startswith(
        "GraphFilterAttentional(in_features=3, out_features=2, filter_taps=3, attention_heads=2, edge_features=1, "
        "bias=False, no GSO stored")


def test_argument_checks_without_a_gpu():
    import gnn_b200
    S = torch.eye(4, dtype=torch.float64).reshape(1, 4, 4)
    x = torch.zeros(2, 3, 4, dtype=torch.float64)
    a, W = torch.zeros(2, 1, 4, dtype=torch.float64), torch.zeros(2, 1, 2, 3, dtype=torch.float64)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        gnn_b200.graphAttention(x, a, W, S)
    with pytest.raises(NotImplementedError, match="slope"):
        gnn_b200.graphAttention(x, a, W, S, negative_slope=0.1)
    with pytest.raises(AssertionError):
        gnn_b200.graphAttention(x, a[:, :, :3], W, S)
    with pytest.raises(AssertionError):
        gnn_b200.graphAttention(x, a, W, torch.eye(5, dtype=torch.float64).reshape(1, 5, 5))


def test_install_attention_is_opt_in():
    import gnn_b200
    names = ("graphAttention", "graphAttentionLSIGF", "graphAttentionEVGF", "GraphAttentional",
             "GraphFilterAttentional", "EdgeVariantAttentional")
    gml = _standin()
    orig = {n: getattr(gml, n) for n in vars(gml) if not n.startswith("__")}
    try:
        gnn_b200.install(gml)
        assert all(getattr(gml, n) is orig[n] for n in names)
        gnn_b200.install(gml, attention=True)
        assert all(getattr(gml, n) is getattr(gnn_b200, n) for n in names)
        assert gml.learnAttentionGSO is orig["learnAttentionGSO"]
    finally:
        gnn_b200.uninstall(gml)
    assert {n: getattr(gml, n) for n in orig} == orig


# ------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-11), (torch.float32, 1e-4)])
def test_fixtures_on_gpu(dtype, tol):
    for kind, tag in FUNCTIONAL_CASES:
        for sparse in (False, True):
            for name, (got, ref) in _functional_case(kind, tag, dtype, "cuda", sparse).items():
                assert _rel(got, ref) < tol, (kind, tag, sparse, name)
    for kind, tag in LAYERS:
        for sparse in (False, True):
            for name, (got, ref) in _layer_case(kind, tag, dtype, "cuda", sparse).items():
                assert _rel(got, ref) < tol, (kind, tag, sparse, name)
    for arch in NETS:
        for name, (got, ref) in _net_case(arch, dtype, "cuda").items():
            assert _rel(got, ref) < tol, (arch, name)


def _er(N, deg, seed, dtype=np.float32):
    """Non-symmetric Erdos-Renyi GSO, rows scaled to absolute sum <= 1, values exact in dtype."""
    rng = np.random.default_rng(seed)
    nnz = N * deg
    m = sp.csr_matrix((rng.standard_normal(nnz), (rng.integers(0, N, nnz), rng.integers(0, N, nnz))), shape=(N, N))
    m.sum_duplicates()
    m.eliminate_zeros()
    m = sp.diags(1.0 / np.maximum(np.abs(m).sum(axis=1).A.ravel(), 1.0)) @ m
    m = sp.csr_matrix(m.astype(dtype).astype(np.float64))
    m.sort_indices()
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["ga", "gl", "ge"])
def test_graphed_forward_backward_is_bit_identical_to_eager(kind):
    import gnn_b200
    N, B, G, F, K, P, E = 20000, 2, 4, 3, 3, 2, 2
    S = gnn_b200.SparseGSO.from_scipy([_er(N, 8, 41), _er(N, 8, 42)], dtype=torch.float32)
    torch.manual_seed(3)
    layer = _make_layer(gnn_b200, kind, G, F, K if kind != "ga" else P, P, E, True, kind != "ge",
                        nn.functional.relu).cuda()
    layer.addGSO(S)
    rng = np.random.default_rng(1)
    x = torch.tensor(rng.standard_normal((B, G, N)), dtype=torch.float32, device="cuda", requires_grad=True)
    tensors = list(layer.parameters()) + [x]

    def step():
        layer(x).square().sum().backward()

    for p in tensors:
        p.grad = None
    step()
    eager = [t.grad.clone() for t in tensors]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            for p in tensors:
                p.grad = None
            step()
    torch.cuda.current_stream().wait_stream(side)
    for p in tensors:
        p.grad = None
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    g.replay()
    torch.cuda.synchronize()
    replay = [t.grad.clone() for t in tensors]
    assert all(torch.equal(a, b) for a, b in zip(eager, replay))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["ga", "gl", "ge"])
def test_at_scale_vs_fp64_restatement(kind):
    """N = 200 000 non-symmetric Erdos-Renyi, degree 16, E = 2, B = 4, P = 4 (B*P = 16), G = F = 4, K = 3: the output
    and every gradient in fp64 against attention_oracle's restatement (run in torch on the GPU) at 1e-10.  The fp32 run
    is held to the same restatement too, at most 8x (+ 1e-6) the error of the restatement itself evaluated in fp32: the
    gradients of x and of the attention parameters pass through the softmax backward, alpha (dalpha - sum alpha
    dalpha), whose cancellation puts the error of any fp32 evaluation at ~1e-3 of the largest element (measured on an
    H100), so a fixed fp32 tolerance would either be loose for the output or fail on a correct kernel; a plain fp32
    evaluation of the same formulas in another summation order is the yardstick."""
    import gnn_b200
    N, B, G, F, K, P, E = 200_000, 4, 4, 4, 3, 4, 2
    mats = [_er(N, 16, 51), _er(N, 16, 52)]
    rng = np.random.default_rng(7)
    stdv = 0.5
    shapes = {"ga": dict(a=(P, E, 2 * F), W=(P, E, F, G)),
              "gl": dict(h=(E, K), a=(P, E, 2 * F), W=(P, E, F, G), b=(F, 1)),
              "ge": dict(a=(P, K, E, 2 * F), W=(P, K, E, F, G), b=(F, 1))}[kind]
    vals = {k: rng.uniform(-stdv, stdv, s).astype(np.float32).astype(np.float64) for k, s in shapes.items()}
    vals["x"] = rng.standard_normal((B, G, N)).astype(np.float32).astype(np.float64)
    dy = rng.standard_normal((B, P, F, N)).astype(np.float32).astype(np.float64)

    def run(fn, S, dtype):
        ts = {k: torch.tensor(v, dtype=dtype, device="cuda", requires_grad=True) for k, v in vals.items()}
        if kind == "ga":
            y = fn["ga"](S, ts["x"], ts["a"], ts["W"])
        elif kind == "gl":
            y = fn["gl"](S, ts["h"], ts["x"], ts["a"], ts["W"], ts["b"])
        else:
            y = fn["ge"](S, ts["x"], ts["a"], ts["W"], ts["b"])
        y.backward(torch.tensor(dy, dtype=dtype, device="cuda"))
        out = {"y": y.detach().double().cpu().numpy()}
        out.update({"d" + k: t.grad.double().cpu().numpy() for k, t in ts.items()})
        return out

    ours = {"ga": lambda S, x, a, W: gnn_b200.graphAttention(x, a, W, S),
            "gl": lambda S, h, x, a, W, b: gnn_b200.graphAttentionLSIGF(h, x, a, W, S, b),
            "ge": lambda S, x, a, W, b: gnn_b200.graphAttentionEVGF(x, a, W, S, b)}
    oracle = {"ga": ao.graph_attention, "gl": ao.graph_attention_lsigf, "ge": ao.graph_attention_evgf}
    ref = run(oracle, ao.CooGSO(mats, "cuda", torch.float64), torch.float64)
    ref32 = run(oracle, ao.CooGSO(mats, "cuda", torch.float32), torch.float32)
    torch.cuda.empty_cache()
    for dtype in (torch.float64, torch.float32):
        S = gnn_b200.SparseGSO.from_scipy(mats, dtype=dtype)
        got = run(ours, S, dtype)
        worst = {k: _rel(got[k], ref[k]) for k in ref}
        print("%s %s at N = %d: worst relative error %s" % (kind, dtype, N, {k: "%.2g" % v for k, v in worst.items()}))
        if dtype == torch.float64:
            assert all(v < 1e-10 for v in worst.values()), worst
        else:
            plain = {k: _rel(ref32[k], ref[k]) for k in ref}
            print("  fp32 restatement: %s" % {k: "%.2g" % v for k, v in plain.items()})
            assert all(worst[k] <= 8 * plain[k] + 1e-6 for k in ref), (worst, plain)


@pytest.mark.gpu
def test_reference_network_trains_one_step_at_100k():
    """A GraphAttentionNetwork-shaped stack (two GraphAttentional layers, an MLP) at N = 100 000 through
    install(attention=True): one optimiser step, finite loss and gradients.  The reference's dense attention would need
    B*P*E*N*N = 2*2*1*1e10 values per layer (160 GB in fp32)."""
    import gnn_b200
    N, B = 100_000, 2
    S = gnn_b200.SparseGSO.from_scipy([_er(N, 16, 61)], dtype=torch.float32)
    gml = gnn_b200.install(_standin(), attention=True)
    try:
        torch.manual_seed(0)
        relu = nn.functional.relu
        net = nn.Sequential(gml.GraphAttentional(2, 4, 2, 1, relu, True), gml.GraphAttentional(8, 3, 2, 1, relu, False))
        mlp = nn.Linear(3 * N, 5)
        net, mlp = net.cuda(), mlp.cuda()
        for layer in net:
            layer.addGSO(S)
        opt = torch.optim.Adam(list(net.parameters()) + list(mlp.parameters()), lr=1e-3)
        x = torch.randn(B, 2, N, device="cuda")
        before = [p.detach().clone() for p in net.parameters()]
        loss = mlp(net(x).reshape(B, 3 * N)).square().mean()
        loss.backward()
        assert bool(torch.isfinite(loss)) and all(bool(torch.isfinite(p.grad).all()) and bool(p.grad.abs().sum() > 0)
                                                  for p in net.parameters())
        opt.step()
        assert all(not torch.equal(a, p) for a, p in zip(before, net.parameters()))
    finally:
        gnn_b200.uninstall(gml)
