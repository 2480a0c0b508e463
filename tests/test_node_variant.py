"""Node-variant graph filters (gnn_b200.nodevariant, csrc/nv/nv.cu) against fixtures produced by the unmodified reference
(tests/golden/nvgf_cases.npz <- oracle/make_golden_nv.py: NVGF, alegnn/utils/graphML.py:293-387; NodeVariantGF
:2317-2509; NodeVariantGNN, alegnn/modules/architectures.py:1485-1719).

CPU tests check the host logic (argument handling, copyNodes, padding, tap map, parameters, install) with a torch
restatement standing in for the CUDA dispatch (`nodevariant._dispatch`); GPU tests run the kernels against the fixtures,
the fp64 oracle's componentwise bound (oracle/nv_oracle.py), GraphFilter, a CUDA graph, and at scale.  Each kernel
branch has a row in tests/test_nv_dispatch.py."""
import os
import types

import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.nn as nn

import lsigf_oracle as orc
import nv_oracle as nvo

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "nvgf_cases.npz"))
NVGF_TAGS = sorted({k.split("_")[1] for k in GOLD.files if k.startswith("nvgf_")})
LAYER_TAGS = sorted({k.split("_")[1] for k in GOLD.files if k.startswith("nvl_")})


def _rel(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def _nvgf_torch(h, S, x, b, taps):
    """Differentiable dense restatement of the dispatch: h[..., node_tap] and the reference's shift / sum order."""
    import gnn_b200
    if isinstance(S, gnn_b200.SparseGSO):
        S = S.to_dense()
    S = S.to(x.dtype)
    ht = h.index_select(4, taps.node_tap.long())
    F_, E, K, G, N = ht.shape
    B = x.shape[0]
    z = x.reshape(B, 1, G, N).repeat(1, E, 1, 1)
    zs = [z]
    for _ in range(1, K):
        z = torch.matmul(z, S.reshape(1, E, N, N))
        zs.append(z)
    Z = torch.stack(zs, dim=2)                                         # [B, E, K, G, N]
    y = (Z.reshape(B, 1, E, K, G, N) * ht.reshape(1, F_, E, K, G, N)).sum(dim=(2, 3, 4))
    return y if b is None else y + b


@pytest.fixture
def torch_dispatch(monkeypatch):
    from gnn_b200 import nodevariant as nvm
    monkeypatch.setattr(nvm, "_dispatch", _nvgf_torch)


def _nvgf_case(tag, dtype, device):
    import gnn_b200
    p = "nvgf_%s_" % tag
    t = lambda k: torch.tensor(GOLD[p + k], dtype=dtype, device=device, requires_grad=True)   # noqa: E731
    h, x = t("h"), t("x")
    b = t("b") if p + "b" in GOLD.files else None
    y = gnn_b200.NVGF(h, torch.tensor(GOLD[p + "S"], dtype=dtype, device=device), x, b)
    y.backward(torch.tensor(GOLD[p + "dy"], dtype=dtype, device=device))
    out = dict(y=(y, "y"), dx=(x.grad, "dx"), dh=(h.grad, "dh"))
    if b is not None:
        out["db"] = (b.grad, "db")
    return {k: (v.detach().cpu().numpy(), GOLD[p + ref]) for k, (v, ref) in out.items()}


def _layer_case(tag, dtype, device, sparse=False):
    import gnn_b200
    p = "nvl_%s_" % tag
    seed, N, B, G, F, K, M, E, bias, Nin = (int(v) for v in GOLD[p + "meta"])
    layer = gnn_b200.NodeVariantGF(G, F, K, M, E, bool(bias))
    S = torch.tensor(GOLD[p + "S"], dtype=dtype, device=device)
    layer.addGSO(gnn_b200.SparseGSO.from_dense(S.cpu()).astype(dtype) if sparse else S)
    assert list(layer.copyNodes.cpu().numpy()) == list(GOLD[p + "copyNodes"])
    sd = {k[len(p) + 2:]: torch.tensor(GOLD[k]) for k in GOLD.files if k.startswith(p + "p_")}
    assert list(sd) == list(layer.state_dict())
    layer.load_state_dict(sd)
    layer = layer.to(device=device, dtype=dtype)
    x = torch.tensor(GOLD[p + "x"], dtype=dtype, device=device, requires_grad=True)
    y = layer(x)
    assert tuple(y.shape) == (B, F, Nin)
    y.backward(torch.tensor(GOLD[p + "dy"], dtype=dtype, device=device))
    out = dict(y=(y, "y"), dx=(x.grad, "dx"))
    for name, prm in layer.named_parameters():
        out[name] = (prm.grad, "g_" + name)
    return {k: (v.detach().cpu().numpy(), GOLD[p + ref]) for k, (v, ref) in out.items()}


def _standin():
    gml = types.ModuleType("graphML_standin")
    for n in ("LSIGF", "GraphFilter", "EVGF", "EdgeVariantGF", "MaxPoolLocal", "MaxLocalActivation",
              "MedianLocalActivation", "HiddenState", "TimeGatedHiddenState", "NodeGatedHiddenState", "LSIGF_DB",
              "GraphFilter_DB", "GRNN_DB", "HiddenState_DB", "EdgeGatedHiddenState", "NVGF", "NodeVariantGF"):
        setattr(gml, n, type(n, (), {}))
    return gml


def _gnn_case(dtype, device):
    """The fixture's NodeVariantGNN([2, 4, 3], [3, 2], [5, 6], True, nn.ReLU, [10, 6], MaxPoolLocal, [1, 2], [5], S)
    rebuilt from the layers install(node_variant=True) puts into a stand-in module, loaded with the reference network's
    parameters."""
    import gnn_b200
    gml = gnn_b200.install(_standin(), node_variant=True)
    try:
        N = int(GOLD["nvgnn_meta"][1])
        B = int(GOLD["nvgnn_meta"][2])
        S = torch.tensor(GOLD["nvgnn_S"], dtype=dtype, device=device).reshape(1, N, N)
        net = nn.Module()
        net.NVGFL = nn.Sequential(gml.NodeVariantGF(2, 4, 3, 5, 1, True), nn.ReLU(), gml.MaxPoolLocal(N, 10, 1),
                                  gml.NodeVariantGF(4, 3, 2, 6, 1, True), nn.ReLU(), gml.MaxPoolLocal(10, 6, 2))
        net.MLP = nn.Sequential(nn.Linear(6 * 3, 5, bias=True))
        for i in (0, 2, 3, 5):
            net.NVGFL[i].addGSO(S)
        assert isinstance(net.NVGFL[0], gnn_b200.NodeVariantGF)
        sd = {k[len("nvgnn_p_"):]: torch.tensor(GOLD[k]) for k in GOLD.files if k.startswith("nvgnn_p_")}
        assert sorted(sd) == sorted(net.state_dict())
        net = net.to(device=device, dtype=dtype)
        net.load_state_dict(sd)
        assert list(net.NVGFL[0].copyNodes.cpu().numpy()) == list(GOLD["nvgnn_copy0"])
        assert list(net.NVGFL[3].copyNodes.cpu().numpy()) == list(GOLD["nvgnn_copy3"])
        x = torch.tensor(GOLD["nvgnn_x"], dtype=dtype, device=device, requires_grad=True)
        y = net.MLP(net.NVGFL(x).reshape(B, 3 * 6))
        y.backward(torch.tensor(GOLD["nvgnn_dy"], dtype=dtype, device=device))
    finally:
        gnn_b200.uninstall(gml)
    out = dict(y=(y.detach(), GOLD["nvgnn_y"]), dx=(x.grad, GOLD["nvgnn_dx"]))
    for name, prm in net.named_parameters():
        out[name] = (prm.grad, GOLD["nvgnn_g_" + name])
    return {k: (v.detach().cpu().numpy(), ref) for k, (v, ref) in out.items()}


# ------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("tag", NVGF_TAGS)
def test_nvgf_host_logic_matches_reference(tag, torch_dispatch):
    for name, (got, ref) in _nvgf_case(tag, torch.float64, "cpu").items():
        assert _rel(got, ref) < 1e-12, name


@pytest.mark.parametrize("sparse", [False, True])
@pytest.mark.parametrize("tag", LAYER_TAGS)
def test_layer_host_logic_matches_reference(tag, sparse, torch_dispatch):
    for name, (got, ref) in _layer_case(tag, torch.float64, "cpu", sparse).items():
        assert _rel(got, ref) < 1e-12, name


def test_gnn_host_logic_matches_reference(torch_dispatch, monkeypatch):
    from gnn_b200 import pooling

    def gather_max(x, nb32, n_out, max_nb):
        B, F, _ = x.shape
        return x.index_select(2, nb32.reshape(-1).long()).reshape(B, F, n_out, max_nb).max(dim=3)[0]
    monkeypatch.setattr(pooling, "_gather_max", gather_max)
    for name, (got, ref) in _gnn_case(torch.float64, "cpu").items():
        assert _rel(got, ref) < 1e-12, name


def test_state_dict_keys_and_seeded_parameters_match_the_reference():
    import gnn_b200
    for tag in LAYER_TAGS:
        p = "nvl_%s_" % tag
        seed, N, B, G, F, K, M, E, bias, Nin = (int(v) for v in GOLD[p + "meta"])
        torch.manual_seed(seed)
        layer = gnn_b200.NodeVariantGF(G, F, K, M, E, bool(bias)).double()
        sd = layer.state_dict()
        ref = {k[len(p) + 2:]: GOLD[k] for k in GOLD.files if k.startswith(p + "p_")}
        assert list(sd) == list(ref)
        for k in ref:
            assert np.array_equal(sd[k].numpy(), ref[k]), (tag, k)
    assert repr(layer).startswith("NodeVariantGF(in_features=%d, out_features=%d, shift_taps=%d, node_taps=%d, "
                                  "edge_features=%d, bias=True, no GSO stored" % (G, F, K, M, E))


def test_tap_map_lists_the_nodes_of_every_tap():
    import gnn_b200
    copy = np.array([0, 1, 2, 3, 3, 0, 0, 0, 0, 0])
    tm = gnn_b200.TapMap(copy, 6)
    rp, nodes = tm.tap_rowptr.numpy(), tm.tap_nodes.numpy()
    assert list(rp) == [0, 6, 7, 8, 10, 10, 10]
    for m in range(6):
        assert list(nodes[rp[m]:rp[m + 1]]) == sorted(np.nonzero(copy == m)[0])
    with pytest.raises(ValueError):
        gnn_b200.TapMap([0, 4], 4)


def test_argument_checks_without_a_gpu():
    import gnn_b200
    h = torch.zeros(2, 1, 2, 3, 5, dtype=torch.float64)
    S = torch.eye(5, dtype=torch.float64).reshape(1, 5, 5)
    x = torch.zeros(1, 3, 5, dtype=torch.float64)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        gnn_b200.NVGF(h, S, x)
    with pytest.raises(RuntimeError, match="bias must be"):
        gnn_b200.NVGF(h, S, x, torch.zeros(3, 1, dtype=torch.float64))
    with pytest.raises(AssertionError):
        gnn_b200.NVGF(h, S, torch.zeros(1, 2, 5, dtype=torch.float64))
    layer = gnn_b200.NodeVariantGF(3, 2, 2, 2)
    with pytest.raises(TypeError, match="Plan"):
        gnn_b200.nodevariant.gso_pattern(gnn_b200.Plan(None, 5, 5, 1, torch.float64, torch.device("cpu")))
    with pytest.raises(ValueError, match="3 node"):               # S = I: nodes 2, 3, 4 reach nothing
        layer.addGSO(S)


def test_install_node_variant_is_opt_in():
    import gnn_b200
    gml = _standin()
    names = list(vars(gml))
    orig = {n: getattr(gml, n) for n in names if not n.startswith("__")}
    try:
        gnn_b200.install(gml)
        assert gml.NVGF is orig["NVGF"] and gml.NodeVariantGF is orig["NodeVariantGF"]
        gnn_b200.install(gml, node_variant=True)
        assert gml.NVGF is gnn_b200.NVGF and gml.NodeVariantGF is gnn_b200.NodeVariantGF
    finally:
        gnn_b200.uninstall(gml)
    assert {n: getattr(gml, n) for n in orig} == orig
    try:
        gnn_b200.install(gml, node_variant=True, edge_gating=True)
        assert gml.NodeVariantGF is gnn_b200.NodeVariantGF
    finally:
        gnn_b200.uninstall(gml)
    assert {n: getattr(gml, n) for n in orig} == orig


# ------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-10), (torch.float32, 1e-4)])
def test_fixtures_on_gpu(dtype, tol):
    for tag in NVGF_TAGS:
        for name, (got, ref) in _nvgf_case(tag, dtype, "cuda").items():
            assert _rel(got, ref) < tol, (tag, name)
    for tag in LAYER_TAGS:
        for sparse in (False, True):
            for name, (got, ref) in _layer_case(tag, dtype, "cuda", sparse).items():
                assert _rel(got, ref) < tol, (tag, sparse, name)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-10), (torch.float32, 1e-4)])
def test_gnn_fixture_on_gpu(dtype, tol):
    for name, (got, ref) in _gnn_case(dtype, "cuda").items():
        assert _rel(got, ref) < tol, name


def _er(N, deg, seed, E=1, dtype=np.float32):
    rng = np.random.default_rng(seed)
    mats = []
    for _ in range(E):
        nnz = N * deg
        m = sp.csr_matrix((rng.standard_normal(nnz), (rng.integers(0, N, nnz), rng.integers(0, N, nnz))), shape=(N, N))
        m.sum_duplicates()
        m = sp.diags(1.0 / np.maximum(np.abs(m).sum(axis=1).A.ravel(), 1.0)) @ m
        m = sp.csr_matrix(m.astype(dtype).astype(np.float64))
        m.sort_indices()
        mats.append(m)
    return mats


@pytest.mark.gpu
def test_m1_agrees_with_graph_filter():
    """M = 1: every node reads tap 0, so NodeVariantGF is GraphFilter with weight[..., 0]; both within the bound."""
    import gnn_b200
    N, B, G, F, K, E = 5000, 3, 6, 5, 3, 2
    mats = _er(N, 8, 5, E)
    S = gnn_b200.SparseGSO.from_scipy(mats, dtype=torch.float32)
    nv = gnn_b200.NodeVariantGF(G, F, K, 1, E).cuda()
    nv.addGSO(S)
    gf = gnn_b200.GraphFilter(G, F, K, E).cuda()
    gf.addGSO(S)
    with torch.no_grad():
        gf.weight.copy_(nv.weight[..., 0])
        gf.bias.copy_(nv.bias)
    rng = np.random.default_rng(0)
    x = rng.standard_normal((B, G, N)).astype(np.float32)
    env = nvo.nv_envelope(nv.weight.detach().double().cpu().numpy(), np.zeros(N, np.int64), mats, x,
                          nv.bias.detach().double().cpu().numpy(), np.ones((B, F, N)), np.float32)
    ref = nvo.nv_forward(nv.weight.detach().double().cpu().numpy(), np.zeros(N, np.int64), mats, x,
                         nv.bias.detach().double().cpu().numpy())
    xt = torch.tensor(x, device="cuda")
    y_nv, y_gf = nv(xt).detach().cpu().numpy(), gf(xt).detach().cpu().numpy()
    assert orc.bound_violation(y_nv, ref, env["y"]) <= 1.0
    assert orc.bound_violation(y_gf, ref, 2 * env["y"]) <= 1.0       # GraphFilter: 3xTF32 or FMA, same envelope x2
    assert orc.bound_violation(y_nv, y_gf, 3 * env["y"]) <= 1.0


@pytest.mark.gpu
def test_graphed_forward_backward_is_bit_identical_to_eager():
    import gnn_b200
    N, B, G, F, K, E, M = 20000, 4, 8, 8, 3, 2, 2000
    S = gnn_b200.SparseGSO.from_scipy(_er(N, 8, 9, E), dtype=torch.float32)
    torch.manual_seed(3)
    layer = gnn_b200.NodeVariantGF(G, F, K, M, E).cuda()
    layer.addGSO(S)
    rng = np.random.default_rng(1)
    x = torch.tensor(rng.standard_normal((B, G, N)), dtype=torch.float32, device="cuda", requires_grad=True)
    dy = torch.tensor(rng.standard_normal((B, F, N)), dtype=torch.float32, device="cuda")

    def step():
        layer(x).backward(dy)

    for p in list(layer.parameters()) + [x]:
        p.grad = None
    step()
    eager = [t.grad.clone() for t in list(layer.parameters()) + [x]]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            for p in list(layer.parameters()) + [x]:
                p.grad = None
            step()
    torch.cuda.current_stream().wait_stream(side)
    for p in list(layer.parameters()) + [x]:
        p.grad = None
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    g.replay()
    torch.cuda.synchronize()
    replay = [t.grad.clone() for t in list(layer.parameters()) + [x]]
    assert all(torch.equal(a, b) for a, b in zip(eager, replay))


@pytest.mark.gpu
def test_at_scale_vs_fp64_oracle():
    """N = 200 000 Erdos-Renyi, degree 16, fp32, E = 2, K = 4, M = N / 10: y, x.grad, weight.grad and bias.grad are each
    held componentwise to the fp64 oracle's bound."""
    import gnn_b200
    N, B, G, F, K, E = 200_000, 4, 8, 6, 4, 2
    M = N // 10
    mats = _er(N, 16, 21, E)
    S = gnn_b200.SparseGSO.from_scipy(mats, dtype=torch.float32)
    torch.manual_seed(4)
    layer = gnn_b200.NodeVariantGF(G, F, K, M, E).cuda()
    layer.addGSO(S)
    rng = np.random.default_rng(2)
    x = orc.biased_uniform(rng, (B, G, N)).astype(np.float32)
    dy = orc.biased_uniform(rng, (B, F, N)).astype(np.float32)
    xt = torch.tensor(x, device="cuda", requires_grad=True)
    y = layer(xt)
    y.backward(torch.tensor(dy, device="cuda"))
    h = layer.weight.detach().double().cpu().numpy()
    b = layer.bias.detach().double().cpu().numpy()
    copy = layer.copyNodes.cpu().numpy()
    env = nvo.nv_envelope(h, copy, mats, x, b, dy, np.float32)
    dxr, dhr, dbr = nvo.nv_backward(h, copy, mats, x, dy, b.shape)
    worst = {}
    for name, got, ref, bound in (("y", y, nvo.nv_forward(h, copy, mats, x, b), env["y"]), ("dx", xt.grad, dxr, env["dx"]),
                                  ("dh", layer.weight.grad, dhr, env["dh"]), ("db", layer.bias.grad, dbr, env["db"])):
        worst[name] = orc.bound_violation(got.detach().double().cpu().numpy(), ref, bound)
    print("at scale, worst error / bound:", worst)
    assert all(v <= 1.0 for v in worst.values()), worst
