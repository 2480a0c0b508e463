"""ARMA graph filters (gnn_b200.arma, csrc/arma/arma.cu) against fixtures produced by the unmodified reference
(tests/golden/arma_cases.npz <- oracle/make_golden_arma.py: jARMA, alegnn/utils/graphML.py:490-638; GraphFilterARMA
:2714-2847; ARMAfilterGNN, alegnn/modules/architectures.py:2243-2555).

CPU tests check the host logic (argument handling, bias forms, padding, parameters, install) with a torch restatement
standing in for the CUDA dispatch (`arma._dispatch`); GPU tests run both paths against the fixtures, against each other,
against the fp64 oracle's componentwise bound at scale (oracle/arma_oracle.py), and in a CUDA graph.  Each kernel launch
branch has a row in tests/test_arma_dispatch.py."""
import os
import types

import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.nn as nn

import arma_oracle as ao
import lsigf_oracle as orc

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "arma_cases.npz"))
TAGS = sorted({k.split("_")[1] for k in GOLD.files if k.startswith("arma_")})
LAYER_TAGS = sorted({k.split("_")[1] for k in GOLD.files if k.startswith("armal_")})


def _rel(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def _jarma_torch(psi, varphi, phi, S, x, b, tMax):
    """Differentiable dense restatement of the dispatch: the per-column Jacobi chains in the column convention, and the
    residue LSIGF in the row convention."""
    import gnn_b200
    if isinstance(S, gnn_b200.SparseGSO):
        S = S.to_dense()
    S = S.to(x.dtype)
    E, N = S.shape[0], S.shape[1]
    d = torch.diagonal(S, dim1=1, dim2=2)                                          # [E, N]
    St = S - torch.diag_embed(d)
    r = 1.0 / (d.reshape(1, E, 1, 1, N) - psi.unsqueeze(-1))                       # [F, E, P, G, N]
    xb = x.reshape(x.shape[0], 1, 1, 1, x.shape[1], N)
    z = r * xb
    zsum = z
    for t in range(1, tMax + 1):
        z = r * torch.einsum("bfepgj,eij->bfepgi", z, St)
        zsum = zsum + (-1.0) ** t * z
    y = xb.expand_as(z)
    for _ in range(tMax + 1):
        y = r * torch.einsum("bfepgj,eij->bfepgi", y, St)
    u = (zsum * varphi.unsqueeze(-1)).sum(dim=(2, 3, 4)) + (-1.0) ** (tMax + 1) * y.sum(dim=(2, 3, 4))
    cur = x.unsqueeze(1).expand(x.shape[0], E, x.shape[1], N)
    for k in range(phi.shape[2]):
        u = u + torch.einsum("begn,feg->bfn", cur, phi[:, :, k])
        cur = torch.matmul(cur, S.unsqueeze(0))
    return u if b is None else u + b


@pytest.fixture
def torch_dispatch(monkeypatch):
    from gnn_b200 import arma
    monkeypatch.setattr(arma, "_dispatch", _jarma_torch)


def _jarma_case(tag, dtype, device, path=None, sparse=False):
    import gnn_b200
    from gnn_b200 import arma
    p = "arma_%s_" % tag
    t = lambda k: torch.tensor(GOLD[p + k], dtype=dtype, device=device, requires_grad=True)   # noqa: E731
    ts = {k: t(k) for k in ("psi", "varphi", "phi", "x")}
    b = t("b") if p + "b" in GOLD.files else None
    S = torch.tensor(GOLD[p + "S"], dtype=dtype, device=device)
    if sparse:
        S = gnn_b200.SparseGSO.from_dense(S.cpu())
    tMax = int(GOLD[p + "meta"][8])
    if path is None:
        u = gnn_b200.jARMA(ts["psi"], ts["varphi"], ts["phi"], S, ts["x"], b, tMax=tMax)
    else:
        u = arma._dispatch_cuda(ts["psi"], ts["varphi"], ts["phi"], S, ts["x"], b, tMax, path=path)
    u.backward(torch.tensor(GOLD[p + "dU"], dtype=dtype, device=device))
    out = dict(u=(u, "u"))
    for k, v in ts.items():
        out["d" + k] = (v.grad, "d" + k)
    if b is not None:
        out["db"] = (b.grad, "db")
    return {k: (v.detach().cpu().numpy(), GOLD[p + ref]) for k, (v, ref) in out.items()}


def _layer_case(tag, dtype, device, sparse=False):
    import gnn_b200
    p = "armal_%s_" % tag
    seed, N, B, G, F, P, K, E, bias, tMax, Nin = (int(v) for v in GOLD[p + "meta"])
    layer = gnn_b200.GraphFilterARMA(G, F, P, K, E, bool(bias), tMax)
    S = torch.tensor(GOLD[p + "S"], dtype=dtype, device=device)
    layer.addGSO(gnn_b200.SparseGSO.from_dense(S.cpu()) if sparse else S)
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
              "GraphFilter_DB", "GRNN_DB", "HiddenState_DB", "EdgeGatedHiddenState", "NVGF", "NodeVariantGF", "jARMA",
              "GraphFilterARMA"):
        setattr(gml, n, type(n, (), {}))
    return gml


def _gnn_case(dtype, device):
    """The fixture's ARMAfilterGNN([2, 4, 3], [2, 1], [3, 2], True, nn.ReLU, [10, 6], MaxPoolLocal, [1, 2], [5], S,
    tMax=3) rebuilt from the layers install(arma=True) puts into a stand-in module, loaded with the reference network's
    parameters."""
    import gnn_b200
    gml = gnn_b200.install(_standin(), arma=True)
    try:
        N = int(GOLD["armagnn_meta"][1])
        B = int(GOLD["armagnn_meta"][2])
        S = torch.tensor(GOLD["armagnn_S"], dtype=dtype, device=device).reshape(1, N, N)
        net = nn.Module()
        net.jARMA = nn.Sequential(gml.GraphFilterARMA(2, 4, 2, 3, 1, True, 3), nn.ReLU(), gml.MaxPoolLocal(N, 10, 1),
                                  gml.GraphFilterARMA(4, 3, 1, 2, 1, True, 3), nn.ReLU(), gml.MaxPoolLocal(10, 6, 2))
        net.MLP = nn.Sequential(nn.Linear(6 * 3, 5, bias=True))
        for i in (0, 2, 3, 5):
            net.jARMA[i].addGSO(S)
        assert isinstance(net.jARMA[0], gnn_b200.GraphFilterARMA)
        sd = {k[len("armagnn_p_"):]: torch.tensor(GOLD[k]) for k in GOLD.files if k.startswith("armagnn_p_")}
        assert sorted(sd) == sorted(net.state_dict())
        net = net.to(device=device, dtype=dtype)
        net.load_state_dict(sd)
        x = torch.tensor(GOLD["armagnn_x"], dtype=dtype, device=device, requires_grad=True)
        y = net.MLP(net.jARMA(x).reshape(B, 3 * 6))
        y.backward(torch.tensor(GOLD["armagnn_dy"], dtype=dtype, device=device))
    finally:
        gnn_b200.uninstall(gml)
    out = dict(y=(y.detach(), GOLD["armagnn_y"]), dx=(x.grad, GOLD["armagnn_dx"]))
    for name, prm in net.named_parameters():
        out[name] = (prm.grad, GOLD["armagnn_g_" + name])
    return {k: (v.detach().cpu().numpy(), ref) for k, (v, ref) in out.items()}


# ------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("tag", TAGS)
def test_jarma_host_logic_matches_reference(tag, torch_dispatch):
    for name, (got, ref) in _jarma_case(tag, torch.float64, "cpu").items():
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


def test_every_bias_form_reaches_the_dispatch_as_lsigf_takes_it(torch_dispatch):
    import gnn_b200
    p = "arma_vt4_"
    args = [torch.tensor(GOLD[p + k]) for k in ("psi", "varphi", "phi")]
    S, x = torch.tensor(GOLD[p + "S"]), torch.tensor(GOLD[p + "x"])
    F_, N = args[0].shape[0], x.shape[2]
    b = torch.tensor(GOLD[p + "b"])                                               # [F, N]
    ref = gnn_b200.jARMA(*args, S, x, b, tMax=4)
    assert torch.allclose(gnn_b200.jARMA(*args, S, x, b.unsqueeze(0), tMax=4), ref, rtol=0, atol=0)
    b1 = b[:, :1]
    ref1 = gnn_b200.jARMA(*args, S, x, b1, tMax=4)
    assert torch.equal(gnn_b200.jARMA(*args, S, x, b1.unsqueeze(0), tMax=4), ref1)
    assert torch.equal(gnn_b200.jARMA(*args, S, x, b[:1].expand(F_, N)[:1], tMax=4),
                       gnn_b200.jARMA(*args, S, x, b[:1].expand(F_, N).contiguous(), tMax=4))
    with pytest.raises(RuntimeError, match="jARMA bias must"):
        gnn_b200.jARMA(*args, S, x, torch.zeros(F_ + 1, 1, dtype=torch.float64), tMax=4)


def test_state_dict_keys_and_seeded_parameters_match_the_reference():
    import gnn_b200
    for tag in LAYER_TAGS:
        p = "armal_%s_" % tag
        seed, N, B, G, F, P, K, E, bias, tMax, Nin = (int(v) for v in GOLD[p + "meta"])
        torch.manual_seed(seed)
        layer = gnn_b200.GraphFilterARMA(G, F, P, K, E, bool(bias), tMax).double()
        sd = layer.state_dict()
        ref = {k[len(p) + 2:]: GOLD[k] for k in GOLD.files if k.startswith(p + "p_")}
        assert list(sd) == list(ref)
        for k in ref:
            assert np.array_equal(sd[k].numpy(), ref[k]), (tag, k)
        assert layer.tMax == tMax and layer.P == P and layer.K == K
    assert repr(layer).startswith("GraphFilterARMA(in_features=%d, out_features=%d, denominator_taps=%d, "
                                  "residue_taps=%d, edge_features=%d, bias=%s, no GSO stored"
                                  % (G, F, P, K, E, bool(bias)))


def test_argument_checks_without_a_gpu():
    import gnn_b200
    psi = torch.full((2, 1, 2, 3), 3.0, dtype=torch.float64)
    phi = torch.zeros(2, 1, 2, 3, dtype=torch.float64)
    S = torch.eye(5, dtype=torch.float64).reshape(1, 5, 5)
    x = torch.zeros(1, 3, 5, dtype=torch.float64)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        gnn_b200.jARMA(psi, psi, phi, S, x)
    with pytest.raises(RuntimeError, match="bias must"):
        gnn_b200.jARMA(psi, psi, phi, S, x, torch.zeros(3, 1, dtype=torch.float64))
    with pytest.raises(AssertionError):                                           # reference's asserts
        gnn_b200.jARMA(psi, psi[:, :, :1], phi, S, x)
    with pytest.raises(AssertionError):
        gnn_b200.jARMA(psi, psi, phi, S, torch.zeros(1, 2, 5, dtype=torch.float64))
    with pytest.raises(ValueError, match="tMax"):
        gnn_b200.jARMA(psi, psi, phi, S, x, tMax=-1)
    with pytest.raises(TypeError, match="Plan"):
        gnn_b200.ArmaOperator(gnn_b200.Plan(None, 5, 5, 1, torch.float64, torch.device("cpu")))


def test_operator_flags_constant_diagonals_bitwise():
    import gnn_b200
    rng = np.random.default_rng(0)
    S = rng.uniform(-0.5, 0.5, (4, 6, 6))
    np.fill_diagonal(S[0], 0.0)
    np.fill_diagonal(S[1], 0.25)
    np.fill_diagonal(S[2], rng.uniform(-1, 1, 6))
    S[3, np.arange(6), np.arange(6)] = 0.25
    S[3, 4, 4] = np.nextafter(0.25, 1.0)                                          # one ulp off
    for gso in (torch.tensor(S), gnn_b200.SparseGSO.from_dense(torch.tensor(S))):
        op = gnn_b200.ArmaOperator(gso)
        assert op.constant == [True, True, False, False]
        assert op.const_value[:2] == [0.0, 0.25]
    St, _ = ao.split_gso([sp.csr_matrix(s) for s in S])
    for e in range(4):                                                           # the plans' CSR holds S~_e^T
        r, c, v = (np.asarray(a.cpu() if isinstance(a, torch.Tensor) else a) for a in op._csr[e])
        assert np.array_equal(sp.csr_matrix((v, c, r), shape=(6, 6)).toarray(), St[e].T.toarray())


def test_install_arma_is_opt_in():
    import gnn_b200
    gml = _standin()
    orig = {n: getattr(gml, n) for n in vars(gml) if not n.startswith("__")}
    try:
        gnn_b200.install(gml)
        assert gml.jARMA is orig["jARMA"] and gml.GraphFilterARMA is orig["GraphFilterARMA"]
        gnn_b200.install(gml, arma=True)
        assert gml.jARMA is gnn_b200.jARMA and gml.GraphFilterARMA is gnn_b200.GraphFilterARMA
    finally:
        gnn_b200.uninstall(gml)
    assert {n: getattr(gml, n) for n in orig} == orig
    try:
        gnn_b200.install(gml, arma=True, node_variant=True)
        assert gml.GraphFilterARMA is gnn_b200.GraphFilterARMA and gml.NodeVariantGF is gnn_b200.NodeVariantGF
    finally:
        gnn_b200.uninstall(gml)
    assert {n: getattr(gml, n) for n in orig} == orig


# ------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-11), (torch.float32, 1e-4)])
def test_fixtures_on_gpu(dtype, tol):
    for tag in TAGS:
        for sparse in (False, True):
            for name, (got, ref) in _jarma_case(tag, dtype, "cuda", sparse=sparse).items():
                assert _rel(got, ref) < tol, (tag, sparse, name)
    for tag in LAYER_TAGS:
        for sparse in (False, True):
            for name, (got, ref) in _layer_case(tag, dtype, "cuda", sparse).items():
                assert _rel(got, ref) < tol, (tag, sparse, name)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-11), (torch.float32, 1e-4)])
def test_both_paths_on_constant_diagonal_gsos(dtype, tol):
    """The general CUDA path run on constant-diagonal GSOs gives what the constant path (the default there) gives."""
    for tag in TAGS:
        if int(GOLD["arma_%s_meta" % tag][9]) not in (0, 1):
            continue
        gen = _jarma_case(tag, dtype, "cuda", path="general")
        con = _jarma_case(tag, dtype, "cuda", path="constant")
        for name in gen:
            assert _rel(gen[name][0], gen[name][1]) < tol, (tag, "general", name)
            assert _rel(con[name][0], con[name][1]) < tol, (tag, "constant", name)
            assert _rel(gen[name][0], con[name][0]) < 2 * tol, (tag, name)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-11), (torch.float32, 1e-4)])
def test_gnn_fixture_on_gpu(dtype, tol):
    for name, (got, ref) in _gnn_case(dtype, "cuda").items():
        assert _rel(got, ref) < tol, name


def _er(N, deg, seed, diag, dtype=np.float32):
    """Erdos-Renyi GSO, rows scaled to absolute sum <= 1, with a zero diagonal or a varying one in [-1, 1]."""
    rng = np.random.default_rng(seed)
    nnz = N * deg
    m = sp.csr_matrix((rng.standard_normal(nnz), (rng.integers(0, N, nnz), rng.integers(0, N, nnz))), shape=(N, N))
    m.sum_duplicates()
    m = sp.csr_matrix(m - sp.diags(m.diagonal()))
    m.eliminate_zeros()
    m = sp.diags(1.0 / np.maximum(np.abs(m).sum(axis=1).A.ravel(), 1.0)) @ m
    if diag == "vary":
        m = m + sp.diags(rng.uniform(-1, 1, N))
    m = sp.csr_matrix(m.astype(dtype).astype(np.float64))
    m.sort_indices()
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("diag", ["zero", "vary"])
def test_at_scale_vs_fp64_oracle(diag):
    """N = 200 000 Erdos-Renyi, degree 8, fp32, B = 2, F = G = 4, P = 2, K = 3, tMax = 3; a zero diagonal (constant
    path) or a varying one (general path): u and the gradients of x, psi, varphi, phi and b each held componentwise to
    the fp64 oracle's bound."""
    import gnn_b200
    N, B, G, F, P, K, tMax = 200_000, 2, 4, 4, 2, 3, 3
    mats = [_er(N, 8, 31, diag)]
    S = gnn_b200.SparseGSO.from_scipy(mats, dtype=torch.float32)
    assert gnn_b200.ArmaOperator(S).constant == [diag == "zero"]
    rng = np.random.default_rng(5)
    stdv = 1. / np.sqrt(G * P)
    r32 = lambda a: np.asarray(a, np.float32)                                    # noqa: E731
    psi = r32(rng.uniform(1 + 1 / stdv, 1 + 2 / stdv, (F, 1, P, G)))
    varphi, phi = r32(rng.uniform(-stdv, stdv, (F, 1, P, G))), r32(rng.uniform(-stdv, stdv, (F, 1, K, G)))
    x, b = r32(orc.biased_uniform(rng, (B, G, N))), r32(rng.uniform(-stdv, stdv, (F, 1)))
    dU = r32(orc.biased_uniform(rng, (B, F, N)))
    dev = lambda a: torch.tensor(a, device="cuda", requires_grad=True)           # noqa: E731
    ts = dict(psi=dev(psi), varphi=dev(varphi), phi=dev(phi), x=dev(x), b=dev(b))
    u = gnn_b200.jARMA(ts["psi"], ts["varphi"], ts["phi"], S, ts["x"], ts["b"], tMax=tMax)
    u.backward(torch.tensor(dU, device="cuda"))
    a64 = [np.asarray(a, np.float64) for a in (psi, varphi, phi, x, b, dU)]
    ref = ao.arma_backward(a64[0], a64[1], a64[2], mats, a64[3], a64[5], tMax, b.shape)
    ref["u"] = ao.arma_forward(a64[0], a64[1], a64[2], mats, a64[3], a64[4], tMax)
    env = ao.arma_envelope(a64[0], a64[1], a64[2], mats, a64[3], a64[4], a64[5], tMax, np.float32)
    env["u"] = env["y"]
    got = dict(u=u, dx=ts["x"].grad, dpsi=ts["psi"].grad, dvarphi=ts["varphi"].grad, dphi=ts["phi"].grad,
               db=ts["b"].grad)
    worst = {k: orc.bound_violation(v.detach().double().cpu().numpy(), ref[k], env[k]) for k, v in got.items()}
    print("at scale (%s diagonal), worst error / bound:" % diag, {k: "%.3g" % v for k, v in worst.items()})
    assert all(v <= 1.0 for v in worst.values()), worst


@pytest.mark.gpu
@pytest.mark.parametrize("diag", ["zero", "vary"])
def test_graphed_forward_backward_is_bit_identical_to_eager(diag):
    import gnn_b200
    N, B, G, F, P, K, E = 20000, 2, 4, 3, 2, 3, 2
    mats = [_er(N, 8, 41, diag), _er(N, 8, 42, "vary")]                         # E = 2: the second always general
    S = gnn_b200.SparseGSO.from_scipy(mats, dtype=torch.float32)
    torch.manual_seed(3)
    layer = gnn_b200.GraphFilterARMA(G, F, P, K, E, True, 3).cuda()
    layer.addGSO(S)
    rng = np.random.default_rng(1)
    x = torch.tensor(rng.standard_normal((B, G, N)), dtype=torch.float32, device="cuda", requires_grad=True)
    dy = torch.tensor(rng.standard_normal((B, F, N)), dtype=torch.float32, device="cuda")
    tensors = list(layer.parameters()) + [x]

    def step():
        layer(x).backward(dy)

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
