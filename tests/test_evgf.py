"""Edge-variant filter (SURVEY.md §8 a-7): EVGF / EdgeVariantGF.
CPU: the numpy oracle vs fixtures produced by the unmodified reference (oracle/make_golden.py::gen_evgf).
GPU: the sparse CUDA execution (csrc/ev.cu through gnn_b200.EVGF / EdgeVariantGF) vs the same fixtures."""
import os

import numpy as np
import pytest
import torch

import lsigf_oracle as orc


def _rel(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


@pytest.fixture(scope="module")
def z(golden_dir):
    return np.load(os.path.join(golden_dir, "evgf_cases.npz"))


def test_oracle_evgf_functional(z):
    y = orc.evgf_dense(z["f_Phi"], z["f_x"], z["f_b"])
    assert _rel(y, z["f_y"]) < 1e-12


@pytest.mark.parametrize("tag", ["full", "hyb"])
def test_oracle_edge_variant_layer(z, tag):
    N, M, E, K, G, F, B, Nin = [int(v) for v in z[tag + "_meta"]]
    x = z[tag + "_x"]
    if Nin < N:
        x = np.concatenate([x, np.zeros((B, G, N - Nin))], axis=2)
    wl = z[tag + "_p_weightLSI"] if (tag + "_p_weightLSI") in z.files else None
    y = orc.edge_variant_gf_forward(z[tag + "_p_weightEV"], wl, z[tag + "_p_bias"], z[tag + "_S"], M, x)[:, :, :Nin]
    assert _rel(y, z[tag + "_y"]) < 1e-12


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-11), (torch.float32, 1e-4)])
def test_evgf_functional_gpu(z, dtype, tol):
    import gnn_b200
    Phi = torch.tensor(z["f_Phi"], dtype=dtype, device="cuda", requires_grad=True)
    x = torch.tensor(z["f_x"], dtype=dtype, device="cuda", requires_grad=True)
    b = torch.tensor(z["f_b"], dtype=dtype, device="cuda", requires_grad=True)
    y = gnn_b200.EVGF(Phi, x, b)
    y.backward(torch.tensor(z["f_dy"], dtype=dtype, device="cuda"))
    assert _rel(y.detach().cpu().numpy(), z["f_y"]) < tol
    assert _rel(x.grad.cpu().numpy(), z["f_dx"]) < tol
    assert _rel(b.grad.cpu().numpy(), z["f_db"]) < tol
    # gradient on the sparsity pattern (entries of Phi that are exactly zero are not parameters of the sparse filter)
    assert _rel(Phi.grad.cpu().numpy(), z["f_dPhi"]) < tol


@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["full", "hyb"])
@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-11), (torch.float32, 1e-4)])
def test_edge_variant_layer_gpu(z, tag, dtype, tol):
    """Reference parameter names/shapes load as a state_dict; output, dx and every parameter gradient match the
    reference layer (hybrid: LSI part through the CUDA LSIGF, bias counted twice as in graphML.py:2682,2686)."""
    import gnn_b200
    N, M, E, K, G, F, B, Nin = [int(v) for v in z[tag + "_meta"]]
    layer = gnn_b200.EdgeVariantGF(G, F, K, M, N, E, True).to("cuda", dtype)
    sd = {k[len(tag) + 3:]: torch.tensor(z[k], dtype=dtype, device="cuda") for k in z.files if k.startswith(tag + "_p_")}
    layer.load_state_dict(sd)
    layer.addGSO(torch.tensor(z[tag + "_S"], dtype=dtype, device="cuda"))
    x = torch.tensor(z[tag + "_x"], dtype=dtype, device="cuda", requires_grad=True)
    y = layer(x)
    assert tuple(y.shape) == z[tag + "_y"].shape
    y.backward(torch.tensor(z[tag + "_dy"], dtype=dtype, device="cuda"))
    assert _rel(y.detach().cpu().numpy(), z[tag + "_y"]) < tol
    assert _rel(x.grad.cpu().numpy(), z[tag + "_dx"]) < tol
    for name, p in layer.named_parameters():
        assert _rel(p.grad.cpu().numpy(), z[tag + "_g_" + name]) < tol, name


@pytest.mark.gpu
def test_hybrid_edge_variant_at_scale():
    """cfg4-shaped hybrid at a size the dense reference cannot hold: the EV part lives on the compact node set; checked
    against the fp64 oracle chain evaluated sparsely on that set."""
    import scipy.sparse as sp
    import gnn_b200
    from gnn_b200 import edgevariant as evm
    rng = np.random.default_rng(5)
    N, M, E, K, G, F, B = 3000, 24, 2, 3, 4, 4, 3
    pats = []
    for e in range(E):
        m = sp.random(N, N, density=8.0 / N, format="csr", random_state=np.random.RandomState(e)) + sp.eye(N)
        pats.append(torch.tensor((m != 0).toarray()))
    pattern = torch.stack(pats).cuda()
    idx = torch.arange(N, device="cuda")
    pattern = pattern & ((idx[:, None] < M) | (idx[None, :] < M))[None]
    st = evm.EVStructure(pattern)
    assert st.NA < N // 2                                   # the compact set is what makes the hybrid layer tractable
    xA = torch.randn(B, G, st.NA, dtype=torch.float64, device="cuda")
    y_ref = torch.zeros(B, F, st.NA, dtype=torch.float64, device="cuda")
    y = torch.zeros_like(y_ref)
    for e in range(E):
        pe = st.per_e[e]
        w = torch.randn(F, K, G, pe["nnz"], dtype=torch.float64, device="cuda") * 0.3
        y = y + evm._EVChain.apply(w, xA, pe, st.NA, False)
        rows, cols = pe["rowidx"].long(), pe["col"].long()
        for f in range(F):
            for g in range(G):
                u = xA[:, g, :]
                for k in range(K):
                    Phi = torch.zeros(st.NA, st.NA, dtype=torch.float64, device="cuda")
                    Phi[rows, cols] = w[f, k, g]
                    u = u @ Phi.t()
                    y_ref[:, f, :] += u
    assert _rel(y.cpu().numpy(), y_ref.cpu().numpy()) < 1e-11


# ------------------------------------------------------------------------------------------------ sparse-parameter layer
def _dense_chain(w, xA, pe, NA, k0_identity=False):
    """torch stand-in for csrc/ev.cu (CPU leg only): scatter the per-non-zero weights into dense NA x NA matrices and run
    the chains u_k = Phi^(k) u_{k-1} of graphML.py:455-478."""
    F_, K, G, nnz = w.shape
    rows, cols = pe["rowidx"].long(), pe["col"].long()
    y = 0
    for k_mask in [None]:
        Phi = torch.zeros(F_, K, G, NA, NA, dtype=w.dtype)
        wk = w
        if k0_identity:
            on = (rows == cols).to(w.dtype)
            wk = torch.cat((w[:, :1] * on, w[:, 1:]), dim=1)
        Phi[:, :, :, rows, cols] = wk
        u = xA.permute(1, 2, 0)[None].expand(F_, G, NA, xA.shape[0])              # [F, G, NA, B]
        for k in range(K):
            u = torch.einsum("fgij,fgjb->fgib", Phi[:, k], u)
            y = y + u.sum(1)
    return y.permute(2, 0, 1)                                                       # [B, F, NA]


def _sparse_layer_from_fixture(z, tag, dtype, device):
    import gnn_b200
    N, M, E, K, G, F, B, Nin = [int(v) for v in z[tag + "_meta"]]
    layer = gnn_b200.SparseEdgeVariantGF(G, F, K, M, N, E, True).to(device, dtype)
    S = torch.tensor(z[tag + "_S"], dtype=dtype, device=device)
    layer.addGSO(S, device=device)
    layer.load_dense_state(torch.tensor(z[tag + "_p_weightEV"], dtype=dtype),
                           torch.tensor(z[tag + "_p_weightLSI"], dtype=dtype) if (tag + "_p_weightLSI") in z.files else None,
                           torch.tensor(z[tag + "_p_bias"], dtype=dtype))
    return layer, (N, M, E, K, G, F, B, Nin)


def _check_sparse_layer(z, tag, layer, dims, dtype, device, tol):
    N, M, E, K, G, F, B, Nin = dims
    x = torch.tensor(z[tag + "_x"], dtype=dtype, device=device, requires_grad=True)
    y = layer(x)
    assert tuple(y.shape) == z[tag + "_y"].shape
    y.backward(torch.tensor(z[tag + "_dy"], dtype=dtype, device=device))
    assert _rel(y.detach().cpu().numpy(), z[tag + "_y"]) < tol
    assert _rel(x.grad.cpu().numpy(), z[tag + "_dx"]) < tol
    gEV = z[tag + "_g_weightEV"]                                                     # dense reference gradient
    for e, (p, pe) in enumerate(zip(layer.weightEV, layer._struct.per_e)):
        want = gEV[:, e].reshape(F, K, G, N * N)[..., pe["lin"].cpu().numpy()]
        assert _rel(p.grad.cpu().numpy(), want) < tol, ("weightEV", e)
        off = (pe["rowidx"] != pe["col"]).cpu().numpy()
        assert np.all(p.grad.cpu().numpy()[:, 0][..., off] == 0)                     # k = 0 off-diagonal slots: no gradient
    if layer.weightLSI is not None:
        assert _rel(layer.weightLSI.grad.cpu().numpy(), z[tag + "_g_weightLSI"]) < tol
    assert _rel(layer.bias.grad.cpu().numpy(), z[tag + "_g_bias"]) < tol
    # everything the reference layer would have as a parameter is there: masked entries only
    dense_live = (z[tag + "_g_weightEV"] != 0).sum()
    assert sum(p.numel() for p in layer.weightEV) >= dense_live


@pytest.mark.parametrize("tag", ["full", "hyb"])
def test_sparse_edge_variant_layer_host_logic(z, tag, monkeypatch):
    """SparseEdgeVariantGF (parameters per masked non-zero) reproduces the reference layer from its dense checkpoint:
    output, dx, and the gradient of every live parameter.  CPU: dense torch chain / oracle LSIGF behind the two hooks."""
    from gnn_b200 import edgevariant as evm, graphML
    monkeypatch.setattr(evm, "_chain", _dense_chain)
    monkeypatch.setattr(graphML, "_dispatch", lambda h, S, x, b, act=0: orc.lsigf_dense_torch(h, S, x, b))
    layer, dims = _sparse_layer_from_fixture(z, tag, torch.float64, "cpu")
    monkeypatch.setattr(evm, "_require_cuda", lambda x: None)                        # the product forward itself runs
    _check_sparse_layer(z, tag, layer, dims, torch.float64, "cpu", 1e-11)
    monkeypatch.undo()
    with pytest.raises(RuntimeError, match="no CPU fallback"):                       # product behaviour on CPU tensors
        layer(torch.zeros(1, dims[4], dims[0], dtype=torch.float64))
    # round trip to the reference's dense parameter
    dense = layer.dense_weightEV().numpy()
    mask = z[tag + "_g_weightEV"] != 0
    assert np.allclose(dense[mask], z[tag + "_p_weightEV"][mask])


@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["full", "hyb"])
@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-11), (torch.float32, 1e-4)])
def test_sparse_edge_variant_layer_gpu(z, tag, dtype, tol):
    layer, dims = _sparse_layer_from_fixture(z, tag, dtype, "cuda")
    _check_sparse_layer(z, tag, layer, dims, dtype, "cuda", tol)


def _twin_fp64(layer, gso, x, dy, absolute):
    """The fp32 layer's parameters and inputs cast to fp64 (absolute values when `absolute`: the run that gives the
    magnitudes M of the error envelope) through the same kernels -> (y, x.grad, [weightEV[e].grad])."""
    import gnn_b200
    f = (lambda t: t.detach().double().abs()) if absolute else (lambda t: t.detach().double())   # noqa: E731
    g64 = gso.astype(torch.float64)
    if absolute:
        g64 = gnn_b200.SparseGSO([(r, c, np.abs(v)) for (r, c, v) in g64.csr], g64.N)
    twin = gnn_b200.SparseEdgeVariantGF(layer.G, layer.F, layer.K, layer.M, layer.N, layer.E, True).to("cuda", torch.float64)
    twin.addGSO(g64, device="cuda")
    with torch.no_grad():
        twin.weightLSI.copy_(f(layer.weightLSI))
        twin.bias.copy_(f(layer.bias))
        for p64, p, pe64, pe in zip(twin.weightEV, layer.weightEV, twin._struct.per_e, layer._struct.per_e):
            assert torch.equal(pe64["col"], pe["col"]) and torch.equal(pe64["rowptr"], pe["rowptr"])
            p64.copy_(f(p))
    x64 = f(x).requires_grad_(True)
    y64 = twin(x64)
    y64.backward(f(dy))
    return y64.detach(), x64.grad, [p.grad for p in twin.weightEV]


@pytest.mark.gpu
def test_sparse_edge_variant_cfg4_size():
    """BASELINE.json config 4 at its stated size: N = 200k, E = 4, K = 3, G = F = 32, hybrid with M = 1024 selected nodes —
    the reference layer would need 32*4*3*32*4e10 parameters.  Constructs, runs forward + backward, and checks the EV part
    against an fp64 evaluation of the same chains on a sub-sample of (f, g) pairs.  y, x.grad and every weightEV[e].grad
    are held componentwise to the envelope of ev_oracle / lsigf_oracle around the same layer run in fp64 through the same
    kernels (their fp64 results are pinned by tests/test_kernel_dispatch.py), M taken from an fp64 run on absolute values."""
    import ev_oracle as evo
    import gnn_b200
    from gnn_b200 import graphs
    N, M, E, K, G, F, B = 200_000, 1024, 4, 3, 32, 32, 8
    gso = graphs.er_gso(N, 16, seed=4, E=E)
    layer = gnn_b200.SparseEdgeVariantGF(G, F, K, M, N, E, True).to("cuda")
    layer.addGSO(gso, device="cuda")
    st = layer._struct
    n_par = sum(p.numel() for p in layer.weightEV)
    assert st.NA < N // 4 and 1e7 < n_par < 1e9
    x = torch.randn(B, G, N, device="cuda", requires_grad=True)
    dy = torch.randn(B, F, N, device="cuda")
    y = layer(x)
    y.backward(dy)
    torch.cuda.synchronize()
    assert tuple(y.shape) == (B, F, N) and torch.isfinite(y).all() and torch.isfinite(x.grad).all()
    assert all(torch.isfinite(p.grad).all() for p in layer.weightEV)
    # componentwise against the fp64 twin.  Depths c: the EV chains' (ev_depths, worst e) and the LSI part's as in
    # lsigf_envelope (3xTF32 tensor cores in fp32), plus the E + 2 sums that join the parts (EV over e, LSI, two biases)
    y64, dx64, dw64 = _twin_fp64(layer, gso, x, dy, absolute=False)
    yM, dxM, dwM = _twin_fp64(layer, gso, x, dy, absolute=True)
    depths = [evo.ev_depths(pe["rowptr"].cpu().numpy(), pe["col"].cpu().numpy(), K, G, F, B) for pe in st.per_e]
    nnz_row = max(max(np.diff(rp).max(), np.bincount(c, minlength=N).max()) for (rp, c, _) in gso.csr)
    hop, T = (K - 1) * int(nnz_row), 1 + E * (K - 1)
    u, tc = orc.unit_roundoff(np.float32), orc.TF32X3_PER_PRODUCT
    checks = [("y", y, y64, yM, max(max(d["Y"] for d in depths), hop + T * G + 2) + E + 2),
              ("x.grad", x.grad, dx64, dxM, max(max(d["dxT"] for d in depths), hop + T * F + 2) + E + 2)]
    checks += [("weightEV[%d].grad" % e, p.grad, dw64[e], dwM[e], depths[e]["dw"]) for e, p in enumerate(layer.weightEV)]
    for name, got, ref, mag, c in checks:
        extra = tc if name in ("y", "x.grad") else 0.0
        bound = (c * u + extra) * mag + 4.0 * np.finfo(np.float32).tiny * (c + 1)
        v = float(((got.double() - ref).abs() / bound).max())
        print("cfg4 %s: worst error / bound %.3g" % (name, v))
        assert v <= 1.0, (name, v)
    # EV part alone (sparse fp64 chains for two (f, g) pairs, every e): Y_ev = layer(x) - LSI part - 2 bias
    with torch.no_grad():
        lsi = gnn_b200.LSIGF(layer.weightLSI, gso, x, layer.bias) + layer.bias
        ev = (y - lsi).index_select(2, st.A).double()                               # [B, F, NA]
        xA = x.detach().index_select(2, st.A).double()
        for f in (0, F - 1):
            want = torch.zeros(B, st.NA, dtype=torch.float64, device="cuda")
            for e in range(E):
                pe = st.per_e[e]
                rows, cols = pe["rowidx"].long(), pe["col"].long()
                for g in range(G):
                    u = xA[:, g, :]
                    for k in range(K):
                        wk = layer.weightEV[e][f, k, g].double()
                        u = torch.zeros_like(u).index_add_(1, rows, wk[None, :] * u[:, cols])
                        want += u
            assert _rel(ev[:, f].cpu().numpy(), want.cpu().numpy()) < 2e-3          # fp32 difference of two large terms
