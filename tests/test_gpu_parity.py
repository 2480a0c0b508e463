"""GPU parity tests (run on an H100: `pytest -m gpu`): the CUDA path behind the C ABI vs
  (1) golden fixtures produced by the UNMODIFIED reference (tests/golden, oracle/make_golden.py),
  (2) the fp64 CPU oracle (oracle/lsigf_oracle.py) on seeded sparse graphs the dense reference could not hold,
  (3) size-independent properties at BASELINE.json's full sizes.
Tolerance (BASELINE.json north_star): max|y - y_ref| / max|y_ref| <= 1e-4 in fp32; fp64 is held to 1e-11.
"""
import os

import numpy as np
import pytest
import torch

import lsigf_oracle as orc

pytestmark = pytest.mark.gpu

TOL32 = 1e-4     # north_star tolerance
TOL64 = 1e-11


def rel(a, b):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


@pytest.fixture(scope="module")
def b200():
    import gnn_b200
    gnn_b200._cabi.load()   # fail loudly if the extension is missing
    return gnn_b200


def _tt(a, dtype, grad=False):
    t = torch.tensor(np.asarray(a), dtype=dtype, device="cuda")
    t.requires_grad_(grad)
    return t


def _case_keys(z, prefix):
    return sorted({k.split("_")[0] for k in z.files if k.startswith(prefix)})


@pytest.mark.parametrize("dtype,tol", [(torch.float64, TOL64), (torch.float32, TOL32)])
def test_lsigf_golden_forward_backward(b200, golden_dir, dtype, tol):
    z = np.load(os.path.join(golden_dir, "lsigf_cases.npz"))
    worst = 0.0
    for c in _case_keys(z, "c"):
        h = _tt(z[c + "_h"], dtype, True)
        x = _tt(z[c + "_x"], dtype, True)
        S = _tt(z[c + "_S"], dtype)
        b = _tt(z[c + "_b"], dtype, True) if (c + "_b") in z.files else None
        y = b200.LSIGF(h, S, x, b)
        assert tuple(y.shape) == z[c + "_y"].shape
        y.backward(_tt(z[c + "_dy"], dtype))
        errs = [rel(y.detach().cpu().numpy(), z[c + "_y"]), rel(h.grad.cpu().numpy(), z[c + "_dh"]),
                rel(x.grad.cpu().numpy(), z[c + "_dx"])]
        if b is not None:
            assert tuple(b.grad.shape) == z[c + "_db"].shape
            errs.append(rel(b.grad.cpu().numpy(), z[c + "_db"]))
        worst = max(worst, max(errs))
        assert max(errs) < tol, (c, errs)
    print("worst rel err %s: %.3e" % (dtype, worst))


@pytest.mark.parametrize("dtype,tol", [(torch.float64, TOL64), (torch.float32, TOL32)])
def test_graphfilter_golden(b200, golden_dir, dtype, tol):
    z = np.load(os.path.join(golden_dir, "graphfilter_cases.npz"))
    for c in _case_keys(z, "g"):
        seed, N, Nin, B, G, F, K, E, bias = [int(v) for v in z[c + "_meta"]]
        layer = b200.GraphFilter(G, F, K, E, bool(bias)).to("cuda", dtype)
        sd = {"weight": _tt(z[c + "_weight"], dtype)}
        if bias:
            sd["bias"] = _tt(z[c + "_bias"], dtype)
        layer.load_state_dict(sd)                       # reference parameter names / shapes
        layer.addGSO(_tt(z[c + "_S"], dtype))
        x = _tt(z[c + "_x"], dtype, True)
        y = layer(x)
        assert tuple(y.shape) == z[c + "_y"].shape      # zero-pad / truncate path when Nin < N
        y.backward(_tt(z[c + "_dy"], dtype))
        assert rel(y.detach().cpu().numpy(), z[c + "_y"]) < tol
        assert rel(x.grad.cpu().numpy(), z[c + "_dx"]) < tol
        assert rel(layer.weight.grad.cpu().numpy(), z[c + "_dweight"]) < tol
        if bias:
            assert rel(layer.bias.grad.cpu().numpy(), z[c + "_dbias"]) < tol


def test_selectiongnn_cfg1_composition(b200, golden_dir):
    """BASELINE configs[0]: GraphFilter -> ReLU -> NoPool -> MLP as composed by the reference's SelectionGNN
    (architectures.py:274-296,445-449), weights and expected outputs/gradients from the reference run (fp64)."""
    z = np.load(os.path.join(golden_dir, "selectiongnn_cfg1.npz"))
    dt = torch.float64
    gfl = b200.GraphFilter(1, 32, 5, 1, True).to("cuda", dt)
    gfl.load_state_dict({"weight": _tt(z["sd_GFL.0.weight"], dt), "bias": _tt(z["sd_GFL.0.bias"], dt)})
    gfl.addGSO(_tt(z["S"][None], dt))
    mlp = torch.nn.Linear(32 * 50, 5).to("cuda", dt)
    mlp.load_state_dict({"weight": _tt(z["sd_MLP.0.weight"], dt), "bias": _tt(z["sd_MLP.0.bias"], dt)})
    x = _tt(z["x"], dt, True)
    u = torch.relu(gfl(x))
    y = mlp(u.reshape(u.shape[0], -1))
    y.backward(_tt(z["dy"], dt))
    assert rel(y.detach().cpu().numpy(), z["y"]) < 1e-11
    assert rel(x.grad.cpu().numpy(), z["dx"]) < 1e-11
    assert rel(gfl.weight.grad.cpu().numpy(), z["grad_GFL.0.weight"]) < 1e-11
    assert rel(gfl.bias.grad.cpu().numpy(), z["grad_GFL.0.bias"]) < 1e-11
    assert rel(mlp.weight.grad.cpu().numpy(), z["grad_MLP.0.weight"]) < 1e-11


# (N, deg, B, G, F, K, E, bias)
SPARSE_CASES = [
    (3000, 8, 1, 64, 64, 5, 1, "F1"),       # headline shape, small N
    (2500, 12, 3, 5, 7, 4, 2, "FN"),        # odd feature counts, tensor GSO, per-node bias
    (4000, 6, 32, 64, 64, 3, 1, "F1"),      # C = 2048: multi-chunk rows (cfg2 shape)
    (1682, 20, 5, 64, 64, 5, 1, "F1"),      # cfg3 (MovieLens-shaped)
    (2000, 40, 2, 1, 32, 5, 1, "F1"),       # G = 1 first layer (cfg1 shape), rows longer than one 32-entry batch
    (1500, 5, 1, 6, 4, 1, 1, None),         # K = 1
    (2048, 10, 2, 32, 16, 3, 4, None),      # cfg4 shape (E = 4, K = 3)
    (2200, 9, 2, 64, 32, 4, 2, "FN"),       # F = 32: 32-column block of the FP64 DMMA contraction, per-node bias
]


@pytest.mark.parametrize("case", SPARSE_CASES)
@pytest.mark.parametrize("dtype,tol", [(torch.float64, TOL64), (torch.float32, TOL32)])
def test_sparse_vs_oracle(b200, case, dtype, tol):
    import scipy.sparse as sp
    N, deg, B, G, F, K, E, bias = case
    rng = np.random.default_rng(N + 7 * G)
    mats = []
    for e in range(E):
        m = sp.random(N, N, density=deg / N, format="csr", random_state=np.random.RandomState(N + e),
                      data_rvs=lambda n: rng.standard_normal(n))
        m = m / max(abs(m).sum(axis=1).max(), 1e-30)   # non-symmetric, spectral radius <= 1
        mats.append(sp.csr_matrix(m))
    x = rng.standard_normal((B, G, N))
    bound = 1 / np.sqrt(G * K)
    h = rng.uniform(-bound, bound, (F, E, K, G))
    b = None if bias is None else rng.uniform(-bound, bound, (F, 1 if bias == "F1" else N))
    dy = rng.standard_normal((B, F, N))
    # oracle works on what the device sees: inputs rounded to the test dtype
    npd = np.float32 if dtype == torch.float32 else np.float64
    mats_r = [sp.csr_matrix((m.data.astype(npd).astype(np.float64), m.indices, m.indptr), shape=m.shape) for m in mats]
    r64 = lambda a: None if a is None else a.astype(npd).astype(np.float64)
    y_ref = orc.lsigf_sparse(r64(h), mats_r, r64(x), r64(b))
    dh_ref, dx_ref, db_ref = orc.lsigf_grads_sparse(r64(h), mats_r, r64(x), r64(dy), None if b is None else b.shape)

    gso = b200.SparseGSO.from_scipy(mats, dtype=dtype)
    ht, xt = _tt(h, dtype, True), _tt(x, dtype, True)
    bt = None if b is None else _tt(b, dtype, True)
    y = b200.LSIGF(ht, gso, xt, bt)
    y.backward(_tt(dy, dtype))
    errs = {"y": rel(y.detach().cpu().numpy(), y_ref), "dh": rel(ht.grad.cpu().numpy(), dh_ref),
            "dx": rel(xt.grad.cpu().numpy(), dx_ref)}
    if b is not None:
        errs["db"] = rel(bt.grad.cpu().numpy(), db_ref)
    print(case, dtype, errs)
    assert max(errs.values()) < tol, errs


def test_node_major_chain_no_transpose(b200):
    """Two stacked GraphFilters with ReLU in between: layer 2 must consume layer 1's node-major view in place."""
    torch.manual_seed(0)
    N = 500
    S = torch.randn(1, N, N, device="cuda") * (torch.rand(1, N, N, device="cuda") < 0.02)
    S = S / S.abs().sum(1).max()
    l1 = b200.GraphFilter(4, 8, 3).cuda(); l1.addGSO(S)
    l2 = b200.GraphFilter(8, 6, 3).cuda(); l2.addGSO(S)
    x = torch.randn(3, 4, N, device="cuda")
    u = torch.relu(l1(x))
    assert b200.node_major_ld(u) is not None            # strides survived the ReLU
    y = l2(u)
    y_ref = orc.lsigf_dense(l2.weight.detach().cpu().double().numpy(), S.cpu().double().numpy(),
                            np.maximum(orc.lsigf_dense(l1.weight.detach().cpu().double().numpy(), S.cpu().double().numpy(),
                                                       x.cpu().double().numpy(), l1.bias.detach().cpu().double().numpy()), 0),
                            l2.bias.detach().cpu().double().numpy())
    assert rel(y.detach().cpu().numpy(), y_ref) < TOL32


def test_errors_are_loud(b200):
    h = torch.randn(2, 1, 2, 3)
    S = torch.eye(5)[None]
    x = torch.randn(1, 3, 5)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        b200.LSIGF(h, S, x)                             # CPU tensors: refuse, never fall back
    with pytest.raises(AssertionError):
        b200.LSIGF(h.cuda(), S.cuda(), torch.randn(1, 4, 5).cuda())     # G mismatch (graphML.py:139)
    with pytest.raises(RuntimeError, match="one dtype"):
        b200.LSIGF(h.cuda().double(), S.cuda(), x.cuda())


@pytest.mark.parametrize("N,deg", [(1_000_000, 32)])
def test_full_size_properties(b200, N, deg):
    """Headline size (ER N=1M, avgDeg 32, K=5, G=F=64, B=1), fp32: properties that need no oracle run.
       (a) sqrt(deg) is a fixed point of x·S for S = D^-1/2 A D^-1/2  => closed-form output;
       (b) linearity in x;  (c) adjoint identities <y, dy> = <x, dx> = <h, dh> for the bias-free filter."""
    from gnn_b200 import graphs
    gso = graphs.er_gso(N, deg, seed=1)
    K, G, F = 5, 64, 64
    g = torch.Generator(device="cpu").manual_seed(5)
    bound = 1 / np.sqrt(G * K)
    h = ((torch.rand(F, 1, K, G, generator=g) * 2 - 1) * bound).cuda()
    b = ((torch.rand(F, 1, generator=g) * 2 - 1) * bound).cuda()
    d = torch.from_numpy(graphs.degrees(gso).astype(np.float64)).sqrt().float().cuda()
    x = d.expand(1, G, N).contiguous()
    y = b200.LSIGF(h, gso, x, b)
    expect = h.double().sum(dim=(1, 2, 3))[None, :, None] * d.double()[None, None, :] + b.double()[None]
    assert rel(y.double().cpu().numpy(), expect.cpu().numpy()) < TOL32
    # linearity
    x1 = torch.randn(1, G, N, device="cuda")
    x2 = torch.randn(1, G, N, device="cuda")
    y12 = b200.LSIGF(h, gso, 0.5 * x1 + x2, None)
    ysum = 0.5 * b200.LSIGF(h, gso, x1, None) + b200.LSIGF(h, gso, x2, None)
    assert rel(y12.cpu().numpy(), ysum.cpu().numpy()) < TOL32
    # adjoints
    hr = h.clone().requires_grad_(True)
    xr = x1.clone().requires_grad_(True)
    yr = b200.LSIGF(hr, gso, xr, None)
    dy = torch.randn(1, F, N, device="cuda")
    yr.backward(dy)
    ydy = (yr.detach().double() * dy.double()).sum().item()
    xdx = (xr.detach().double() * xr.grad.double()).sum().item()
    hdh = (hr.detach().double() * hr.grad.double()).sum().item()
    assert abs(ydy - xdx) / abs(ydy) < TOL32 and abs(ydy - hdh) / abs(ydy) < TOL32, (ydy, xdx, hdh)


def test_forward_is_cuda_graph_capturable(b200):
    """include/b200gf.h promises no allocation and no host synchronisation inside b200gf_forward: capture one call
    (hops + wgmma contraction) in a CUDA graph, replay it on new input values, compare with an eager call."""
    from gnn_b200 import graphs, _cabi
    lib = _cabi.load()
    N, K, G, F, B = 20000, 4, 64, 64, 1
    gso = graphs.er_gso(N, 12, seed=7)
    plan = gso.plan("cuda")
    gen = torch.Generator(device="cuda").manual_seed(3)
    h = torch.randn(F, 1, K, G, device="cuda", generator=gen) * 0.1
    bias = torch.randn(F, device="cuda", generator=gen)
    xn = torch.randn(N, G, device="cuda", generator=gen)           # node-major operands: the C call does everything
    y = torch.empty(N, F, device="cuda")
    wsb = lib.b200gf_workspace_bytes(plan.handle, B, G, F, K, _cabi.NODE_MAJOR, 0)
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")

    def call(stream):
        rc = lib.b200gf_forward(plan.handle, xn.data_ptr(), _cabi.NODE_MAJOR, G, h.data_ptr(), bias.data_ptr(), 0,
                                y.data_ptr(), _cabi.NODE_MAJOR, F, ws.data_ptr(), wsb, B, G, F, K, stream)
        assert rc == 0, lib.b200gf_strerror(rc)

    call(torch.cuda.current_stream().cuda_stream)                  # warm-up (function attributes, tensor-map encoder)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        call(torch.cuda.current_stream().cuda_stream)
    xn.copy_(torch.randn(N, G, device="cuda", generator=gen))      # new values, same buffers
    graph.replay()
    torch.cuda.synchronize()
    y_graph = y.clone()
    call(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert torch.equal(y_graph, y)                                 # deterministic kernels: bit-identical
    ref = b200.LSIGF(h, gso, xn.t().reshape(1, G, N).contiguous(), bias.view(F, 1))
    assert rel(y.t().reshape(1, F, N).cpu().numpy(), ref.cpu().numpy()) < 1e-5
