"""MaxLocalActivation / MedianLocalActivation on CUDA tensors (graph-neural-networks_b200/activations.py) against the
reference layers' stored results (tests/golden/local_activation_cases.npz, oracle/make_golden_local_activation.py) and
oracle/local_activation_oracle.py: layer results, a LocalActivationGNN, the node-major hand-off from a GraphFilter,
CUDA-graph capture, operand checks, and a graph whose padded neighbourhood matrices would not fit on the card."""
import os

import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.nn as nn

import local_activation_oracle as lao
import lsigf_oracle as orc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "local_activation_cases.npz")
CASES = sorted({k[:-len("_y")] for k in np.load(GOLDEN).files if k.startswith("la_") and k.endswith("_y")})
pytestmark = pytest.mark.gpu


def _layer(kind, K, S, weight, dtype, device="cuda"):
    from gnn_b200 import activations
    m = getattr(activations, kind + "LocalActivation")(K).to(device=device, dtype=dtype)
    m.load_state_dict({"weight": torch.tensor(weight, dtype=dtype)})
    m.addGSO(torch.tensor(S, dtype=dtype))
    return m


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("case", CASES)
def test_layer_matches_reference(case, dtype):
    z = np.load(GOLDEN)
    g = lambda n: z[case + "_" + n]                          # noqa: E731
    kind = "Max" if "_Max_" in case else "Median"
    K = g("weight").shape[1] - 1
    m = _layer(kind, K, g("S"), g("weight"), dtype)
    x = torch.tensor(g("x"), dtype=dtype, device="cuda", requires_grad=True)
    y = m(x)
    dx, dw = torch.autograd.grad(y, [x, m.weight], torch.tensor(g("dy"), dtype=dtype, device="cuda"))
    if dtype == torch.float64:
        for name, out in (("y", y), ("dx", dx), ("dw", dw)):
            assert np.allclose(out.detach().cpu().numpy(), g(name), rtol=0, atol=1e-12), name
        return
    # fp32: the oracle on the rounded inputs, within its componentwise bounds
    from gnn_b200.graphtools_sparse import ring_neighborhoods
    B, F, N = g("x").shape
    rnd = lambda a: a.astype(np.float32).astype(np.float64)  # noqa: E731
    nm = lambda t: t.reshape(B * F, N).T                     # noqa: E731
    rings = ring_neighborhoods([sp.csr_matrix(s) for s in g("S")], K)
    op = lao.MAX if kind == "Max" else lao.MEDIAN
    yr, yb, agg, arg = lao.forward(nm(rnd(g("x"))), rnd(g("weight")), *rings, K, op, np.float32)
    dxr, dxb, dwr, dwb = lao.backward(nm(rnd(g("x"))), nm(rnd(g("dy"))), rnd(g("weight")), agg, arg, np.float32)
    assert orc.bound_violation(nm(y.detach().double().cpu().numpy()), yr, yb) <= 1
    assert orc.bound_violation(nm(dx.double().cpu().numpy()), dxr, dxb) <= 1
    assert orc.bound_violation(dw.double().cpu().numpy(), dwr, dwb) <= 1


@pytest.mark.parametrize("kind", ["Max", "Median"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_ties_give_the_torch_path_values(kind, dtype):
    """Values on a coarse grid: the max and the median are unambiguous values even where nodes tie, and equal the
    torch path's (CPU) results."""
    rng = np.random.default_rng(3)
    N, K = 300, 2
    S = orc.random_sparse_gso(rng, N, 3, 1)
    w = rng.uniform(-1, 1, (1, K + 1))
    x0 = np.round(rng.standard_normal((2, 5, N)) * 2) / 2 + 0.0
    cpu = _layer(kind, K, S, w, dtype, "cpu")(torch.tensor(x0, dtype=dtype))
    gpu = _layer(kind, K, S, w, dtype)(torch.tensor(x0, dtype=dtype, device="cuda"))
    tol = 1e-5 if dtype == torch.float32 else 1e-13
    assert torch.allclose(gpu.cpu(), cpu, rtol=0, atol=tol)


def test_local_activation_gnn_matches_reference():
    """The fixture's LocalActivationGNN rebuilt from this package's layers under the same GFL.<i> / MLP.<i> keys."""
    import gnn_b200
    z = np.load(GOLDEN)
    g = lambda n: z["lagnn_" + n]                            # noqa: E731
    _, N, B = g("meta")
    S = torch.tensor(g("S")).reshape(1, N, N).cuda()

    class Net(nn.Module):
        def __init__(self):
            super().__init__()
            self.GFL = nn.Sequential(gnn_b200.GraphFilter(2, 3, 2, 1, True), gnn_b200.MaxLocalActivation(2),
                                     gnn_b200.MaxPoolLocal(N, N, 1), gnn_b200.GraphFilter(3, 2, 3, 1, True),
                                     gnn_b200.MedianLocalActivation(1), gnn_b200.MaxPoolLocal(N, N, 2))
            self.MLP = nn.Sequential(nn.Linear(N * 2, 4, bias=True))

        def forward(self, x):
            y = self.GFL(x)
            return self.MLP(y.reshape(x.shape[0], -1))

    net = Net().double()
    for layer in net.GFL:
        layer.addGSO(S)
    state = {k[len("p_"):]: torch.tensor(z["lagnn_" + k]) for k in (f[len("lagnn_"):] for f in z.files)
             if k.startswith("p_")}
    net.load_state_dict(state)
    net.cuda()
    x = torch.tensor(g("x"), device="cuda", requires_grad=True)
    y = net(x)
    y.backward(torch.tensor(g("dy"), device="cuda"))
    assert np.allclose(y.detach().cpu().numpy(), g("y"), rtol=0, atol=1e-11)
    assert np.allclose(x.grad.cpu().numpy(), g("dx"), rtol=0, atol=1e-11)
    for name, prm in net.named_parameters():
        assert np.allclose(prm.grad.cpu().numpy(), g("g_" + name), rtol=0, atol=1e-10), name


@pytest.mark.parametrize("kind", ["Max", "Median"])
def test_graph_filter_output_is_consumed_in_place(kind):
    """GraphFilter -> LocalActivation -> MaxPoolLocal: the activation reads the filter's node-major output with no
    layout launch (one library launch), and hands the pool a node-major view it reads in place too."""
    import gnn_b200
    from gnn_b200 import activations
    lib = gnn_b200._cabi.load()
    rng = np.random.default_rng(4)
    N = 500
    S = torch.tensor(orc.random_sparse_gso(rng, N, 4, 1)).cuda()
    gf = gnn_b200.GraphFilter(3, 6, 3, 1, True).double().cuda()
    act = getattr(activations, kind + "LocalActivation")(2).double().cuda()
    pool = gnn_b200.MaxPoolLocal(N, N, 1)
    for m in (gf, act, pool):
        m.addGSO(S)
    x = torch.randn(2, 3, N, dtype=torch.float64, device="cuda")
    h = gf(x)
    assert gnn_b200.node_major_ld(h) is not None
    act(h)
    pool(act(h))                                              # warm-up: device neighbourhood copies
    torch.cuda.synchronize()
    lib.b200gf_launch_count(1)
    a = act(h)
    assert lib.b200gf_launch_count(1) == 1
    assert gnn_b200.node_major_ld(a) is not None
    pool(a)
    assert lib.b200gf_launch_count(1) == 1


@pytest.mark.parametrize("kind", ["Max", "Median"])
def test_forward_and_backward_replay_in_a_cuda_graph(kind):
    rng = np.random.default_rng(6)
    N, K = 400, 2
    S = orc.random_sparse_gso(rng, N, 3, 1)
    m = _layer(kind, K, S, rng.uniform(-1, 1, (1, K + 1)), torch.float32)
    x = torch.randn(3, 4, N, device="cuda", requires_grad=True)
    dy = torch.randn(3, 4, N, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            x.grad, m.weight.grad = None, None
            m(x).backward(dy)
    torch.cuda.current_stream().wait_stream(s)
    x.grad, m.weight.grad = None, None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y = m(x)
        y.backward(dy)
    with torch.no_grad():
        x.copy_(torch.randn_like(x))
        m.weight.copy_(torch.tensor(rng.uniform(-1, 1, (1, K + 1)), dtype=torch.float32))
    graph.replay()
    torch.cuda.synchronize()
    y_r, dx_r, dw_r = y.clone(), x.grad.clone(), m.weight.grad.clone()
    xe = x.detach().clone().requires_grad_(True)
    ye = m(xe)
    dxe, dwe = torch.autograd.grad(ye, [xe, m.weight], dy)
    assert torch.equal(y_r, ye)                               # the forward is deterministic
    assert torch.allclose(dx_r, dxe, rtol=1e-5, atol=1e-6)   # atomics: last bits may differ
    assert torch.allclose(dw_r, dwe, rtol=1e-5, atol=1e-5)


def test_operand_checks():
    rng = np.random.default_rng(7)
    N = 20
    S = orc.random_sparse_gso(rng, N, 3, 1)
    m = _layer("Max", 2, S, rng.uniform(-1, 1, (1, 3)), torch.float64)
    with pytest.raises(RuntimeError, match="one dtype"):
        m(torch.randn(1, 2, N, device="cuda", dtype=torch.float32))
    xc = torch.randn(1, 2, N, dtype=torch.float64)
    y_cpu = m.cpu()(xc)                                        # a CPU x takes the torch path
    assert y_cpu.device.type == "cpu" and m._padded is not None
    y_gpu = m.cuda()(xc.cuda())
    assert torch.allclose(y_gpu.cpu(), y_cpu, rtol=0, atol=1e-13)


@pytest.mark.parametrize("kind", ["Max", "Median"])
def test_graph_beyond_the_padded_path(kind):
    """N = 100k, degree 16, K = 2, B = 4, F = 8, and a hub of 2000 neighbours: the padded [B, F, N, M_2] tensor of the
    torch path would exceed the card's memory.  Every 997th node (and the hub) against the oracle."""
    from gnn_b200 import activations
    N, K, B, F = 100_000, 2, 4, 8
    rng = np.random.default_rng(8)
    rows = np.concatenate([np.repeat(np.arange(N), 16), np.zeros(2000, dtype=np.int64)])
    cols = np.concatenate([rng.integers(0, N, 16 * N), rng.choice(np.arange(1, N), 2000, replace=False)])
    A = sp.csr_matrix((np.ones(len(rows)), (rows, cols)), shape=(N, N))
    import gnn_b200
    m = getattr(activations, kind + "LocalActivation")(K).cuda()
    m.addGSO(gnn_b200.SparseGSO.from_scipy([A]))
    padded = B * F * N * max(m.maxNeighborhoodSizes) * 4
    assert padded > torch.cuda.get_device_properties(0).total_memory, padded
    x = torch.randn(B, F, N, device="cuda", requires_grad=True)
    y = m(x)
    y.backward(torch.randn_like(y))
    torch.cuda.synchronize()
    assert m._padded is None                                    # the CUDA path never built the padded matrices
    rows = np.arange(0, N, 997)
    xn = x.detach().double().cpu().numpy().reshape(B * F, N).T
    yr, yb, _, _ = lao.forward(xn, m.weight.detach().double().cpu().numpy(), *m._rings, K,
                               lao.MAX if kind == "Max" else lao.MEDIAN, np.float32, rows)
    yn = y.detach().double().cpu().numpy().reshape(B * F, N).T[rows]
    assert orc.bound_violation(yn, yr, yb) <= 1
    assert torch.isfinite(x.grad).all() and torch.isfinite(m.weight.grad).all()
