"""The aggregation GNNs (aggregation.py) on the GPU: parity with the reference's stored results
(tests/golden/aggregation_cases.npz) for AggregationGNN, MultiNodeAggregationGNN and order='Degree' in float64 and
float32, determinism and CUDA-graph replay, a 200k-node graph whose dense GSO would not fit the card, and a maxN past
the graph's diameter, where rows saturate and the split reaches 3 levels."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.nn as nn

import aggregation_oracle as aao
import lsigf_oracle as orc
from test_aggregation_oracle import GOLDEN, build, close

pytestmark = pytest.mark.gpu


def _load(net, z, name):
    net.load_state_dict({k[len(name) + 3:]: torch.tensor(z[k]) for k in z.files if k.startswith(name + "_p_")})


@pytest.fixture
def no_tf32():
    """float32 convolutions in float32 arithmetic: cuDNN's default TF32 would round their products to 10 bits."""
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-11), (torch.float32, 2e-5)])
@pytest.mark.parametrize("name", ["agg_n1", "agg_n3_aggmlp", "agg_n3", "agg_n1_e2", "agg_degree", "multi"])
def test_matches_reference_fixtures(name, dtype, tol, no_tf32):
    """y, dx and every parameter gradient of the fixed loss against the reference's float64 results (float32 is an
    extension: the reference raises there)."""
    z = np.load(GOLDEN)
    g = lambda k: z[name + "_" + k]                           # noqa: E731
    net = build(name, g("S"))
    _load(net, z, name)
    net = net.to(device="cuda", dtype=dtype)
    x = torch.tensor(g("x"), dtype=dtype, device="cuda", requires_grad=True)
    y = net(x)
    y.backward(torch.tensor(g("dy"), dtype=dtype, device="cuda"))
    assert close(y.detach().double().cpu().numpy(), g("y"), tol)
    assert close(x.grad.double().cpu().numpy(), g("dx"), tol)
    for k, prm in net.named_parameters():
        assert close(prm.grad.double().cpu().numpy(), g("g_" + k), tol), k


def _random_graph(N, deg, seed):
    rng = np.random.default_rng(seed)
    rows = np.repeat(np.arange(N), deg)
    A = sp.csr_matrix((rng.uniform(-1, 1, N * deg) / deg, (rows, rng.integers(0, N, N * deg))), shape=(N, N))
    A.sum_duplicates()
    return A


def _net(S, dtype, **kw):
    from gnn_b200 import aggregation
    torch.manual_seed(0)
    return aggregation.AggregationGNN([3, 4], [2], True, nn.ReLU, nn.MaxPool1d, [1], [5], S, **kw).to(
        device="cuda", dtype=dtype)


def test_reruns_and_graph_replay_are_bit_identical():
    import gnn_b200
    S = gnn_b200.SparseGSO.from_scipy([_random_graph(3000, 6, 1)])
    net = _net(S, torch.float32, maxN=8, nNodes=20, dimLayersAggMLP=[3])
    x = torch.randn(4, 3, 3000, device="cuda", requires_grad=True)
    dy = torch.randn(4, 3, device="cuda")

    def step():
        x.grad = None
        net.zero_grad(set_to_none=True)
        y = net(x)
        y.backward(dy)
        return y.detach().clone(), x.grad.clone()

    y1, dx1 = step()
    y2, dx2 = step()
    assert torch.equal(y1, y2) and torch.equal(dx1, dx2)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    x.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y = net(x)
        y.backward(dy)
    with torch.no_grad():
        x.copy_(torch.randn_like(x))
    graph.replay()
    torch.cuda.synchronize()
    y_r, dx_r = y.detach().clone(), x.grad.clone()
    ye, dxe = step()
    assert torch.equal(y_r, ye) and torch.equal(dx_r, dxe)


def _check_product(A, sel, maxN, B, F, dtype, seed):
    """z and dx of one product against the oracle's bounds; returns the operator."""
    import gnn_b200
    from gnn_b200 import aggregation
    N = A.shape[0]
    op = aggregation.AggregationOperator(gnn_b200.SparseGSO.from_scipy([A]), sel, maxN)
    npd = np.float32 if dtype == torch.float32 else np.float64
    rng = np.random.default_rng(seed)
    xh = rng.standard_normal((B, F, N)).astype(npd).astype(np.float64)
    x = torch.tensor(xh, dtype=dtype, device="cuda", requires_grad=True)
    z = aggregation._aggregate_cuda(op, x)
    dzh = rng.standard_normal(tuple(z.shape)).astype(npd).astype(np.float64)
    z.backward(torch.tensor(dzh, dtype=dtype, device="cuda"))
    R, Rabs, r_err = aao.operator([A], sel, maxN)
    zr, zb = aao.forward(R, Rabs, r_err, xh, 1, maxN, npd)
    dxr, dxb = aao.backward(R, Rabs, r_err, dzh, 1, maxN, N, npd)
    assert orc.bound_violation(z.detach().double().cpu().numpy(), zr, zb) <= 1
    assert orc.bound_violation(x.grad.double().cpu().numpy(), dxr, dxb) <= 1
    return op


def test_graph_whose_dense_gso_would_not_fit():
    """N = 200k, degree 16, nNodes = 8, maxN = 5: the reference's dense GSO alone would take 320 GB."""
    N = 200_000
    assert N * N * 8 > 3 * torch.cuda.get_device_properties(0).total_memory
    A = _random_graph(N, 16, 2)
    sel = np.random.default_rng(3).choice(N, 8, replace=False)
    op = _check_product(A, sel, 5, 4, 2, torch.float32, 4)
    fwd, bwd = op.levels(torch.device("cuda"), torch.float32)
    assert sum(p.nnz for p in fwd) >= op.host(torch.device("cuda"))[0][0][-1]


def test_max_n_past_the_diameter_saturates_rows():
    """maxN = 12 on a 70k-node graph of degree 8 plus a ring: the last rows of R reach every node, R splits into 3
    levels, and R^T (rows up to nNodes maxN = 768) into 2."""
    N = 70_000
    A = _random_graph(N, 8, 5) + sp.csr_matrix((np.full(N, 0.5), (np.arange(N), (np.arange(N) + 1) % N)), shape=(N, N))
    A = sp.csr_matrix(A)
    A.sort_indices()
    sel = np.random.default_rng(6).choice(N, 64, replace=False)
    op = _check_product(A, sel, 12, 2, 3, torch.float64, 7)
    (rp, _, _), _ = op.host(torch.device("cuda"))
    assert np.diff(rp).max() == N
    fwd, bwd = op.levels(torch.device("cuda"), torch.float64)
    assert (len(fwd), len(bwd)) == (3, 2)


def test_operator_is_built_once_per_device_and_dtype():
    import gnn_b200
    net = _net(gnn_b200.SparseGSO.from_scipy([_random_graph(500, 4, 8)]), torch.float64, maxN=4, nNodes=2)
    x = torch.randn(2, 3, 500, dtype=torch.float64, device="cuda")
    net(x)
    host, levels = dict(net.operator._host), dict(net.operator._levels)
    net(x)
    net.float()(x.float())
    assert all(net.operator._host[k] is v for k, v in host.items()) and len(net.operator._host) == len(host)
    assert all(net.operator._levels[k] is v for k, v in levels.items())
    assert len(net.operator._levels) == len(levels) + 1
    with pytest.raises(RuntimeError, match="needs CUDA tensors"):
        net(x.cpu().float())
