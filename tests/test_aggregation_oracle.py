"""CPU checks behind the aggregation GNNs (aggregation.py): the float64 oracle (oracle/aggregation_oracle.py) and the
layers' host code, with the graph product swapped for the oracle, against the reference's stored results
(tests/golden/aggregation_cases.npz, oracle/make_golden_aggregation.py); the level split of long operator rows; the GSO
forms, orders and install()."""
import os
import types

import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.nn as nn

import aggregation_oracle as aao
import make_golden_aggregation as mga

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "aggregation_cases.npz")


def _oracle_aggregate(op, x):
    mats = [sp.csr_matrix((v, c, r), shape=(op.N, op.N)) for (r, c, v) in op.gso.csr]
    R, _, _ = aao.operator(mats, op.sel, op.maxN)
    return aao.aggregate_torch(R, op.E, op.maxN, x)


@pytest.fixture
def oracle_product(monkeypatch):
    from gnn_b200 import aggregation
    monkeypatch.setattr(aggregation, "_aggregate", _oracle_aggregate)


def build(name, S):
    """Our layer for fixture case `name`, built like the reference under the case's seed, in float64."""
    from gnn_b200 import aggregation
    kind, seed, _, _, _, kw = mga.CASES[name]
    cls = aggregation.AggregationGNN if kind == "agg" else aggregation.MultiNodeAggregationGNN
    torch.manual_seed(seed)
    return cls(nonlinearity=nn.ReLU, poolingFunction=nn.MaxPool1d, GSO=S, **kw).double()


def close(out, ref, tol):
    """Componentwise: |out - ref| <= tol (|ref| + max |ref|)."""
    ref = np.asarray(ref)
    return np.all(np.abs(np.asarray(out) - ref) <= tol * (np.abs(ref) + np.abs(ref).max()))


def _fixture():
    return np.load(GOLDEN)


@pytest.mark.parametrize("name", sorted(mga.CASES))
def test_layers_on_the_oracle_match_the_reference(name, oracle_product):
    """Same seed -> same state_dict keys and values as the reference; y, dx and every parameter gradient of the fixed
    loss agree with the reference's in float64."""
    z = _fixture()
    g = lambda k: z[name + "_" + k]                           # noqa: E731
    net = build(name, g("S"))
    state = net.state_dict()
    ref_keys = sorted(k[len(name) + 3:] for k in z.files if k.startswith(name + "_p_"))
    assert sorted(state) == ref_keys
    for k, v in state.items():
        assert np.array_equal(v.numpy(), g("p_" + k)), k
    assert list(net.order) == g("order").tolist()
    x = torch.tensor(g("x"), requires_grad=True)
    y = net(x)
    y.backward(torch.tensor(g("dy")))
    assert y.shape == g("y").shape
    assert close(y.detach().numpy(), g("y"), 1e-12)
    assert close(x.grad.numpy(), g("dx"), 1e-12)
    for k, prm in net.named_parameters():
        assert close(prm.grad.numpy(), g("g_" + k), 1e-12), k


def test_conv_output_lengths_and_max_n():
    """self.N (the conv output lengths) and maxN capped at N, as architectures.py:3064-3077 computes them."""
    from gnn_b200 import aggregation
    S = mga.gso(1, 10, 1)
    for maxN, want in ((None, 10), (4, 4), (30, 10)):
        m = aggregation.AggregationGNN([1, 2, 2], [3, 2], True, nn.ReLU, nn.MaxPool1d, [2, 1], [3], S, maxN=maxN)
        n = [want, (want - 2 - 1) // 2 + 1]
        n.append(n[1] - 1)
        assert m.maxN == want and m.N == n and m.operator.maxN == want


@pytest.mark.parametrize("nNodes,agg", [(1, []), (3, []), (3, [4])])
def test_output_shapes(nNodes, agg, oracle_product):
    from gnn_b200 import aggregation
    S = mga.gso(2, 8, 2)
    m = aggregation.AggregationGNN([2, 3], [2], True, nn.ReLU, nn.MaxPool1d, [1], [5], S, maxN=3, nNodes=nNodes,
                                   dimLayersAggMLP=agg)
    y = m(torch.randn(4, 2, 8))
    assert tuple(y.shape) == ((4, 5) if nNodes == 1 else (4, 4) if agg else (4, 5, nNodes))


def test_multinode_pads_outputs_at_the_selected_nodes(monkeypatch):
    """The second outer layer's input is zero except at nodes order[:P[0]], where it holds the first layer's outputs
    in order; the caller's lists are left as they were."""
    from gnn_b200 import aggregation
    seen = []

    def record(op, x):
        seen.append(x.detach().clone())
        return _oracle_aggregate(op, x)

    monkeypatch.setattr(aggregation, "_aggregate", record)
    S = mga.gso(3, 9, 1)
    dims, sel = [[2, 3], [3, 2]], [3, 2]
    m = aggregation.MultiNodeAggregationGNN(sel, [3, 2], dims, [[2], [1]], True, nn.ReLU, nn.MaxPool1d,
                                            [[1], [1]], [4], S, order="Degree")
    assert dims == [[2, 3], [3, 2]] and sel == [3, 2]
    assert [len(mods) for mods in m.aggGNNmodules] == [3, 2]
    assert all(op.sel.tolist() == m.order[:p] for op, p in zip(m.operators, m.P))
    m(torch.randn(2, 2, 9))
    x1 = seen[1]
    keep = np.zeros(9, dtype=bool)
    keep[m.order[:3]] = True
    assert torch.all(x1[:, :, torch.from_numpy(~keep)] == 0) and torch.all(x1[:, :, torch.from_numpy(keep)] != 0)


def test_oracle_is_the_reference_sn_without_its_zeros():
    """R against the reference's own SN (live reference only), and against the definition on a case with an isolated
    selected node, whose rows q >= 1 are empty."""
    import ref_import
    S = mga.gso(4, 11, 2)
    S[:, 1, :] = 0
    S[:, :, 1] = 0                                           # node 1: no edges
    sel = [1, 0, 5]
    R, Rabs, _ = aao.operator(S, sel, 4)
    assert R.shape == (3 * 2 * 4, 11)
    for p in range(3):
        for e in range(2):
            for q in range(4):
                col = np.linalg.matrix_power(S[e], q)[:, sel[p]]
                row = R[(p * 2 + e) * 4 + q].toarray().ravel()
                assert np.allclose(row, col, rtol=0, atol=1e-15)
                if p == 0:
                    assert R[(p * 2 + e) * 4 + q].nnz == (1 if q == 0 else 0)
    assert np.all(Rabs.toarray() >= np.abs(R.toarray()))
    if not ref_import.reference_available():
        pytest.skip("reference checkout not available (B200GF_REFERENCE_ROOT)")
    ref_import.import_reference()
    import alegnn.modules.architectures as archit
    perm = sel + [i for i in range(11) if i not in sel]
    Sp = S[:, perm][:, :, perm]
    m = archit.AggregationGNN([1, 1], [1], False, nn.ReLU, nn.MaxPool1d, [1], [], Sp, maxN=4, nNodes=3)
    SN = m.SN.numpy()                                         # [nNodes, E, N, maxN] in the reordered numbering
    dense = R.toarray().reshape(3, 2, 4, 11)[:, :, :, perm].transpose(0, 1, 3, 2)
    assert np.allclose(SN, dense, rtol=0, atol=1e-15)


def _random_operator(n_rows, n_cols, lens, seed):
    rng = np.random.default_rng(seed)
    rows = np.repeat(np.arange(n_rows), lens)
    cols = np.concatenate([rng.choice(n_cols, L, replace=False) for L in lens]) if len(rows) else np.zeros(0, int)
    return sp.csr_matrix((rng.standard_normal(len(rows)), (rows, cols)), shape=(n_rows, n_cols))


def _chain_product(levels):
    out = None
    for (rp, c, v, n, nc) in levels:
        M = sp.csr_matrix((v, c, rp), shape=(n, nc))
        out = M if out is None else M @ out
    return out


@pytest.mark.parametrize("n_rows,n_cols,L,depth", [(5, 3000, 16, 3), (40, 700, 16, 3), (700, 40, 8, 2),
                                                   (6, 50, 64, 1), (300, 300, 4, 5)])
def test_split_levels_multiply_back_to_the_operator(n_rows, n_cols, L, depth):
    """No level has a row past L, the chain's product is the operator (exactly: a sum of the same terms, grouped), and
    the same input gives the same arrays.  Rows of length 0, 1, L, L + 1 and the longest the shape allows."""
    from gnn_b200.aggregation import split_levels
    rng = np.random.default_rng(n_rows + n_cols)
    lens = rng.integers(0, min(n_cols, 3 * L), n_rows)
    lens[:4] = [0, 1, min(L, n_cols), min(L + 1, n_cols)][:min(4, n_rows)]
    lens[-1] = n_cols
    R = _random_operator(n_rows, n_cols, lens, n_rows)
    levels = split_levels(R.indptr, R.indices.astype(np.int32), R.data, n_cols, L)
    assert len(levels) == depth
    assert levels[0][4] == n_cols and levels[-1][3] == n_rows
    for (rp, c, v, n, nc) in levels:
        assert rp[0] == 0 and len(rp) == n + 1 and np.diff(rp).max() <= L and c.max() < nc
    assert np.allclose(_chain_product(levels).toarray(), R.toarray(), rtol=1e-14, atol=1e-14)
    again = split_levels(R.indptr, R.indices.astype(np.int32), R.data, n_cols, L)
    for a, b in zip(levels, again):
        assert all(np.array_equal(x, y) for x, y in zip(a[:3], b[:3])) and a[3:] == b[3:]


def test_split_levels_of_a_saturated_row_at_the_library_width():
    """A row of a million entries at ROW_SPLIT = 256 takes 3 levels; one of 256 entries stays whole."""
    from gnn_b200.aggregation import ROW_SPLIT, split_levels
    n = 1_000_000
    rp = np.array([0, n, n + ROW_SPLIT], dtype=np.int64)
    col = np.concatenate([np.arange(n), np.arange(ROW_SPLIT)]).astype(np.int32)
    levels = split_levels(rp, col, np.ones(n + ROW_SPLIT), n)
    assert [lv[3] for lv in levels] == [3907 + 1, 16 + 1, 2]
    assert len(split_levels(rp[1:] - n, col[n:], np.ones(ROW_SPLIT), n)) == 1


def test_gso_forms_give_one_operator():
    """numpy [N, N] / [E, N, N], torch dense, torch sparse (never densified) and SparseGSO all give the same CSR."""
    import gnn_b200
    from gnn_b200.aggregation import as_sparse_gso
    S = mga.gso(5, 7, 1)
    want = as_sparse_gso(gnn_b200.SparseGSO.from_scipy([sp.csr_matrix(S[0])]))
    forms = [S, S[0], torch.tensor(S), torch.tensor(S[0]), torch.tensor(S[0]).to_sparse(),
             torch.tensor(S).to_sparse()]
    for f in forms:
        g = as_sparse_gso(f)
        assert g.N == 7 and g.E == 1
        for a, b in zip(g.csr[0], want.csr[0]):
            assert np.array_equal(a, b)
    with pytest.raises(TypeError):
        as_sparse_gso([[0.0]])


def test_orders_and_operands():
    from gnn_b200 import aggregation
    from gnn_b200.graphtools_sparse import perm_degree
    S = mga.gso(6, 9, 1)
    args = ([1, 2], [2], True, nn.ReLU, nn.MaxPool1d, [1], [3], S)
    m = aggregation.AggregationGNN(*args, order="Degree", nNodes=2, maxN=3)
    assert m.order == perm_degree(sp.csr_matrix(S[0]))[1] and m.operator.sel.tolist() == m.order[:2]
    for order in ("EDS", "SpectralProxies"):
        with pytest.raises(NotImplementedError, match="eigendecomposition"):
            aggregation.AggregationGNN(*args, order=order)
    with pytest.raises(ValueError, match="nNodes"):
        aggregation.AggregationGNN(*args, nNodes=10)
    with pytest.raises(RuntimeError, match="needs CUDA tensors"):
        m(torch.randn(2, 1, 9, dtype=torch.float64))
    assert m.to("cpu") is m                                   # the reference's .to() returns None


def test_install_points_both_architectures_at_the_package():
    import gnn_b200
    from gnn_b200 import aggregation
    from gnn_b200.graphML import install, uninstall
    names = ("LSIGF", "GraphFilter", "EVGF", "EdgeVariantGF", "MaxPoolLocal", "MaxLocalActivation",
             "MedianLocalActivation", "HiddenState", "TimeGatedHiddenState", "NodeGatedHiddenState", "LSIGF_DB",
             "GraphFilter_DB", "GRNN_DB", "HiddenState_DB")
    gml = types.ModuleType("gml_standin")
    for n in names:
        setattr(gml, n, object())
    archit = types.ModuleType("archit_standin")
    archit.AggregationGNN, archit.MultiNodeAggregationGNN = object(), object()
    before = (archit.AggregationGNN, archit.MultiNodeAggregationGNN)
    install(gml, archit=archit)
    assert (archit.AggregationGNN, archit.MultiNodeAggregationGNN) == before     # off by default
    uninstall(gml)
    install(gml, aggregation=True, archit=archit)
    try:
        assert archit.AggregationGNN is aggregation.AggregationGNN is gnn_b200.AggregationGNN
        assert archit.MultiNodeAggregationGNN is aggregation.MultiNodeAggregationGNN
    finally:
        uninstall(gml)
    assert (archit.AggregationGNN, archit.MultiNodeAggregationGNN) == before
