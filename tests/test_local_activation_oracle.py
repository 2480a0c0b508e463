"""CPU checks behind the localized activations' CUDA path: the ring-ordered K-hop lists
(graphtools_sparse.ring_neighborhoods) against compute_neighborhood, and the float64 oracle
(oracle/local_activation_oracle.py) against the reference layers' stored results (tests/golden/local_activation_cases.npz,
oracle/make_golden_local_activation.py)."""
import os

import numpy as np
import pytest
import scipy.sparse as sp

import local_activation_oracle as lao

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "local_activation_cases.npz")


def _graphs():
    rng = np.random.default_rng(5)
    directed = sp.random(40, 40, density=0.06, random_state=1, format="csr")
    sym = sp.csr_matrix(directed + directed.T)
    iso = sym.tolil()
    iso[7, :] = 0
    iso[:, 7] = 0                                          # node 7: no edges at all
    two = [sp.random(30, 30, density=0.04, random_state=2, format="csr"),
           sp.random(30, 30, density=0.04, random_state=3, format="csr")]
    tiny = sp.csr_matrix(np.array([[rng.standard_normal()]]))
    cancel = [sp.csr_matrix(np.array([[0, 1e-10], [2.0, 0]])), sp.csr_matrix(np.array([[0, -1e-10], [0, 0]]))]
    return {"directed": directed, "symmetric": sym, "isolated": sp.csr_matrix(iso), "E2": two, "N1": tiny,
            "below-tolerance": cancel, "empty": sp.csr_matrix((5, 5))}


@pytest.mark.parametrize("name", sorted(_graphs()))
@pytest.mark.parametrize("K", [1, 2, 3])
def test_ring_prefixes_are_the_k_hop_neighbourhoods(name, K):
    from gnn_b200.graphtools_sparse import compute_neighborhood, ring_neighborhoods
    S = _graphs()[name]
    rowptr, col, ring_end = ring_neighborhoods(S, K)
    N = (S[0] if isinstance(S, list) else S).shape[0]
    assert rowptr.dtype == np.int64 and col.dtype == np.int32 and ring_end.dtype == np.int32
    assert rowptr.shape == (N + 1,) and ring_end.shape == (N, K + 1) and rowptr[-1] == len(col)
    assert np.array_equal(np.diff(rowptr), ring_end[:, K])
    for k in range(K + 1):
        ref = compute_neighborhood(S, k)
        for i in range(N):
            lst = col[rowptr[i]:rowptr[i] + ring_end[i, k]]
            assert sorted(lst.tolist()) == ref[i], (k, i)
    for i in range(N):
        lst = col[rowptr[i]:rowptr[i + 1]]
        assert lst[0] == i and ring_end[i, 0] == 1
        for k in range(1, K + 1):                           # each ring ascending, and new at its distance
            ring = lst[ring_end[i, k - 1]:ring_end[i, k]]
            assert np.all(np.diff(ring) > 0)
    if name == "isolated":
        assert np.all(ring_end[7] == 1)
    if name == "below-tolerance":
        assert np.array_equal(ring_end[:, 1], [1, 2])       # |1e-10| + |-1e-10| is no edge, 2.0 is


def _cases():
    if not os.path.exists(GOLDEN):
        return []
    z = np.load(GOLDEN)
    return sorted({k[:-len("_y")] for k in z.files if k.startswith("la_") and k.endswith("_y")})


@pytest.mark.parametrize("case", _cases())
def test_oracle_matches_reference_fixtures(case):
    from gnn_b200.graphtools_sparse import ring_neighborhoods
    z = np.load(GOLDEN)
    g = lambda n: z[case + "_" + n]                          # noqa: E731
    S, w, x, dy = g("S"), g("weight"), g("x"), g("dy")
    K = w.shape[1] - 1
    op = lao.MAX if "_Max_" in case else lao.MEDIAN
    B, F, N = x.shape
    rings = ring_neighborhoods([sp.csr_matrix(s) for s in S], K)
    node_major = lambda t: t.reshape(B * F, N).T             # noqa: E731
    y, ybound, agg, arg = lao.forward(node_major(x), w, *rings, K, op, np.float64)
    assert np.allclose(y.T.reshape(B, F, N), g("y"), rtol=0, atol=1e-13)
    dx, _, dw, _ = lao.backward(node_major(x), node_major(dy), w, agg, arg, np.float64)
    assert np.allclose(dx.T.reshape(B, F, N), g("dx"), rtol=0, atol=1e-13)
    assert np.allclose(dw, g("dw"), rtol=0, atol=1e-12)
    assert np.all(ybound > 0)


def test_oracle_tie_rules():
    """Max: the smallest node holding the maximum; median: the lower median, at the smallest node holding it."""
    rowptr = np.array([0, 5], dtype=np.int64)
    col = np.array([0, 4, 2, 3, 1], dtype=np.int32)         # ring order is not index order
    ring_end = np.array([[1, 5]], dtype=np.int32)
    x = np.array([[1.0], [2.0], [2.0], [0.5], [2.0]])
    agg, arg = lao.select(x, rowptr, col, ring_end, 1, lao.MAX)
    assert agg[0, 0, 0] == 2.0 and arg[0, 0, 0] == 1
    agg, arg = lao.select(x, rowptr, col, ring_end, 1, lao.MEDIAN)   # sorted 0.5 1 2 2 2: rank 2 -> 2.0 at node 1
    assert agg[0, 0, 0] == 2.0 and arg[0, 0, 0] == 1
    x2 = np.array([[3.0], [1.0], [4.0], [1.0], [5.0]])
    agg, arg = lao.select(x2, rowptr, col, np.array([[1, 4]], dtype=np.int32), 1, lao.MEDIAN)
    assert agg[0, 0, 0] == 3.0 and arg[0, 0, 0] == 0       # nodes 0 4 2 3 hold 3 5 4 1: lower median of 1 3 4 5


@pytest.mark.parametrize("kind", ["Max", "Median"])
def test_add_gso_keeps_the_padded_matrices_for_the_cpu_path(kind):
    """addGSO builds only the ring lists; `neighborhood` (the torch path's padded matrices) is built on first use
    and equals compute_neighborhood's 'matrix' form, and maxNeighborhoodSizes is its widths."""
    import gnn_b200
    from gnn_b200 import activations
    from gnn_b200.graphtools_sparse import compute_neighborhood
    S = _graphs()["isolated"]
    layer = getattr(activations, kind + "LocalActivation")(3)
    assert layer.extra_repr() == "neighborhood stored" and layer.neighborhood == "None"
    layer.addGSO(gnn_b200.SparseGSO.from_scipy([S]))
    assert layer._padded is None
    ref = [compute_neighborhood(S, k, outputType="matrix") for k in (1, 2, 3)]
    assert layer.maxNeighborhoodSizes == [m.shape[1] for m in ref]
    for k, ((idx, lens), m) in enumerate(zip(layer.neighborhood, ref), start=1):
        assert np.array_equal(idx.numpy(), m)
        assert lens.tolist() == [len(r) for r in compute_neighborhood(S, k)]
    assert layer.extra_repr() == "neighborhood stored"
