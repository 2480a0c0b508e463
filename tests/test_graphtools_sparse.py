"""CSR-native graph utilities (graph-neural-networks_b200/graphtools_sparse.py) against the UNMODIFIED reference's dense
`alegnn.utils.graphTools` (CPU; the reference's results are stored in tests/golden, oracle/ref_golden.py), plus
reference-free properties."""
import numpy as np
import pytest
import scipy.sparse as sp

from ref_golden import pack_lists, reference, unpack_lists


def _graph(seed, N=24, p=0.18, directed=False, weights=True):
    rng = np.random.default_rng(seed)
    A = (rng.random((N, N)) < p).astype(float)
    np.fill_diagonal(A, 0.0)
    if weights:
        A = A * rng.uniform(0.2, 1.5, (N, N))
    if not directed:
        A = np.triu(A, 1)
        A = A + A.T
    ring = np.roll(np.eye(N), 1, axis=1) * 0.7       # a ring keeps every graph connected and every degree positive
    return A + (ring if directed else ring + ring.T)


def _gt():
    import ref_import
    ref_import.import_reference()
    import alegnn.utils.graphTools as graphTools
    return graphTools


@pytest.fixture(scope="module")
def gs():
    import gnn_b200  # noqa: F401
    import gnn_b200.graphtools_sparse as g
    return g


@pytest.mark.parametrize("seed,directed", [(0, False), (1, False), (2, True), (3, True)])
def test_normalisations_and_spectrum(gs, seed, directed):
    W = _graph(seed, directed=directed)
    Ws = sp.csr_matrix(W)

    def run_reference():
        gt = _gt()
        L = gt.adjacencyToLaplacian(W)
        E, _ = gt.computeGFT(W)                                   # what the examples divide by (sourceLocGNN.py:752)
        return dict(L=L, A=gt.normalizeAdjacency(W), Ln=gt.normalizeLaplacian(L), lam=np.max(np.real(np.diag(E))))

    r = reference("graphtools_normalisations_%d_%d" % (seed, directed), run_reference)
    assert np.allclose(gs.adjacency_to_laplacian(Ws).toarray(), r["L"], atol=1e-13)
    assert np.allclose(gs.normalize_adjacency(Ws).toarray(), r["A"], atol=1e-13)
    assert np.allclose(gs.normalize_laplacian(sp.csr_matrix(r["L"])).toarray(), r["Ln"], atol=1e-13)
    lam = float(r["lam"])
    assert abs(gs.largest_real_eigenvalue(Ws) - lam) < 1e-8 * abs(lam)
    assert np.allclose(gs.spectral_normalize(Ws).toarray(), W / lam, atol=1e-8)


def test_connectivity(gs):
    graphs = [_graph(seed, directed=seed % 2 == 1) for seed in range(4)]
    two = np.zeros((10, 10))
    two[:5, :5] = _graph(7, N=5)
    two[5:, 5:] = _graph(8, N=5)
    one_way = np.diag(np.ones(5), 1)                             # a directed path counts as connected (:570-574)
    graphs += [two, one_way]
    r = reference("graphtools_connectivity", lambda: dict(connected=np.array([_gt().isConnected(W) for W in graphs])))
    assert r["connected"].tolist() == [True] * 4 + [False, True]
    assert [gs.is_connected(sp.csr_matrix(W)) for W in graphs] == r["connected"].tolist()


@pytest.mark.parametrize("K", [0, 1, 2, 3])
@pytest.mark.parametrize("seed,directed", [(0, False), (5, True)])
def test_neighbourhoods(gs, K, seed, directed):
    W = _graph(seed, N=20, p=0.1, directed=directed)
    # edge-feature GSO: an edge exists where any S_e is non-zero (:424-432)
    S3 = np.stack([W * (np.arange(20)[:, None] % 2 == 0), W * (np.arange(20)[:, None] % 2 == 1)])

    def run_reference():
        gt = _gt()
        nb, nb_len = pack_lists([sorted(int(j) for j in r) for r in gt.computeNeighborhood(W, K)])
        nb3, nb3_len = pack_lists([sorted(int(j) for j in r) for r in gt.computeNeighborhood(S3, K)])
        return dict(nb=nb, nb_len=nb_len, m=gt.computeNeighborhood(W, K, N=7, nb=15, outputType="matrix"),
                    nb3=nb3, nb3_len=nb3_len)

    r = reference("graphtools_neighbourhoods_K%d_%d_%d" % (K, seed, directed), run_reference)
    got = gs.compute_neighborhood(sp.csr_matrix(W), K)
    assert unpack_lists(r["nb"], r["nb_len"]) == got
    # first N nodes only, neighbours restricted to nodes < nb, matrix output padded with the node's own index
    ref_m = r["m"]
    got_m = gs.compute_neighborhood(sp.csr_matrix(W), K, N=7, nb=15, outputType="matrix")
    assert ref_m.shape == got_m.shape
    assert [sorted(set(r.tolist())) for r in ref_m] == [sorted(set(r.tolist())) for r in got_m]
    got3 = gs.compute_neighborhood([sp.csr_matrix(S3[0]), sp.csr_matrix(S3[1])], K)
    assert unpack_lists(r["nb3"], r["nb3_len"]) == got3


def test_perm_degree(gs):
    W = _graph(11, directed=True)
    S3 = np.stack([W, W.T * 0.5])

    def run_reference():
        gt = _gt()
        refS, refOrder = gt.permDegree(W)
        ref3, order3 = gt.permDegree(S3)
        return dict(S=refS, order=np.asarray(refOrder), S3=ref3, order3=np.asarray(order3))

    r = reference("graphtools_perm_degree", run_reference)
    gotS, gotOrder = gs.perm_degree(sp.csr_matrix(W))
    assert r["order"].tolist() == list(gotOrder) and np.array_equal(gotS.toarray(), r["S"])
    got3, gorder3 = gs.perm_degree([sp.csr_matrix(S3[0]), sp.csr_matrix(S3[1])])
    assert r["order3"].tolist() == list(gorder3) and np.array_equal(np.stack([m.toarray() for m in got3]), r["S3"])


@pytest.mark.parametrize("directed", [False, True])
def test_edge_fail_sampling_matches_reference_rng(gs, directed):
    W = _graph(13, directed=directed)

    def run_reference():
        np.random.seed(5)
        return dict(W=_gt().edgeFailSampling(W, 0.3))

    r = reference("graphtools_edge_fail_%d" % directed, run_reference)
    np.random.seed(5)
    got = gs.edge_fail_sampling(sp.csr_matrix(W), 0.3, dense_rng_compat=True)
    assert np.array_equal(got.toarray(), r["W"])


def test_edge_fail_sampling_scalable_mode(gs):
    W = sp.csr_matrix(_graph(17, N=200, p=0.05))
    out = gs.edge_fail_sampling(W, 0.4, rng=np.random.default_rng(1))
    assert abs(out - out.T).max() == 0                            # stays undirected
    assert (out != 0).multiply(W == 0).nnz == 0                   # never creates an edge
    frac = out.nnz / W.nnz
    assert 0.5 < frac < 0.7                                       # ~60 % of the edges survive
    assert gs.edge_fail_sampling(W, 0.0, rng=np.random.default_rng(1)).nnz == W.nnz


@pytest.mark.parametrize("kind,p", [("threshold", 0.6), ("threshold", 1.2), ("NN", 3), ("NN", 1)])
@pytest.mark.parametrize("directed", [False, True])
def test_sparsify(gs, kind, p, directed):
    W = _graph(19, N=18, p=0.35, directed=directed)
    r = reference("graphtools_sparsify_%s_%s_%d" % (kind, p, directed), lambda: dict(W=_gt().sparsifyGraph(W, kind, p)))
    got = gs.sparsify_graph(sp.csr_matrix(W), kind, p)
    assert np.allclose(got.toarray(), r["W"], atol=1e-13)


def test_large_graph_pipeline_feeds_the_filter(gs):
    """The sparse pipeline at a size the dense reference cannot hold: build, check, normalise, wrap as a SparseGSO."""
    import gnn_b200
    from gnn_b200 import graphs
    g = graphs.er_gso(200_000, 8, seed=3)
    r, c, v = g.csr[0]
    A = sp.csr_matrix((np.ones_like(v, dtype=np.float64), c, r), shape=(g.N, g.N))
    assert gs.is_connected(A) in (True, False)
    S = gs.spectral_normalize(A)
    assert abs(gs.largest_real_eigenvalue(S) - 1.0) < 1e-6
    nb = gs.compute_neighborhood(A, 2, N=5)
    assert all(i in nb[i] for i in range(5))
    gso = gs.to_sparse_gso(S, dtype="torch.float32")
    assert gso.shape == (1, 200_000, 200_000) and gso.nnz() == A.nnz
